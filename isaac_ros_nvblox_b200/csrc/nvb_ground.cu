// nvb_ground.cu -- the ground-plane estimator (GroundPlaneEstimator::computeGroundPlane,
// src/experimental/ground_plane/ground_plane_estimator.cpp:27-62):
//   * zero crossings from above (TsdfZeroCrossingsExtractor::computeZeroCrossingsFromAboveOnGPU,
//     tsdf_zero_crossings_extractor.cu:24-146) and the ground-candidate z filter (getPointsWithinMinMaxZCPU,
//     ground_plane_estimator.cpp:109-125), as count -> scan -> emit over the blocks in (x, y, z) order, so that both point
//     lists come out in a canonical order (block index lexicographically, then voxel (x, y, z)) instead of the reference's
//     atomicAdd order;
//   * the MSAC plane fit (RansacPlaneFitter::fit, ransac_plane_fitter.cu:29-144): one thread per iteration, XORWOW
//     states curand_init(1234, iteration, 0) cached by the caller, the points streamed through shared memory by cp.async
//     (double-buffered, every lane reads the same point: a broadcast), and the argmin on the device.
#include <cfloat>

#include <cub/device/device_radix_sort.cuh>
#include <curand_kernel.h>

#include "nvb_internal.cuh"

namespace nvb {

namespace {

constexpr int kPairThreads = kVpb;   // one thread per (voxel, voxel above) pair of a block
constexpr int kScanThreads = 1024;
constexpr int kFitThreads = 32;      // one warp per CTA: 1 000 iterations spread over 32 SMs
constexpr int kFitTile = 512;        // points per shared-memory tile (8 KB; two tiles in flight)
constexpr int kArgminThreads = 1024;

// The crossing between voxel v = (x, y, z) of the block in `slot` and the voxel above it, and whether it is a ground
// candidate. Pairs at z = 7 read z = 0 of the block above (`above` slot, -1: no block -> no pair).
__device__ __forceinline__ bool crossingAt(const GroundExtractArgs& a, int slot, int above, const int bidx[3], int v, float3* p,
                                           bool* candidate) {
  const int vx = v >> 6, vy = (v >> 3) & 7, vz = v & 7;
  const float2* blk = reinterpret_cast<const float2*>(a.tsdf.blocks + (size_t)slot * kTsdfBlockBytes);
  float2 below = blk[v], up;
  if (vz < kVps - 1) {
    up = blk[v + 1];
  } else {
    if (above < 0) return false;
    up = reinterpret_cast<const float2*>(a.tsdf.blocks + (size_t)above * kTsdfBlockBytes)[v - (kVps - 1)];
  }
  // TsdfVoxel {distance, weight}
  if (!(up.y >= a.min_tsdf_weight && below.y >= a.min_tsdf_weight)) return false;
  if (!(up.x > 0.0f && below.x <= 0.0f)) return false;
  // getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:51-81)
  const float vs = a.block_size * 0.125f, hvs = a.block_size * 0.0625f;
  const float px = (a.block_size * (float)bidx[0] + vs * (float)vx) + hvs;
  const float py = (a.block_size * (float)bidx[1] + vs * (float)vy) + hvs;
  const float pz = (a.block_size * (float)bidx[2] + vs * (float)vz) + hvs;
  const float dz = (-below.x * a.voxel_size) / (up.x - below.x);
  *p = make_float3(px, py, pz + dz);
  *candidate = isfinite(p->x) && isfinite(p->y) && isfinite(p->z) && p->z >= a.min_z && p->z <= a.max_z;
  return true;
}

// Sort keys of the slab's slots below the high-water mark: packIndex orders like Index3D's lexicographic comparison;
// free slots get the largest key and the value -1, so they sort last and are skipped.
__global__ void groundKeysKernel(DevLayer L, int hw, unsigned long long* keys, int* slots) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += gridDim.x * blockDim.x) {
    const int x = L.block_index[3 * i];
    const bool live = x != kDeadSlotX;
    keys[i] = live ? packIndex(x, L.block_index[3 * i + 1], L.block_index[3 * i + 2]) : ~0ull;
    slots[i] = live ? i : -1;
  }
}

// Slot of block i of the sorted list (-1: a free slot) and of the block above it (one lookup per CTA, in the device hash).
__device__ __forceinline__ void loadBlock(const GroundExtractArgs& a, int i, int* s_slot, int* s_above, int* s_idx) {
  if (threadIdx.x == 0) {
    const int slot = a.slots[i];
    *s_slot = slot;
    if (slot >= 0) {
      s_idx[0] = a.tsdf.block_index[3 * slot], s_idx[1] = a.tsdf.block_index[3 * slot + 1], s_idx[2] = a.tsdf.block_index[3 * slot + 2];
      *s_above = s_idx[2] + 1 < kIndexBias ? hashFind(a.tsdf.hash, s_idx[0], s_idx[1], s_idx[2] + 1) : -1;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kPairThreads) groundCountKernel(GroundExtractArgs a) {
  __shared__ int s_slot, s_above, s_idx[3];
  loadBlock(a, blockIdx.x, &s_slot, &s_above, s_idx);
  if (s_slot < 0) {
    if (threadIdx.x == 0) a.counts[blockIdx.x] = make_int2(0, 0);
    return;
  }
  float3 p;
  bool cand = false;
  const bool hit = crossingAt(a, s_slot, s_above, s_idx, threadIdx.x, &p, &cand);
  const int n_hit = __syncthreads_count(hit);
  const int n_cand = __syncthreads_count(hit && cand);
  if (threadIdx.x == 0) a.counts[blockIdx.x] = make_int2(n_hit, n_cand);
}

// Exclusive scan of n int2 counts in place (one CTA); totals -> totals[0..1]. Shared with nvb_dynamics.cu.
__global__ void __launch_bounds__(kScanThreads) exclusiveScanInt2Kernel(int2* counts, int n, int* totals) {
  __shared__ int2 s_warp[kScanThreads / 32];
  __shared__ int2 s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = make_int2(0, 0);
  __syncthreads();
  for (int base = 0; base < n; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int2 c = i < n ? counts[i] : make_int2(0, 0);
    int2 incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, incl.x, o), y = __shfl_up_sync(0xffffffffu, incl.y, o);
      if (lane >= o) incl.x += x, incl.y += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int2 w = s_warp[lane];
      int2 wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, wi.x, o), y = __shfl_up_sync(0xffffffffu, wi.y, o);
        if (lane >= o) wi.x += x, wi.y += y;
      }
      s_warp[lane] = make_int2(wi.x - w.x, wi.y - w.y);
    }
    __syncthreads();
    const int2 carry = s_carry, wo = s_warp[warp];
    if (i < n) counts[i] = make_int2(carry.x + wo.x + incl.x - c.x, carry.y + wo.y + incl.y - c.y);
    __syncthreads();
    if (threadIdx.x == kScanThreads - 1) s_carry = make_int2(carry.x + wo.x + incl.x, carry.y + wo.y + incl.y);
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[0] = s_carry.x, totals[1] = s_carry.y;
}

// Block-wide exclusive rank of `flag` in thread order; 16 warps.
__device__ __forceinline__ int blockRank(bool flag, int* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned int b = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) s_warp[warp] = __popc(b);
  __syncthreads();
  int before = 0;
  for (int w = 0; w < warp; w++) before += s_warp[w];
  __syncthreads();
  return before + __popc(b & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kPairThreads) groundEmitKernel(GroundExtractArgs a) {
  __shared__ int s_slot, s_above, s_idx[3];
  __shared__ int s_warp[kPairThreads / 32];
  loadBlock(a, blockIdx.x, &s_slot, &s_above, s_idx);
  if (s_slot < 0) return;
  float3 p = make_float3(0.0f, 0.0f, 0.0f);
  bool cand = false;
  const bool hit = crossingAt(a, s_slot, s_above, s_idx, threadIdx.x, &p, &cand);
  const int2 off = a.counts[blockIdx.x];
  const int r_hit = blockRank(hit, s_warp);
  const int r_cand = blockRank(hit && cand, s_warp);
  if (hit) a.crossings[off.x + r_hit] = p;
  if (hit && cand) a.candidates[off.y + r_cand] = make_float4(p.x, p.y, p.z, 0.0f);
}

__global__ void packPointsKernel(const float* xyz, int n, float4* out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    out[i] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], 0.0f);
}

__global__ void ransacInitKernel(curandState* states, int first, int n) {
  const int i = first + blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) curand_init(1234ull, (unsigned long long)i, 0ull, &states[i]);  // kSeed (ransac_plane_fitter.cu:26)
}

// Eigen's fixed-size-3 expressions, evaluated as the rest of the library does (sum3 order, one rounding per operation).
__device__ __forceinline__ float3 normalized3(float3 v) {  // MatrixBase::normalized: v / sqrt(squaredNorm) if > 0
  const float z = sum3(v.x * v.x, v.y * v.y, v.z * v.z);
  if (z > 0.0f) {
    const float s = sqrtf(z);
    return make_float3(v.x / s, v.y / s, v.z / s);
  }
  return v;
}

// Plane::planeFromPoints (geometry/internal/impl/plane_impl.h:34-52) with Plane(normal, point) -> Plane(normal, d): the
// normal is normalised three times and d taken from the second one, as the reference's constructor chain does.
__device__ __forceinline__ bool planeFromPoints(float4 a, float4 b, float4 c, float4* out) {
  auto eq = [](float4 u, float4 w) { return u.x == w.x && u.y == w.y && u.z == w.z; };
  if (eq(a, b) || eq(a, c) || eq(b, c)) return false;
  const float3 ab = make_float3(b.x - a.x, b.y - a.y, b.z - a.z);
  const float3 ac = make_float3(c.x - a.x, c.y - a.y, c.z - a.z);
  const float3 v = make_float3(ab.y * ac.z - ab.z * ac.y, ab.z * ac.x - ab.x * ac.z, ab.x * ac.y - ab.y * ac.x);
  if (fabsf(v.x) <= 1e-6f && fabsf(v.y) <= 1e-6f && fabsf(v.z) <= 1e-6f) return false;  // isZero(1e-6): collinear
  const float3 n1 = normalized3(v);
  const float3 n2 = normalized3(n1);
  const float d = -sum3(a.x * n2.x, a.y * n2.y, a.z * n2.z);
  const float3 n3 = normalized3(n2);
  *out = make_float4(n3.x, n3.y, n3.z, d);
  return true;
}

__device__ __forceinline__ void cpAsync16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cpAsyncCommit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cpAsyncWaitPrior1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

__device__ __forceinline__ void stageTile(float4* dst, const float4* pts, int n, int tile) {
  const int base = tile * kFitTile;
  const int m = min(kFitTile, n - base);
  for (int j = threadIdx.x; j < m; j += kFitThreads) cpAsync16(dst + j, pts + base + j);
}

// ransacKernel (ransac_plane_fitter.cu:37-85): three draws curand() % n, the plane, then the MSAC cost summed over the
// points in list order in float. Rejected samples keep the cost FLT_MAX.
__device__ __forceinline__ bool samplePlane(const float4* pts, int n, int it, int iterations, const curandState* states,
                                            float4* pl) {
  if (it >= iterations) return false;
  curandState st = states[it];
  const unsigned int un = (unsigned int)n;
  const unsigned int i1 = curand(&st) % un, i2 = curand(&st) % un, i3 = curand(&st) % un;
  return planeFromPoints(pts[i1], pts[i2], pts[i3], pl);
}

__device__ __forceinline__ float msacTerm(const float4& pl, const float4& q, float thr, float thr2) {
  // Plane::signedDistance = normal.dot(p) + d
  const float dist = fabsf(sum3(pl.x * q.x, pl.y * q.y, pl.z * q.z) + pl.w);
  return dist < thr ? dist * dist : thr2;
}

__global__ void __launch_bounds__(kFitThreads) ransacFitKernel(const float4* pts, int n, int iterations, float thr,
                                                              const curandState* states, float* costs, float4* planes) {
  __shared__ __align__(16) float4 s_pts[2][kFitTile];
  const int it = blockIdx.x * kFitThreads + threadIdx.x;
  float4 pl = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  const bool ok = samplePlane(pts, n, it, iterations, states, &pl);
  // Whole CTA rejected: nothing to sum (the threads agree, so the exit is uniform).
  if (__syncthreads_or(ok) == 0) {
    if (it < iterations) costs[it] = FLT_MAX;
    return;
  }
  const float thr2 = thr * thr;
  float cost = 0.0f;
  const int tiles = (n + kFitTile - 1) / kFitTile;
  stageTile(s_pts[0], pts, n, 0);
  cpAsyncCommit();
  for (int t = 0; t < tiles; t++) {
    if (t + 1 < tiles) stageTile(s_pts[(t + 1) & 1], pts, n, t + 1);
    cpAsyncCommit();
    cpAsyncWaitPrior1();
    __syncthreads();
    const float4* s = s_pts[t & 1];
    const int m = min(kFitTile, n - t * kFitTile);
#pragma unroll 8
    for (int j = 0; j < m; j++) cost += msacTerm(pl, s[j], thr, thr2);
    __syncthreads();
  }
  if (it < iterations) {
    costs[it] = ok ? cost : FLT_MAX;
    if (ok) planes[it] = pl;
  }
}

// std::min_element over the costs (lowest cost, lowest index on ties: the costs are never NaN, every summand being
// d^2 < t^2 or t^2) -> {nx, ny, nz, d, found}.
__global__ void __launch_bounds__(kArgminThreads) ransacArgminKernel(const float* costs, const float4* planes, int iterations,
                                                                     float* out) {
  __shared__ float s_c[kArgminThreads];
  __shared__ int s_i[kArgminThreads];
  float bc = FLT_MAX;
  int bi = -1;
  for (int i = threadIdx.x; i < iterations; i += kArgminThreads)
    if (bi < 0 || costs[i] < bc) bc = costs[i], bi = i;
  s_c[threadIdx.x] = bc, s_i[threadIdx.x] = bi;
  __syncthreads();
  for (int h = kArgminThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      const float oc = s_c[threadIdx.x + h];
      const int oi = s_i[threadIdx.x + h];
      const int mi = s_i[threadIdx.x];
      if (oi >= 0 && (mi < 0 || oc < s_c[threadIdx.x] || (oc == s_c[threadIdx.x] && oi < mi)))
        s_c[threadIdx.x] = oc, s_i[threadIdx.x] = oi;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int i = s_i[0];
    const bool found = i >= 0 && s_c[0] != FLT_MAX;
    const float4 pl = found ? planes[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    out[0] = pl.x, out[1] = pl.y, out[2] = pl.z, out[3] = pl.w;
    reinterpret_cast<int*>(out)[4] = found ? 1 : 0;
  }
}

}  // namespace

size_t ransacStateBytes() { return sizeof(curandState); }

size_t groundSortTempBytes(int n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n, 0, 64);
  return bytes;
}

cudaError_t launchGroundSortBlocks(const DevLayer& tsdf, int hw, unsigned long long* keys, int* slots, void* temp,
                                   size_t temp_bytes, cudaStream_t stream) {
  groundKeysKernel<<<std::min((hw + 255) / 256, 4 * kHelperCtas), 256, 0, stream>>>(tsdf, hw, keys, slots);
  return cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys + hw, slots, slots + hw, hw, 0, 64, stream);
}

void launchGroundCount(const GroundExtractArgs& a, cudaStream_t stream) {
  groundCountKernel<<<a.num_blocks, kPairThreads, 0, stream>>>(a);
  exclusiveScanInt2Kernel<<<1, kScanThreads, 0, stream>>>(a.counts, a.num_blocks, a.totals);
}

void launchExclusiveScanInt2(int2* counts, int n, int* totals, cudaStream_t stream) {
  exclusiveScanInt2Kernel<<<1, kScanThreads, 0, stream>>>(counts, n, totals);
}

void launchGroundEmit(const GroundExtractArgs& a, cudaStream_t stream) {
  groundEmitKernel<<<a.num_blocks, kPairThreads, 0, stream>>>(a);
}

void launchPackPoints(const float* xyz, int n, float4* out, cudaStream_t stream) {
  packPointsKernel<<<std::min((n + 255) / 256, 4 * kHelperCtas), 256, 0, stream>>>(xyz, n, out);
}

void launchRansacInit(void* states, int first, int n, cudaStream_t stream) {
  if (n <= first) return;
  ransacInitKernel<<<(n - first + 127) / 128, 128, 0, stream>>>(static_cast<curandState*>(states), first, n);
}

void launchRansacFit(const float4* pts, int n, int iterations, float threshold, const void* states, float* costs,
                     float4* planes, float* out5, cudaStream_t stream) {
  const curandState* st = static_cast<const curandState*>(states);
  ransacFitKernel<<<(iterations + kFitThreads - 1) / kFitThreads, kFitThreads, 0, stream>>>(pts, n, iterations, threshold, st,
                                                                                              costs, planes);
  ransacArgminKernel<<<1, kArgminThreads, 0, stream>>>(costs, planes, iterations, out5);
}

}  // namespace nvb
