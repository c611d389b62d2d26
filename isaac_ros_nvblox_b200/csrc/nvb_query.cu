// nvb_query.cu -- reading the map at arbitrary points: voxel lookups (VoxelBlockLayer::getVoxels, queryVoxelsKernel,
// map/internal/cuda/impl/layer_impl.cuh:29-80), trilinear interpolation (interpolation::interpolateOnCPU,
// src/interpolation/interpolation_3d.cpp, interpolation/internal/impl/interpolation_3d_impl.h) and nvblox_torch's
// sphere / point queries (nvblox_torch/cpp/src/sdf_query.cu:63-354).
//
// One grid-stride kernel per query kind, 64-bit point offsets. A query reads the map and never writes it. Each point
// resolves its block through hashFind and reads only the voxel words the query needs (a distance-only ESDF query skips the
// parent words).
//
// Deviations from the reference, where its behaviour is undefined or accidental:
//  - a point with a non-finite coordinate, or whose block index lies outside the hash's +-2^20 key range, is a miss (the
//    reference's float -> int conversion would alias it to some other block);
//  - interpolation does not abort when the corner offsets leave [0, 1] by rounding (getQVector3D's CHECKs); it evaluates the
//    same polynomial.
#include "nvb_esdf_block.cuh"

namespace nvb {

namespace {

constexpr int kQueryThreads = 256;
constexpr float kMaxDistance = 100.0f;       // nvblox_torch/sdf_query.cuh:30-31 (kMaxDistance, kESDFUnknownDistance)
constexpr float kTsdfMinWeight = 1e-4f;      // interpolation_3d.cpp:31
constexpr float kGradientEpsilon = 1e-6f;    // sdf_query.cu:106

__device__ __forceinline__ bool finite3(const Vec3& p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

// getVoxelAtPosition (gpu_hash/internal/cuda/gpu_indexing.cuh:56-64): the block holding p (null if it is not allocated)
// and the voxel's index v in it.
__device__ __forceinline__ const unsigned char* voxelAt(const QueryLayer& q, const Vec3& p, int* v) {
  if (!finite3(p)) return nullptr;
  int3 b, vi;
  blockAndVoxelIndexFromPosition(q.block_size, q.voxel_size_inv, p, b, vi);
  const int slot = hashFind(q.layer.hash, b.x, b.y, b.z);
  if (slot < 0) return nullptr;
  *v = (vi.x * kVps + vi.y) * kVps + vi.z;
  return q.layer.blocks + (size_t)slot * q.layer.block_bytes;
}

__device__ __forceinline__ Vec3 loadPoint(const float* xyz, long long i, int stride) {
  const float* p = xyz + i * stride;
  return Vec3{p[0], p[1], p[2]};
}

// ESDF voxels are returned as the reference's 20-byte records (nvb_esdf_block.cuh).
__global__ void __launch_bounds__(kQueryThreads) queryVoxelsKernel(const __grid_constant__ QueryLayer q, int voxel_words, bool esdf,
                                                                  const float* __restrict__ xyz, long long n,
                                                                  unsigned int* __restrict__ out,
                                                                  unsigned char* __restrict__ found) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int v = 0;
    const unsigned char* blk = voxelAt(q, loadPoint(xyz, i, 3), &v);
    found[i] = blk != nullptr;
    if (!blk) continue;
    const unsigned int* words = reinterpret_cast<const unsigned int*>(blk);
    if (esdf) {
      esdfVoxelToRecord(words, v, out + i * voxel_words);
    } else {
      for (int w = 0; w < voxel_words; w++) out[i * voxel_words + w] = words[(size_t)v * voxel_words + w];
    }
  }
}

// The member interpolated and the validity rule of each layer (interpolation_3d.cpp:21-69).
template <int kKind>
__device__ __forceinline__ bool interpMember(const unsigned char* blk, int v, float* value) {
  if (kKind == kInterpTsdf) {
    const float2 t = reinterpret_cast<const float2*>(blk)[v];
    *value = t.x;
    return t.y > kTsdfMinWeight;
  } else if (kKind == kInterpEsdf) {
    const unsigned int* b = reinterpret_cast<const unsigned int*>(blk);
    if ((*esdfFlag(b, v) & 0xff00u) == 0) return false;  // observed
    *value = sqrtf(__uint_as_float(*esdfCell(b, v)));
    return true;
  } else {
    const float lo = reinterpret_cast<const float*>(blk)[v];
    *value = expf(lo) / (1.0f + expf(lo));  // probabilityFromLogOdds (core/log_odds.h:32-34)
    return true;
  }
}

// interpolateMemberOnCPU (interpolation_3d_impl.h:127-165) with getSurroundingVoxels3D (:57-125). The sums of the 8x8 table
// product and of the q-vector product run left to right over the table's non-zero entries (the order the restatement fixes).
template <int kKind>
__device__ __forceinline__ bool interpolateAt(const QueryLayer& q, Vec3 p, float* result) {
  if (!finite3(p)) return false;
  const float half = q.voxel_size * 0.5f;
  int3 b, v;
  blockAndVoxelIndexFromPosition(q.block_size, q.voxel_size_inv, Vec3{p.x - half, p.y - half, p.z - half}, b, v);
  if (!indexInRange(b.x, b.y, b.z)) return false;
  // getPositionFromBlockIndexAndVoxelIndex (indexing_impl.h:51-57) + half a voxel; the offset in voxels
  const float ox = (p.x - ((q.block_size * (float)b.x + q.voxel_size * (float)v.x) + half)) / q.voxel_size;
  const float oy = (p.y - ((q.block_size * (float)b.y + q.voxel_size * (float)v.y) + half)) / q.voxel_size;
  const float oz = (p.z - ((q.block_size * (float)b.z + q.voxel_size * (float)v.z) + half)) / q.voxel_size;
  // The 8 neighbours lie in up to 8 blocks: block (cx, cy, cz) is needed when the low corner sits on the block's last voxel
  // along every axis with c = 1. Slots are kept in registers (key = cx << 2 | cy << 1 | cz, picked by branch-free selects).
  const int ex = v.x == kVps - 1, ey = v.y == kVps - 1, ez = v.z == kVps - 1;
  int slots[8];
#pragma unroll
  for (int key = 0; key < 8; key++) {
    const int cx = key >> 2, cy = (key >> 1) & 1, cz = key & 1;
    const bool needed = (!cx || ex) && (!cy || ey) && (!cz || ez);
    slots[key] = needed ? hashFind(q.layer.hash, b.x + cx, b.y + cy, b.z + cz) : -1;
  }
  float m[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int dx = i >> 2, dy = (i >> 1) & 1, dz = i & 1;
    const int cx = dx & ex, cy = dy & ey, cz = dz & ez;
    const int slot = cx ? (cy ? (cz ? slots[7] : slots[6]) : (cz ? slots[5] : slots[4]))
                        : (cy ? (cz ? slots[3] : slots[2]) : (cz ? slots[1] : slots[0]));
    if (slot < 0) return false;
    const int vx = cx ? 0 : v.x + dx, vy = cy ? 0 : v.y + dy, vz = cz ? 0 : v.z + dz;
    if (!interpMember<kKind>(q.layer.blocks + (size_t)slot * q.layer.block_bytes, (vx * kVps + vy) * kVps + vz, &m[i]))
      return false;
  }
  // interpolation_table * member_vector (rows of the table, non-zero entries in column order)
  const float t0 = m[0];
  const float t1 = -m[0] + m[4];
  const float t2 = -m[0] + m[2];
  const float t3 = -m[0] + m[1];
  const float t4 = ((m[0] - m[2]) - m[4]) + m[6];
  const float t5 = ((m[0] - m[1]) - m[2]) + m[3];
  const float t6 = ((m[0] - m[1]) - m[4]) + m[5];
  const float t7 = ((((((-m[0] + m[1]) + m[2]) - m[3]) + m[4]) - m[5]) - m[6]) + m[7];
  // getQVector3D (interpolation_3d.cpp:73-95)
  const float qv[8] = {1.0f, ox, oy, oz, ox * oy, oy * oz, oz * ox, (ox * oy) * oz};
  const float tv[8] = {t0, t1, t2, t3, t4, t5, t6, t7};
  float r = qv[0] * tv[0];
#pragma unroll
  for (int k = 1; k < 8; k++) r = r + qv[k] * tv[k];
  *result = r;
  return true;
}

template <int kKind>
__global__ void __launch_bounds__(kQueryThreads) interpolateKernel(const __grid_constant__ QueryLayer q, const float* __restrict__ xyz,
                                                                  long long n, float* __restrict__ out,
                                                                  unsigned char* __restrict__ success) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float r = 0.0f;  // the vector overload's value of a failed point (interpolation_3d_impl.h:33-37)
    const bool ok = interpolateAt<kKind>(q, loadPoint(xyz, i, 3), &r);
    out[i] = ok ? r : 0.0f;
    success[i] = ok;
  }
}

// queryESDFKernel / queryESDFMultiMapperKernel with extractEsdf (sdf_query.cu:63-115,155-205). Spheres {x, y, z, r}; out
// {gx, gy, gz, d} with the gradient, {d} without. Only the last write of each output matters, so they are kept in registers
// and stored once: the outputs a point never writes keep what the caller put there.
// (The minimum of 4 CTAs per SM lifts ptxas' register budget above the 32 at which the multi-mapper gradient variant spills.)
template <bool kMulti, bool kGrad>
__global__ void __launch_bounds__(kQueryThreads, 4) queryEsdfKernel(const __grid_constant__ QueryLayers q,
                                                                const float* __restrict__ spheres, long long n,
                                                                float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float4 s = make_float4(spheres[4 * i], spheres[4 * i + 1], spheres[4 * i + 2], spheres[4 * i + 3]);
    const Vec3 p{s.x, s.y, s.z};
    float min_distance = kMaxDistance;  // over all mappers
    bool write_d = false, write_g = false;
    float d = 0.0f, gx = 0.0f, gy = 0.0f, gz = 0.0f;
    const int nm = kMulti ? q.n : 1;
    for (int k = 0; k < nm; k++) {
      const QueryLayer& L = q.l[k];
      int v = 0;
      const unsigned char* blk = voxelAt(L, p, &v);
      if (!blk) continue;
      const unsigned int* e = esdfCell(reinterpret_cast<const unsigned int*>(blk), v);
      const unsigned int flags = *esdfFlag(reinterpret_cast<const unsigned int*>(blk), v);
      write_d = true;
      if ((flags & 0xff00u) == 0) {  // not observed
        d = kMaxDistance;
        continue;
      }
      float distance = L.voxel_size * sqrtf(__uint_as_float(e[0]));
      if (flags & 0xffu) distance = -distance;  // is_inside
      const float sphere_distance = distance - s.w;
      if (kMulti) {
        if (sphere_distance > min_distance) {
          d = min_distance;
          continue;
        }
        min_distance = sphere_distance;
      }
      d = sphere_distance;
      if (kGrad) {
        write_g = true;
        if (distance > kGradientEpsilon) {
          const float f = -L.voxel_size / distance;
          gx = f * (float)(int)e[1], gy = f * (float)(int)e[2], gz = f * (float)(int)e[3];
        } else {
          gx = gy = gz = 0.0f;
        }
      }
    }
    if (kGrad) {
      if (write_g) out[4 * i] = gx, out[4 * i + 1] = gy, out[4 * i + 2] = gz;
      if (write_d) out[4 * i + 3] = d;
    } else if (write_d) {
      out[i] = d;
    }
  }
}

// queryTSDFKernel / queryTSDFMultiMapperKernel (sdf_query.cu:240-318): out {distance, weight}. Single mapper: written on a hit
// only. Several: the smallest distance and the weight at it, {100, 0} when no mapper has the voxel.
template <bool kMulti>
__global__ void __launch_bounds__(kQueryThreads) queryTsdfKernel(const __grid_constant__ QueryLayers q, const float* __restrict__ xyz,
                                                                long long n, float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const Vec3 p = loadPoint(xyz, i, 3);
    if (!kMulti) {
      int v = 0;
      const unsigned char* blk = voxelAt(q.l[0], p, &v);
      if (blk) {
        const float2 t = reinterpret_cast<const float2*>(blk)[v];
        out[2 * i] = t.x, out[2 * i + 1] = t.y;
      }
      continue;
    }
    float min_distance = kMaxDistance, weight_at_min = 0.0f;
    for (int k = 0; k < q.n; k++) {
      int v = 0;
      const unsigned char* blk = voxelAt(q.l[k], p, &v);
      if (!blk) continue;
      const float2 t = reinterpret_cast<const float2*>(blk)[v];
      if (t.x < min_distance) min_distance = t.x, weight_at_min = t.y;
    }
    out[2 * i] = min_distance, out[2 * i + 1] = weight_at_min;
  }
}

// queryOccupancyMultiMapperKernel (sdf_query.cu:320-351): the largest log-odds over the mappers that have the voxel,
// starting from logOddsFromProbability(0). (nvblox_torch has no single-mapper occupancy kernel: one mapper is the same loop.)
template <bool kMulti>
__global__ void __launch_bounds__(kQueryThreads) queryOccupancyKernel(const __grid_constant__ QueryLayers q, float initial,
                                                                     const float* __restrict__ xyz, long long n,
                                                                     float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const Vec3 p = loadPoint(xyz, i, 3);
    float max_log_odds = initial;
    const int nm = kMulti ? q.n : 1;
    for (int k = 0; k < nm; k++) {
      int v = 0;
      const unsigned char* blk = voxelAt(q.l[k], p, &v);
      if (!blk) continue;
      const float lo = reinterpret_cast<const float*>(blk)[v];
      if (lo > max_log_odds) max_log_odds = lo;
    }
    out[i] = max_log_odds;
  }
}

int queryGrid(long long n, int num_sms) {
  const long long want = (n + kQueryThreads - 1) / kQueryThreads;
  const long long cap = (long long)num_sms * 16;
  return (int)(want < cap ? want : cap);
}

}  // namespace

void launchQueryVoxels(const QueryLayer& q, int voxel_bytes, bool esdf, const float* xyz, long long n, void* out, unsigned char* found,
                       int num_sms, cudaStream_t stream) {
  if (n <= 0) return;
  queryVoxelsKernel<<<queryGrid(n, num_sms), kQueryThreads, 0, stream>>>(q, voxel_bytes / 4, esdf, xyz, n,
                                                                         static_cast<unsigned int*>(out), found);
}

void launchInterpolate(const QueryLayer& q, int kind, const float* xyz, long long n, float* out, unsigned char* success,
                       int num_sms, cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = queryGrid(n, num_sms);
  if (kind == kInterpTsdf) interpolateKernel<kInterpTsdf><<<grid, kQueryThreads, 0, stream>>>(q, xyz, n, out, success);
  else if (kind == kInterpEsdf) interpolateKernel<kInterpEsdf><<<grid, kQueryThreads, 0, stream>>>(q, xyz, n, out, success);
  else interpolateKernel<kInterpOccupancy><<<grid, kQueryThreads, 0, stream>>>(q, xyz, n, out, success);
}

void launchQueryEsdf(const QueryLayers& q, bool multi, const float* spheres_xyzr, long long n, bool with_gradient, float* out,
                     int num_sms, cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = queryGrid(n, num_sms);
  if (multi && with_gradient) queryEsdfKernel<true, true><<<grid, kQueryThreads, 0, stream>>>(q, spheres_xyzr, n, out);
  else if (multi) queryEsdfKernel<true, false><<<grid, kQueryThreads, 0, stream>>>(q, spheres_xyzr, n, out);
  else if (with_gradient) queryEsdfKernel<false, true><<<grid, kQueryThreads, 0, stream>>>(q, spheres_xyzr, n, out);
  else queryEsdfKernel<false, false><<<grid, kQueryThreads, 0, stream>>>(q, spheres_xyzr, n, out);
}

void launchQueryTsdf(const QueryLayers& q, bool multi, const float* xyz, long long n, float* out, int num_sms,
                     cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = queryGrid(n, num_sms);
  if (multi) queryTsdfKernel<true><<<grid, kQueryThreads, 0, stream>>>(q, xyz, n, out);
  else queryTsdfKernel<false><<<grid, kQueryThreads, 0, stream>>>(q, xyz, n, out);
}

void launchQueryOccupancy(const QueryLayers& q, bool multi, float initial_log_odds, const float* xyz, long long n, float* out,
                          int num_sms, cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = queryGrid(n, num_sms);
  if (multi) queryOccupancyKernel<true><<<grid, kQueryThreads, 0, stream>>>(q, initial_log_odds, xyz, n, out);
  else queryOccupancyKernel<false><<<grid, kQueryThreads, 0, stream>>>(q, initial_log_odds, xyz, n, out);
}

}  // namespace nvb
