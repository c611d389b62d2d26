// nvb_tsdf.cu -- projective TSDF update of the frame's VoxelBlocks.
//
// Replaces integrateBlocksKernel<TsdfVoxel, UpdateTsdfVoxelFunctor, Camera>
// (nvblox/include/nvblox/integrators/internal/cuda/impl/projective_integrator_impl.cuh:59-114)
// with its functor (projective_tsdf_integrator_impl.cuh:30-90) and weighting
// function (internal/impl/weighting_function_impl.h:29-117).
//
// Kernel shape: a persistent grid (multiple of the SM count) walks the device-side
// block list -- the host never learns the block count. A 256-thread CTA owns one
// 4 KiB VoxelBlock per iteration; every thread owns two z-adjacent voxels = one
// 128-bit word, so a warp moves 512 contiguous bytes per LDG.128/STG.128 and a
// block is exactly 256 vector accesses each way. The next block's word is
// prefetched before the current one is processed. Blocks are addressed by slot in
// the layer slab (no pointer table). Update parameters arrive as __grid_constant__
// kernel arguments (the reference dereferences a device pointer to a functor it
// re-uploads every frame). Unchanged words are not written back.
#include "nvb_internal.cuh"

namespace nvb {

namespace {

struct TsdfArgs {
  const int4* frame_blocks;
  const int* frame_count;
  unsigned char* tsdf_blocks;
  const float* depth;
  const unsigned char* mask;
  int mask_mode;
  int rows, cols;
  Rigid T_C_L;
  NvbCamera cam;
  TsdfKernelParams p;
  unsigned int* bits_to_clear;  // view bitset of this frame: consumed by the compaction, zeroed here
  int num_words;
};

// WeightingFunction (weighting_function_impl.h:29-117)
__device__ __forceinline__ float dropoff(float measured, float voxel_depth, float trunc) {
  if (trunc <= 1e-2f) return 0.0f;
  if (voxel_depth > measured) {
    const float behind = voxel_depth - measured;
    if (behind > trunc) return 0.0f;
    return (trunc - behind) / trunc;
  }
  return 1.0f;
}
__device__ __forceinline__ float inverseSquare(float measured, float voxel_depth, float trunc) {
  if (voxel_depth <= 1e-2f) return 1.0f;
  if (voxel_depth - measured >= trunc) return 0.0f;
  return 1.0f / (voxel_depth * voxel_depth);
}
__device__ __forceinline__ float tsdfDistancePenalty(float measured, float voxel_depth, float trunc) {
  return (fabsf(measured - voxel_depth) >= trunc) ? 0.1f : 1.0f;
}
__device__ __forceinline__ float weighting(int type, float measured, float voxel_depth, float trunc) {
  switch (type) {
    case NVB_WEIGHT_CONSTANT:
      return 1.0f;
    case NVB_WEIGHT_CONSTANT_DROPOFF:
      return 1.0f * dropoff(measured, voxel_depth, trunc);
    case NVB_WEIGHT_INVERSE_SQUARE:
      return inverseSquare(measured, voxel_depth, trunc);
    case NVB_WEIGHT_INVERSE_SQUARE_DROPOFF:
      return inverseSquare(measured, voxel_depth, trunc) * dropoff(measured, voxel_depth, trunc);
    case NVB_WEIGHT_INVERSE_SQUARE_TSDF_DISTANCE_PENALTY:
      return inverseSquare(measured, voxel_depth, trunc) * tsdfDistancePenalty(measured, voxel_depth, trunc);
    default:  // NVB_WEIGHT_LINEAR_WITH_MAX
      return (voxel_depth > 1.0f) ? 1.0f / voxel_depth : 1.0f;
  }
}

// Shared front end of integrateBlocksKernel (projective_integrator_impl.cuh:59-114): project the voxel centre,
// look the depth (and the mask) up. Returns false if the voxel is not updated at all.
template <bool kDistort>
__device__ __forceinline__ bool sampleVoxel(const TsdfArgs& a, const int4& blk, int vx, int vy, int vz, float& d,
                                            float& voxel_depth, bool& is_active) {
  // getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:51-81)
  Vec3 p_L;
  p_L.x = (a.p.block_size * (float)blk.x + a.p.voxel_size * (float)vx) + a.p.half_voxel_size;
  p_L.y = (a.p.block_size * (float)blk.y + a.p.voxel_size * (float)vy) + a.p.half_voxel_size;
  p_L.z = (a.p.block_size * (float)blk.z + a.p.voxel_size * (float)vz) + a.p.half_voxel_size;
  const Vec3 p_C = transformPoint(a.T_C_L, p_L);
  // Camera::project (sensors/internal/impl/camera_impl.h:37-76)
  if (!(isfinite(p_C.x) && isfinite(p_C.y) && isfinite(p_C.z))) return false;
  if (!(p_C.z >= 1e-6f)) return false;
  float un = p_C.x / p_C.z, vn = p_C.y / p_C.z;
  if (kDistort) applyDistortion(a.cam, un, vn);
  const float u = un * a.cam.fu + a.cam.cu;
  const float v = vn * a.cam.fv + a.cam.cv;
  if (u > (float)a.cam.width || v > (float)a.cam.height || u < 0.0f || v < 0.0f) return false;
  voxel_depth = p_C.z;
  // projectThreadVoxel max-depth test (projective_integrators_common_impl.cuh:42-45)
  if (a.p.max_integration_distance_m > 0.0f && voxel_depth > a.p.max_integration_distance_m) return false;
  // interpolate2DClosest (interpolation/internal/impl/interpolation_2d_impl.h:125-150)
  const int ux = floatToIntRz(floorf(u)), uy = floatToIntRz(floorf(v));
  if (ux < 0 || uy < 0 || ux >= a.cols || uy >= a.rows) return false;
  const size_t pix = (size_t)uy * a.cols + ux;
  d = __ldg(a.depth + pix);
  if (!(isfinite(d) && d > 1e-6f)) d = 0.0f;  // PixelIsValidDepth (interpolation_2d_impl.h:99-104)
  is_active = true;  // MaskedImageView::isMasked (sensors/internal/impl/image_impl.h:250-259)
  if (a.mask != nullptr) {
    const unsigned char mv = __ldg(a.mask + pix);
    is_active = (a.mask_mode == NVB_MASK_NON_INVERTED) ? (mv != 0) : (mv == 0);
  }
  return true;
}

// UpdateTsdfVoxelFunctor (projective_tsdf_integrator_impl.cuh:30-90) on a sampled voxel. Returns true if (dist, weight) changed.
__device__ __forceinline__ bool fuseVoxel(const TsdfArgs& a, float d, float voxel_depth, bool is_active, float& dist,
                                          float& wgt) {
  const float trunc = a.p.truncation_distance_m;
  if (d <= 0.0f) {
    if (a.p.invalid_depth_decay_factor >= 0.0f) {
      wgt = wgt * a.p.invalid_depth_decay_factor;
      return true;
    }
    return false;
  }
  const float sdf = d - voxel_depth;
  if (sdf < -trunc) return false;
  if (!is_active && sdf < trunc) return false;
  const float w = weighting(a.p.weighting_type, d, voxel_depth, trunc);
  float fused = (sdf * w + dist * wgt) / (w + wgt);
  if (fused > 0.0f) {
    fused = fminf(trunc, fused);
  } else {
    fused = fmaxf(-trunc, fused);
  }
  dist = fused;
  wgt = fminf(w + wgt, a.p.max_weight);
  return true;
}

// One TSDF voxel: sample, fuse. Returns true if (dist, weight) changed.
template <bool kDistort>
__device__ __forceinline__ bool updateVoxel(const TsdfArgs& a, const int4& blk, int vx, int vy, int vz, float& dist,
                                            float& wgt) {
  float d, voxel_depth;
  bool is_active;
  if (!sampleVoxel<kDistort>(a, blk, vx, vy, vz, d, voxel_depth, is_active)) return false;
  return fuseVoxel(a, d, voxel_depth, is_active, dist, wgt);
}

// One occupancy voxel: UpdateOccupancyVoxelFunctor (projective_occupancy_integrator_impl.cuh:27-73).
template <bool kDistort>
__device__ __forceinline__ bool updateOccupancyVoxel(const TsdfArgs& a, const OccKernelParams& o, const int4& blk, int vx,
                                                     int vy, int vz, float& log_odds) {
  float d, voxel_depth;
  bool is_active;
  if (!sampleVoxel<kDistort>(a, blk, vx, vy, vz, d, voxel_depth, is_active)) return false;
  if (d <= 0.0f) return false;
  float upd;
  if (!is_active || voxel_depth > d + o.occupied_half_width_m) {
    upd = o.unobserved_log_odds;
  } else if (voxel_depth > d - o.occupied_half_width_m) {
    upd = o.occupied_log_odds;
  } else {
    upd = o.free_log_odds;
  }
  const float updated = log_odds + upd;
  log_odds = fmaxf(o.min_log_odds, fminf(updated, o.max_log_odds));
  return true;
}

// Occupancy twin of tsdfIntegrateKernel: a block is 2 KiB (512 floats); 128 threads, four z-adjacent voxels
// (one 128-bit word) per thread, two blocks per 256-thread CTA iteration.
template <bool kDistort>
__global__ void __launch_bounds__(256) occupancyIntegrateKernel(const __grid_constant__ TsdfArgs a,
                                                                const __grid_constant__ OccKernelParams o) {
  const int n = *a.frame_count;
  const int tid = threadIdx.x;
  for (int w = blockIdx.x * blockDim.x + tid; w < a.num_words; w += gridDim.x * blockDim.x) a.bits_to_clear[w] = 0;
  const int half = tid >> 7, t = tid & 127;
  // voxels 4t .. 4t+3 : linear offset = x*64 + y*8 + z
  const int vx = t >> 4, vy = (t >> 1) & 7, vz = (t & 1) * 4;
  for (int i = blockIdx.x * 2 + half; i < n; i += gridDim.x * 2) {
    const int4 blk = a.frame_blocks[i];
    if (blk.w < 0) continue;
    float4* gp = reinterpret_cast<float4*>(a.tsdf_blocks + (size_t)blk.w * kOccBlockBytes) + t;
    float4 word = *gp;
    bool c = updateOccupancyVoxel<kDistort>(a, o, blk, vx, vy, vz, word.x);
    c |= updateOccupancyVoxel<kDistort>(a, o, blk, vx, vy, vz + 1, word.y);
    c |= updateOccupancyVoxel<kDistort>(a, o, blk, vx, vy, vz + 2, word.z);
    c |= updateOccupancyVoxel<kDistort>(a, o, blk, vx, vy, vz + 3, word.w);
    if (c) *gp = word;
  }
}

template <bool kDistort>
__global__ void __launch_bounds__(256) tsdfIntegrateKernel(const __grid_constant__ TsdfArgs a) {
  const int n = *a.frame_count;
  const int tid = threadIdx.x;
  for (int w = blockIdx.x * blockDim.x + tid; w < a.num_words; w += gridDim.x * blockDim.x) a.bits_to_clear[w] = 0;
  // voxel pair owned by this thread: linear voxel offset 2*tid = x*64 + y*8 + z
  const int vx = tid >> 5, vy = (tid >> 2) & 7, vz = (tid & 3) * 2;
  int i = blockIdx.x;
  if (i >= n) return;
  int4 blk = a.frame_blocks[i];
  float4 word = make_float4(0.f, 0.f, 0.f, 0.f);
  if (blk.w >= 0) word = __ldcs(reinterpret_cast<const float4*>(a.tsdf_blocks + (size_t)blk.w * kTsdfBlockBytes) + tid);
  while (true) {
    // prefetch the next block's word before working on this one
    const int inext = i + gridDim.x;
    int4 nblk = make_int4(0, 0, 0, -1);
    float4 nword = make_float4(0.f, 0.f, 0.f, 0.f);
    if (inext < n) {
      nblk = a.frame_blocks[inext];
      if (nblk.w >= 0)
        nword = __ldcs(reinterpret_cast<const float4*>(a.tsdf_blocks + (size_t)nblk.w * kTsdfBlockBytes) + tid);
    }
    if (blk.w >= 0) {
      const bool c0 = updateVoxel<kDistort>(a, blk, vx, vy, vz, word.x, word.y);
      const bool c1 = updateVoxel<kDistort>(a, blk, vx, vy, vz + 1, word.z, word.w);
      if (c0 || c1) *(reinterpret_cast<float4*>(a.tsdf_blocks + (size_t)blk.w * kTsdfBlockBytes) + tid) = word;
    }
    if (inext >= n) break;
    i = inext, blk = nblk, word = nword;
  }
}

// ProjectiveIntegrator::markUnobservedFreeInsideRadiusTemplate (projective_integrator_impl.cuh:408-462): a warp per block of
// the box around the sphere: exterior distance of the block's box to the centre (getBlocksWithinRadius,
// src/geometry/bounding_spheres.cpp:24-67), find-or-insert, tracker append, setUnobservedVoxel (:377-392) on its 512 voxels.
__global__ void __launch_bounds__(256) markFreeSphereKernel(const __grid_constant__ MarkFreeArgs a) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const float c[3] = {a.cx, a.cy, a.cz};
  for (int cell = warp; cell < a.cells; cell += nwarps) {
    const int idx[3] = {a.lo.x + cell / (a.size.y * a.size.z), a.lo.y + (cell / a.size.z) % a.size.y, a.lo.z + cell % a.size.z};
    if (!(blockExteriorDistance(idx, a.block_size, c) < a.radius)) continue;
    int slot = -1;
    if (lane == 0) {
      bool was_new;
      slot = hashFindOrInsert(a.layer, idx[0], idx[1], idx[2], a.error, &was_new);
      if (slot >= 0) {
        trackerAdd(a.tracker, slot);  // addBlocksToUpdate(updated_blocks) (src/mapper/mapper.cpp:506)
        a.out[atomicAdd(a.out_count, 1)] = make_int4(idx[0], idx[1], idx[2], slot);
      }
    }
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (slot < 0) continue;
    if (a.occupancy) {
      float* lo = reinterpret_cast<float*>(a.layer.blocks + (size_t)slot * kOccBlockBytes);
#pragma unroll 4
      for (int k = 0; k < kVpb / 32; k++) {
        const float v = lo[lane + 32 * k];
        if (fabsf(v - 0.0f) < 1e-4f) lo[lane + 32 * k] = -2e-4f;
      }
    } else {
      float2* t = reinterpret_cast<float2*>(a.layer.blocks + (size_t)slot * kTsdfBlockBytes);
#pragma unroll 4
      for (int k = 0; k < kVpb / 32; k++) {
        const float2 v = t[lane + 32 * k];
        if (v.y < 0.001f) t[lane + 32 * k] = make_float2(a.trunc_m, 0.1f);
      }
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------
// VoxelDecayer::decay (decayer_impl.cuh:84-262) with TsdfDecayFunctor (tsdf_decay_integrator_impl.cuh:25-75) or
// OccupancyDecayFunctor (occupancy_decay_integrator_impl.cuh:26-70). Persistent CTAs over the slab's slots, one
// block per iteration, two voxels per thread. A block whose voxels are all fully decayed is deallocated on the
// spot: its bytes go back to zero (the slab invariant), its slot onto the layer's free stack, its index into
// the `dead` list (the host rebuilds the hash afterwards and removes the ESDF twin).
// ---------------------------------------------------------------------------
template <bool kDistort>
__device__ __forceinline__ bool voxelHasDepthMeasurement(const TsdfArgs& v, const int4& blk, int vx, int vy, int vz) {
  // doesVoxelHaveDepthMeasurement (projective_integrators_common_impl.cuh:58-101)
  float d, voxel_depth;
  bool is_active;
  if (!sampleVoxel<kDistort>(v, blk, vx, vy, vz, d, voxel_depth, is_active)) return false;
  if (!(d > 0.0f)) return false;  // invalid depth (sampleVoxel maps it to 0): not in view
  return !(d - voxel_depth < -v.p.truncation_distance_m);
}

template <bool kDistort>
__global__ void __launch_bounds__(256) decayKernel(const __grid_constant__ DecayArgs a) {
  const int tid = threadIdx.x;
  const int n = *a.layer.count < a.layer.capacity ? *a.layer.count : a.layer.capacity;
  TsdfArgs v;  // view description for sampleVoxel
  v.depth = a.depth, v.mask = nullptr, v.mask_mode = 0, v.rows = a.rows, v.cols = a.cols;
  v.T_C_L = a.T_C_L, v.cam = a.cam, v.p = a.p;
  // voxels 2 tid, 2 tid + 1 (z-adjacent): linear offset = x*64 + y*8 + z
  const int vx = tid >> 5, vy = (tid >> 2) & 7, vz = (tid & 3) * 2;
  for (int slot = blockIdx.x; slot < n; slot += gridDim.x) {
    const int bx = a.layer.block_index[3 * slot];
    if (bx == kDeadSlotX) continue;
    const int by = a.layer.block_index[3 * slot + 1], bz = a.layer.block_index[3 * slot + 2];
    // getBlockIndicesToDecay (decayer_impl.cuh:38-80)
    if (a.skip_stamp && a.skip_stamp[slot] == a.skip_seq) continue;
    if (a.has_sphere) {
      // getPositionFromBlockIndex = block origin; squaredNorm in Eigen's a0 + (a1 + a2) order
      const float dx = a.p.block_size * (float)bx - a.cx, dy = a.p.block_size * (float)by - a.cy,
                  dz = a.p.block_size * (float)bz - a.cz;
      const float d2 = sum3(dx * dx, dy * dy, dz * dz);
      if (!(d2 > a.r2)) continue;
    }
    const int4 blk = make_int4(bx, by, bz, slot);
    bool decay0 = true, decay1 = true;
    if (a.depth) {
      decay0 = !voxelHasDepthMeasurement<kDistort>(v, blk, vx, vy, vz);
      decay1 = !voxelHasDepthMeasurement<kDistort>(v, blk, vx, vy, vz + 1);
    }
    bool fully;
    if (a.occupancy) {
      float2* gp = reinterpret_cast<float2*>(a.layer.blocks + (size_t)slot * kOccBlockBytes) + tid;
      float2 w = *gp;
      const float2 old = w;
      auto is_fully = [&](float lo) {
        return lo >= a.to_log_odds ? (lo + a.occupied_log_odds < a.to_log_odds) : (lo + a.free_log_odds >= a.to_log_odds);
      };
      auto step = [&](float lo) {
        if (is_fully(lo)) return a.to_log_odds;
        return lo >= 0.0f ? lo + a.occupied_log_odds : lo + a.free_log_odds;
      };
      if (decay0) w.x = step(w.x);
      if (decay1) w.y = step(w.y);
      fully = is_fully(w.x) && is_fully(w.y);
      const bool all = __syncthreads_and(fully);
      if (all && a.deallocate) *gp = make_float2(0.0f, 0.0f);
      else if (w.x != old.x || w.y != old.y) *gp = w;
      fully = all;
    } else {
      float4* gp = reinterpret_cast<float4*>(a.layer.blocks + (size_t)slot * kTsdfBlockBytes) + tid;
      float4 w = *gp;  // {distance0, weight0, distance1, weight1}
      const float4 old = w;
      auto step = [&](float& dist, float& weight) {
        if (weight < (a.weight_threshold - 1e-6f)) return;
        weight = fmaxf(weight * a.decay_factor, a.weight_threshold);
        if (a.set_free_distance && weight < (a.weight_threshold + 1e-6f)) dist = a.free_distance_m;
      };
      if (decay0) step(w.x, w.y);
      if (decay1) step(w.z, w.w);
      fully = (w.y < (a.weight_threshold + 1e-6f)) && (w.w < (a.weight_threshold + 1e-6f));
      const bool all = __syncthreads_and(fully);
      if (all && a.deallocate) *gp = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      else if (w.x != old.x || w.y != old.y || w.z != old.z || w.w != old.w) *gp = w;
      fully = all;
    }
    if (fully && a.deallocate && tid == 0) {
      a.layer.block_index[3 * slot] = kDeadSlotX;
      a.dead[atomicAdd(a.dead_count, 1)] = make_int4(slot, bx, by, bz);
      a.layer.free_slots[atomicAdd(a.layer.free_count, 1)] = slot;
    }
  }
}

// DecayBlockExclusionOptions::block_indices_to_exclude: stamp the slots of the listed blocks.
__global__ void markSkippedKernel(DevLayer L, const int* xyz, int n, int* skip_stamp, int skip_seq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int slot = hashFind(L.hash, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
  if (slot >= 0) skip_stamp[slot] = skip_seq;
}

// ---------------------------------------------------------------------------
// FreespaceIntegrator::updateFreespaceLayer (freespace_integrator_impl.cuh:324-383): allocate the freespace twins of
// the blocks to update, then updateFreespaceLayerKernel (:99-246) -- the dynablox freespace state machine, one CTA
// (512 threads, one voxel each) per block.
// ---------------------------------------------------------------------------
__global__ void freespaceAllocateKernel(FreespaceArgs a) {
  const int n = a.todo.count ? *a.todo.count : a.n_explicit;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *a.work_count = n;
  if (i >= n) return;
  int x, y, z, tslot;
  if (a.todo.slots) {
    tslot = a.todo.slots[i];
    a.todo.dirty[tslot] = 0;
    x = a.tsdf.block_index[3 * tslot], y = a.tsdf.block_index[3 * tslot + 1], z = a.tsdf.block_index[3 * tslot + 2];
  } else {
    x = a.in_xyz[3 * i], y = a.in_xyz[3 * i + 1], z = a.in_xyz[3 * i + 2];
    tslot = hashFind(a.tsdf.hash, x, y, z);
  }
  bool was_new;
  const int fslot = hashFindOrInsert(a.fs, x, y, z, a.error, &was_new);  // allocateBlocksAtIndices (:343-345)
  a.work[i] = make_int4(tslot, fslot, 0, 0);
}

struct FsVoxel {
  long long last_occupied, consecutive;
  unsigned long long flag;  // byte 0: is_high_confidence_freespace
};

template <bool kDistort>
__global__ void __launch_bounds__(512) freespaceUpdateKernel(const __grid_constant__ FreespaceArgs a) {
  __shared__ unsigned char s_free[512];
  const int tid = threadIdx.x;
  const int n = *a.work_count;
  if (blockIdx.x == 0 && tid == 0 && a.todo.count) *a.todo.count = 0;  // tracker list consumed
  TsdfArgs v;
  v.depth = a.depth, v.mask = nullptr, v.mask_mode = 0, v.rows = a.rows, v.cols = a.cols;
  v.T_C_L = a.T_C_L, v.cam = a.cam, v.p = a.p;
  const int vx = tid >> 6, vy = (tid >> 3) & 7, vz = tid & 7;
  for (int item = blockIdx.x; item < n; item += gridDim.x) {
    const int4 w = a.work[item];
    if (w.x < 0 || w.y < 0) continue;  // no TSDF block / slab exhausted
    s_free[tid] = 0;
    __syncthreads();
    FsVoxel* gp = reinterpret_cast<FsVoxel*>(a.fs.blocks + (size_t)w.y * kFreespaceBlockBytes) + tid;
    FsVoxel f = *gp;
    const float2 t = reinterpret_cast<const float2*>(a.tsdf.blocks + (size_t)w.x * kTsdfBlockBytes)[tid];  // {distance, weight}
    bool update_voxel = true;
    if (a.depth) {
      const int4 blk = make_int4(a.tsdf.block_index[3 * w.x], a.tsdf.block_index[3 * w.x + 1], a.tsdf.block_index[3 * w.x + 2], w.x);
      update_voxel = voxelHasDepthMeasurement<kDistort>(v, blk, vx, vy, vz);
    }
    const bool init = f.last_occupied == 0;
    if (init) {  // all voxels are initialised to being occupied
      f.last_occupied = a.now_ms;
      f.consecutive = 0;
      f.flag = (f.flag & ~0xffull) | (a.init_high_confidence ? 1ull : 0ull);
    }
    bool is_free = false;
    if (update_voxel && !init) {
      // dynablox Eq. (9): consecutive occupancy duration
      if (a.now_ms - f.last_occupied <= a.max_unobserved_ms) f.consecutive += a.now_ms - a.last_update_ms;
      else f.consecutive = 0;
      // Eq. (8): last occupied timestamp
      if (t.x <= a.max_tsdf_distance_for_occupancy_m) f.last_occupied = a.now_ms;
      // isVoxelFree (:36-44); `weight > 1e-6` is a float compared with a double literal
      is_free = ((double)t.y > 1e-6) && (f.last_occupied != 0) && (f.last_occupied <= a.now_ms - a.min_free_ms);
      s_free[tid] = is_free ? 1 : 0;
    }
    __syncthreads();
    if (update_voxel && !init) {
      if (a.check_neighborhood && is_free) {  // isVoxelNeighborhoodFree (:46-83): 3x3x3, inside this block only
        for (int dx = -1; dx <= 1; dx++)
          for (int dy = -1; dy <= 1; dy++)
            for (int dz = -1; dz <= 1; dz++) {
              const int x = vx + dx, y = vy + dy, z = vz + dz;
              if ((dx | dy | dz) == 0) continue;
              if (x < 0 || x > 7 || y < 0 || y > 7 || z < 0 || z > 7) continue;
              is_free = is_free && s_free[(x * 8 + y) * 8 + z];
            }
      }
      // Eq. (12) / (11): high confidence freespace
      const bool hc = (f.flag & 0xffull) != 0;
      const bool nhc = (f.consecutive >= a.min_reset_ms) ? false : (hc || is_free);
      f.flag = (f.flag & ~0xffull) | (nhc ? 1ull : 0ull);
    }
    if (update_voxel || init) *gp = f;
    __syncthreads();
  }
}

// Resident CTAs per SM of the projective update kernels: 8 x 256 threads fill an SM's thread slots (one full wave). That
// keeps the cooperative ESDF wavefront of the previous frame (side stream, one 256-thread CTA per SM) from starting until
// this kernel drains.
constexpr int kProjectiveCtasPerSm = 8;

static TsdfArgs projectiveArgs(const int4* frame_blocks, const int* frame_count, unsigned char* blocks, const float* depth,
                               const unsigned char* mask, int mask_mode, int rows, int cols, const Rigid& T_C_L,
                               const NvbCamera& cam, const TsdfKernelParams& p, unsigned int* bits_to_clear, int num_words) {
  TsdfArgs a;
  a.frame_blocks = frame_blocks;
  a.frame_count = frame_count;
  a.tsdf_blocks = blocks;
  a.depth = depth;
  a.mask = mask;
  a.mask_mode = mask_mode;
  a.rows = rows, a.cols = cols;
  a.T_C_L = T_C_L;
  a.cam = cam;
  a.p = p;
  a.bits_to_clear = bits_to_clear;
  a.num_words = num_words;
  return a;
}

void launchMarkFreeSphere(const MarkFreeArgs& a, int num_sms, cudaStream_t stream) {
  markFreeSphereKernel<<<num_sms * 4, 256, 0, stream>>>(a);
}

void launchTsdfIntegrate(const int4* frame_blocks, const int* frame_count, unsigned char* tsdf_blocks,
                         const float* depth, const unsigned char* mask, int mask_mode, int rows, int cols,
                         const Rigid& T_C_L, const NvbCamera& cam, const TsdfKernelParams& p, int num_sms,
                         unsigned int* bits_to_clear, int num_words, cudaStream_t stream) {
  const TsdfArgs a = projectiveArgs(frame_blocks, frame_count, tsdf_blocks, depth, mask, mask_mode, rows, cols, T_C_L, cam, p,
                                    bits_to_clear, num_words);
  // the lens-distortion variant is a separate instantiation so the pinhole path keeps its register budget
  const int grid = num_sms * kProjectiveCtasPerSm;
  if (cam.has_distortion) tsdfIntegrateKernel<true><<<grid, 256, 0, stream>>>(a);
  else tsdfIntegrateKernel<false><<<grid, 256, 0, stream>>>(a);
}

void launchOccupancyIntegrate(const int4* frame_blocks, const int* frame_count, unsigned char* occ_blocks,
                              const float* depth, const unsigned char* mask, int mask_mode, int rows, int cols,
                              const Rigid& T_C_L, const NvbCamera& cam, const TsdfKernelParams& p,
                              const OccKernelParams& op, int num_sms, unsigned int* bits_to_clear, int num_words,
                              cudaStream_t stream) {
  const TsdfArgs a = projectiveArgs(frame_blocks, frame_count, occ_blocks, depth, mask, mask_mode, rows, cols, T_C_L, cam, p,
                                    bits_to_clear, num_words);
  const int grid = num_sms * kProjectiveCtasPerSm;
  if (cam.has_distortion) occupancyIntegrateKernel<true><<<grid, 256, 0, stream>>>(a, op);
  else occupancyIntegrateKernel<false><<<grid, 256, 0, stream>>>(a, op);
}

void launchFreespaceUpdate(const FreespaceArgs& a, int upper, int num_sms, cudaStream_t stream) {
  if (upper < 1) upper = 1;
  freespaceAllocateKernel<<<(upper + 255) / 256, 256, 0, stream>>>(a);
  int grid = num_sms * 4;
  if (upper < grid) grid = upper;
  if (a.depth && a.cam.has_distortion) freespaceUpdateKernel<true><<<grid, 512, 0, stream>>>(a);
  else freespaceUpdateKernel<false><<<grid, 512, 0, stream>>>(a);
}

void launchDecay(const DecayArgs& a, int num_sms, cudaStream_t stream) {
  const int grid = num_sms * 8;
  if (a.depth && a.cam.has_distortion) decayKernel<true><<<grid, 256, 0, stream>>>(a);
  else decayKernel<false><<<grid, 256, 0, stream>>>(a);
}
void launchMarkSkipped(const DevLayer& layer, const int* xyz_dev, int n, int* skip_stamp, int skip_seq, cudaStream_t stream) {
  if (n > 0) markSkippedKernel<<<(n + 255) / 256, 256, 0, stream>>>(layer, xyz_dev, n, skip_stamp, skip_seq);
}

}  // namespace nvb
