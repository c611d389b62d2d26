// nvb_clear.cu -- map clearing: the block selection of Mapper::clearOutsideRadius (src/mapper/mapper.cpp:473-492), the
// tracker pass that follows its deallocation (BlocksToUpdateTracker::removeClearedBlocksFromTracking,
// src/map/blocks_to_update_tracker.cpp:75-90) and ShapeClearer::clear (integrators/internal/cuda/impl/shape_clearer_impl.cuh:22-127).
// The deallocation itself is the decay's (removeBlocksKernel, esdfRemoveBlocksKernel, hash rebuild).
#include "nvb_internal.cuh"

namespace nvb {

namespace {

constexpr int kShapeTile = 256;  // shapes staged in shared memory per pass of the voxel kernel (7 KB)

// getBlocksOutsideRadius (src/geometry/bounding_spheres.cpp:47-50,69-74): exteriorDistance(center) > radius, strict.
// One thread per slot below the high-water mark, warp-ballot append like todoAllKernel.
__global__ void selectOutsideRadiusKernel(DevLayer L, float cx, float cy, float cz, float radius, float block_size, int4* dead,
                                          int* dead_count) {
  const int n = *L.count < L.capacity ? *L.count : L.capacity;
  const int lane = threadIdx.x & 31;
  const float c[3] = {cx, cy, cz};
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) - lane; base < n; base += gridDim.x * blockDim.x) {
    const int i = base + lane;
    int idx[3] = {kDeadSlotX, 0, 0};
    if (i < n) idx[0] = L.block_index[3 * i], idx[1] = L.block_index[3 * i + 1], idx[2] = L.block_index[3 * i + 2];
    const bool out = idx[0] != kDeadSlotX && blockExteriorDistance(idx, block_size, c) > radius;
    const unsigned int ballot = __ballot_sync(0xffffffffu, out);
    int pos = 0;
    if (lane == 0 && ballot) pos = atomicAdd(dead_count, __popc(ballot));
    pos = __shfl_sync(0xffffffffu, pos, 0);
    if (out) dead[pos + __popc(ballot & ((1u << lane) - 1u))] = make_int4(i, idx[0], idx[1], idx[2]);
  }
}

__global__ void trackerDropDeadKernel(const int4* dead, const int* dead_count, const TrackerLists t) {
  const int n = *dead_count;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int slot = dead[i].x;
#pragma unroll
    for (const TrackerList& l : t.list)
      if (l.dirty) l.dirty[slot] = 0;
  }
}

// BoundingShape::touchesBlock (src/geometry/bounding_shape.cpp:48-66): sphere -> isBlockWithinRadius (exteriorDistance <
// radius); AABB -> AlignedBox::intersects(getAABBOfBlock) (bounding_boxes_impl.h:22-26), inclusive on both sides.
__device__ __forceinline__ bool shapeTouchesBlock(const NvbBoundingShape& s, const int idx[3], float block_size) {
  if (s.type == NVB_SHAPE_SPHERE) return blockExteriorDistance(idx, block_size, s.a) < s.b[0];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float bmin = (float)idx[k] * block_size, bmax = ((float)idx[k] + 1.0f) * block_size;
    if (!(s.a[k] <= bmax && bmin <= s.b[k])) return false;
  }
  return true;
}

// BoundingShape::contains: sphere (center - p).norm() <= radius (bounding_spheres.h:29-32; squaredNorm in Eigen's
// a0 + (a1 + a2) order); AABB AlignedBox::contains, inclusive.
__device__ __forceinline__ bool shapeContains(const NvbBoundingShape& s, const float p[3]) {
  if (s.type == NVB_SHAPE_SPHERE) {
    const float dx = s.a[0] - p[0], dy = s.a[1] - p[1], dz = s.a[2] - p[2];
    return sqrtf(sum3(dx * dx, dy * dy, dz * dz)) <= s.b[0];
  }
  return s.a[0] <= p[0] && s.a[1] <= p[1] && s.a[2] <= p[2] && p[0] <= s.b[0] && p[1] <= s.b[1] && p[2] <= s.b[2];
}

// BlockLayer::getBlockIndicesIf(any shape touches the block) (shape_clearer_impl.cuh:67-77), then addBlocksToUpdate of the
// touched blocks for every tracker consumer that is told (Mapper::clearTsdfInsideShapes, src/mapper/mapper.cpp:364-368).
__global__ void shapeSelectKernel(const __grid_constant__ ShapeClearArgs a) {
  const int n = *a.layer.count < a.layer.capacity ? *a.layer.count : a.layer.capacity;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int idx[3] = {a.layer.block_index[3 * i], a.layer.block_index[3 * i + 1], a.layer.block_index[3 * i + 2]};
    if (idx[0] == kDeadSlotX) continue;
    bool touched = false;
    for (int s = 0; s < a.num_shapes && !touched; s++) touched = shapeTouchesBlock(a.shapes[s], idx, a.block_size);
    if (!touched) continue;
    a.sel[atomicAdd(a.sel_count, 1)] = make_int4(i, idx[0], idx[1], idx[2]);
    trackerAdd(a.tracker, i);
  }
}

// clearShapesKernel (:38-59) with clearVoxel (:22-36): one CTA per selected block (grid-stride over the device count), one
// thread per voxel, the shape list in shared-memory tiles. Clearing is idempotent, so the tiles are independent passes.
__global__ void __launch_bounds__(kVpb) shapeClearKernel(const __grid_constant__ ShapeClearArgs a) {
  __shared__ NvbBoundingShape s_shapes[kShapeTile];
  const int tid = threadIdx.x;
  const int vidx[3] = {tid >> 6, (tid >> 3) & 7, tid & 7};  // linear voxel offset (x * 8 + y) * 8 + z
  const float voxel_size = a.block_size * (1.0f / kVps), half_voxel_size = a.block_size * (0.5f / kVps);
  const int n = *a.sel_count;
  for (int first = 0; first < a.num_shapes; first += kShapeTile) {
    const int tile = a.num_shapes - first < kShapeTile ? a.num_shapes - first : kShapeTile;
    __syncthreads();
    for (int s = tid; s < tile; s += blockDim.x) s_shapes[s] = a.shapes[first + s];
    __syncthreads();
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
      const int4 b = a.sel[i];
      const int bidx[3] = {b.y, b.z, b.w};
      float p[3];  // getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:51-81)
#pragma unroll
      for (int k = 0; k < 3; k++) p[k] = (a.block_size * (float)bidx[k] + voxel_size * (float)vidx[k]) + half_voxel_size;
      bool inside = false;
      for (int s = 0; s < tile && !inside; s++) inside = shapeContains(s_shapes[s], p);
      if (!inside) continue;
      unsigned char* blk = a.layer.blocks + (size_t)b.x * a.layer.block_bytes;
      if (a.voxel_kind == 0) {
        reinterpret_cast<float2*>(blk)[tid] = make_float2(0.0f, 0.0f);
      } else if (a.voxel_kind == 1) {
        reinterpret_cast<float*>(blk)[tid] = 0.0f;
      } else {  // Color::Gray() (core/color.h:59), weight 0; the pad byte is left alone
        unsigned char* v = blk + (size_t)tid * 8;
        v[0] = 127, v[1] = 127, v[2] = 127;
        *reinterpret_cast<float*>(v + 4) = 0.0f;
      }
    }
  }
}

}  // namespace

void launchSelectOutsideRadius(const DevLayer& layer, const float center[3], float radius, float block_size, int4* dead,
                               int* dead_count, cudaStream_t stream) {
  selectOutsideRadiusKernel<<<4 * kHelperCtas, 256, 0, stream>>>(layer, center[0], center[1], center[2], radius, block_size,
                                                                 dead, dead_count);
}

void launchTrackerDropDead(const int4* dead, const int* dead_count, int upper, const TrackerLists& t, cudaStream_t stream) {
  const int grid = upper < 1 ? 1 : (upper + 255) / 256 < kHelperCtas ? (upper + 255) / 256 : kHelperCtas;
  trackerDropDeadKernel<<<grid, 256, 0, stream>>>(dead, dead_count, t);
}

void launchShapeSelect(const ShapeClearArgs& a, cudaStream_t stream) {
  shapeSelectKernel<<<4 * kHelperCtas, 256, 0, stream>>>(a);
}

void launchShapeClear(const ShapeClearArgs& a, int num_sms, cudaStream_t stream) {
  shapeClearKernel<<<4 * num_sms, kVpb, 0, stream>>>(a);
}

}  // namespace nvb
