// nvb_util.cu -- small service kernels of the layer storage (gather / scatter of
// blocks for host access, hash maintenance, ESDF "blocks to update" tracker).
//
// These back the BlockLayer queries the reference answers from its host-side
// unordered_map (nvblox/include/nvblox/map/layer.h:76-217): here the map lives in
// HBM, so host access is an explicit gather.
#include "nvb_esdf_block.cuh"

namespace nvb {

namespace {

// ESDF blocks (`esdf`) leave in the reference's 20-byte voxel records and come back from them (nvb_esdf_block.cuh).
__global__ void gatherBlocksKernel(DevLayer L, bool esdf, const int* xyz, int n, unsigned char* out, unsigned char* found) {
  const int i = blockIdx.x;
  if (i >= n) return;
  __shared__ int s_slot;
  if (threadIdx.x == 0) {
    s_slot = hashFind(L.hash, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    found[i] = s_slot >= 0 ? 1 : 0;
  }
  __syncthreads();
  const int slot = s_slot;
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)i * L.block_bytes);
  const int nvec = L.block_bytes / 16;
  if (slot >= 0 && esdf) {
    const unsigned int* src = reinterpret_cast<const unsigned int*>(L.blocks + (size_t)slot * L.block_bytes);
    unsigned int* rec = reinterpret_cast<unsigned int*>(dst);
    for (int v = threadIdx.x; v < kVpb; v += blockDim.x) esdfVoxelToRecord(src, v, rec + kEsdfRecordWords * v);
  } else if (slot >= 0) {
    const uint4* src = reinterpret_cast<const uint4*>(L.blocks + (size_t)slot * L.block_bytes);
    for (int k = threadIdx.x; k < nvec; k += blockDim.x) dst[k] = src[k];
  } else {
    for (int k = threadIdx.x; k < nvec; k += blockDim.x) dst[k] = make_uint4(0, 0, 0, 0);
  }
}

__global__ void scatterBlocksKernel(DevLayer L, bool esdf, const int* xyz, int n, const unsigned char* in, int* error) {
  const int i = blockIdx.x;
  if (i >= n) return;
  __shared__ int s_slot;
  if (threadIdx.x == 0) {
    bool was_new;
    s_slot = hashFindOrInsert(L, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], error, &was_new);
  }
  __syncthreads();
  const int slot = s_slot;
  if (slot < 0) return;
  if (esdf) {
    const unsigned int* rec = reinterpret_cast<const unsigned int*>(in + (size_t)i * L.block_bytes);
    unsigned int* dst = reinterpret_cast<unsigned int*>(L.blocks + (size_t)slot * L.block_bytes);
    for (int v = threadIdx.x; v < kVpb; v += blockDim.x) esdfVoxelFromRecord(rec + kEsdfRecordWords * v, dst, v);
    return;
  }
  const uint4* src = reinterpret_cast<const uint4*>(in + (size_t)i * L.block_bytes);
  uint4* dst = reinterpret_cast<uint4*>(L.blocks + (size_t)slot * L.block_bytes);
  const int nvec = L.block_bytes / 16;
  for (int k = threadIdx.x; k < nvec; k += blockDim.x) dst[k] = src[k];
}

// DepthPreprocessor::dilateInvalidRegionsAsync (src/sensors/depth_preprocessing.cpp): mask = depth < threshold, N x 3x3
// dilations with a replicated border, masked pixels set to the invalid value. N 3x3 dilations with replicated borders
// are one (2N+1)^2 maximum over clamped coordinates, and a clamped coordinate never leaves the window, so the out-of-
// image taps can simply be dropped. Separable in shared memory: rows first, then columns; one pass over the image.
constexpr int kDilateTileW = 32, kDilateTileH = 8;
__global__ void dilateInvalidKernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols, int n,
                                    float threshold, float invalid_value) {
  extern __shared__ unsigned char s_flags[];
  const int tw = kDilateTileW + 2 * n, th = kDilateTileH + 2 * n;
  unsigned char* s_in = s_flags;             // th x tw : depth < threshold
  unsigned char* s_row = s_flags + tw * th;  // th x kDilateTileW : OR over the row window
  const int x0 = blockIdx.x * kDilateTileW - n, y0 = blockIdx.y * kDilateTileH - n;
  const int tid = threadIdx.y * kDilateTileW + threadIdx.x, nthreads = kDilateTileW * kDilateTileH;
  for (int i = tid; i < tw * th; i += nthreads) {
    const int x = x0 + i % tw, y = y0 + i / tw;
    unsigned char f = 0;
    if (x >= 0 && x < cols && y >= 0 && y < rows) f = in[(size_t)y * cols + x] < threshold ? 1 : 0;  // NaN compares false
    s_in[i] = f;
  }
  __syncthreads();
  for (int i = tid; i < kDilateTileW * th; i += nthreads) {
    const int x = i % kDilateTileW, y = i / kDilateTileW;
    unsigned char f = 0;
    for (int k = 0; k <= 2 * n; k++) f |= s_in[y * tw + x + k];
    s_row[i] = f;
  }
  __syncthreads();
  const int x = blockIdx.x * kDilateTileW + threadIdx.x, y = blockIdx.y * kDilateTileH + threadIdx.y;
  if (x >= cols || y >= rows) return;
  unsigned char f = 0;
  for (int k = 0; k <= 2 * n; k++) f |= s_row[(threadIdx.y + k) * kDilateTileW + threadIdx.x];
  out[(size_t)y * cols + x] = f ? invalid_value : in[(size_t)y * cols + x];
}

__global__ void fillU64Kernel(unsigned long long* p, unsigned long long v, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

// Re-insert every live slot into a freshly emptied hash (after a capacity change).
__global__ void rehashKernel(DevLayer L, int count) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= count) return;
  if (L.block_index[3 * slot] == kDeadSlotX) return;  // deallocated slot
  const unsigned long long key = packIndex(L.block_index[3 * slot], L.block_index[3 * slot + 1],
                                           L.block_index[3 * slot + 2]);
  unsigned int p = hashKey(key) & L.hash.mask;
  while (true) {
    const unsigned long long old = atomicCAS(&L.hash.keys[p], kEmptyKey, key);
    if (old == kEmptyKey) {
      L.hash.vals[p] = slot;
      return;
    }
    p = (p + 1) & L.hash.mask;
  }
}

// BlocksToUpdateState::setUpdateAllBlocks (map/blocks_to_update_tracker.h): the todo
// list becomes every allocated TSDF slot. The kernel only appends: the caller zeroes *todo_count first, which drops the
// pending entries like setUpdateAllBlocks clears the pending set. Deallocated slots are skipped.
__global__ void todoAllKernel(DevLayer tsdf, int* dirty, int* todo_slots, int* todo_count) {
  const int n = *tsdf.count < tsdf.capacity ? *tsdf.count : tsdf.capacity;
  const int lane = threadIdx.x & 31;
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) - lane; base < n; base += gridDim.x * blockDim.x) {
    const int i = base + lane;
    const bool live = i < n && tsdf.block_index[3 * i] != kDeadSlotX;
    const unsigned int ballot = __ballot_sync(0xffffffffu, live);
    int pos = 0;
    if (lane == 0 && ballot) pos = atomicAdd(todo_count, __popc(ballot));
    pos = __shfl_sync(0xffffffffu, pos, 0);
    if (live) {
      todo_slots[pos + __popc(ballot & ((1u << lane) - 1u))] = i;
      dirty[i] = 1;
    }
  }
}

// Generic twin of a deallocation (Mapper::clearBlocksInLayers for a layer without side tables): zero the block,
// mark the slot dead, give it back. One CTA per dead block. The host rebuilds the hash afterwards.
__global__ void removeBlocksKernel(DevLayer L, const int4* dead, const int* dead_count) {
  __shared__ int s_slot;
  const int n = *dead_count;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int4 d = dead[i];
    if (threadIdx.x == 0) s_slot = hashFind(L.hash, d.y, d.z, d.w);
    __syncthreads();
    const int slot = s_slot;
    if (slot >= 0) {
      uint4* g = reinterpret_cast<uint4*>(L.blocks + (size_t)slot * L.block_bytes);
      for (int k = threadIdx.x; k < L.block_bytes / 16; k += blockDim.x) g[k] = make_uint4(0, 0, 0, 0);
      if (threadIdx.x == 0) {
        L.block_index[3 * slot] = kDeadSlotX;
        L.free_slots[atomicAdd(L.free_count, 1)] = slot;
      }
    }
    __syncthreads();
  }
}

// Drops the slots that are dead in L from a list of its slots, keeping the order of the others (the ESDF's persistent cleared
// list, the tracker's todo lists). In place, one CTA: a chunk is read completely before any of it is written, and the write
// position never passes the read position.
__global__ void __launch_bounds__(1024) dropDeadSlotsKernel(DevLayer L, int* list, int* count) {
  __shared__ int s_base, s_warp[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = *count;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int first = 0; first < n; first += blockDim.x) {
    const int i = first + tid;
    const int slot = i < n ? list[i] : -1;
    const bool keep = slot >= 0 && L.block_index[3 * slot] != kDeadSlotX;
    const unsigned int ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int before = s_base;
    for (int w = 0; w < warp; w++) before += s_warp[w];
    if (keep) list[before + __popc(ballot & ((1u << lane) - 1u))] = slot;
    __syncthreads();
    if (tid == 0) {
      int total = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); w++) total += s_warp[w];
      s_base += total;
    }
    __syncthreads();
  }
  if (tid == 0) *count = s_base;
}

// EsdfSlicer::getAabbOfLayerAtHeight (src/integrators/esdf_slicer.cu:112-135): extreme x / y block indices at height zb.
__global__ void sliceAabbKernel(DevLayer L, int zb, int* out4) {
  const int n = *L.count < L.capacity ? *L.count : L.capacity;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
    const int x = L.block_index[3 * s];
    if (x == kDeadSlotX || L.block_index[3 * s + 2] != zb) continue;
    const int y = L.block_index[3 * s + 1];
    atomicMin(out4 + 0, x), atomicMin(out4 + 1, y), atomicMax(out4 + 2, x), atomicMax(out4 + 3, y);
  }
}

// populateSliceFromLayerKernel (:25-67) + occupancyGridFromSliceImageKernel (:78-110), one thread per pixel.
__global__ void sliceImageKernel(DevLayer L, float block_size, float min_x, float min_y, float slice_height,
                                 float unobserved_value, int rows, int cols, float* image, signed char* grid) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y * blockDim.y + threadIdx.y;
  if (col >= cols || row >= rows) return;
  const float voxel_size = block_size / (float)kVps;
  const Vec3 p{min_x + voxel_size / 2.0f + voxel_size * (float)col, min_y + voxel_size / 2.0f + voxel_size * (float)row,
               slice_height};
  int3 b, v;
  blockAndVoxelIndexFromPosition(block_size, voxelSizeInv(block_size), p, b, v);
  float d = unobserved_value;
  const int slot = hashFind(L.hash, b.x, b.y, b.z);
  if (slot >= 0) {
    const unsigned int* blk = reinterpret_cast<const unsigned int*>(L.blocks + (size_t)slot * kEsdfBlockBytes);
    const int vi = (v.x * kVps + v.y) * kVps + v.z;
    const unsigned int fl = *esdfFlag(blk, vi);
    if ((fl & 0xff00u) != 0) {  // observed
      d = voxel_size * sqrtf(__uint_as_float(*esdfCell(blk, vi)));
      if ((fl & 0xffu) != 0) d = -d;  // is_inside
    }
  }
  const size_t pix = (size_t)row * cols + col;
  if (image) image[pix] = d;
  if (grid) {
    signed char g = (signed char)((d < 1e-2f) * 100);
    if (fabsf(d - unobserved_value) < 1e-2f) g = -1;
    grid[pix] = g;
  }
}

// voxelLayerToDenseVoxelGridInAABBAsync (nvblox map/internal/cuda/impl/layer_to_3d_grid_impl.cuh) with nvblox_ros's
// SignedDistanceFunctor (conversions/esdf_and_gradients_conversions.cu): one CTA per block overlapping the grid, one thread per
// voxel; a cell is the voxel's distance in metres (negative inside), `default_value` where the voxel is unobserved or its block
// is not allocated. Cells in z-fastest order over the grid (min_vox, dims), as Unified3DGrid stores them.
__global__ void __launch_bounds__(kVpb) esdfDenseGridKernel(DevLayer L, int3 min_block, int3 min_vox, int3 dims, float voxel_size,
                                                           float default_value, float* out) {
  __shared__ int s_slot;
  const int bx = min_block.x + (int)blockIdx.x, by = min_block.y + (int)blockIdx.y, bz = min_block.z + (int)blockIdx.z;
  if (threadIdx.x == 0) s_slot = hashFind(L.hash, bx, by, bz);
  __syncthreads();
  const int v = threadIdx.x;
  const int gx = bx * kVps + (v >> 6) - min_vox.x, gy = by * kVps + ((v >> 3) & 7) - min_vox.y, gz = bz * kVps + (v & 7) - min_vox.z;
  if (gx < 0 || gy < 0 || gz < 0 || gx >= dims.x || gy >= dims.y || gz >= dims.z) return;
  float d = default_value;
  if (s_slot >= 0) {
    const unsigned int* blk = reinterpret_cast<const unsigned int*>(L.blocks + (size_t)s_slot * kEsdfBlockBytes);
    const unsigned int fl = *esdfFlag(blk, v);
    if ((fl & 0xff00u) != 0) {  // observed
      d = sqrtf(__uint_as_float(*esdfCell(blk, v))) * voxel_size;
      if ((fl & 0xffu) != 0) d = -d;  // is_inside
    }
  }
  out[((size_t)gx * dims.y + gy) * dims.z + gz] = d;
}

}  // namespace

void launchEsdfDenseGrid(const DevLayer& esdf, int3 min_vox, int3 dims, float voxel_size, float default_value, float* out,
                         cudaStream_t stream) {
  // the blocks holding the grid's first and last voxel (floor division)
  const int3 lo = make_int3(min_vox.x >> 3, min_vox.y >> 3, min_vox.z >> 3);
  const int3 hi = make_int3((min_vox.x + dims.x - 1) >> 3, (min_vox.y + dims.y - 1) >> 3, (min_vox.z + dims.z - 1) >> 3);
  const dim3 grid(hi.x - lo.x + 1, hi.y - lo.y + 1, hi.z - lo.z + 1);
  esdfDenseGridKernel<<<grid, kVpb, 0, stream>>>(esdf, lo, min_vox, dims, voxel_size, default_value, out);
}

void launchSliceAabb(const DevLayer& esdf, int zb, int* out4, cudaStream_t stream) {
  sliceAabbKernel<<<296, 256, 0, stream>>>(esdf, zb, out4);
}
void launchSliceImage(const DevLayer& esdf, float block_size, float min_x, float min_y, float slice_height, float unobserved_value,
                      int rows, int cols, float* image, signed char* grid, cudaStream_t stream) {
  const dim3 threads(16, 16);
  const dim3 blocks((cols + 15) / 16, (rows + 15) / 16);
  sliceImageKernel<<<blocks, threads, 0, stream>>>(esdf, block_size, min_x, min_y, slice_height, unobserved_value, rows, cols,
                                                   image, grid);
}

void launchRemoveBlocks(const DevLayer& layer, const int4* dead, const int* dead_count, int upper, cudaStream_t stream) {
  int grid = upper < 1184 ? (upper < 1 ? 1 : upper) : 1184;
  removeBlocksKernel<<<grid, 256, 0, stream>>>(layer, dead, dead_count);
}

void launchDropDeadSlots(const DevLayer& layer, int* list, int* count, cudaStream_t stream) {
  dropDeadSlotsKernel<<<1, 1024, 0, stream>>>(layer, list, count);
}

void launchGatherBlocks(const DevLayer& layer, bool esdf, const int* xyz_dev, int n, unsigned char* out, unsigned char* found,
                        cudaStream_t stream) {
  if (n > 0) gatherBlocksKernel<<<n, 128, 0, stream>>>(layer, esdf, xyz_dev, n, out, found);
}
void launchScatterBlocks(const DevLayer& layer, bool esdf, const int* xyz_dev, int n, const unsigned char* in, int* error,
                         cudaStream_t stream) {
  if (n > 0) scatterBlocksKernel<<<n, 128, 0, stream>>>(layer, esdf, xyz_dev, n, in, error);
}
void launchDilateInvalid(const float* in, float* out, int rows, int cols, int num_dilations, float threshold,
                         float invalid_value, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return;
  const int tw = kDilateTileW + 2 * num_dilations, th = kDilateTileH + 2 * num_dilations;
  const size_t smem = (size_t)tw * th + (size_t)kDilateTileW * th;
  const dim3 grid((cols + kDilateTileW - 1) / kDilateTileW, (rows + kDilateTileH - 1) / kDilateTileH);
  dilateInvalidKernel<<<grid, dim3(kDilateTileW, kDilateTileH), smem, stream>>>(in, out, rows, cols, num_dilations, threshold,
                                                                            invalid_value);
}
void launchFillU64(unsigned long long* p, unsigned long long v, size_t n, cudaStream_t stream) {
  if (n > 0) fillU64Kernel<<<1184, 256, 0, stream>>>(p, v, n);
}
void launchRehash(const DevLayer& layer, int count, cudaStream_t stream) {
  if (count > 0) rehashKernel<<<(count + 255) / 256, 256, 0, stream>>>(layer, count);
}
void launchTodoAll(const DevLayer& tsdf, const TrackerList& t, cudaStream_t stream) {
  todoAllKernel<<<296, 256, 0, stream>>>(tsdf, t.dirty, t.slots, t.count);
}

}  // namespace nvb
