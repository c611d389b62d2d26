// nvb_view.cu -- which VoxelBlocks does a depth frame touch?
//
// Replaces ViewCalculator::getBlocksInImageViewRaycast
// (nvblox/include/nvblox/integrators/internal/cuda/impl/view_calculator_impl.cuh:62-233,
//  nvblox/src/integrators/view_calculator.cu:157-195) with a device-only chain:
//   viewRaycastKernel      one thread per subsampled pixel, Amanatides-Woo walk over
//                          the block grid, marks a BITSET (1 bit per AABB cell; the
//                          reference marks one byte per cell and copies it to the host)
//   compactAllocateKernel  ordered (x-fastest) compaction of the bitset into the frame's
//                          block list with warp ballots/popc + a chained tile scan, fused
//                          with allocate-if-absent in the TSDF layer's device hash and the
//                          ESDF "blocks to update" tracker. The reference does this part on
//                          the host (D2H copy, sync, host loop, unordered_map inserts).
// Nothing returns to the host; the list and its count stay in HBM for the TSDF kernel.
#include "nvb_internal.cuh"

namespace nvb {

namespace {

__device__ __forceinline__ int signum(float x) { return (x > 0.0f) ? 1 : ((x < 0.0f) ? -1 : 0); }

// setIndexUpdated (view_calculator_impl.cuh:46-56): the linear index is computed in
// int arithmetic and only guarded by lin < linear_size (negative values fail the
// guard; out-of-AABB cells whose linear index lands in range alias, as in the reference).
// The bitset lives in shared memory when it fits (kSmem): a CTA of 16x8 neighbouring rays
// crosses mostly the same cells, so the marks are shared-memory atomics and each CTA
// merges only its non-zero words into the global bitset at the end.
template <bool kSmem>
__device__ __forceinline__ void markCell(int x, int y, int z, const ViewGrid& g, unsigned int* bits) {
  const unsigned int sx = (unsigned int)x - (unsigned int)g.min_index.x;
  const unsigned int sy = (unsigned int)y - (unsigned int)g.min_index.y;
  const unsigned int sz = (unsigned int)z - (unsigned int)g.min_index.z;
  const unsigned int lin = sx + sy * (unsigned int)g.size.x + sz * (unsigned int)g.size.x * (unsigned int)g.size.y;
  if ((int)lin >= 0 && lin < (unsigned int)g.linear_size) {
    const unsigned int bit = 1u << (lin & 31);
    unsigned int* w = bits + (lin >> 5);
    // Many rays cross the same cells: test first (a stale read only costs an extra atomic).
    if (!(*(volatile unsigned int*)w & bit)) atomicOr(w, bit);
  }
}

constexpr int kRayTileCols = 16, kRayTileRows = 8;  // rays per CTA
constexpr int kMaxSmemWords = 12288;                 // 48 KiB of bitset (393 216 cells)

// combinedBlockIndicesInImageKernel (view_calculator_impl.cuh:62-115) + RayCaster
// (rays/internal/impl/ray_caster_impl.h:26-72).
template <bool kSmem>
__global__ void __launch_bounds__(kRayTileCols* kRayTileRows)
    viewRaycastKernel(const float* __restrict__ depth, int rows, int cols, Rigid T_L_C, NvbCamera cam,
                      float block_size, float trunc_m, float max_dist, int f, int ray_rows, int ray_cols,
                      int tiles_x, ViewGrid g, unsigned int* gbits) {
  extern __shared__ unsigned int s_bits[];
  unsigned int* bits = kSmem ? s_bits : gbits;
  const int tid = threadIdx.x;
  if (kSmem) {
    for (int w = tid; w < g.num_words; w += blockDim.x) s_bits[w] = 0;
    __syncthreads();
  }
  const int tile_y = blockIdx.x / tiles_x, tile_x = blockIdx.x - tile_y * tiles_x;
  const int rr = tile_y * kRayTileRows + tid / kRayTileCols;
  const int rc = tile_x * kRayTileCols + tid % kRayTileCols;
  bool active = rr < ray_rows && rc < ray_cols;
  float d = 0.0f;
  int pixel_row = 0, pixel_col = 0;
  if (active) {
    pixel_row = rr * f, pixel_col = rc * f;
    if (pixel_row >= rows) pixel_row = rows - 1;  // overhanging rays are pulled back to the border
    if (pixel_col >= cols) pixel_col = cols - 1;
    d = __ldg(depth + (size_t)pixel_row * cols + pixel_col);
    if (d <= 0.0f) active = false;  // NaN passes this test, exactly like the reference
  }
  if (active) {
    if (max_dist > 0.0f && d > max_dist) d = max_dist;
    // Camera::vectorFromPixelIndices (sensors/internal/impl/camera_impl.h:89-112)
    float vx = (((float)pixel_col + 0.5f) - cam.cu) / cam.fu;
    float vy = (((float)pixel_row + 0.5f) - cam.cv) / cam.fv;
    if (cam.has_distortion) removeDistortion(cam, vx, vy);
    const float s = d + trunc_m;
    Vec3 p_C = {s * vx, s * vy, s * 1.0f};
    const Vec3 p_L = transformPoint(T_L_C, p_C);

    const int3 b = blockIndexFromPosition(block_size, p_L);
    markCell<kSmem>(b.x, b.y, b.z, g, bits);

    // RayCaster(T_L_C.translation() / block_size, p_L / block_size), scale 1.
    const float o[3] = {T_L_C.t[0] / block_size, T_L_C.t[1] / block_size, T_L_C.t[2] / block_size};
    const float e[3] = {p_L.x / block_size, p_L.y / block_size, p_L.z / block_size};
    int cur[3], sgn[3];
    float t_next[3], t_step[3];
    unsigned int length = 0;
#pragma unroll
    for (int i = 0; i < 3; i++) {
      cur[i] = floatToIntRz(floorf(o[i] / 1.0f));
      const int end = floatToIntRz(floorf(e[i] / 1.0f));
      const int diff = (int)((unsigned int)end - (unsigned int)cur[i]);
      length += (diff < 0) ? (0u - (unsigned int)diff) : (unsigned int)diff;
      const float ray_i = e[i] - o[i];
      sgn[i] = signum(ray_i);
      const int corrected = sgn[i] > 0 ? sgn[i] : 0;
      const float shifted = o[i] - (float)cur[i];
      t_next[i] = ((float)corrected - shifted) / ray_i;  // NaN / inf allowed
      t_step[i] = (float)sgn[i] / ray_i;
    }
    // nextRayIndex returns length+1 cells.
    for (int step = 0; step <= (int)length; step++) {
      markCell<kSmem>(cur[0], cur[1], cur[2], g, bits);
      // Eigen minCoeff: start at element 0, replace on strict '<'.
      float best = t_next[0];
      int k = 0;
      if (t_next[1] < best) best = t_next[1], k = 1;
      if (t_next[2] < best) k = 2;
      if (k == 0) {
        cur[0] = (int)((unsigned int)cur[0] + (unsigned int)sgn[0]);
        t_next[0] = t_next[0] + t_step[0];
      } else if (k == 1) {
        cur[1] = (int)((unsigned int)cur[1] + (unsigned int)sgn[1]);
        t_next[1] = t_next[1] + t_step[1];
      } else {
        cur[2] = (int)((unsigned int)cur[2] + (unsigned int)sgn[2]);
        t_next[2] = t_next[2] + t_step[2];
      }
    }
  }
  if (kSmem) {
    __syncthreads();
    for (int w = tid; w < g.num_words; w += blockDim.x) {
      const unsigned int v = s_bits[w];
      if (v && (*(volatile unsigned int*)(gbits + w) & v) != v) atomicOr(gbits + w, v);
    }
  }
}

constexpr int kCompactThreads = 256;
constexpr int kTileWords = 64;                       // 2048 cells per tile
constexpr int kTileCells = kTileWords * 32;
constexpr int kChainedThresholdWords = 1 << 16;      // above this the redundant prefix would be quadratic

// Ordered compaction + allocation. The emitted list is in ascending linear-index order =
// the order convertAabbUpdatedToVector produces (view_calculator.cu:185-195): x fastest,
// then y, then z.
//   * A tile is 64 bitset words. Its output offset is the popcount of ALL preceding words,
//     which every tile recomputes for itself (the whole bitset is a few KB in L2), so tiles
//     are independent: no chained scan, no tickets, and the hash work of all tiles overlaps.
//     (Bitsets beyond 2^16 words fall back to a ticketed chained scan.)
//   * Inside a tile the set bits are dealt round-robin to the 256 threads (binary search over
//     the popcount scan + find-n-th-set-bit): the dependent hash probes run in parallel.
//   * Entries are staged in shared memory and written out coalesced.
// The bitset is NOT cleared here (other tiles still read it); the TSDF kernel that follows
// zeroes it for the next frame.
__global__ void __launch_bounds__(kCompactThreads) compactAllocateKernel(CompactArgs a) {
  __shared__ int s_incl[kTileWords];
  __shared__ unsigned int s_word[kTileWords];
  __shared__ int s_red[kCompactThreads / 32];
  __shared__ int s_prefix;
  __shared__ unsigned int s_tile;
  __shared__ int4 s_out[kTileCells];
  const int tid = threadIdx.x;
  const bool chained = a.grid.num_words > kChainedThresholdWords;
  unsigned int tile = blockIdx.x;
  if (chained) {
    if (tid == 0) s_tile = atomicAdd(a.ticket, 1u) - a.ticket_base;
    __syncthreads();
    tile = s_tile;
  }
  const int num_tiles = (a.grid.num_words + kTileWords - 1) / kTileWords;
  const int w0 = (int)tile * kTileWords;

  // popcount scan of this tile's words (2 warps)
  unsigned int word = 0;
  if (tid < kTileWords && w0 + tid < a.grid.num_words) word = a.bits[w0 + tid];
  if (tid < kTileWords) {
    s_word[tid] = word;
    int incl = __popc(word);
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, incl, off);
      if ((tid & 31) >= off) incl += n;
    }
    s_incl[tid] = incl;
  }
  // offset of the tile = popcount of every preceding word
  int part = 0;
  if (!chained)
    for (int w = tid; w < w0; w += kCompactThreads) part += __popc(a.bits[w]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) part += __shfl_down_sync(0xffffffffu, part, off);
  if ((tid & 31) == 0) s_red[tid >> 5] = part;
  __syncthreads();
  if (tid >= 32 && tid < kTileWords) s_incl[tid] += s_incl[31];  // second warp continues the first
  __syncthreads();
  const int total = s_incl[kTileWords - 1];
  if (tid == 0) {
    int prefix = 0;
    if (!chained) {
      for (int q = 0; q < kCompactThreads / 32; q++) prefix += s_red[q];
    } else if (tile > 0) {
      volatile unsigned long long* prev = a.tile_state + (tile - 1);
      unsigned long long st;
      do {
        st = *prev;
      } while ((unsigned int)(st >> 32) != a.epoch);
      prefix = (int)(unsigned int)st;
    }
    if (chained) {
      __threadfence();
      atomicExch(a.tile_state + tile, ((unsigned long long)a.epoch << 32) | (unsigned int)(prefix + total));
    }
    if ((int)tile == num_tiles - 1) *a.frame_count = prefix + total;
    s_prefix = prefix;
  }
  const int sx = a.grid.size.x, sxy = a.grid.size.x * a.grid.size.y;
  for (int j = tid; j < total; j += kCompactThreads) {
    // first word whose inclusive count exceeds j
    int lo = 0, hi = kTileWords - 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (s_incl[mid] > j) hi = mid;
      else lo = mid + 1;
    }
    const unsigned int wv = s_word[lo];
    const int rank = j - (s_incl[lo] - __popc(wv));  // 0-based rank of the bit inside the word
    const int bit = (int)__fns(wv, 0, rank + 1);     // position of the (rank+1)-th set bit
    const int lin = (w0 + lo) * 32 + bit;
    // aabbLinearIndexToLayerIndex (view_calculator_impl.cuh:38-44)
    const int x = lin % sx + a.grid.min_index.x;
    const int y = (lin / sx) % a.grid.size.y + a.grid.min_index.y;
    const int z = lin / sxy + a.grid.min_index.z;
    int slot = -1;
    if (a.allocate) {
      bool was_new;
      slot = hashFindOrInsert(a.layer, x, y, z, a.error, &was_new);
      if (slot >= 0) trackerAdd(a.tracker, slot);
    }
    s_out[j] = make_int4(x, y, z, slot);
  }
  __syncthreads();
  const int prefix = s_prefix;
  for (int j = tid; j < total; j += kCompactThreads) a.frame_blocks[prefix + j] = s_out[j];
}

// Union of block-index lists (multi-GPU merge): every valid entry marks its cell of the union AABB.
__global__ void markListKernel(const int* __restrict__ xyz, int n, ViewGrid g, unsigned int* bits) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
  if (x == INT32_MIN) return;  // padding entry
  const int sx = x - g.min_index.x, sy = y - g.min_index.y, sz = z - g.min_index.z;
  if (sx < 0 || sy < 0 || sz < 0 || sx >= g.size.x || sy >= g.size.y || sz >= g.size.z) return;
  const int lin = sx + sy * g.size.x + sz * g.size.x * g.size.y;
  atomicOr(bits + (lin >> 5), 1u << (lin & 31));
}
__global__ void unpackListKernel(const int4* __restrict__ in, const int* __restrict__ count, int* out, int cap) {
  const int n = *count < cap ? *count : cap;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int4 v = in[i];
    out[3 * i] = v.x, out[3 * i + 1] = v.y, out[3 * i + 2] = v.z;
  }
}

__global__ void clearWordsKernel(unsigned int* bits, int n) {
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n; w += gridDim.x * blockDim.x) bits[w] = 0;
}

}  // namespace

int compactNumTiles(const ViewGrid& grid) {
  const int t = (grid.num_words + kTileWords - 1) / kTileWords;
  return t < 1 ? 1 : t;
}

void launchMarkList(const int* xyz_dev, int n, const ViewGrid& grid, unsigned int* bits, cudaStream_t stream) {
  if (n > 0) markListKernel<<<(n + 255) / 256, 256, 0, stream>>>(xyz_dev, n, grid, bits);
}
void launchUnpackList(const int4* in, const int* count, int* out, int cap, cudaStream_t stream) {
  unpackListKernel<<<kHelperCtas, 256, 0, stream>>>(in, count, out, cap);
}

bool compactUsesTickets(const ViewGrid& grid) { return grid.num_words > kChainedThresholdWords; }

void launchClearBits(unsigned int* bits, int num_words, cudaStream_t stream) {
  if (num_words > 0)
    clearWordsKernel<<<(num_words + 1023) / 1024 < kHelperCtas ? (num_words + 1023) / 1024 : kHelperCtas, 1024, 0, stream>>>(bits, num_words);
}

void launchViewRaycast(const float* depth, int rows, int cols, const Rigid& T_L_C, const NvbCamera& cam,
                       float block_size, float trunc_m, float max_dist, int f, const ViewGrid& grid,
                       unsigned int* bits, cudaStream_t stream) {
  // Launch shape of getBlocksByRaycastingPixelsAsync (view_calculator_impl.cuh:200-233):
  // ceil((dim + 1) / f) rays rounded up to 16-thread tiles, then the in-kernel guard
  // pixel < dim + f - 1 decides which of those threads cast a ray.
  const int rows_s = (int)ceilf((float)(rows + 1) / (float)f);
  const int cols_s = (int)ceilf((float)(cols + 1) / (float)f);
  const int thr_rows = ((rows_s + 15) / 16) * 16;
  const int thr_cols = ((cols_s + 15) / 16) * 16;
  int ray_rows = (rows + f - 2) / f + 1;
  int ray_cols = (cols + f - 2) / f + 1;
  if (ray_rows > thr_rows) ray_rows = thr_rows;
  if (ray_cols > thr_cols) ray_cols = thr_cols;
  if (ray_rows <= 0 || ray_cols <= 0) return;
  const int tiles_x = (ray_cols + kRayTileCols - 1) / kRayTileCols;
  const int tiles_y = (ray_rows + kRayTileRows - 1) / kRayTileRows;
  const int threads = kRayTileCols * kRayTileRows;
  if (grid.num_words <= kMaxSmemWords) {
    viewRaycastKernel<true><<<tiles_x * tiles_y, threads, (size_t)grid.num_words * sizeof(unsigned int), stream>>>(
        depth, rows, cols, T_L_C, cam, block_size, trunc_m, max_dist, f, ray_rows, ray_cols, tiles_x, grid, bits);
  } else {
    viewRaycastKernel<false><<<tiles_x * tiles_y, threads, 0, stream>>>(
        depth, rows, cols, T_L_C, cam, block_size, trunc_m, max_dist, f, ray_rows, ray_cols, tiles_x, grid, bits);
  }
}

void launchCompactAllocate(const CompactArgs& args, cudaStream_t stream) {
  compactAllocateKernel<<<compactNumTiles(args.grid), kCompactThreads, 0, stream>>>(args);
}

}  // namespace nvb
