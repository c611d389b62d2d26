// nvb_dynamics.cu -- dynamics detection and the connected-component mask filter of the kDynamic MultiMapper:
//   * DynamicsDetection::computeDynamics (findDynamicPointsKernel, dynamics/internal/cuda/impl/dynamics_detection_impl.cuh:
//     26-87): a depth pixel is dynamic when its surface point falls into a high-confidence freespace voxel. Count -> scan ->
//     emit (the scan is nvb_ground.cu's), so that the points come out in row-major pixel order instead of the reference's
//     atomicAdd order, and their count stays on the device;
//   * MaskPreprocessor::removeSmallConnectedComponents (src/sensors/mask_preprocessor.cpp:140-183, image.cu:323-404): the
//     reference labels the 2x-downscaled mask with a BFS on the host; here it is a union-find on the GPU in four launches
//     whatever the mask holds: tile-local union-find in shared memory (fused with the downscale), a lock-free merge across
//     tile borders, flatten + component sizes, erase + upscale.
#include "nvb_internal.cuh"

namespace nvb {

namespace {

constexpr int kDetectThreads = 256;  // one tile of the compaction = 256 consecutive pixels (row-major)
constexpr int kTile = 32;            // label tile: 32 x 32 downscaled pixels, one CTA of 1024 threads
constexpr int kCcThreads = 256;

// ---------------------------------------------------------------------------------------------------------------------
// Detection
// ---------------------------------------------------------------------------------------------------------------------

// unprojectFromPixelIndices (sensors/internal/impl/camera_impl.h:84-113) and T_L_C * p_C.
__device__ __forceinline__ Vec3 pixelToLayer(const DynamicsArgs& a, int r, int c, float depth) {
  float u = ((float)c + 0.5f - a.cam.cu) / a.cam.fu;
  float v = ((float)r + 0.5f - a.cam.cv) / a.cam.fv;
  if (a.cam.has_distortion) removeDistortion(a.cam, u, v);
  Vec3 p_C;
  p_C.x = depth * u, p_C.y = depth * v, p_C.z = depth * 1.0f;
  return transformPoint(a.T_L_C, p_C);
}

// The pixel's mask and overlay; returns is_dynamic.
__device__ __forceinline__ bool detectPixel(const DynamicsArgs& a, int pix) {
  const int r = pix / a.cols, c = pix - r * a.cols;
  a.mask[pix] = 0;
  unsigned char* ov = a.overlay + 3 * (size_t)pix;
  ov[0] = 255, ov[1] = 255, ov[2] = 255;  // Color::White()
  const float depth = a.depth[pix];
  if (depth <= 0.0f) return false;  // NaN goes on, like the reference's
  const Vec3 p = pixelToLayer(a, r, c, depth);
  int3 b, vi;
  blockAndVoxelIndexFromPosition(a.block_size, a.voxel_size_inv, p, b, vi);
  const int slot = hashFind(a.fs.hash, b.x, b.y, b.z);
  if (slot < 0) return false;
  const int v = (vi.x * kVps + vi.y) * kVps + vi.z;
  const bool dyn = isVoxelFreespace(a.fs, slot, v);  // FreespaceVoxel::is_high_confidence_freespace
  // getOverlayColor (:26-34): red for dynamics, grey scaled by depth
  constexpr float kMaxDisplayDepthM = 10.f;
  constexpr float kDepthScaleFactor = 255.0f / kMaxDisplayDepthM;
  const unsigned char s = (unsigned char)(unsigned int)fminf(kDepthScaleFactor * depth, 255.0f);
  a.mask[pix] = dyn ? 255 : 0;  // is_dynamic * image::kMaskedValue
  ov[0] = dyn ? 255 : 0, ov[1] = s, ov[2] = s;
  return dyn;
}

__global__ void __launch_bounds__(kDetectThreads) dynamicsDetectKernel(DynamicsArgs a) {
  const int pix = blockIdx.x * kDetectThreads + threadIdx.x;
  const bool dyn = pix < a.rows * a.cols && detectPixel(a, pix);
  const int n = __syncthreads_count(dyn);
  if (threadIdx.x == 0) a.counts[blockIdx.x] = make_int2(n, 0);
}

// The dynamic pixels of each tile at the tile's offset, in pixel order; the mask tells which ones (no second lookup).
__global__ void __launch_bounds__(kDetectThreads) dynamicsEmitKernel(DynamicsArgs a) {
  __shared__ int s_warp[kDetectThreads / 32];
  const int pix = blockIdx.x * kDetectThreads + threadIdx.x;
  const bool dyn = pix < a.rows * a.cols && a.mask[pix] != 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned int bal = __ballot_sync(0xffffffffu, dyn);
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  if (!dyn) return;
  int rank = __popc(bal & ((1u << lane) - 1u));
  for (int w = 0; w < warp; w++) rank += s_warp[w];
  const int r = pix / a.cols, c = pix - r * a.cols;
  const Vec3 p = pixelToLayer(a, r, c, a.depth[pix]);
  float* out = a.points + 3 * (size_t)(a.counts[blockIdx.x].x + rank);
  out[0] = p.x, out[1] = p.y, out[2] = p.z;
}

// ---------------------------------------------------------------------------------------------------------------------
// Connected components (4-connected) of the downscaled mask: union-find with lock-free unions (link the larger root to
// the smaller with atomicMin, retry from the value found when another thread linked it first). Parents are always smaller
// indices than their children, so the trees have no cycles whatever the interleaving; a label only ever decreases, so a
// stale read is an older ancestor and the union's retry loop corrects it.
// ---------------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ int ufFind(const int* L, int i) {
  int p = *(volatile const int*)(L + i);
  while (p != i) {
    i = p;
    p = *(volatile const int*)(L + i);
  }
  return i;
}

__device__ __forceinline__ void ufUnion(int* L, int a, int b) {
  bool done;
  do {
    a = ufFind(L, a);
    b = ufFind(L, b);
    if (a < b) {
      const int old = atomicMin(L + b, a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(L + a, b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

// Pass 1: downscale (pixel (2r, 2c), naiveDownscaleKernel), threshold (> 0 is set), label the tile in shared memory, and
// write each set pixel's tile root as a global linear index (-1: not set). Zeroes the size counters.
__global__ void __launch_bounds__(kTile * kTile) ccLocalKernel(CcArgs a) {
  __shared__ int s_L[kTile * kTile];
  const int lx = threadIdx.x, ly = threadIdx.y, li = ly * kTile + lx;
  const int c = blockIdx.x * kTile + lx, r = blockIdx.y * kTile + ly;
  const bool in = r < a.drows && c < a.dcols;
  const bool set = in && a.in[(size_t)(2 * r) * a.cols + 2 * c] > 0;
  s_L[li] = set ? li : -1;
  __syncthreads();
  if (set && lx > 0 && s_L[li - 1] >= 0) ufUnion(s_L, li, li - 1);
  __syncthreads();
  if (set && ly > 0 && s_L[li - kTile] >= 0) ufUnion(s_L, li, li - kTile);
  __syncthreads();
  if (!in) return;
  const int i = r * a.dcols + c;
  a.sizes[i] = 0;
  if (set) {
    const int root = ufFind(s_L, li);
    a.labels[i] = (blockIdx.y * kTile + root / kTile) * a.dcols + blockIdx.x * kTile + root % kTile;
  } else {
    a.labels[i] = -1;
  }
}

// Pass 2: the pixels on a tile's left or top border join their neighbour across it.
__global__ void __launch_bounds__(kCcThreads) ccMergeKernel(CcArgs a) {
  const int i = blockIdx.x * kCcThreads + threadIdx.x;
  if (i >= a.drows * a.dcols) return;
  const int r = i / a.dcols, c = i - r * a.dcols;
  if ((c % kTile != 0 || c == 0) && (r % kTile != 0 || r == 0)) return;
  if (a.labels[i] < 0) return;
  if (c % kTile == 0 && c > 0 && a.labels[i - 1] >= 0) ufUnion(a.labels, i, i - 1);
  if (r % kTile == 0 && r > 0 && a.labels[i - a.dcols] >= 0) ufUnion(a.labels, i, i - a.dcols);
}

// Pass 3: every set pixel points at its root; sizes counted on the roots, one atomic per root and warp.
__global__ void __launch_bounds__(kCcThreads) ccCountKernel(CcArgs a) {
  const int i = blockIdx.x * kCcThreads + threadIdx.x;
  const bool set = i < a.drows * a.dcols && a.labels[i] >= 0;
  const unsigned int active = __ballot_sync(0xffffffffu, set);
  if (!set) return;
  const int root = ufFind(a.labels, i);
  a.labels[i] = root;
  const unsigned int peers = __match_any_sync(active, root);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(a.sizes + root, __popc(peers));
}

// Pass 4: erase the components smaller than min_size, upscale (upscaleKernel: pixel (r / 2, c / 2)); survivors hold 254,
// the reference's 255 with its visited bit 0x01 cleared. A trailing odd row / column has no source pixel and is 0.
__global__ void __launch_bounds__(kCcThreads) ccOutputKernel(CcArgs a) {
  const size_t n = (size_t)a.rows * a.cols;
  for (size_t k = (size_t)blockIdx.x * kCcThreads + threadIdx.x; k < n; k += (size_t)gridDim.x * kCcThreads) {
    const int r = (int)(k / a.cols), c = (int)(k - (size_t)r * a.cols);
    unsigned char v = 0;
    if ((r >> 1) < a.drows && (c >> 1) < a.dcols) {
      const int root = a.labels[(r >> 1) * a.dcols + (c >> 1)];
      if (root >= 0 && a.sizes[root] >= a.min_size) v = 254;
    }
    a.out[k] = v;
  }
}

}  // namespace

int dynamicsNumTiles(int pixels) { return (pixels + kDetectThreads - 1) / kDetectThreads; }

void launchDynamicsDetect(const DynamicsArgs& a, int* totals, cudaStream_t stream) {
  const int tiles = dynamicsNumTiles(a.rows * a.cols);
  dynamicsDetectKernel<<<tiles, kDetectThreads, 0, stream>>>(a);
  launchExclusiveScanInt2(a.counts, tiles, totals, stream);
  dynamicsEmitKernel<<<tiles, kDetectThreads, 0, stream>>>(a);
}

void launchRemoveSmallComponents(const CcArgs& a, int num_sms, cudaStream_t stream) {
  if (a.drows > 0 && a.dcols > 0) {
    const dim3 grid((a.dcols + kTile - 1) / kTile, (a.drows + kTile - 1) / kTile);
    ccLocalKernel<<<grid, dim3(kTile, kTile), 0, stream>>>(a);
    const int n = a.drows * a.dcols, ctas = (n + kCcThreads - 1) / kCcThreads;
    ccMergeKernel<<<ctas, kCcThreads, 0, stream>>>(a);
    ccCountKernel<<<ctas, kCcThreads, 0, stream>>>(a);
  }
  const long long n = (long long)a.rows * a.cols;
  const int ctas = (int)std::min<long long>((n + kCcThreads - 1) / kCcThreads, 8ll * num_sms);
  ccOutputKernel<<<ctas, kCcThreads, 0, stream>>>(a);
}

}  // namespace nvb
