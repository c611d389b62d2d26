// nvb_masker.cu -- ImageMasker (semantics/image_masker.h, src/semantics/image_masker.cu): split a depth frame by a mask
// seen from another camera, with occlusion, and split a colour image by a mask lying on top of it. One thread per pixel.
//   * fill: the mask-sized min-depth image <- FLT_MAX (initializeImageKernel);
//   * min depth: every depth pixel is unprojected, moved into the mask camera by T_CM_CD and projected; its z is
//     min-reduced into the 5 x 5 patch around the projection (getMinimumDepthKernel<5>). The patch column is
//     (int)((u + patch_col) - 2.0f), truncated toward zero, so at the left and top edges the patch is asymmetric;
//   * split: a depth pixel goes to the masked output when it projects, the mask is set at (int)(u, v) and it is not
//     occluded (min_depth + occlusion_threshold_m < z); every other pixel goes to the unmasked output
//     (splitDepthImageKernel);
//   * colour: splitColorImageKernel.
// Two deviations where the reference reads out of bounds or is undefined:
//   * a projection with u == width or v == height passes Camera::project's viewport test, and the reference then reads
//     column `width` or row `height` of the mask; here such a pixel is a miss and goes to the unmasked output;
//   * the overlay's grey level converts a negative double to uint8_t for a negative depth (undefined in C++); here it is 0.
//     NaN and +inf give 255, as fmin does in the reference.
#include <cfloat>

#include "nvb_internal.cuh"

namespace nvb {

namespace {

constexpr int kMaskerThreads = 256;
constexpr int kPatchSize = 5;

__host__ __device__ __forceinline__ int numCtas(long long n) { return (int)((n + kMaskerThreads - 1) / kMaskerThreads); }

// unprojectFromPixelIndices (sensors/internal/impl/camera_impl.h:84-113), T_CM_CD * p_CD and Camera::project
// (camera_impl.h:37-76) into the mask camera. Returns false when the projection fails.
__device__ __forceinline__ bool projectIntoMask(const MaskerArgs& a, int r, int c, float depth, float& z, float& u, float& v) {
  float x = ((float)c + 0.5f - a.depth_cam.cu) / a.depth_cam.fu;
  float y = ((float)r + 0.5f - a.depth_cam.cv) / a.depth_cam.fv;
  if (a.depth_cam.has_distortion) removeDistortion(a.depth_cam, x, y);
  Vec3 p_CD;
  p_CD.x = depth * x, p_CD.y = depth * y, p_CD.z = depth * 1.0f;
  const Vec3 p = transformPoint(a.T_CM_CD, p_CD);
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return false;
  if (!(p.z >= 1e-6f)) return false;
  float un = p.x / p.z, vn = p.y / p.z;
  if (a.mask_cam.has_distortion) applyDistortion(a.mask_cam, un, vn);
  u = un * a.mask_cam.fu + a.mask_cam.cu;
  v = vn * a.mask_cam.fv + a.mask_cam.cv;
  if (u > (float)a.mask_cam.width || v > (float)a.mask_cam.height || u < 0.0f || v < 0.0f) return false;
  z = p.z;
  return true;
}

__global__ void __launch_bounds__(kMaskerThreads) maskerFillKernel(float* img, long long n) {
  for (long long k = (long long)blockIdx.x * kMaskerThreads + threadIdx.x; k < n; k += (long long)gridDim.x * kMaskerThreads)
    img[k] = FLT_MAX;
}

__global__ void __launch_bounds__(kMaskerThreads) maskerMinDepthKernel(MaskerArgs a) {
  const int pix = blockIdx.x * kMaskerThreads + threadIdx.x;
  if (pix >= a.rows * a.cols) return;
  const int r = pix / a.cols, c = pix - r * a.cols;
  float z, u, v;
  if (!projectIntoMask(a, r, c, a.depth[pix], z, u, v)) return;
  // z >= 1e-6 > 0: the minimum of positive floats is the minimum of their bit patterns as ints. Values only decrease, so
  // a plain read that already holds <= z makes the atomic a no-op.
  const int zi = __float_as_int(z);
  for (int pr = 0; pr < kPatchSize; pr++) {
    const int row = floatToIntRz((v + (float)pr) - (float)(kPatchSize / 2));
    if (row < 0 || row >= a.mrows) continue;
    for (int pc = 0; pc < kPatchSize; pc++) {
      const int col = floatToIntRz((u + (float)pc) - (float)(kPatchSize / 2));
      if (col < 0 || col >= a.mcols) continue;
      int* cell = reinterpret_cast<int*>(a.min_depth + (size_t)row * a.mcols + col);
      if (*cell > zi) atomicMin(cell, zi);
    }
  }
}

// Grey level of the overlay: fmin(12.75f * depth, 255) converted to uint8_t; 0 for a negative value (see the header).
__device__ __forceinline__ unsigned char overlayGrey(float depth) {
  const float x = (255.0f / 20.0f) * depth;  // 255u / max_depth_display_m
  if (!(x <= 255.0f)) return 255;           // NaN, +inf and everything above 255
  return x > 0.0f ? (unsigned char)(unsigned int)x : 0;
}

__global__ void __launch_bounds__(kMaskerThreads) maskerSplitDepthKernel(MaskerArgs a) {
  const int pix = blockIdx.x * kMaskerThreads + threadIdx.x;
  if (pix >= a.rows * a.cols) return;
  const int r = pix / a.cols, c = pix - r * a.cols;
  const float depth = a.depth[pix];
  unsigned char grey = 0;
  if (a.overlay) grey = overlayGrey(depth);
  bool masked = false;
  float z, u, v;
  if (!isinf(depth) && projectIntoMask(a, r, c, depth, z, u, v)) {
    const int ui = floatToIntRz(u), vi = floatToIntRz(v);
    if (ui < a.mcols && vi < a.mrows) {
      const size_t m = (size_t)vi * a.mcols + ui;
      const bool occluded = a.min_depth[m] + a.occlusion_threshold_m < z;
      masked = a.mask[m] != 0 && !occluded;
    }
  }
  a.unmasked[pix] = masked ? a.unmasked_invalid : depth;
  a.masked[pix] = masked ? depth : a.masked_invalid;
  if (a.overlay) {
    unsigned char* ov = a.overlay + 3 * (size_t)pix;
    ov[0] = masked ? 255 : grey, ov[1] = grey, ov[2] = grey;
  }
}

__global__ void __launch_bounds__(kMaskerThreads) maskerSplitColorKernel(ColorSplitArgs a) {
  const long long pix = (long long)blockIdx.x * kMaskerThreads + threadIdx.x;
  if (pix >= a.pixels) return;
  const bool masked = a.mask[pix] != 0;
  const unsigned char* in = a.rgb + 3 * pix;
  const unsigned char r = in[0], g = in[1], b = in[2];
  unsigned char* keep = (masked ? a.masked : a.unmasked) + 3 * pix;
  unsigned char* drop = (masked ? a.unmasked : a.masked) + 3 * pix;
  keep[0] = r, keep[1] = g, keep[2] = b;
  drop[0] = 0, drop[1] = 0, drop[2] = 0;  // Color(0, 0, 0): the reference has no setter for the colour invalid pixel
  if (a.overlay) {
    unsigned char* ov = a.overlay + 3 * pix;
    ov[0] = masked ? 255 : r, ov[1] = g, ov[2] = b;
  }
}

}  // namespace

void launchSplitDepth(const MaskerArgs& a, int num_sms, cudaStream_t stream) {
  const long long mask_pixels = (long long)a.mrows * a.mcols;
  maskerFillKernel<<<std::min<long long>(numCtas(mask_pixels), 8ll * num_sms), kMaskerThreads, 0, stream>>>(a.min_depth,
                                                                                                         mask_pixels);
  const int ctas = numCtas((long long)a.rows * a.cols);
  maskerMinDepthKernel<<<ctas, kMaskerThreads, 0, stream>>>(a);
  maskerSplitDepthKernel<<<ctas, kMaskerThreads, 0, stream>>>(a);
}

void launchSplitColor(const ColorSplitArgs& a, cudaStream_t stream) {
  maskerSplitColorKernel<<<numCtas(a.pixels), kMaskerThreads, 0, stream>>>(a);
}

}  // namespace nvb
