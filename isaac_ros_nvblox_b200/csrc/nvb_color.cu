// nvb_color.cu -- colour integration: ProjectiveAppearanceIntegrator<ColorLayer>::integrateFrame
// (nvblox/src/integrators/projective_appearance_integrator.cu:68-165) with its SphereTracer
// (nvblox/src/rays/sphere_tracer.cu:31-173, 422-485), and the SphereTracer's depth and RGBD renders (:239-300), which share the
// tracer's ray and cast with the colour integrator.
//
// The reference enumerates every block of the view AABB on the host, projects the block centres on the host, looks
// the survivors up in the TSDF layer on the host, uploads their pointers, runs checkBlocksInTruncationBand, downloads
// the flags, filters on the host, allocates on the host and uploads pointers again. Here one kernel walks the TSDF
// slab: a warp per allocated block does the AABB-range test, the centre projection, the truncation-band scan,
// the colour-block allocation (device hash + Gray initialisation) and appends to the frame's work list; nothing
// returns to the host. The sphere tracer is a thread per ray over the device hash; the appearance update is the
// TSDF kernel's shape: a persistent grid, a 256-thread CTA per 4 KiB ColorBlock, two z-adjacent voxels (one 128-bit
// word) per thread, unchanged words not written back.
#include "nvb_internal.cuh"

#include <cuda_fp16.h>

namespace nvb {

namespace {

constexpr unsigned int kGrayVoxelWord = 0x007f7f7fu;  // ColorVoxel(): Color::Gray() + one padding byte (map/voxels.h:77-83)

// ---------------------------------------------------------------------------
// getBlocksInImageViewProjection (view_calculator_impl.h:29-78) + getVisibleBlocksByProjection<Camera>
// (src/integrators/view_calculator.cu:380-417) + reduceBlocksToThoseInTruncationBand (:378-481) +
// allocateBlocksWhereRequired, over the allocated TSDF blocks.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colorSelectKernel(const __grid_constant__ ColorArgs a) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n = min(*(volatile int*)a.tsdf.count, a.tsdf.capacity);
  for (int slot = warp; slot < n; slot += nwarps) {
    const int bx = a.tsdf.block_index[3 * slot], by = a.tsdf.block_index[3 * slot + 1], bz = a.tsdf.block_index[3 * slot + 2];
    if (bx == kDeadSlotX) continue;
    // getBlockIndicesTouchedByBoundingBox (geometry/internal/impl/bounding_boxes_impl.h:28-53)
    if (bx < a.aabb_lo.x || bx > a.aabb_hi.x || by < a.aabb_lo.y || by > a.aabb_hi.y || bz < a.aabb_lo.z || bz > a.aabb_hi.z)
      continue;
    // getCenterPositionFromBlockIndex (core/internal/impl/indexing_impl.h:65-69)
    const Vec3 c_L{a.block_size * ((float)bx + 0.5f), a.block_size * ((float)by + 0.5f), a.block_size * ((float)bz + 0.5f)};
    const Vec3 p = transformPoint(a.T_C_L, c_L);
    if (!(p.z > 1e-6f)) continue;
    if (!(p.z >= 1e-6f)) continue;  // projectToNormalizedCoordinates (camera_impl.h:65-75)
    const float un = p.x / p.z, vn = p.y / p.z;
    if (!(a.vmin_x <= un && a.vmin_y <= vn && un <= a.vmax_x && vn <= a.vmax_y)) continue;  // AlignedBox::contains
    // checkBlocksInTruncationBand (:378-392)
    const float2* blk = reinterpret_cast<const float2*>(a.tsdf.blocks + (size_t)slot * kTsdfBlockBytes);
    bool in_band = false;
#pragma unroll 4
    for (int k = 0; k < kVpb / 32; k++) {
      const float2 t = blk[lane + 32 * k];
      if (t.y > 0.0f && fabsf(t.x) < a.trunc_m) in_band = true;
    }
    if (!__any_sync(0xffffffffu, in_band)) continue;
    int cslot = -1;
    bool was_new = false;
    if (lane == 0) cslot = hashFindOrInsert(a.color, bx, by, bz, a.error, &was_new);
    cslot = __shfl_sync(0xffffffffu, cslot, 0);
    was_new = __shfl_sync(0xffffffffu, (int)was_new, 0) != 0;
    if (cslot < 0) continue;
    if (was_new) {
      uint2* cb = reinterpret_cast<uint2*>(a.color.blocks + (size_t)cslot * kColorBlockBytes);
#pragma unroll 4
      for (int k = 0; k < kVpb / 32; k++) cb[lane + 32 * k] = make_uint2(kGrayVoxelWord, 0u);
    }
    if (lane == 0) a.work[atomicAdd(a.work_count, 1)] = make_int4(bx, by, bz, cslot);
  }
}

// ---------------------------------------------------------------------------
// SphereTracer (src/rays/sphere_tracer.cu): the cast of one pixel's ray (pixelRay, nvb_internal.cuh), shared by the colour
// integrator's synthetic depth and the public render kernels.
// ---------------------------------------------------------------------------
// cast (:31-100): march from o along u by the TSDF distance of the voxel under the point. Returns whether the ray converged;
// t is then the refined distance along the ray.
__device__ __forceinline__ bool sphereTraceCast(const DevLayer& tsdf, float block_size, float voxel_size_inv, const float o[3],
                                                const Vec3& u, float trunc_m, int max_steps, float max_ray_len, float eps_m,
                                                float& t) {
  int first = 0;  // 0 not yet known, 1 positive, 2 negative
  t = 0.0f;
  bool ok = false, done = false;
  int last_bx = INT32_MIN, last_by = 0, last_bz = 0, last_slot = -1;
  for (int i = 0; (i < max_steps) && (t < max_ray_len) && !done; i++) {
    const float plx = o[0] + t * u.x, ply = o[1] + t * u.y, plz = o[2] + t * u.z;
    int3 bi, vi;
    blockAndVoxelIndexFromPosition(block_size, voxel_size_inv, Vec3{plx, ply, plz}, bi, vi);
    const int bx = bi.x, by = bi.y, bz = bi.z, vx = vi.x, vy = vi.y, vz = vi.z;
    // consecutive samples mostly stay in one block (a step is at most the truncation distance): remember its slot
    if (bx != last_bx || by != last_by || bz != last_bz) {
      last_slot = hashFind(tsdf.hash, bx, by, bz);
      last_bx = bx, last_by = by, last_bz = bz;
    }
    const int slot = last_slot;
    float dist = 0.0f, wgt = 0.0f;
    if (slot >= 0) {
      const float2 v = *reinterpret_cast<const float2*>(tsdf.blocks + (size_t)slot * kTsdfBlockBytes +
                                                       (size_t)((vx * kVps + vy) * kVps + vz) * 8);
      dist = v.x, wgt = v.y;
    }
    float step;
    if (slot < 0 || !(wgt > 1e-4f)) {  // isTsdfVoxelValid (:26-29)
      if (first == 0) {
        step = trunc_m;
      } else {
        done = true;
        continue;
      }
    } else {
      if (first == 0) first = (dist >= 0.0f) ? 1 : 2;
      if (first == 1) {
        if (dist < eps_m) {
          t += dist;
          ok = true, done = true;
          continue;
        }
        step = dist;
      } else {
        if (dist > -eps_m) {
          t -= dist;
          ok = true, done = true;
          continue;
        }
        step = -dist;
      }
    }
    t += step;
  }
  return ok;
}

// sphereTracingKernel (:134-173) for the colour integrator's occlusion test
template <bool kDistort>
__global__ void __launch_bounds__(128) sphereTraceKernel(const __grid_constant__ ColorArgs a) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y * blockDim.y + threadIdx.y;
  if (r >= a.drows || c >= a.dcols) return;
  float dz, t;
  Vec3 u;
  pixelRay<kDistort>(a.cam, a.T_L_C, a.subsample, r, c, dz, u);
  const bool ok = sphereTraceCast(a.tsdf, a.block_size, a.voxel_size_inv, a.T_L_C.t, u, a.trunc_m, a.max_steps, a.max_ray_len,
                                  a.eps_m, t);
  a.synth[(size_t)r * a.dcols + c] = ok ? t * dz : -1.0f;
}

// sphereTracingKernel / sphereTracingKernelWithColor (:134-173, 239-300): depth, and with kRgb the colour of the voxel that
// holds the hit point p_L = origin + t * u in the colour layer, whatever its weight. A miss, or a hit without a colour block,
// is -1 and black.
template <bool kDistort, bool kRgb>
__global__ void __launch_bounds__(128) renderKernel(const __grid_constant__ RenderArgs a) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y * blockDim.y + threadIdx.y;
  if (r >= a.drows || c >= a.dcols) return;
  float dz, t;
  Vec3 u;
  pixelRay<kDistort>(a.cam, a.T_L_C, a.subsample, r, c, dz, u);
  const bool ok = sphereTraceCast(a.tsdf, a.block_size, a.voxel_size_inv, a.T_L_C.t, u, a.trunc_m, a.max_steps, a.max_ray_len,
                                  a.eps_m, t);
  const size_t i = (size_t)r * a.dcols + c;
  a.depth[i] = ok ? t * dz : -1.0f;
  if (!kRgb) return;
  unsigned int rgb = 0u;
  if (ok && a.color.blocks != nullptr) {
    // Ray::pointAt, then getVoxelAtPosition (gpu_hash/internal/cuda/gpu_indexing.cuh) on the colour layer's hash
    const Rigid& T = a.T_L_C;
    int3 bi, vi;
    blockAndVoxelIndexFromPosition(a.block_size, a.voxel_size_inv, Vec3{T.t[0] + t * u.x, T.t[1] + t * u.y, T.t[2] + t * u.z},
                                   bi, vi);
    const int slot = hashFind(a.color.hash, bi.x, bi.y, bi.z);
    if (slot >= 0)
      rgb = *reinterpret_cast<const unsigned int*>(a.color.blocks + (size_t)slot * kColorBlockBytes +
                                                   (size_t)((vi.x * kVps + vi.y) * kVps + vi.z) * 8);
  }
  unsigned char* px = a.rgb + 3 * i;
  px[0] = (unsigned char)rgb, px[1] = (unsigned char)(rgb >> 8), px[2] = (unsigned char)(rgb >> 16);
}

// ---------------------------------------------------------------------------
// integrateBlocksKernel for appearance voxels (projective_integrator_impl.cuh:117-185) with
// UpdateAppearanceVoxelFunctor<ColorVoxel> (projective_appearance_integrator.cu:312-348)
// ---------------------------------------------------------------------------
// interpolatePixels<float> (interpolation/internal/impl/interpolation_2d_impl.h:26-36)
__device__ __forceinline__ float interpolatePixels(float x, float y, float f00, float f01, float f10, float f11) {
  const float dx = f10 - f00;
  return f00 + x * dx + y * (f01 - f00) + x * y * (f11 - f01 - dx);
}

// One ColorVoxel {rgb + pad, weight}. Returns true if the voxel changed.
template <bool kDistort>
__device__ __forceinline__ bool updateColorVoxel(const ColorArgs& a, const int4& blk, int vx, int vy, int vz, unsigned int& rgb,
                                                 float& wgt) {
  Vec3 p_L;
  p_L.x = (a.block_size * (float)blk.x + a.voxel_size * (float)vx) + a.half_voxel_size;
  p_L.y = (a.block_size * (float)blk.y + a.voxel_size * (float)vy) + a.half_voxel_size;
  p_L.z = (a.block_size * (float)blk.z + a.voxel_size * (float)vz) + a.half_voxel_size;
  const Vec3 p_C = transformPoint(a.T_C_L, p_L);
  // Camera::project (camera_impl.h:37-76) + projectThreadVoxel's max-depth test
  if (!(isfinite(p_C.x) && isfinite(p_C.y) && isfinite(p_C.z))) return false;
  if (!(p_C.z >= 1e-6f)) return false;
  float un = p_C.x / p_C.z, vn = p_C.y / p_C.z;
  if (kDistort) applyDistortion(a.cam, un, vn);
  const float u = un * a.cam.fu + a.cam.cu;
  const float v = vn * a.cam.fv + a.cam.cv;
  if (u > (float)a.cam.width || v > (float)a.cam.height || u < 0.0f || v < 0.0f) return false;
  const float voxel_depth = p_C.z;
  if (a.max_integration_distance_m > 0.0f && voxel_depth > a.max_integration_distance_m) return false;
  // occlusion test against the synthetic depth: interpolate2DClosest on the subsampled image
  const float ud = u / (float)a.depth_subsample, vd = v / (float)a.depth_subsample;
  const int dxi = floatToIntRz(floorf(ud)), dyi = floatToIntRz(floorf(vd));
  if (dxi < 0 || dyi < 0 || dxi >= a.dcols || dyi >= a.drows) return false;
  const float surface_depth = a.synth[(size_t)dyi * a.dcols + dxi];
  if (!(isfinite(surface_depth) && surface_depth > 1e-6f)) return false;  // PixelIsValidDepth
  if (fabsf(surface_depth - voxel_depth) > a.trunc_m) return false;
  // interpolate2DLinear<Color> (interpolation_2d_impl.h:152-199)
  const float ucx = u - 0.5f, ucy = v - 0.5f;
  const int lx = floatToIntRz(floorf(ucx)), ly = floatToIntRz(floorf(ucy));
  if (lx < 0 || ly < 0 || (lx + 1) > (a.cols - 1) || (ly + 1) > (a.rows - 1)) return false;
  const float ox = ucx - (float)lx, oy = ucy - (float)ly;
  const unsigned char* c00 = a.color_image + ((size_t)ly * a.cols + lx) * 3;
  const unsigned char* c01 = c00 + (size_t)a.cols * 3;
  const unsigned char* c10 = c00 + 3;
  const unsigned char* c11 = c01 + 3;
  unsigned int meas[3];
#pragma unroll
  for (int ch = 0; ch < 3; ch++)
    meas[ch] = (unsigned int)(unsigned char)roundf(
        interpolatePixels(ox, oy, (float)__ldg(c00 + ch), (float)__ldg(c01 + ch), (float)__ldg(c10 + ch), (float)__ldg(c11 + ch)));
  // isMasked(u_px.y(), u_px.x()): float -> int by truncation
  if (a.mask != nullptr) {
    const unsigned char mv = __ldg(a.mask + (size_t)floatToIntRz(v) * a.cols + floatToIntRz(u));
    const bool is_active = (a.mask_mode == NVB_MASK_NON_INVERTED) ? (mv != 0) : (mv == 0);
    if (!is_active) return false;
  }
  const unsigned int old_rgb = rgb;
  const float old_wgt = wgt;
  if (__half2float(__float2half_rn(wgt)) == 0.0f) {
    rgb = (rgb & 0xff000000u) | meas[0] | (meas[1] << 8) | (meas[2] << 16);
  } else {
    unsigned int out = rgb & 0xff000000u;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {  // weightedSum(uint8_t, float, uint8_t, float) (:277-285), weights rounded through __half
      const float cur = (float)((rgb >> (8 * ch)) & 0xffu);
      const unsigned int fused = (unsigned int)(unsigned char)roundf(cur * a.w_old_h + (float)meas[ch] * a.w_new_h);
      out |= fused << (8 * ch);
    }
    rgb = out;
  }
  wgt = fminf(a.measurement_weight + old_wgt, a.max_weight);
  return rgb != old_rgb || __float_as_uint(wgt) != __float_as_uint(old_wgt);
}

template <bool kDistort>
__global__ void __launch_bounds__(256) colorIntegrateKernel(const __grid_constant__ ColorArgs a) {
  const int n = *a.work_count;
  const int tid = threadIdx.x;
  // thread -> voxels (vx, vy, 2 * zp) and (vx, vy, 2 * zp + 1): one 16-byte word of the block
  const int vx = tid >> 5, vy = (tid >> 2) & 7, vz0 = (tid & 3) * 2;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int4 blk = a.work[i];
    uint4* word = reinterpret_cast<uint4*>(a.color.blocks + (size_t)blk.w * kColorBlockBytes) + tid;
    uint4 w = *word;
    float w0 = __uint_as_float(w.y), w1 = __uint_as_float(w.w);
    const bool c0 = updateColorVoxel<kDistort>(a, blk, vx, vy, vz0, w.x, w0);
    const bool c1 = updateColorVoxel<kDistort>(a, blk, vx, vy, vz0 + 1, w.z, w1);
    if (c0 || c1) {
      w.y = __float_as_uint(w0), w.w = __float_as_uint(w1);
      *word = w;
    }
  }
}

}  // namespace

void launchColorSelect(const ColorArgs& a, int num_sms, cudaStream_t stream) {
  colorSelectKernel<<<num_sms * 4, 256, 0, stream>>>(a);
}

void launchSphereTrace(const ColorArgs& a, cudaStream_t stream) {
  const dim3 threads(16, 8, 1);
  const dim3 grid((a.dcols + threads.x - 1) / threads.x, (a.drows + threads.y - 1) / threads.y, 1);
  if (a.cam.has_distortion)
    sphereTraceKernel<true><<<grid, threads, 0, stream>>>(a);
  else
    sphereTraceKernel<false><<<grid, threads, 0, stream>>>(a);
}

void launchRender(const RenderArgs& a, cudaStream_t stream) {
  const dim3 threads(16, 8, 1);
  const dim3 grid((a.dcols + threads.x - 1) / threads.x, (a.drows + threads.y - 1) / threads.y, 1);
  const bool d = a.cam.has_distortion != 0;
  if (a.rgb)
    d ? renderKernel<true, true><<<grid, threads, 0, stream>>>(a) : renderKernel<false, true><<<grid, threads, 0, stream>>>(a);
  else
    d ? renderKernel<true, false><<<grid, threads, 0, stream>>>(a) : renderKernel<false, false><<<grid, threads, 0, stream>>>(a);
}

void launchColorIntegrate(const ColorArgs& a, int num_sms, cudaStream_t stream) {
  if (a.cam.has_distortion)
    colorIntegrateKernel<true><<<num_sms * 4, 256, 0, stream>>>(a);
  else
    colorIntegrateKernel<false><<<num_sms * 4, 256, 0, stream>>>(a);
}

}  // namespace nvb
