// Replays nvblox_ros' human-mapping calls through nvblox/nvblox.h only: integrateDepth(depth, mask, T_L_C, T_CM_CD,
// depth_camera, mask_camera) with the mask from a separate 1280 x 720 colour camera (1 degree rotation, 5 cm baseline),
// then getLastDepthFrameForeground / getLastDepthFrameMaskOverlay (publishHumanDebugOutput) and updateEsdf.
// The depth frame holds a box face at 1.5 m and zero (invalid) depth elsewhere; the mask is a rectangle of the colour
// camera that covers part of the box. Expected: the foreground frame holds exactly the box pixels whose points project
// into the rectangle; the background frame holds the others; the foreground occupancy is observed only around the box.
// Then the kept deviation: T_CM_CD = identity with the depth camera as mask camera integrates exactly like two masked-view
// integrations. Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <cstring>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

constexpr int kRows = 480, kCols = 640, kMaskRows = 720, kMaskCols = 1280;
constexpr int kBoxR0 = 120, kBoxR1 = 300, kBoxC0 = 250, kBoxC1 = 450;
constexpr int kMaskR0 = 200, kMaskR1 = 520, kMaskC0 = 400, kMaskC1 = 800;  // even bounds: the 2x filter keeps them
constexpr float kBox = 1.5f;

static long observedOccupancy(const OccupancyLayer& layer, float* max_z) {
  long n = 0;
  for (const Index3D& b : layer.getAllBlockIndices()) {
    auto blk = layer.getBlockAtIndexHost(b);
    for (int x = 0; x < 8; x++) for (int y = 0; y < 8; y++) for (int z = 0; z < 8; z++)
      if (blk->voxels[x][y][z].log_odds != 0.0f) {
        n++;
        *max_z = std::fmax(*max_z, (b[2] * 8 + z) * 0.05f);
      }
  }
  return n;
}

static bool sameTsdf(const TsdfLayer& a, const TsdfLayer& b) {
  if (a.numBlocks() != b.numBlocks()) return false;
  for (const Index3D& idx : a.getAllBlockIndices()) {
    if (!b.getBlockAtIndex(idx)) return false;
    auto x = a.getBlockAtIndexHost(idx), y = b.getBlockAtIndexHost(idx);
    if (std::memcmp(x->voxels, y->voxels, sizeof(x->voxels)) != 0) return false;
  }
  return true;
}

static bool sameOccupancy(const OccupancyLayer& a, const OccupancyLayer& b) {
  if (a.numBlocks() != b.numBlocks()) return false;
  for (const Index3D& idx : a.getAllBlockIndices()) {
    if (!b.getBlockAtIndex(idx)) return false;
    auto x = a.getBlockAtIndexHost(idx), y = b.getBlockAtIndexHost(idx);
    if (std::memcmp(x->voxels, y->voxels, sizeof(x->voxels)) != 0) return false;
  }
  return true;
}

int main() {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  // the depth / colour pair of tests/camera_pose_cases.py
  const Camera depth_camera(290.f, 320.f, 320.f + 0.12f * 640.f, 240.f - 0.11f * 480.f, kCols, kRows);
  const Camera mask_camera(610.f, 560.f, 640.f - 0.13f * 1280.f, 360.f + 0.12f * 720.f, kMaskCols, kMaskRows);
  const float a = 1.0f * 3.14159265f / 180.f, ca = std::cos(a), sa = std::sin(a);
  Transform T_CM_CD = Transform::Identity();  // 1 degree about y, 5 cm along x; t.z = 0, so zero depth does not project
  T_CM_CD(0, 0) = ca, T_CM_CD(0, 2) = sa, T_CM_CD(2, 0) = -sa, T_CM_CD(2, 2) = ca, T_CM_CD(0, 3) = -0.05f;
  const Transform T_L_C = Transform::Identity();

  DepthImage depth(kRows, kCols, MemoryType::kUnified);
  for (int r = 0; r < kRows; r++)
    for (int c = 0; c < kCols; c++) depth(r, c) = (r >= kBoxR0 && r < kBoxR1 && c >= kBoxC0 && c < kBoxC1) ? kBox : 0.0f;
  MonoImage mask(kMaskRows, kMaskCols, MemoryType::kUnified);
  for (int r = 0; r < kMaskRows; r++)
    for (int c = 0; c < kMaskCols; c++) mask(r, c) = (r >= kMaskR0 && r < kMaskR1 && c >= kMaskC0 && c < kMaskC1) ? 1 : 0;

  MultiMapper mm(0.05f, MappingType::kHumanWithStaticTsdf, EsdfMode::k3D);
  mm.setMultiMapperParams(MultiMapperParams());  // the filter is on (threshold 2000): the rectangle survives it
  mm.image_masker().occlusion_threshold_m(0.25f);
  EXPECT(mm.image_masker().occlusion_threshold_m() == 0.25f && mm.image_masker().depth_masked_image_invalid_pixel() == -1.0f);
  mm.integrateDepth(depth, mask, T_L_C, T_CM_CD, depth_camera, mask_camera);
  mm.updateEsdf();

  const DepthImage& fg = mm.getLastDepthFrameForeground();
  const DepthImage& bgf = mm.getLastDepthFrameBackground();
  const ColorImage& overlay = mm.getLastDepthFrameMaskOverlay();
  EXPECT(fg.rows() == kRows && fg.cols() == kCols && bgf.rows() == kRows && overlay.rows() == kRows && overlay.cols() == kCols);
  long n_fg = 0, n_checked = 0;
  for (int r = 0; r < kRows; r++)
    for (int c = 0; c < kCols; c++) {
      const float d = depth(r, c), f = fg(r, c), b = bgf(r, c);
      const bool in_fg = f != -1.0f;
      EXPECT(in_fg ? (f == d && b == -1.0f) : (b == d && f == -1.0f));
      EXPECT((overlay(r, c).r == 255) == in_fg || (d >= 20.0f));
      n_fg += in_fg;
      if (d == 0.0f) { EXPECT(!in_fg); continue; }
      // the box point in the mask camera
      const float x = ((c + 0.5f) - depth_camera.cu()) / depth_camera.fu() * d, y = ((r + 0.5f) - depth_camera.cv()) / depth_camera.fv() * d;
      const float px = T_CM_CD(0, 0) * x + T_CM_CD(0, 2) * d + T_CM_CD(0, 3), py = y, pz = T_CM_CD(2, 0) * x + T_CM_CD(2, 2) * d;
      const float u = px / pz * mask_camera.fu() + mask_camera.cu(), v = py / pz * mask_camera.fv() + mask_camera.cv();
      const float margin = 0.01f;
      const bool inside = u > kMaskC0 + margin && u < kMaskC1 - margin && v > kMaskR0 + margin && v < kMaskR1 - margin;
      const bool outside = u < kMaskC0 - margin || u > kMaskC1 + margin || v < kMaskR0 - margin || v > kMaskR1 + margin;
      if (inside) { EXPECT(in_fg); n_checked++; }
      if (outside) { EXPECT(!in_fg); n_checked++; }
    }
  std::printf("foreground pixels: %ld of %d box pixels; checked %ld\n", n_fg, (kBoxR1 - kBoxR0) * (kBoxC1 - kBoxC0), n_checked);
  EXPECT(n_fg > 5000 && n_fg < (kBoxR1 - kBoxR0) * (kBoxC1 - kBoxC0) - 5000);
  EXPECT(n_checked > (kBoxR1 - kBoxR0) * (kBoxC1 - kBoxC0) - 2000);
  float max_z = 0.0f;
  EXPECT(observedOccupancy(mm.foreground_mapper()->occupancy_layer(), &max_z) > 1000);
  EXPECT(max_z < kBox + 0.5f);  // the foreground reaches no further than the box's truncation band
  EXPECT(mm.background_mapper()->tsdf_layer().numBlocks() > 0 && mm.background_mapper()->esdf_layer().numBlocks() > 0);

  {  // the kept deviation: identity T_CM_CD with the depth camera as mask camera integrates through masked views
    MonoImage same_mask(kRows, kCols, MemoryType::kUnified);
    for (int r = 0; r < kRows; r++) for (int c = 0; c < kCols; c++) same_mask(r, c) = c < 350 ? 1 : 0;
    DepthImage wall(kRows, kCols, MemoryType::kUnified);
    for (int r = 0; r < kRows; r++) for (int c = 0; c < kCols; c++) wall(r, c) = 3.0f + 0.001f * c - (c > 300 && c < 400 ? 1.2f : 0.0f);
    MultiMapper human(0.05f, MappingType::kHumanWithStaticTsdf, EsdfMode::k3D);
    human.integrateDepth(wall, same_mask, T_L_C, Transform::Identity(), depth_camera, depth_camera);
    Mapper tsdf(0.05f, MemoryType::kDevice), occupancy(0.05f, BlockMemoryPoolParams(), ProjectiveLayerType::kOccupancy);
    occupancy.integrateDepth(MaskedDepthImageConstView(wall, MonoImageConstView(same_mask)), T_L_C, depth_camera);
    tsdf.integrateDepth(MaskedDepthImageConstView(wall, MonoImageConstView(same_mask), MaskMode::kInverted), T_L_C, depth_camera);
    EXPECT(tsdf.tsdf_layer().numBlocks() > 100 && occupancy.occupancy_layer().numBlocks() > 100);
    EXPECT(sameTsdf(human.background_mapper()->tsdf_layer(), tsdf.tsdf_layer()));
    EXPECT(sameOccupancy(human.foreground_mapper()->occupancy_layer(), occupancy.occupancy_layer()));
    // the split still ran: the getters describe this frame
    const DepthImage& f = human.getLastDepthFrameForeground();
    EXPECT(f.rows() == kRows && f.cols() == kCols && f(240, 100) == wall(240, 100) && f(240, 600) == -1.0f);

    // identity T_CM_CD, but a mask camera of the same size with other intrinsics: the mask is re-projected, not applied
    // pixel for pixel (with a 20 % longer focal length the mask's edge at column 350 falls on depth column 357, and the
    // top and bottom rows of the depth frame fall outside the mask image)
    const Camera zoomed(depth_camera.fu() * 1.2f, depth_camera.fv() * 1.2f, depth_camera.cu(), depth_camera.cv(), kCols, kRows);
    MultiMapper reproj(0.05f, MappingType::kHumanWithStaticTsdf, EsdfMode::k3D);
    reproj.integrateDepth(wall, same_mask, T_L_C, Transform::Identity(), depth_camera, zoomed);
    const DepthImage& g = reproj.getLastDepthFrameForeground();
    long differ = 0;
    for (int r = 0; r < kRows; r++) for (int c = 0; c < kCols; c++) differ += (g(r, c) != -1.0f) != (same_mask(r, c) != 0);
    std::printf("re-projected mask differs from the pixel-for-pixel mask at %ld pixels\n", differ);
    EXPECT(differ > 1000 && g(240, 100) == wall(240, 100) && g(240, 600) == -1.0f);
    EXPECT(!sameOccupancy(reproj.foreground_mapper()->occupancy_layer(), occupancy.occupancy_layer()));
  }
  std::printf("human mapping drop-in ok\n");
  return 0;
}
