// Replays nvblox_ros' kDynamic calls through nvblox/nvblox.h only, with no setDynamicMask: the node integrates every depth
// frame with MultiMapper::integrateDepth(depth, T_L_C, camera, update_time_ms), calls updateEsdf, and publishes
// getLastDynamicPointcloud (~/dynamic_points) and getLastDynamicFrameMaskOverlay (~/dynamic_depth_frame_overlay).
// A static camera sees a wall at 3 m for 1.6 s (its freespace turns high-confidence), then a box moves through the view
// at 1.5 m. Expected: dynamic points only on the box, an overlay of the frame's size, and foreground occupancy blocks only
// around the box. Then image::MaskPreprocessor on a small mask. Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <vector>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

constexpr int kRows = 480, kCols = 640;
constexpr float kWall = 3.0f, kBox = 1.5f;
constexpr int kBoxR0 = 180, kBoxR1 = 300;  // box rows [r0, r1), columns [c0, c0 + 120)

// Foreground blocks with an observed voxel (log odds != 0). The view raycast allocates blocks for the whole view, masked or
// not; only the masked pixels update voxels.
static std::vector<Index3D> observedBlocks(const OccupancyLayer& layer) {
  std::vector<Index3D> out;
  for (const Index3D& b : layer.getAllBlockIndices()) {
    auto blk = layer.getBlockAtIndexHost(b);
    bool any = false;
    for (int x = 0; x < 8; x++) for (int y = 0; y < 8; y++) for (int z = 0; z < 8; z++) any |= blk->voxels[x][y][z].log_odds != 0.0f;
    if (any) out.push_back(b);
  }
  return out;
}

static void render(DepthImage* d, int box_c0) {
  for (int r = 0; r < kRows; r++)
    for (int c = 0; c < kCols; c++)
      (*d)(r, c) = (box_c0 >= 0 && r >= kBoxR0 && r < kBoxR1 && c >= box_c0 && c < box_c0 + 120) ? kBox : kWall;
}

int main() {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  Camera camera(300.f, 300.f, 320.f, 240.f, kCols, kRows);
  const Transform T_L_C = Transform::Identity();  // the camera looks along +z
  MultiMapper mm(0.05f, MappingType::kDynamic, EsdfMode::k3D);
  MultiMapperParams params;  // remove_small_connected_components, threshold 2000 (the node's defaults)
  mm.setMultiMapperParams(params);
  DepthImage depth(kRows, kCols, MemoryType::kUnified);

  render(&depth, -1);
  for (int i = 0; i < 17; i++) {  // the static wall, 100 ms apart
    mm.integrateDepth(depth, T_L_C, camera, std::optional<Time>(Time(100 * i)));
    mm.updateEsdf();
    EXPECT(mm.getLastDynamicPointcloud().size() == 0);
  }
  EXPECT(observedBlocks(mm.foreground_mapper()->occupancy_layer()).empty());

  int total = 0;
  for (int k = 0; k < 3; k++) {  // the box moves right by 40 pixels per frame
    const int c0 = 220 + 40 * k;
    render(&depth, c0);
    mm.integrateDepth(depth, T_L_C, camera, std::optional<Time>(Time(1700 + 100 * k)));
    mm.updateEsdf();
    const Pointcloud& cloud = mm.getLastDynamicPointcloud();
    const ColorImage& overlay = mm.getLastDynamicFrameMaskOverlay();
    EXPECT(overlay.rows() == kRows && overlay.cols() == kCols);
    EXPECT(cloud.size() > 2000);
    total += cloud.size();
    for (const Vector3f& p : cloud.points()) {
      // on the box's front face, inside its frustum
      EXPECT(std::fabs(p[2] - kBox) <= 1e-4f);
      const float c = p[0] / p[2] * 300.f + 320.f, r = p[1] / p[2] * 300.f + 240.f;
      EXPECT(c >= c0 - 1e-2f && c <= c0 + 120 + 1e-2f && r >= kBoxR0 - 1e-2f && r <= kBoxR1 + 1e-2f);
    }
    int red = 0;
    for (int r = 0; r < kRows; r++)
      for (int c = 0; c < kCols; c++) red += overlay(r, c).r == 255 && overlay(r, c).g != 255;
    EXPECT(red == cloud.size());
  }
  // foreground occupancy: only the box's frustum in front of the wall
  const std::vector<Index3D> blocks = observedBlocks(mm.foreground_mapper()->occupancy_layer());
  EXPECT(!blocks.empty());
  const float bs = 0.4f;
  for (const Index3D& b : blocks) {
    const float x0 = b[0] * bs, y0 = b[1] * bs, z0 = b[2] * bs;
    EXPECT(z0 < kWall - 0.2f);                                          // nothing at the wall
    EXPECT(x0 + bs > -0.6f && x0 < 0.9f && y0 + bs > -0.6f && y0 < 0.6f);  // the box's frustum up to 2 m
  }
  std::printf("points over 3 frames: %d, foreground blocks: %zu\n", total, blocks.size());

  // image::MaskPreprocessor: a 4 x 4 blob survives threshold 8, a single pixel does not; the odd last row / column is 0
  image::MaskPreprocessor pre(std::make_shared<CudaStreamOwning>());
  MonoImage mask(11, 11, MemoryType::kHost), out(11, 11, MemoryType::kHost);
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) mask(r, c) = 255;
  mask(8, 8) = 255;
  pre.removeSmallConnectedComponents(mask, 8, &out);
  EXPECT(out.rows() == 11 && out.cols() == 11);
  EXPECT(out(0, 0) == 254 && out(3, 3) == 254 && out(8, 8) == 0 && out(10, 10) == 0);
  std::printf("dynamics drop-in ok\n");
  return 0;
}
