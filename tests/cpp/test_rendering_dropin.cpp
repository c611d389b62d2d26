// Rendering through nvblox/nvblox.h only, with the calls nvblox_torch's py_rendering.cpp makes: a SphereTracer with
// maximum_ray_length_m / maximum_steps set, renderImageOnGPU into a DepthImageView and renderRgbdImageOnGPU into depth and
// colour views, on the TSDF and colour layers of a mapper that saw a red wall 3 m ahead. The rays along the optical axis hit
// the wall within a voxel; a hit is red, grey (a voxel of a coloured block that the frame did not reach) or black (a block
// without colour), most hits are red, a miss is black; the
// RGBD render's depth is the depth render's, and the owning-image overloads agree with the view overloads.
// Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <cstring>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  constexpr float kVoxel = 0.05f;
  constexpr int W = 640, H = 480;
  Camera camera(570.f, 570.f, 320.f, 240.f, W, H);
  DepthImage depth(H, W, MemoryType::kUnified);
  ColorImage red(H, W, MemoryType::kUnified);
  for (int r = 0; r < H; r++)
    for (int c = 0; c < W; c++) depth(r, c) = 3.0f, red(r, c) = Color::Red();
  Mapper mapper(kVoxel);
  mapper.integrateDepth(depth, Transform::Identity(), camera);
  mapper.integrateColor(red, Transform::Identity(), camera);
  const TsdfLayer& tsdf_layer = mapper.tsdf_layer();
  const ColorLayer& color_layer = mapper.color_layer();
  const float truncation_distance_m = tsdf_layer.voxel_size() * 4.0;

  SphereTracer sphere_tracer_gpu;
  EXPECT(sphere_tracer_gpu.maximum_steps() == 100 && sphere_tracer_gpu.maximum_ray_length_m() == 15.0f &&
         sphere_tracer_gpu.surface_distance_epsilon_vox() == 0.1f);
  sphere_tracer_gpu.maximum_ray_length_m(20.0);
  sphere_tracer_gpu.maximum_steps(100);
  EXPECT(sphere_tracer_gpu.maximum_ray_length_m() == 20.0f);
  const auto size = sphere_tracer_gpu.getSubsampledImageSize(camera, 4);
  EXPECT(size.rows == H / 4 && size.cols == W / 4);

  DepthImage d_img(H, W, MemoryType::kDevice);
  DepthImageView depth_image_view(d_img);
  sphere_tracer_gpu.renderImageOnGPU(camera, Transform::Identity(), tsdf_layer, truncation_distance_m, &depth_image_view,
                                     MemoryType::kDevice);
  DepthImage d2_img(H, W, MemoryType::kDevice);
  ColorImage c_img(H, W, MemoryType::kDevice);
  DepthImageView d2_view(d2_img);
  ColorImageView color_image_view(c_img);
  sphere_tracer_gpu.renderRgbdImageOnGPU(camera, Transform::Identity(), tsdf_layer, color_layer, truncation_distance_m,
                                         &d2_view, &color_image_view, MemoryType::kDevice);
  int hits = 0, red_hits = 0;
  for (int r = 0; r < H; r++)
    for (int c = 0; c < W; c++) {
      const float z = d_img(r, c);
      EXPECT(std::memcmp(&z, &d2_img(r, c), sizeof(float)) == 0);
      const Color& col = c_img(r, c);
      if (z > 0.0f) {
        hits++;
        EXPECT(std::fabs(z - 3.0f) < kVoxel);
        EXPECT(col == Color::Red() || col == Color::Gray() || col == Color(0, 0, 0));
        red_hits += col == Color::Red();
      } else {
        EXPECT(z == -1.0f && col == Color(0, 0, 0));
      }
    }
  EXPECT(hits > W * H / 2 && red_hits > hits / 2);

  // the owning-image overloads allocate the subsampled size and render the same rays as a view of that size
  DepthImage d4(1, 1, MemoryType::kDevice);
  ColorImage c4(1, 1, MemoryType::kDevice);
  sphere_tracer_gpu.renderRgbdImageOnGPU(camera, Transform::Identity(), tsdf_layer, color_layer, truncation_distance_m, &d4,
                                         &c4, MemoryType::kDevice, 4);
  EXPECT(d4.rows() == H / 4 && d4.cols() == W / 4 && c4.rows() == H / 4 && c4.cols() == W / 4);
  DepthImage d4v(H / 4, W / 4);
  DepthImageView d4_view(d4v);
  sphere_tracer_gpu.renderImageOnGPU(camera, Transform::Identity(), tsdf_layer, truncation_distance_m, &d4_view,
                                     MemoryType::kDevice, 4);
  EXPECT(std::memcmp(d4.dataPtr(), d4v.dataPtr(), sizeof(float) * d4.numel()) == 0);
  // a view of another size is left alone
  DepthImage wrong(2, 2);
  wrong(0, 0) = 42.0f;
  DepthImageView wrong_view(wrong);
  sphere_tracer_gpu.renderImageOnGPU(camera, Transform::Identity(), tsdf_layer, truncation_distance_m, &wrong_view,
                                     MemoryType::kDevice);
  EXPECT(wrong(0, 0) == 42.0f);
  std::printf("rendering drop-in ok: %d hits, %d red\n", hits, red_hits);
  return 0;
}
