// Replays nvblox_ros' ground-plane calls through nvblox/nvblox.h only: a MultiMapper (kStaticTsdf, kStaticOccupancy,
// kDynamic) with and without experimental_use_ground_plane_estimation and a 2-D ESDF, updateEsdf, then the node's publishers
// read ground_plane_estimator().tsdf_zero_crossings_ground_candidates() (nvblox_node.cpp:1456) and
// ground_plane_estimator().ground_plane() (:1474). Every ESDF slice block of both mappers is compared byte for byte with
// single mappers sliced by hand on the same plane (or at constant z without one). Then RansacPlaneFitter::fit on a Pointcloud
// (T/test_ransac_plane_fitter.cpp, FitToKnownPlanarPoints). Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <map>
#include <tuple>
#include <vector>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

using Blocks = std::map<std::tuple<int, int, int>, std::vector<unsigned char>>;

// Every block of a layer, bytes and all, keyed by block index (read through the C ABI).
static Blocks layerBytes(NvbMapper* m, int layer) {
  int32_t n = 0;
  nvb_layer_num_blocks(m, layer, &n);
  std::vector<int32_t> idx((size_t)n * 3);
  if (n) nvb_layer_block_indices(m, layer, idx.data(), n, &n);
  const size_t bytes = (size_t)nvb_layer_block_bytes(layer);
  std::vector<unsigned char> raw(bytes * n);
  std::vector<uint8_t> found((size_t)n);
  if (n) nvb_layer_get_blocks(m, layer, idx.data(), n, raw.data(), found.data());
  Blocks out;
  for (int i = 0; i < n; i++)
    out[std::make_tuple(idx[3 * i], idx[3 * i + 1], idx[3 * i + 2])] =
        std::vector<unsigned char>(raw.begin() + i * bytes, raw.begin() + (i + 1) * bytes);
  return out;
}

int main() {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  Camera camera(300.f, 300.f, 320.f, 240.f, 640, 480);
  // a camera 1.5 m above the floor z = 0, looking straight down at it and at a 0.6 m high box
  DepthImage depth(480, 640, MemoryType::kUnified);
  for (int r = 0; r < 480; r++)
    for (int c = 0; c < 640; c++) depth(r, c) = (r > 180 && r < 300 && c > 260 && c < 380) ? 0.9f : 1.5f;
  MonoImage mask(480, 640, MemoryType::kUnified);  // kDynamic: the left half of the image is dynamic
  for (int r = 0; r < 480; r++) for (int c = 0; c < 640; c++) mask(r, c) = c < 320 ? 255 : 0;
  Transform T_L_C = Transform::Identity();
  T_L_C(1, 1) = -1.0f, T_L_C(2, 2) = -1.0f;
  T_L_C.setTranslation(Vector3f(0.0f, 0.0f, 1.5f));
  const Time t_ms = 1000;

  // --- MultiMapper::updateEsdf with and without experimental_use_ground_plane_estimation, 2-D ESDF, against single
  // mappers driven by hand: the estimated plane on the background mapper, handed to both mappers' planar slices
  for (MappingType type : {MappingType::kStaticTsdf, MappingType::kStaticOccupancy, MappingType::kDynamic}) {
    Blocks slice_off;
    for (int use_plane = 0; use_plane < 2; use_plane++) {
      MultiMapper mm(0.05f, type, EsdfMode::k2D);
      MultiMapperParams params;
      params.experimental_use_ground_plane_estimation = use_plane == 1;
      params.ground_plane_estimator_params.num_ransac_iterations = 500;
      mm.setMultiMapperParams(params);
      EXPECT(mm.ground_plane_estimator().ransac_plane_fitter().num_ransac_iterations() == 500);
      EXPECT(mm.ground_plane_estimator().tsdf_zero_crossings_extractor().max_crossings() == 360000);
      if (type == MappingType::kDynamic) mm.setDynamicMask(MonoImageConstView(mask));
      mm.integrateDepth(depth, T_L_C, camera, std::optional<Time>(t_ms));
      mm.updateEsdf();
      // nvblox_node.cpp:1456 and :1474
      const std::optional<std::vector<Vector3f>> candidates =
          mm.ground_plane_estimator().tsdf_zero_crossings_ground_candidates();
      const std::optional<Plane> plane = mm.ground_plane_estimator().ground_plane();

      // the same by hand
      const ProjectiveLayerType bg = type == MappingType::kStaticOccupancy ? ProjectiveLayerType::kOccupancy
                                     : type == MappingType::kDynamic     ? ProjectiveLayerType::kTsdfWithFreespace
                                                                          : ProjectiveLayerType::kTsdf;
      Mapper back(0.05f, MemoryType::kDevice, bg);
      back.integrateDepth(depth, T_L_C, camera);
      if (type == MappingType::kDynamic) back.updateFreespace(t_ms, T_L_C, camera, DepthImageConstView(depth));
      std::optional<Plane> want;
      if (use_plane) {
        GroundPlaneEstimator est(back.c_abi());
        est.ransac_plane_fitter().num_ransac_iterations(500);
        want = est.computeGroundPlane(back.tsdf_layer());
      }
      EXPECT(plane.has_value() == want.has_value());
      if (want) EXPECT(plane->normal() == want->normal() && plane->d() == want->d());
      if (want) back.updateEsdfSlice(UpdateFullLayer::kNo, *want);
      else back.updateEsdfSlice();
      const Blocks got = layerBytes(mm.background_mapper()->c_abi(), NVB_LAYER_ESDF);
      EXPECT(!got.empty());
      EXPECT(got == layerBytes(back.c_abi(), NVB_LAYER_ESDF));
      if (type == MappingType::kDynamic) {
        Mapper fore(0.05f, MemoryType::kDevice, ProjectiveLayerType::kOccupancy);
        fore.integrateDepth(MaskedDepthImageConstView(depth, MonoImageConstView(mask)), T_L_C, camera);
        if (want) fore.updateEsdfSlice(UpdateFullLayer::kNo, *want);
        else fore.updateEsdfSlice();
        const Blocks fg = layerBytes(mm.foreground_mapper()->c_abi(), NVB_LAYER_ESDF);
        EXPECT(!fg.empty() && fg == layerBytes(fore.c_abi(), NVB_LAYER_ESDF));
      }

      if (!use_plane) {
        EXPECT(!candidates && !plane);  // never computed
        slice_off = got;
        continue;
      }
      if (type == MappingType::kStaticOccupancy) {
        EXPECT(!candidates && !plane && got == slice_off);  // no TSDF layer: no plane, the constant-z slice
        continue;
      }
      EXPECT(candidates && candidates->size() > 1000);
      for (const Vector3f& p : *candidates) EXPECT(p[2] >= -0.1f && p[2] <= 0.15f && std::fabs(p[2]) < 0.01f);
      EXPECT(plane);
      EXPECT(std::fabs(std::fabs(plane->normal()[2]) - 1.0f) < 1e-3f && std::fabs(plane->d()) < 0.01f);
      EXPECT(got != slice_off);  // the planar slice is not the constant-z one
    }
  }

  // RansacPlaneFitter on a Pointcloud: seven points on z = 0.1 (sign-flip rule of verifyPlaneFit)
  Mapper mapper(0.05f);
  GroundPlaneEstimator est(mapper.c_abi());
  RansacPlaneFitter fitter = est.ransac_plane_fitter();
  fitter.num_ransac_iterations(1000);
  fitter.ransac_distance_threshold_m(0.2f);
  Pointcloud cloud(MemoryType::kDevice);
  CudaStreamOwning stream;
  cloud.copyPointsFromAsync({Vector3f(0.f, 0.f, .1f), Vector3f(1.f, 0.f, .1f), Vector3f(2.f, 0.f, .1f), Vector3f(0.f, 1.f, .1f),
                             Vector3f(1.f, 1.f, .1f), Vector3f(2.f, 1.f, .1f), Vector3f(.5f, .5f, .1f)},
                            stream);
  const std::optional<Plane> fit = fitter.fit(cloud);
  EXPECT(fit);
  const float s = fit->d() == -0.1f ? 1.0f : -1.0f;
  EXPECT(std::fabs(fit->normal()[0]) < 1e-4f && std::fabs(fit->normal()[1]) < 1e-4f && std::fabs(s * fit->normal()[2] - 1.0f) < 1e-4f);
  EXPECT(std::fabs(s * fit->d() + 0.1f) < 1e-4f);
  Pointcloud two;
  two.copyPointsFrom({Vector3f(0.f, 0.f, 0.f), Vector3f(1.f, 0.f, 0.f)});
  EXPECT(!fitter.fit(two));
  std::printf("ground plane drop-in ok\n");
  return 0;
}
