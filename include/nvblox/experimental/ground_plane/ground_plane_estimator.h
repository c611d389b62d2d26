// nvblox/experimental/ground_plane/ground_plane_estimator.h -- GroundPlaneEstimator (reference:
// nvblox/include/nvblox/experimental/ground_plane/ground_plane_estimator.h, ground_plane_estimator_params.h) as a view of
// one mapper's estimator (nvb_mapper_compute_ground_plane and its getters). Point lists come in canonical order: block
// index (x, y, z) lexicographically, then voxel (x, y, z).
#pragma once
#include <optional>
#include <vector>
#include "nvblox/experimental/ground_plane/ransac_plane_fitter.h"
#include "nvblox/experimental/ground_plane/tsdf_zero_crossings_extractor.h"
namespace nvblox {

// GroundPlaneEstimatorParams (ground_plane_estimator_params.h) with the defaults of the reference
struct GroundPlaneEstimatorParams {
  float ground_points_candidates_min_z_m = -0.1f;
  float ground_points_candidates_max_z_m = 0.15f;
  float ransac_distance_threshold_m = 0.2f;
  int num_ransac_iterations = 1000;
  float min_tsdf_weight = 0.1f;
  int max_crossings = 360000;
};

class GroundPlaneEstimator {
 public:
  explicit GroundPlaneEstimator(NvbMapper* m) : m_(m) {}
  // computeGroundPlane(tsdf_layer): the layer must be the TSDF layer of this estimator's mapper.
  std::optional<Plane> computeGroundPlane(const TsdfLayer& tsdf_layer) {
    if (tsdf_layer.mapper_handle() != m_)
      b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "GroundPlaneEstimator::computeGroundPlane", "the layer belongs to another mapper");
    float pl[4];
    int32_t found = 0;
    b200_detail::check(nvb_mapper_compute_ground_plane(m_, pl, &found), "computeGroundPlane", nvb_last_error());
    if (!found) return std::nullopt;
    return Plane::fromCoefficients(Vector3f(pl[0], pl[1], pl[2]), pl[3]);
  }
  std::optional<Plane> ground_plane() const {
    float pl[4];
    int32_t found = 0;
    b200_detail::check(nvb_mapper_ground_plane(m_, pl, &found), "ground_plane", nvb_last_error());
    if (!found) return std::nullopt;
    return Plane::fromCoefficients(Vector3f(pl[0], pl[1], pl[2]), pl[3]);
  }
  std::optional<std::vector<Vector3f>> tsdf_zero_crossings() const { return points(NVB_GROUND_POINTS_CROSSINGS); }
  std::optional<std::vector<Vector3f>> tsdf_zero_crossings_ground_candidates() const {
    return points(NVB_GROUND_POINTS_CANDIDATES);
  }
  float ground_points_candidates_min_z_m() const { return b200_detail::groundParams(m_).ground_points_candidates_min_z_m; }
  float ground_points_candidates_max_z_m() const { return b200_detail::groundParams(m_).ground_points_candidates_max_z_m; }
  void ground_points_candidates_min_z_m(float v) {
    auto p = b200_detail::groundParams(m_);
    p.ground_points_candidates_min_z_m = v;
    b200_detail::setGroundParams(m_, p);
  }
  void ground_points_candidates_max_z_m(float v) {
    auto p = b200_detail::groundParams(m_);
    p.ground_points_candidates_max_z_m = v;
    b200_detail::setGroundParams(m_, p);
  }
  RansacPlaneFitter ransac_plane_fitter() const { return RansacPlaneFitter(m_); }
  TsdfZeroCrossingsExtractor tsdf_zero_crossings_extractor() const { return TsdfZeroCrossingsExtractor(m_); }
  // All parameters at once (MultiMapper::setMultiMapperParams, multi_mapper.cpp:121-128)
  void setParams(const GroundPlaneEstimatorParams& q) {
    NvbGroundPlaneParams p{q.ground_points_candidates_min_z_m, q.ground_points_candidates_max_z_m, q.ransac_distance_threshold_m,
                           q.num_ransac_iterations, q.min_tsdf_weight, q.max_crossings};
    b200_detail::setGroundParams(m_, p);
  }

 private:
  std::optional<std::vector<Vector3f>> points(int which) const {
    int32_t n = 0, valid = 0;
    b200_detail::check(nvb_mapper_ground_plane_points(m_, which, nullptr, 0, &n, &valid), "ground plane points", nvb_last_error());
    if (!valid) return std::nullopt;
    std::vector<float> xyz((size_t)n * 3);
    if (n) b200_detail::check(nvb_mapper_ground_plane_points(m_, which, xyz.data(), n, &n, &valid), "ground plane points", nvb_last_error());
    std::vector<Vector3f> out((size_t)n);
    for (int i = 0; i < n; i++) out[i] = Vector3f(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]);
    return out;
  }
  NvbMapper* m_;
};
}  // namespace nvblox
