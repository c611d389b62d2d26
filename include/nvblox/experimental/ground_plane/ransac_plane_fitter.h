// nvblox/experimental/ground_plane/ransac_plane_fitter.h -- RansacPlaneFitter (reference:
// nvblox/include/nvblox/experimental/ground_plane/ransac_plane_fitter.h): MSAC plane fit on the GPU through
// nvb_ransac_fit_plane. The parameters live in the owning mapper's NvbGroundPlaneParams, so the fitter of
// GroundPlaneEstimator and the estimator see the same values.
#pragma once
#include <optional>
#include <vector>
#include "nvblox/geometry/plane.h"
#include "nvblox/mapper/mapper.h"
#include "nvblox/sensors/pointcloud.h"
namespace nvblox {
namespace b200_detail {
inline NvbGroundPlaneParams groundParams(NvbMapper* m) {
  NvbGroundPlaneParams p;
  check(nvb_mapper_get_ground_plane_params(m, &p), "ground plane params", nvb_last_error());
  return p;
}
inline void setGroundParams(NvbMapper* m, const NvbGroundPlaneParams& p) {
  check(nvb_mapper_set_ground_plane_params(m, &p), "ground plane params", nvb_last_error());
}
}  // namespace b200_detail

class RansacPlaneFitter {
 public:
  explicit RansacPlaneFitter(NvbMapper* m) : m_(m) {}
  // fit(point_cloud) (ransac_plane_fitter.h): the plane of the lowest MSAC cost, std::nullopt for < 3 points or when every
  // sample is degenerate.
  std::optional<Plane> fit(const Pointcloud& point_cloud) const {
    std::vector<float> xyz((size_t)point_cloud.size() * 3);
    for (int i = 0; i < point_cloud.size(); i++)
      for (int k = 0; k < 3; k++) xyz[3 * (size_t)i + k] = point_cloud.points()[i][k];
    float pl[4];
    int32_t found = 0;
    b200_detail::check(nvb_ransac_fit_plane(m_, xyz.data(), NVB_MEM_HOST, point_cloud.size(), num_ransac_iterations(),
                                            ransac_distance_threshold_m(), pl, &found),
                       "RansacPlaneFitter::fit", nvb_last_error());
    if (!found) return std::nullopt;
    return Plane::fromCoefficients(Vector3f(pl[0], pl[1], pl[2]), pl[3]);
  }
  void ransac_distance_threshold_m(float v) {
    auto p = b200_detail::groundParams(m_);
    p.ransac_distance_threshold_m = v;
    b200_detail::setGroundParams(m_, p);
  }
  float ransac_distance_threshold_m() const { return b200_detail::groundParams(m_).ransac_distance_threshold_m; }
  void num_ransac_iterations(int v) {
    auto p = b200_detail::groundParams(m_);
    p.num_ransac_iterations = v;
    b200_detail::setGroundParams(m_, p);
  }
  int num_ransac_iterations() const { return b200_detail::groundParams(m_).num_ransac_iterations; }

 private:
  NvbMapper* m_;
};
}  // namespace nvblox
