// nvblox/experimental/ground_plane/tsdf_zero_crossings_extractor.h -- TsdfZeroCrossingsExtractor's parameter surface
// (reference: nvblox/include/nvblox/experimental/ground_plane/tsdf_zero_crossings_extractor.h). The extraction itself runs
// inside GroundPlaneEstimator::computeGroundPlane (nvb_mapper_compute_ground_plane).
#pragma once
#include "nvblox/experimental/ground_plane/ransac_plane_fitter.h"
namespace nvblox {
class TsdfZeroCrossingsExtractor {
 public:
  explicit TsdfZeroCrossingsExtractor(NvbMapper* m) : m_(m) {}
  // A layer with max_crossings crossings or more gives no plane.
  void max_crossings(int v) {
    auto p = b200_detail::groundParams(m_);
    p.max_crossings = v;
    b200_detail::setGroundParams(m_, p);
  }
  int max_crossings() const { return b200_detail::groundParams(m_).max_crossings; }
  // Both voxels of a crossing need a weight >= min_tsdf_weight.
  void min_tsdf_weight(float v) {
    auto p = b200_detail::groundParams(m_);
    p.min_tsdf_weight = v;
    b200_detail::setGroundParams(m_, p);
  }
  float min_tsdf_weight() const { return b200_detail::groundParams(m_).min_tsdf_weight; }

 private:
  NvbMapper* m_;
};
}  // namespace nvblox
