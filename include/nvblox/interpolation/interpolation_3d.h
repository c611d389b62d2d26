// nvblox/interpolation/interpolation_3d.h -- interpolation::interpolateOnCPU (reference: nvblox/include/nvblox/interpolation/
// interpolation_3d.h, src/interpolation/interpolation_3d.cpp). The names are the reference's, but the work runs on the GPU
// (nvb_layer_interpolate) and the result is returned to the host: trilinear interpolation of the 8 voxels around each point
// -- TSDF distance (weight > 1e-4), ESDF sqrt(squared_distance_vox) in voxels (observed), occupancy probability. A point
// fails when a neighbour's block is missing or a neighbour is invalid; the vector overloads then store 0.
#pragma once
#include <vector>
#include "nvblox/map/layer.h"
namespace nvblox {
namespace interpolation {
namespace b200_detail_interp {
template <typename VoxelType>
inline void interpolate(const std::vector<Vector3f>& points_L, const VoxelBlockLayer<VoxelType>& layer,
                        std::vector<float>* values_ptr, std::vector<bool>* success_flags_ptr) {
  const size_t n = points_L.size();
  std::vector<float> xyz(n * 3);
  for (size_t i = 0; i < n; i++) xyz[3 * i] = points_L[i][0], xyz[3 * i + 1] = points_L[i][1], xyz[3 * i + 2] = points_L[i][2];
  values_ptr->assign(n, 0.0f);
  std::vector<uint8_t> ok(n, 0);
  ::nvblox::b200_detail::check(nvb_layer_interpolate(layer.mapper_handle(), layer.layer_id(), xyz.data(), NVB_MEM_HOST, (int64_t)n,
                                                     values_ptr->data(), ok.data()),
                               "interpolateOnCPU", nvb_last_error());
  success_flags_ptr->assign(ok.begin(), ok.end());
}
template <typename VoxelType>
inline bool interpolateOne(const Vector3f& p_L, const VoxelBlockLayer<VoxelType>& layer, float* value_ptr) {
  std::vector<float> values;
  std::vector<bool> ok;
  interpolate(std::vector<Vector3f>{p_L}, layer, &values, &ok);
  if (ok[0]) *value_ptr = values[0];  // the single-point overload leaves the output alone on failure
  return ok[0];
}
}  // namespace b200_detail_interp

inline bool interpolateOnCPU(const Vector3f& p_L, const TsdfLayer& layer, float* distance) {
  return b200_detail_interp::interpolateOne(p_L, layer, distance);
}
inline bool interpolateOnCPU(const Vector3f& p_L, const EsdfLayer& layer, float* distance) {
  return b200_detail_interp::interpolateOne(p_L, layer, distance);
}
inline bool interpolateOnCPU(const Vector3f& p_L, const OccupancyLayer& layer, float* probability) {
  return b200_detail_interp::interpolateOne(p_L, layer, probability);
}
template <typename VoxelType>
void interpolateOnCPU(const std::vector<Vector3f>& points_L, const VoxelBlockLayer<VoxelType>& layer,
                      std::vector<float>* distances_ptr, std::vector<bool>* success_flags_ptr) {
  b200_detail_interp::interpolate(points_L, layer, distances_ptr, success_flags_ptr);
}
}  // namespace interpolation
}  // namespace nvblox
