// nvblox/io/pointcloud_io.h -- io::outputVoxelLayerToPly (reference: nvblox/include/nvblox/io/pointcloud_io.h,
// src/io/pointcloud_io.cpp:23-73) for the TSDF, ESDF, occupancy and freespace layers: the kept voxels' centres and
// intensities from nvb_layer_export_points (computed on the GPU), blocks in (x, y, z) order, then voxels in x, y, z order.
#pragma once
#include <string>
#include <vector>
#include "nvblox/io/ply_writer.h"
#include "nvblox/map/layer.h"
namespace nvblox {
namespace io {
namespace b200_detail_io {
template <typename VoxelType>
inline bool outputLayerPoints(const VoxelBlockLayer<VoxelType>& layer, const std::string& filename) {
  int64_t n = 0;
  b200_detail::check(nvb_layer_export_points(layer.c_abi(), layer.layer_id(), NVB_MEM_HOST, nullptr, 0, &n),
                     "outputVoxelLayerToPly", nvb_last_error());
  std::vector<float> xyzi((size_t)n * 4 + 4);
  b200_detail::check(nvb_layer_export_points(layer.c_abi(), layer.layer_id(), NVB_MEM_HOST, xyzi.data(), n, &n),
                     "outputVoxelLayerToPly", nvb_last_error());
  std::vector<Vector3f> points((size_t)n);
  std::vector<float> intensities((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    points[i] = Vector3f(xyzi[4 * i], xyzi[4 * i + 1], xyzi[4 * i + 2]);
    intensities[i] = xyzi[4 * i + 3];
  }
  PlyWriter writer(filename);
  writer.setPoints(&points);
  writer.setIntensities(&intensities);
  return writer.write();
}
}  // namespace b200_detail_io
inline bool outputVoxelLayerToPly(const TsdfLayer& layer, const std::string& filename) {
  return b200_detail_io::outputLayerPoints(layer, filename);
}
inline bool outputVoxelLayerToPly(const EsdfLayer& layer, const std::string& filename) {
  return b200_detail_io::outputLayerPoints(layer, filename);
}
inline bool outputVoxelLayerToPly(const OccupancyLayer& layer, const std::string& filename) {
  return b200_detail_io::outputLayerPoints(layer, filename);
}
inline bool outputVoxelLayerToPly(const FreespaceLayer& layer, const std::string& filename) {
  return b200_detail_io::outputLayerPoints(layer, filename);
}
}  // namespace io
}  // namespace nvblox
