// nvblox/sensors/pointcloud.h -- the subset of Pointcloud (reference: nvblox/include/nvblox/sensors/pointcloud.h) that
// RansacPlaneFitter::fit takes: a list of points. Kept on the host here; the fit copies it to the device.
#pragma once
#include <vector>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/core/types.h"
namespace nvblox {
class Pointcloud {
 public:
  Pointcloud() = default;
  explicit Pointcloud(MemoryType) {}
  void copyPointsFromAsync(const std::vector<Vector3f>& points, const CudaStream&) { points_ = points; }
  void copyPointsFrom(const std::vector<Vector3f>& points) { points_ = points; }
  int size() const { return (int)points_.size(); }
  const std::vector<Vector3f>& points() const { return points_; }

 private:
  std::vector<Vector3f> points_;
};
}  // namespace nvblox
