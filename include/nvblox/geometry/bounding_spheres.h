// nvblox/geometry/bounding_spheres.h -- BoundingSphere and the block-radius tests (reference:
// nvblox/include/nvblox/geometry/bounding_spheres.h:22-60, src/geometry/bounding_spheres.cpp:23-74).
#pragma once
#include <cmath>
#include <vector>
#include "nvblox/geometry/bounding_boxes.h"
namespace nvblox {
class BoundingSphere {
 public:
  BoundingSphere() : center_(0.0f, 0.0f, 0.0f), radius_(0.0f) {}
  BoundingSphere(const Vector3f& center, float radius) : center_(center), radius_(radius) {}
  const Vector3f& center() const { return center_; }
  float radius() const { return radius_; }
  // (center - point).norm() <= radius; the squared norm in Eigen's a0 + (a1 + a2) order
  bool contains(const Vector3f& point) const {
    const float dx = center_[0] - point[0], dy = center_[1] - point[1], dz = center_[2] - point[2];
    return std::sqrt(dx * dx + (dy * dy + dz * dz)) <= radius_;
  }

 private:
  Vector3f center_;
  float radius_;
};
// exteriorDistance of the block's box to the centre: < radius (within) / > radius (outside), both strict
inline bool isBlockWithinRadius(const Index3D& block_index, float block_size, const Vector3f& center, float radius) {
  return getAABBOfBlock(block_size, block_index).exteriorDistance(center) < radius;
}
inline bool isBlockOutsideRadius(const Index3D& block_index, float block_size, const Vector3f& center, float radius) {
  return getAABBOfBlock(block_size, block_index).exteriorDistance(center) > radius;
}
inline std::vector<Index3D> getBlocksWithinRadius(const std::vector<Index3D>& blocks, float block_size, const Vector3f& center,
                                                  float radius) {
  std::vector<Index3D> out;
  for (const Index3D& b : blocks)
    if (isBlockWithinRadius(b, block_size, center, radius)) out.push_back(b);
  return out;
}
inline std::vector<Index3D> getBlocksOutsideRadius(const std::vector<Index3D>& blocks, float block_size, const Vector3f& center,
                                                   float radius) {
  std::vector<Index3D> out;
  for (const Index3D& b : blocks)
    if (isBlockOutsideRadius(b, block_size, center, radius)) out.push_back(b);
  return out;
}
}  // namespace nvblox
