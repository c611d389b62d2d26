// nvblox/geometry/bounding_boxes.h -- block boxes (reference: nvblox/include/nvblox/geometry/bounding_boxes.h,
// internal/impl/bounding_boxes_impl.h:20-60). AxisAlignedBoundingBox itself lives in plane.h.
#pragma once
#include "nvblox/geometry/plane.h"
namespace nvblox {
// getAABBOfBlock (bounding_boxes_impl.h:55-60): [index * block_size, (index + 1) * block_size] per axis, in float
inline AxisAlignedBoundingBox getAABBOfBlock(float block_size, const Index3D& block_index) {
  Vector3f mn, mx;
  for (int k = 0; k < 3; k++) mn[k] = (float)block_index[k] * block_size, mx[k] = ((float)block_index[k] + 1.0f) * block_size;
  return AxisAlignedBoundingBox(mn, mx);
}
// isBlockTouchedByBoundingBox (bounding_boxes_impl.h:22-26)
inline bool isBlockTouchedByBoundingBox(const Index3D& block_index, float block_size, const AxisAlignedBoundingBox& aabb_L) {
  return aabb_L.intersects(getAABBOfBlock(block_size, block_index));
}
}  // namespace nvblox
