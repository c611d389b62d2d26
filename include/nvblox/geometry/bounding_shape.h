// nvblox/geometry/bounding_shape.h -- BoundingShape, a sphere or an axis-aligned box (reference:
// nvblox/include/nvblox/geometry/bounding_shape.h:26-110, src/geometry/bounding_shape.cpp:20-66).
#pragma once
#include <cstdio>
#include <cstdlib>
#include "nvblox/geometry/bounding_boxes.h"
#include "nvblox/geometry/bounding_spheres.h"
#include "nvblox_b200.h"
namespace nvblox {
enum class ShapeType { kSphere, kAABB };

class BoundingShape {
 public:
  BoundingShape(const BoundingSphere& sphere) : type_(ShapeType::kSphere), sphere_(sphere) {}  // NOLINT (implicit, like the reference)
  BoundingShape(const AxisAlignedBoundingBox& aabb) : type_(ShapeType::kAABB), aabb_(aabb) {}  // NOLINT
  ShapeType type() const { return type_; }
  const BoundingSphere& sphere() const { check(ShapeType::kSphere); return sphere_; }
  const AxisAlignedBoundingBox& aabb() const { check(ShapeType::kAABB); return aabb_; }
  bool contains(const Vector3f& point) const {
    return type_ == ShapeType::kSphere ? sphere_.contains(point) : aabb_.contains(point);
  }
  // sphere: isBlockWithinRadius; box: isBlockTouchedByBoundingBox
  bool touchesBlock(const Index3D& block_index, float block_size) const {
    return type_ == ShapeType::kSphere ? isBlockWithinRadius(block_index, block_size, sphere_.center(), sphere_.radius())
                                       : isBlockTouchedByBoundingBox(block_index, block_size, aabb_);
  }
  // (not in the reference) the C-ABI description of the shape
  NvbBoundingShape toNvb() const {
    NvbBoundingShape s;
    if (type_ == ShapeType::kSphere) {
      s.type = NVB_SHAPE_SPHERE;
      for (int k = 0; k < 3; k++) s.a[k] = sphere_.center()[k], s.b[k] = 0.0f;
      s.b[0] = sphere_.radius();
    } else {
      s.type = NVB_SHAPE_AABB;
      for (int k = 0; k < 3; k++) s.a[k] = aabb_.min()[k], s.b[k] = aabb_.max()[k];
    }
    return s;
  }

 private:
  void check(ShapeType t) const {  // CHECK(type_ == ...) of the reference's accessors
    if (type_ != t) std::fprintf(stderr, "BoundingShape: wrong shape type\n"), std::abort();
  }
  ShapeType type_;
  BoundingSphere sphere_;
  AxisAlignedBoundingBox aabb_;
};
}  // namespace nvblox
