// nvblox/primitives/scene.h -- nvblox::primitives::Scene (reference: nvblox/include/nvblox/primitives/scene.h,
// src/primitives/scene.cpp, internal/impl/scene_impl.h). Construction, getSignedDistanceToPoint and getRayIntersection run on
// the host; generateDepthImageFromScene and generateLayerFromScene run on the GPU (nvb_scene_render_depth,
// nvb_scene_generate_layer) and return once their outputs are written. The layers are a mapper's TSDF, occupancy or freespace
// layer; the reference's setVoxel exists for those three voxel types only.
#pragma once
#include <memory>
#include <vector>
#include "nvblox/geometry/plane.h"
#include "nvblox/map/layer.h"
#include "nvblox/primitives/primitives.h"
#include "nvblox/sensors/camera.h"
#include "nvblox/sensors/image.h"
#include "nvblox_b200.h"
namespace nvblox {
namespace primitives {

class Scene {
 public:
  Scene() : aabb_(Vector3f(-5.0f, -5.0f, -1.0f), Vector3f(5.0f, 5.0f, 9.0f)) {}

  /// Create an environment by adding primitives, which are then owned by the scene.
  void addPrimitive(std::unique_ptr<Primitive> primitive) { primitives_.emplace_back(std::move(primitive)); }
  /// A ground plane (normal up) at a height on the z axis.
  void addGroundLevel(float height) { primitives_.emplace_back(new Plane(Vector3f(0.0f, 0.0f, height), Vector3f(0.0f, 0.0f, 1.0f))); }
  /// A ceiling (normal down) at a height on the z axis.
  void addCeiling(float height) { primitives_.emplace_back(new Plane(Vector3f(0.0f, 0.0f, height), Vector3f(0.0f, 0.0f, -1.0f))); }
  /// Four infinite walls facing inwards: x_min, x_max, y_min, y_max in that order.
  void addPlaneBoundaries(float x_min, float x_max, float y_min, float y_max) {
    primitives_.emplace_back(new Plane(Vector3f(x_min, 0.0f, 0.0f), Vector3f(1.0f, 0.0f, 0.0f)));
    primitives_.emplace_back(new Plane(Vector3f(x_max, 0.0f, 0.0f), Vector3f(-1.0f, 0.0f, 0.0f)));
    primitives_.emplace_back(new Plane(Vector3f(0.0f, y_min, 0.0f), Vector3f(0.0f, 1.0f, 0.0f)));
    primitives_.emplace_back(new Plane(Vector3f(0.0f, y_max, 0.0f), Vector3f(0.0f, -1.0f, 0.0f)));
  }
  /// Deletes all objects.
  void clear() { primitives_.clear(); }

  /// The camera-frame depth of each pixel's nearest hit within max_dist, invalid_depth elsewhere. The image is resized to
  /// the camera; it holds host memory, as the reference requires.
  void generateDepthImageFromScene(const Camera& sensor, const Transform& T_S_C, float max_dist, DepthImage* depth_frame,
                                   const float invalid_depth = 0.f) const {
    if (!depth_frame) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "generateDepthImageFromScene", "null image");
    if (depth_frame->rows() != sensor.height() || depth_frame->cols() != sensor.width())
      *depth_frame = DepthImage(sensor.height(), sensor.width(), depth_frame->memory_type());
    std::vector<NvbPrimitive> prims;
    const NvbScene s = c_abi(&prims);
    b200_detail::check(nvb_scene_render_depth(&s, sensor.c_abi(), T_S_C.data(), max_dist, invalid_depth, NVB_MEM_HOST,
                                              depth_frame->dataPtr(), nullptr),
                       "generateDepthImageFromScene", nvb_last_error());
  }

  /// The ground-truth layer: every block the AABB touches is allocated, and every voxel inside the AABB written.
  template <typename VoxelType>
  void generateLayerFromScene(float max_dist, VoxelBlockLayer<VoxelType>* layer) const {
    if (!layer) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "generateLayerFromScene", "null layer");
    std::vector<NvbPrimitive> prims;
    const NvbScene s = c_abi(&prims);
    b200_detail::check(nvb_scene_generate_layer(layer->mapper_handle(), layer->layer_id(), &s, max_dist),
                       "generateLayerFromScene", nvb_last_error());
  }

  /// Distance to the nearest primitive, starting at max_dist: positive distances are capped there, negative ones are not.
  float getSignedDistanceToPoint(const Vector3f& coords, float max_dist) const {
    float min_dist = max_dist;
    for (const std::unique_ptr<Primitive>& primitive : primitives_) {
      const float d = primitive->getDistanceToPoint(coords);
      if (d < min_dist) min_dist = d;
    }
    return min_dist;
  }

  /// The first primitive with the nearest intersection of the ray within max_dist.
  bool getRayIntersection(const Vector3f& ray_origin, const Vector3f& ray_direction, float max_dist,
                          Vector3f* ray_intersection, float* ray_dist) const {
    *ray_intersection = Vector3f::Zero();
    *ray_dist = max_dist;
    bool ray_valid = false;
    for (const std::unique_ptr<Primitive>& primitive : primitives_) {
      Vector3f p;
      float d;
      if (primitive->getRayIntersection(ray_origin, ray_direction, max_dist, &p, &d) && (!ray_valid || d < *ray_dist)) {
        ray_valid = true;
        *ray_dist = d;
        *ray_intersection = p;
      }
    }
    return ray_valid;
  }

  const AxisAlignedBoundingBox& aabb() const { return aabb_; }
  AxisAlignedBoundingBox& aabb() { return aabb_; }

  std::vector<Primitive::Type> getPrimitiveTypeList() const {
    std::vector<Primitive::Type> types;
    for (const std::unique_ptr<Primitive>& primitive : primitives_) types.push_back(primitive->getType());
    return types;
  }

 protected:
  NvbScene c_abi(std::vector<NvbPrimitive>* prims) const {
    for (const std::unique_ptr<Primitive>& primitive : primitives_) prims->push_back(primitive->c_abi());
    NvbScene s{};
    s.primitives = prims->data();
    s.num_primitives = (int32_t)prims->size();
    for (int k = 0; k < 3; k++) s.aabb_min[k] = aabb_.min()[k], s.aabb_max[k] = aabb_.max()[k];
    return s;
  }

  std::vector<std::unique_ptr<Primitive>> primitives_;
  AxisAlignedBoundingBox aabb_;
};

}  // namespace primitives
}  // namespace nvblox
