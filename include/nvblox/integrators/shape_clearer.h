// nvblox/integrators/shape_clearer.h -- ShapeClearer<LayerType> (reference: nvblox/include/nvblox/integrators/shape_clearer.h,
// internal/cuda/impl/shape_clearer_impl.cuh:22-127), on the TSDF, occupancy and colour layers of a mapper.
#pragma once
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/geometry/bounding_shape.h"
#include "nvblox/map/layer.h"
#include "nvblox_b200.h"
namespace nvblox {
namespace b200_detail {
// Runs the shape clearer of the C ABI; returns the touched blocks in (x, y, z) order.
inline std::vector<Index3D> clearShapes(NvbMapper* m, int layer_id, const std::vector<BoundingShape>& shapes, int cap,
                                        bool mapper_tsdf) {
  std::vector<NvbBoundingShape> s;
  for (const BoundingShape& b : shapes) s.push_back(b.toNvb());
  std::vector<int32_t> raw(3 * (size_t)(cap > 0 ? cap : 1));
  int32_t n = 0;
  const int32_t rc = mapper_tsdf ? nvb_mapper_clear_tsdf_inside_shapes(m, s.data(), (int32_t)s.size(), raw.data(), cap, &n)
                                 : nvb_layer_clear_shapes(m, layer_id, s.data(), (int32_t)s.size(), raw.data(), cap, &n);
  if (rc != NVB_OK) throw std::runtime_error(std::string("ShapeClearer: ") + nvb_last_error());
  std::vector<Index3D> out;
  for (int i = 0; i < n && i < cap; i++) out.push_back(Index3D(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]));
  return out;
}
}  // namespace b200_detail

template <typename LayerType>
class ShapeClearer {
 public:
  ShapeClearer() = default;
  explicit ShapeClearer(std::shared_ptr<CudaStream>) {}
  // Resets the voxels whose centre lies in a shape, in the blocks a shape touches; returns those blocks. Synchronous.
  std::vector<Index3D> clear(const std::vector<BoundingShape>& bounding_shapes, LayerType* layer_ptr) {
    if (layer_ptr == nullptr) throw std::invalid_argument("ShapeClearer::clear: null layer");
    return b200_detail::clearShapes(layer_ptr->mapper_handle(), layer_ptr->layer_id(), bounding_shapes, layer_ptr->numBlocks(),
                                    false);
  }
};
}  // namespace nvblox
