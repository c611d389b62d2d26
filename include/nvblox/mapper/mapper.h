// nvblox/mapper/mapper.h -- nvblox::Mapper restricted to the depth-integration path
// (reference: nvblox/include/nvblox/mapper/mapper.h:107-836), forwarding to libnvblox_b200.so.
//   Mapper(voxel_size_m, BlockMemoryPoolParams, ProjectiveLayerType, shared_ptr<CudaStream>)   mapper.h:119-124
//   integrateDepth(depth, T_L_C, camera)                   mapper.h:167-172
//   updateEsdf(UpdateFullLayer)                            mapper.h:326
//   tsdf_layer() / esdf_layer()                            mapper.h:372,393
//   tsdf_integrator() / esdf_integrator()                  mapper.h:442,534
//   Mapper(voxel_size_m, memory_type, ProjectiveLayerType::kOccupancy), occupancy_layer(), occupancy_integrator()
//                                                          mapper.h:52-53,119-124,374,456
//   decayTsdfAllVoxels / decayTsdfExcludeLastView / decayOccupancy...   mapper.h:218-233
//   tsdf_decay_integrator() / occupancy_decay_integrator()  mapper.h:496-504
//   clearOutsideRadius / clearTsdfInsideShapes / getClearedBlocks  mapper.h:237,350,713
#pragma once
#include <memory>
#include <type_traits>
#include <vector>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/integrators/weighting_function.h"
#include "nvblox/geometry/plane.h"
#include "nvblox/integrators/shape_clearer.h"
#include "nvblox/io/mesh_io.h"
#include "nvblox/io/pointcloud_io.h"
#include "nvblox/map/layer.h"
#include "nvblox/mesh/mesh_integrator.h"
#include "nvblox/sensors/camera.h"
#include "nvblox/sensors/image.h"
#include "nvblox_b200.h"
namespace nvblox {

enum class UpdateFullLayer { kNo, kYes };

// BlockMemoryPoolParams (map/internal/block_memory_pool_params.h:35-45): how the reference's block pools are sized. Here a layer
// is one slab (DESIGN.md section 5): num_preallocated_blocks becomes the slabs' initial capacity (0: the library's default),
// growth is by doubling whatever expansion_factor says, and blocks always live in device memory.
struct BlockMemoryPoolParams {
  BlockMemoryPoolParams() = default;
  BlockMemoryPoolParams(const MemoryType _memory_type) : memory_type(_memory_type) {}  // NOLINT (implicit, like the reference)
  MemoryType memory_type = MemoryType::kDevice;
  int num_preallocated_blocks = 0;
  float expansion_factor = 2.0f;
};

// MapperParams (mapper/mapper_params.h:46-70), the members this path consumes; applied with Mapper::setMapperParams.
struct EsdfIntegratorParams {
  float esdf_integrator_max_distance_m = 2.0f;
  float esdf_integrator_max_site_distance_vox = 1.0f;
  float esdf_integrator_min_weight = 1e-4f;
  float esdf_slice_min_height = 0.0f, esdf_slice_max_height = 1.0f, esdf_slice_height = 1.0f;
};
struct ProjectiveIntegratorParams {
  float projective_integrator_max_integration_distance_m = 7.0f;
  float projective_integrator_truncation_distance_vox = 4.0f;
  WeightingFunctionType projective_integrator_weighting_mode = WeightingFunctionType::kInverseSquareWeight;
  float projective_integrator_max_weight = 5.0f;
};
struct OccupancyIntegratorParams {
  float free_region_occupancy_probability = 0.3f, occupied_region_occupancy_probability = 0.7f;
  float unobserved_region_occupancy_probability = 0.5f, occupied_region_half_width_m = 0.1f;
};
struct MapperParams {
  MeshIntegratorParams mesh_integrator_params;  // mapper_params.h:54
  bool do_depth_preprocessing = false;          // mapper_params.h:33-37
  int depth_preprocessing_num_dilations = 4;    // mapper_params.h:39-42
  EsdfIntegratorParams esdf_integrator_params;
  ProjectiveIntegratorParams projective_integrator_params;
  OccupancyIntegratorParams occupancy_integrator_params;
};
enum class ProjectiveLayerType { kTsdf, kOccupancy, kTsdfWithFreespace, kNone };
enum class EsdfMode { k3D, k2D, kUnset };

namespace b200_detail {
// integrateFrame(depth_frame, T_L_C, camera, layer, updated_blocks) of either projective integrator.
inline void integrateFrame(NvbMapper* m, const MaskedDepthImageConstView& depth, const Transform& T_L_C,
                           const Camera& camera, std::vector<Index3D>* updated_blocks) {
  const MonoImageConstView& mk = depth.mask();
  int32_t n = 0;
  std::vector<int32_t> raw;
  int32_t cap = 0;
  if (updated_blocks) { cap = 1 << 16; raw.resize((size_t)cap * 3); }
  check(nvb_mapper_integrate_depth(m, depth.dataConstPtr(), mk.dataConstPtr(), (int)depth.mode(),
                                   depth.on_device() ? NVB_MEM_DEVICE : NVB_MEM_HOST, depth.rows(), depth.cols(),
                                   T_L_C.data(), camera.c_abi(), cap ? raw.data() : nullptr, cap, &n),
        "integrateFrame", nvb_last_error());
  if (updated_blocks) {
    if (n > cap) {
      raw.resize((size_t)n * 3);
      check(nvb_mapper_last_frame_blocks(m, raw.data(), n, &n), "integrateFrame", nvb_last_error());
    }
    updated_blocks->resize((size_t)n);
    for (int i = 0; i < n; i++) (*updated_blocks)[i] = Index3D(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
  }
}
}  // namespace b200_detail

// ViewCalculator's parameter surface (integrators/view_calculator.h:115-190): the workspace bounds and the raycast subsampling.
enum class WorkspaceBoundsType { kUnbounded, kHeightBounds, kBoundingBox };  // geometry/workspace_bounds.h:24
class ViewCalculator {
 public:
  explicit ViewCalculator(NvbMapper* m) : m_(m) {}
  WorkspaceBoundsType workspace_bounds_type() const { return (WorkspaceBoundsType)get().workspace_bounds_type; }
  void workspace_bounds_type(WorkspaceBoundsType t) { auto p = get(); p.workspace_bounds_type = (int)t; set(p); }
  Vector3f workspace_bounds_min_corner_m() const { auto p = get(); return Vector3f(p.workspace_min[0], p.workspace_min[1], p.workspace_min[2]); }
  void workspace_bounds_min_corner_m(const Vector3f& v) { auto p = get(); for (int a = 0; a < 3; a++) p.workspace_min[a] = v[a]; set(p); }
  Vector3f workspace_bounds_max_corner_m() const { auto p = get(); return Vector3f(p.workspace_max[0], p.workspace_max[1], p.workspace_max[2]); }
  void workspace_bounds_max_corner_m(const Vector3f& v) { auto p = get(); for (int a = 0; a < 3; a++) p.workspace_max[a] = v[a]; set(p); }
  bool cache_last_viewpoint() const { return nvb_mapper_get_cache_last_viewpoint(m_) != 0; }  // view_calculator.h:146-151
  void cache_last_viewpoint(bool v) { b200_detail::check(nvb_mapper_set_cache_last_viewpoint(m_, v ? 1 : 0), "cache_last_viewpoint", nvb_last_error()); }
  unsigned int raycast_subsampling_factor() const { return (unsigned int)get().raycast_subsampling; }
  void raycast_subsampling_factor(unsigned int f) { auto p = get(); p.raycast_subsampling = (int)f; set(p); }
 private:
  NvbTsdfParams get() const { NvbTsdfParams p; b200_detail::check(nvb_mapper_get_tsdf_params(m_, &p), "view calculator params", nvb_last_error()); return p; }
  void set(const NvbTsdfParams& p) { b200_detail::check(nvb_mapper_set_tsdf_params(m_, &p), "view calculator params", nvb_last_error()); }
  NvbMapper* m_;
};

// ProjectiveTsdfIntegrator's parameter surface + integrateFrame
// (integrators/projective_tsdf_integrator.h:48-121, internal/projective_integrator.h:56-85).
class ProjectiveTsdfIntegrator {
 public:
  explicit ProjectiveTsdfIntegrator(NvbMapper* m) : m_(m) {}
  float truncation_distance_vox() const { return get().truncation_distance_vox; }
  void truncation_distance_vox(float v) { auto p = get(); p.truncation_distance_vox = v; set(p); }
  float max_integration_distance_m() const { return get().max_integration_distance_m; }
  void max_integration_distance_m(float v) { auto p = get(); p.max_integration_distance_m = v; set(p); }
  float max_weight() const { return get().max_weight; }
  void max_weight(float v) { auto p = get(); p.max_weight = v; set(p); }
  float invalid_depth_decay_factor() const { return get().invalid_depth_decay_factor; }
  void invalid_depth_decay_factor(float v) { auto p = get(); p.invalid_depth_decay_factor = v; set(p); }
  WeightingFunctionType weighting_function_type() const { return (WeightingFunctionType)get().weighting_type; }
  void weighting_function_type(WeightingFunctionType t) { auto p = get(); p.weighting_type = (int)t; set(p); }
  float get_truncation_distance_m(float voxel_size) const { return truncation_distance_vox() * voxel_size; }
  ViewCalculator view_calculator() const { return ViewCalculator(m_); }  // internal/projective_integrator.h:118-119
  // integrateFrame(depth_frame, T_L_C, camera, layer, updated_blocks)
  void integrateFrame(const MaskedDepthImageConstView& depth, const Transform& T_L_C, const Camera& camera,
                      TsdfLayer* /*layer of this mapper*/, std::vector<Index3D>* updated_blocks = nullptr) {
    b200_detail::integrateFrame(m_, depth, T_L_C, camera, updated_blocks);
  }
 private:
  NvbTsdfParams get() const { NvbTsdfParams p; b200_detail::check(nvb_mapper_get_tsdf_params(m_, &p), "tsdf params", nvb_last_error()); return p; }
  void set(const NvbTsdfParams& p) { b200_detail::check(nvb_mapper_set_tsdf_params(m_, &p), "tsdf params", nvb_last_error()); }
  NvbMapper* m_;
};

// ProjectiveOccupancyIntegrator (integrators/projective_occupancy_integrator.h:36-131): sensor model + integrateFrame.
class ProjectiveOccupancyIntegrator {
 public:
  explicit ProjectiveOccupancyIntegrator(NvbMapper* m) : m_(m) {}
  float free_region_occupancy_probability() const { return get().free_region_occupancy_probability; }
  void free_region_occupancy_probability(float v) { auto p = get(); p.free_region_occupancy_probability = v; set(p); }
  float occupied_region_occupancy_probability() const { return get().occupied_region_occupancy_probability; }
  void occupied_region_occupancy_probability(float v) { auto p = get(); p.occupied_region_occupancy_probability = v; set(p); }
  float unobserved_region_occupancy_probability() const { return get().unobserved_region_occupancy_probability; }
  void unobserved_region_occupancy_probability(float v) { auto p = get(); p.unobserved_region_occupancy_probability = v; set(p); }
  float occupied_region_half_width_m() const { return get().occupied_region_half_width_m; }
  void occupied_region_half_width_m(float v) { auto p = get(); p.occupied_region_half_width_m = v; set(p); }
  float truncation_distance_vox() const { return ProjectiveTsdfIntegrator(m_).truncation_distance_vox(); }
  void truncation_distance_vox(float v) { ProjectiveTsdfIntegrator(m_).truncation_distance_vox(v); }
  float max_integration_distance_m() const { return ProjectiveTsdfIntegrator(m_).max_integration_distance_m(); }
  void max_integration_distance_m(float v) { ProjectiveTsdfIntegrator(m_).max_integration_distance_m(v); }
  void integrateFrame(const MaskedDepthImageConstView& depth, const Transform& T_L_C, const Camera& camera,
                      OccupancyLayer* /*layer of this mapper*/, std::vector<Index3D>* updated_blocks = nullptr) {
    b200_detail::integrateFrame(m_, depth, T_L_C, camera, updated_blocks);
  }
 private:
  NvbOccupancyParams get() const { NvbOccupancyParams p; b200_detail::check(nvb_mapper_get_occupancy_params(m_, &p), "occupancy params", nvb_last_error()); return p; }
  void set(const NvbOccupancyParams& p) { b200_detail::check(nvb_mapper_set_occupancy_params(m_, &p), "occupancy params", nvb_last_error()); }
  NvbMapper* m_;
};

// ProjectiveColorIntegrator (integrators/projective_appearance_integrator.h:44-194): parameters; integrateFrame is reached
// through Mapper::integrateColor (the integrator reads the mapper's TSDF layer and writes its colour layer).
class ProjectiveColorIntegrator {
 public:
  explicit ProjectiveColorIntegrator(NvbMapper* m) : m_(m) {}
  float max_integration_distance_m() const { return get().max_integration_distance_m; }
  void max_integration_distance_m(float v) { auto p = get(); p.max_integration_distance_m = v; set(p); }
  float truncation_distance_vox() const { return get().truncation_distance_vox; }
  void truncation_distance_vox(float v) { auto p = get(); p.truncation_distance_vox = v; set(p); }
  float get_truncation_distance_m(float voxel_size) const { return get().truncation_distance_vox * voxel_size; }
  float max_weight() const { return get().max_weight; }
  void max_weight(float v) { auto p = get(); p.max_weight = v; set(p); }
  float measurement_weight() const { return get().measurement_weight; }
  void measurement_weight(float v) { auto p = get(); p.measurement_weight = v; set(p); }
  int sphere_tracing_ray_subsampling_factor() const { return get().sphere_tracing_ray_subsampling_factor; }
  void sphere_tracing_ray_subsampling_factor(int v) { auto p = get(); p.sphere_tracing_ray_subsampling_factor = v; set(p); }
 private:
  NvbColorParams get() const { NvbColorParams p; b200_detail::check(nvb_mapper_get_color_params(m_, &p), "color params", nvb_last_error()); return p; }
  void set(const NvbColorParams& p) { b200_detail::check(nvb_mapper_set_color_params(m_, &p), "color params", nvb_last_error()); }
  NvbMapper* m_;
};

// FreespaceIntegrator (integrators/freespace_integrator.h:36-175): parameters + updateFreespaceLayer on a block list.
class FreespaceIntegrator {
 public:
  explicit FreespaceIntegrator(NvbMapper* m) : m_(m) {}
  float max_tsdf_distance_for_occupancy_m() const { return get().max_tsdf_distance_for_occupancy_m; }
  void max_tsdf_distance_for_occupancy_m(float v) { auto p = get(); p.max_tsdf_distance_for_occupancy_m = v; set(p); }
  Time max_unobserved_to_keep_consecutive_occupancy_ms() const { return get().max_unobserved_to_keep_consecutive_occupancy_ms; }
  void max_unobserved_to_keep_consecutive_occupancy_ms(Time v) { auto p = get(); p.max_unobserved_to_keep_consecutive_occupancy_ms = v; set(p); }
  Time min_duration_since_occupied_for_freespace_ms() const { return get().min_duration_since_occupied_for_freespace_ms; }
  void min_duration_since_occupied_for_freespace_ms(Time v) { auto p = get(); p.min_duration_since_occupied_for_freespace_ms = v; set(p); }
  Time min_consecutive_occupancy_duration_for_reset_ms() const { return get().min_consecutive_occupancy_duration_for_reset_ms; }
  void min_consecutive_occupancy_duration_for_reset_ms(Time v) { auto p = get(); p.min_consecutive_occupancy_duration_for_reset_ms = v; set(p); }
  bool check_neighborhood() const { return get().check_neighborhood != 0; }
  void check_neighborhood(bool v) { auto p = get(); p.check_neighborhood = v ? 1 : 0; set(p); }
  bool initialize_to_high_confidence_freespace() const { return get().initialize_to_high_confidence_freespace != 0; }
  void initialize_to_high_confidence_freespace(bool v) { auto p = get(); p.initialize_to_high_confidence_freespace = v ? 1 : 0; set(p); }
  // updateFreespaceLayer(block_indices, update_time_ms, tsdf_layer, {} /* no view */, freespace_layer)
  void updateFreespaceLayer(const std::vector<Index3D>& block_indices, Time update_time_ms, const TsdfLayer&, FreespaceLayer*) {
    std::vector<int32_t> raw(block_indices.size() * 3 + 3);
    for (size_t i = 0; i < block_indices.size(); i++) for (int a = 0; a < 3; a++) raw[3 * i + a] = block_indices[i][a];
    b200_detail::check(nvb_freespace_update_blocks(m_, raw.data(), (int32_t)block_indices.size(), update_time_ms, nullptr, 0, 0, 0,
                                                   nullptr, nullptr, 0.0f, 0.0f), "updateFreespaceLayer", nvb_last_error());
  }
 private:
  NvbFreespaceParams get() const { NvbFreespaceParams p; b200_detail::check(nvb_mapper_get_freespace_params(m_, &p), "freespace params", nvb_last_error()); return p; }
  void set(const NvbFreespaceParams& p) { b200_detail::check(nvb_mapper_set_freespace_params(m_, &p), "freespace params", nvb_last_error()); }
  NvbMapper* m_;
};

// TsdfDecayIntegrator / OccupancyDecayIntegrator parameter surfaces (integrators/tsdf_decay_integrator.h:73-101,
// occupancy_decay_integrator.h:72-101, internal/decay_integrator_base.h:50-58).
class TsdfDecayIntegrator {
 public:
  explicit TsdfDecayIntegrator(NvbMapper* m) : m_(m) {}
  bool deallocate_decayed_blocks() const { return get().deallocate_decayed_blocks != 0; }
  void deallocate_decayed_blocks(bool v) { auto p = get(); p.deallocate_decayed_blocks = v ? 1 : 0; set(p); }
  float decay_factor() const { return get().decay_factor; }
  void decay_factor(float v) { auto p = get(); p.decay_factor = v; set(p); }
  float decayed_weight_threshold() const { return get().decayed_weight_threshold; }
  void decayed_weight_threshold(float v) { auto p = get(); p.decayed_weight_threshold = v; set(p); }
  bool set_free_distance_on_decayed() const { return get().set_free_distance_on_decayed != 0; }
  void set_free_distance_on_decayed(bool v) { auto p = get(); p.set_free_distance_on_decayed = v ? 1 : 0; set(p); }
  float free_distance_vox() const { return get().free_distance_vox; }
  void free_distance_vox(float v) { auto p = get(); p.free_distance_vox = v; set(p); }
 private:
  NvbTsdfDecayParams get() const { NvbTsdfDecayParams p; b200_detail::check(nvb_mapper_get_tsdf_decay_params(m_, &p), "tsdf decay params", nvb_last_error()); return p; }
  void set(const NvbTsdfDecayParams& p) { b200_detail::check(nvb_mapper_set_tsdf_decay_params(m_, &p), "tsdf decay params", nvb_last_error()); }
  NvbMapper* m_;
};
class OccupancyDecayIntegrator {
 public:
  static constexpr float kDefaultProbabilityUnknown = 0.5f;
  static constexpr float kDefaultProbabilityFree = 0.49f;
  explicit OccupancyDecayIntegrator(NvbMapper* m) : m_(m) {}
  bool deallocate_decayed_blocks() const { return get().deallocate_decayed_blocks != 0; }
  void deallocate_decayed_blocks(bool v) { auto p = get(); p.deallocate_decayed_blocks = v ? 1 : 0; set(p); }
  float free_region_decay_probability() const { return get().free_region_decay_probability; }
  void free_region_decay_probability(float v) { auto p = get(); p.free_region_decay_probability = v; set(p); }
  float occupied_region_decay_probability() const { return get().occupied_region_decay_probability; }
  void occupied_region_decay_probability(float v) { auto p = get(); p.occupied_region_decay_probability = v; set(p); }
  float decay_to_probability() const { return get().decay_to_probability; }
  void decay_to_probability(float v) { auto p = get(); p.decay_to_probability = v; set(p); }
  void decay_to_free(bool v) { decay_to_probability(v ? kDefaultProbabilityFree : kDefaultProbabilityUnknown); }
 private:
  NvbOccupancyDecayParams get() const { NvbOccupancyDecayParams p; b200_detail::check(nvb_mapper_get_occupancy_decay_params(m_, &p), "occupancy decay params", nvb_last_error()); return p; }
  void set(const NvbOccupancyDecayParams& p) { b200_detail::check(nvb_mapper_set_occupancy_decay_params(m_, &p), "occupancy decay params", nvb_last_error()); }
  NvbMapper* m_;
};

// EsdfIntegrator (integrators/esdf_integrator.h:45-401): parameters + integrateBlocks.
class EsdfIntegrator {
 public:
  explicit EsdfIntegrator(NvbMapper* m) : m_(m) {}
  float max_esdf_distance_m() const { return get().max_esdf_distance_m; }
  void max_esdf_distance_m(float v) { auto p = get(); p.max_esdf_distance_m = v; set(p); }
  float max_site_distance_vox() const { return get().max_site_distance_vox; }
  void max_site_distance_vox(float v) { auto p = get(); p.max_site_distance_vox = v; set(p); }
  float min_weight() const { return get().min_weight; }
  void min_weight(float v) { auto p = get(); p.min_weight = v; set(p); }
  // the constant-z slice of the 2-D ESDF (esdf_integrator.h:216-256)
  float esdf_slice_min_height() const { return getSlice().slice_min_height_m; }
  void esdf_slice_min_height(float v) { auto p = getSlice(); p.slice_min_height_m = v; setSlice(p); }
  float esdf_slice_max_height() const { return getSlice().slice_max_height_m; }
  void esdf_slice_max_height(float v) { auto p = getSlice(); p.slice_max_height_m = v; setSlice(p); }
  float esdf_slice_height() const { return getSlice().slice_height_m; }
  void esdf_slice_height(float v) { auto p = getSlice(); p.slice_height_m = v; setSlice(p); }
  // integrateSlice(layer, block_indices, esdf_layer) (esdf_integrator.h:96-118)
  template <typename LayerT>
  void integrateSlice(const LayerT&, const std::vector<Index3D>& block_indices, EsdfLayer*) {
    std::vector<int32_t> raw(block_indices.size() * 3 + 3);
    for (size_t i = 0; i < block_indices.size(); i++) for (int a = 0; a < 3; a++) raw[3 * i + a] = block_indices[i][a];
    b200_detail::check(nvb_esdf_integrate_slice_blocks(m_, raw.data(), (int32_t)block_indices.size()), "integrateSlice", nvb_last_error());
  }
  // integrateSlice(layer, block_indices, ground_plane, esdf_layer) (esdf_integrator.h:136-173)
  template <typename LayerT>
  void integrateSlice(const LayerT&, const std::vector<Index3D>& block_indices, const Plane& ground_plane, EsdfLayer*) {
    std::vector<int32_t> raw(block_indices.size() * 3 + 3);
    for (size_t i = 0; i < block_indices.size(); i++) for (int a = 0; a < 3; a++) raw[3 * i + a] = block_indices[i][a];
    const float pl[4] = {ground_plane.normal()[0], ground_plane.normal()[1], ground_plane.normal()[2], ground_plane.d()};
    b200_detail::check(nvb_esdf_integrate_slice_planar_blocks(m_, pl, raw.data(), (int32_t)block_indices.size()), "integrateSlice",
                       nvb_last_error());
  }
  float slice_height_above_plane_m() const { return getSlice().slice_height_above_plane_m; }
  void slice_height_above_plane_m(float v) { auto p = getSlice(); p.slice_height_above_plane_m = v; setSlice(p); }
  float slice_height_thickness_m() const { return getSlice().slice_height_thickness_m; }
  void slice_height_thickness_m(float v) { auto p = getSlice(); p.slice_height_thickness_m = v; setSlice(p); }
  float occupied_threshold() const { return get().occupied_threshold; }
  void occupied_threshold(float v) { auto p = get(); p.occupied_threshold = v; set(p); }
  // integrateBlocks(const TsdfLayer&, const std::vector<Index3D>&, EsdfLayer*)
  void integrateBlocks(const OccupancyLayer&, const std::vector<Index3D>& block_indices, EsdfLayer* e) {
    integrateBlocksImpl(block_indices, e);
  }
  void integrateBlocks(const TsdfLayer&, const std::vector<Index3D>& block_indices, EsdfLayer* e) {
    integrateBlocksImpl(block_indices, e);
  }
 private:
  void integrateBlocksImpl(const std::vector<Index3D>& block_indices, EsdfLayer*) {
    std::vector<int32_t> raw(block_indices.size() * 3 + 3);
    for (size_t i = 0; i < block_indices.size(); i++) for (int a = 0; a < 3; a++) raw[3 * i + a] = block_indices[i][a];
    b200_detail::check(nvb_esdf_integrate_blocks(m_, raw.data(), (int32_t)block_indices.size()), "integrateBlocks", nvb_last_error());
  }
  NvbEsdfSliceParams getSlice() const { NvbEsdfSliceParams p; b200_detail::check(nvb_mapper_get_esdf_slice_params(m_, &p), "esdf slice params", nvb_last_error()); return p; }
  void setSlice(const NvbEsdfSliceParams& p) { b200_detail::check(nvb_mapper_set_esdf_slice_params(m_, &p), "esdf slice params", nvb_last_error()); }
  NvbEsdfParams get() const { NvbEsdfParams p; b200_detail::check(nvb_mapper_get_esdf_params(m_, &p), "esdf params", nvb_last_error()); return p; }
  void set(const NvbEsdfParams& p) { b200_detail::check(nvb_mapper_set_esdf_params(m_, &p), "esdf params", nvb_last_error()); }
  NvbMapper* m_;
};

class Mapper {
 public:
  Mapper() = delete;
  // Mapper(voxel_size_m, block_memory_pool_params, projective_layer_type, cuda_stream) -- mapper/mapper.h:119-124.
  // (BlockMemoryPoolParams converts from a MemoryType, so the older Mapper(voxel, MemoryType, layer type) spelling still works.)
  explicit Mapper(float voxel_size_m, BlockMemoryPoolParams block_memory_pool_params = BlockMemoryPoolParams(),
                  ProjectiveLayerType projective_layer_type = ProjectiveLayerType::kTsdf,
                  std::shared_ptr<CudaStream> cuda_stream = std::make_shared<CudaStreamOwning>())
      : projective_layer_type_(projective_layer_type), cuda_stream_(std::move(cuda_stream)) {
    NvbMapperOptions o;
    nvb_default_mapper_options(&o);
    o.voxel_size_m = voxel_size_m;
    if (block_memory_pool_params.num_preallocated_blocks > 0)
      o.tsdf_capacity_blocks = o.esdf_capacity_blocks = block_memory_pool_params.num_preallocated_blocks;
    o.keep_last_view = 1;  // Mapper::integrateDepth keeps the last posed depth image for the decay (mapper_impl.h:70-78)
    // ProjectiveLayerType::kNone has no projective layer to integrate into: nvb_mapper_create rejects it (-1).
    o.projective_layer_type = projective_layer_type == ProjectiveLayerType::kTsdf                 ? NVB_PROJECTIVE_TSDF
                              : projective_layer_type == ProjectiveLayerType::kOccupancy          ? NVB_PROJECTIVE_OCCUPANCY
                              : projective_layer_type == ProjectiveLayerType::kTsdfWithFreespace ? NVB_PROJECTIVE_TSDF_WITH_FREESPACE
                                                                                                  : -1;
    b200_detail::check(nvb_mapper_create(&o, &m_), "Mapper", nvb_last_error());
  }
  // Mapper(map_filepath, block_memory_pool_params, cuda_stream) -- mapper/mapper.h:128-134: a TSDF mapper holding the map of
  // the file (loadMap; a file that cannot be loaded leaves the mapper empty, as in the reference).
  Mapper(const std::string& map_filepath, BlockMemoryPoolParams block_memory_pool_params = BlockMemoryPoolParams(),
         std::shared_ptr<CudaStream> cuda_stream = std::make_shared<CudaStreamOwning>())
      : Mapper(0.05f, block_memory_pool_params, ProjectiveLayerType::kTsdf, std::move(cuda_stream)) {
    loadMap(map_filepath, block_memory_pool_params);
  }
  ~Mapper() { nvb_mapper_destroy(m_); }
  Mapper(const Mapper&) = delete;
  Mapper& operator=(const Mapper&) = delete;

  // template <typename SensorType> integrateDepth(depth_frame, T_L_C, sensor) -- mapper/mapper.h:167-180, mapper_impl.h:28-81.
  // SensorType = Camera is built (the Lidar model of sensors/lidar.h is not on this path).
  template <typename SensorType>
  void integrateDepth(const DepthImage& depth_frame, const Transform& T_L_C, const SensorType& sensor) {
    integrateDepth(MaskedDepthImageConstView(depth_frame, kMaskActiveEverywhere), T_L_C, sensor);
  }
  template <typename SensorType>
  void integrateDepth(const MaskedDepthImageConstView& depth_frame, const Transform& T_L_C, const SensorType& sensor) {
    static_assert(std::is_same<SensorType, Camera>::value, "only the Camera sensor model is built on this path");
    // Mapper::integrateDepth dispatches on the projective layer type (mapper_impl.h:28-81)
    b200_detail::integrateFrame(m_, depth_frame, T_L_C, sensor, nullptr);
  }
  // Mapper::setMapperParams (mapper/mapper.h:131): the members of MapperParams this path consumes
  void setMapperParams(const MapperParams& p) {
    do_depth_preprocessing(p.do_depth_preprocessing);
    color_mesh_integrator().min_weight(p.mesh_integrator_params.mesh_integrator_min_weight);
    color_mesh_integrator().weld_vertices(p.mesh_integrator_params.mesh_integrator_weld_vertices);
    depth_preprocessing_num_dilations(p.depth_preprocessing_num_dilations);
    auto ti = tsdf_integrator();
    ti.max_integration_distance_m(p.projective_integrator_params.projective_integrator_max_integration_distance_m);
    ti.truncation_distance_vox(p.projective_integrator_params.projective_integrator_truncation_distance_vox);
    ti.weighting_function_type(p.projective_integrator_params.projective_integrator_weighting_mode);
    ti.max_weight(p.projective_integrator_params.projective_integrator_max_weight);
    auto ei = esdf_integrator();
    ei.max_esdf_distance_m(p.esdf_integrator_params.esdf_integrator_max_distance_m);
    ei.max_site_distance_vox(p.esdf_integrator_params.esdf_integrator_max_site_distance_vox);
    ei.min_weight(p.esdf_integrator_params.esdf_integrator_min_weight);
    ei.esdf_slice_min_height(p.esdf_integrator_params.esdf_slice_min_height);
    ei.esdf_slice_max_height(p.esdf_integrator_params.esdf_slice_max_height);
    ei.esdf_slice_height(p.esdf_integrator_params.esdf_slice_height);
    if (projective_layer_type_ == ProjectiveLayerType::kOccupancy) {
      auto oi = occupancy_integrator();
      oi.free_region_occupancy_probability(p.occupancy_integrator_params.free_region_occupancy_probability);
      oi.occupied_region_occupancy_probability(p.occupancy_integrator_params.occupied_region_occupancy_probability);
      oi.unobserved_region_occupancy_probability(p.occupancy_integrator_params.unobserved_region_occupancy_probability);
      oi.occupied_region_half_width_m(p.occupancy_integrator_params.occupied_region_half_width_m);
    }
  }
  std::shared_ptr<CudaStream> cuda_stream() const { return cuda_stream_; }
  // Mapper::do_depth_preprocessing / depth_preprocessing_num_dilations (mapper.h; mapper.cpp:335-352): dilation of the
  // invalid regions of every depth image before it is integrated
  bool do_depth_preprocessing() const {
    int32_t en = 0, n = 0;
    b200_detail::check(nvb_mapper_get_depth_preprocessing(m_, &en, &n), "do_depth_preprocessing", nvb_last_error());
    return en != 0;
  }
  void do_depth_preprocessing(bool v) {
    b200_detail::check(nvb_mapper_set_depth_preprocessing(m_, v ? 1 : 0, depth_preprocessing_num_dilations()),
                       "do_depth_preprocessing", nvb_last_error());
  }
  int depth_preprocessing_num_dilations() const {
    int32_t en = 0, n = 0;
    b200_detail::check(nvb_mapper_get_depth_preprocessing(m_, &en, &n), "depth_preprocessing_num_dilations", nvb_last_error());
    return n;
  }
  void depth_preprocessing_num_dilations(int v) {
    b200_detail::check(nvb_mapper_set_depth_preprocessing(m_, do_depth_preprocessing() ? 1 : 0, v),
                       "depth_preprocessing_num_dilations", nvb_last_error());
  }
  // Mapper::markUnobservedTsdfFreeInsideRadius (mapper.h:352-356)
  void markUnobservedTsdfFreeInsideRadius(const Vector3f& center, float radius) {
    const float c[3] = {center[0], center[1], center[2]};
    b200_detail::check(nvb_mapper_mark_unobserved_free_inside_radius(m_, c, radius, nullptr, 0, nullptr),
                       "markUnobservedTsdfFreeInsideRadius", nvb_last_error());
  }
  // Mapper::clearOutsideRadius (mapper.h:350, src/mapper/mapper.cpp:473-492): the projective blocks farther than `radius` from
  // `center` are deallocated with their ESDF, freespace, colour and mesh twins, and join getClearedBlocks' set.
  void clearOutsideRadius(const Vector3f& center, float radius) {
    const float c[3] = {center[0], center[1], center[2]};
    b200_detail::check(nvb_mapper_clear_outside_radius(m_, c, radius, nullptr, 0, nullptr), "clearOutsideRadius", nvb_last_error());
  }
  // Mapper::clearTsdfInsideShapes (mapper.h:237, mapper.cpp:364-368): ShapeClearer<TsdfLayer> + addBlocksToUpdate
  void clearTsdfInsideShapes(const std::vector<BoundingShape>& shapes) {
    if (projective_layer_type_ == ProjectiveLayerType::kOccupancy) return;  // the TSDF layer is empty: nothing to clear
    b200_detail::clearShapes(m_, NVB_LAYER_TSDF, shapes, tsdf_layer().numBlocks(), true);
  }
  // Mapper::getClearedBlocks (mapper.h:713, mapper.cpp:509-521): the blocks deallocated since the last call (by
  // clearOutsideRadius or a decay), minus blocks_to_ignore, in (x, y, z) order; empties the set.
  std::vector<Index3D> getClearedBlocks(const std::vector<Index3D>& blocks_to_ignore) {
    std::vector<int32_t> ign;
    for (const Index3D& k : blocks_to_ignore) ign.push_back(k[0]), ign.push_back(k[1]), ign.push_back(k[2]);
    int32_t n = 0;
    b200_detail::check(nvb_mapper_get_cleared_blocks(m_, nullptr, 0, nullptr, 0, &n), "getClearedBlocks", nvb_last_error());
    std::vector<int32_t> raw(3 * (size_t)(n > 0 ? n : 1));
    b200_detail::check(nvb_mapper_get_cleared_blocks(m_, ign.empty() ? nullptr : ign.data(), (int32_t)(ign.size() / 3), raw.data(),
                                                     n, &n),
                       "getClearedBlocks", nvb_last_error());
    std::vector<Index3D> out;
    for (int i = 0; i < n; i++) out.push_back(Index3D(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]));
    return out;
  }
  // Mapper::integrateColor (mapper.h:202-207, mapper_impl.h:104-130)
  void integrateColor(const ColorImage& color_frame, const Transform& T_L_C, const Camera& camera) {
    integrateColor(MaskedColorImageConstView(color_frame, kMaskActiveEverywhere), T_L_C, camera);
  }
  void integrateColor(const MaskedColorImageConstView& color_frame, const Transform& T_L_C, const Camera& camera) {
    const MonoImageConstView& mask = color_frame.mask();
    b200_detail::check(nvb_mapper_integrate_color(m_, reinterpret_cast<const uint8_t*>(color_frame.dataConstPtr()), mask.dataConstPtr(),
                                                  color_frame.mode() == MaskMode::kInverted ? NVB_MASK_INVERTED : NVB_MASK_NON_INVERTED,
                                                  color_frame.on_device() ? NVB_MEM_DEVICE : NVB_MEM_HOST, color_frame.rows(),
                                                  color_frame.cols(), T_L_C.data(), camera.c_abi(), nullptr, 0, nullptr),
                       "integrateColor", nvb_last_error());
  }
  ColorLayer color_layer() const { return ColorLayer(m_, NVB_LAYER_COLOR); }
  // Mapper::color_mesh_layer / color_mesh_integrator / updateColorMesh (mapper.h; src/mapper/mapper.cpp:371-406)
  ColorMeshLayer color_mesh_layer() const { return ColorMeshLayer(m_); }
  ColorMeshIntegrator color_mesh_integrator() const { return ColorMeshIntegrator(m_); }
  void updateColorMesh(UpdateFullLayer full = UpdateFullLayer::kNo) {
    b200_detail::check(nvb_mapper_update_mesh(m_, full == UpdateFullLayer::kYes ? 1 : 0), "updateColorMesh", nvb_last_error());
  }
  ProjectiveColorIntegrator color_integrator() const { return ProjectiveColorIntegrator(m_); }
  void updateEsdf(UpdateFullLayer full = UpdateFullLayer::kNo) {
    b200_detail::check(nvb_mapper_update_esdf(m_, full == UpdateFullLayer::kYes ? 1 : 0), "updateEsdf", nvb_last_error());
  }
  // Mapper::updateEsdfSlice (mapper.h:343): the 2-D ESDF on the slice layer
  void updateEsdfSlice(UpdateFullLayer full = UpdateFullLayer::kNo) {
    b200_detail::check(nvb_mapper_update_esdf_slice(m_, full == UpdateFullLayer::kYes ? 1 : 0), "updateEsdfSlice", nvb_last_error());
  }
  // Mapper::updateEsdfSlice(update_full_layer, ground_plane) (mapper.h:338-344): the band follows the ground plane
  void updateEsdfSlice(UpdateFullLayer full, const Plane& ground_plane) {
    const float pl[4] = {ground_plane.normal()[0], ground_plane.normal()[1], ground_plane.normal()[2], ground_plane.d()};
    b200_detail::check(nvb_mapper_update_esdf_slice_planar(m_, pl, full == UpdateFullLayer::kYes ? 1 : 0), "updateEsdfSlice",
                       nvb_last_error());
  }
  void clear() { b200_detail::check(nvb_mapper_clear(m_), "clear", nvb_last_error()); }
  // Mapper::saveLayerCake / loadMap (mapper.h:662-671, mapper.cpp:636-687): the map in the reference's .nvblx file. loadMap
  // takes the voxel size from the file and returns false (the map unchanged) on a file it cannot load; nvb_last_error()
  // says why. Tables this mapper cannot hold are skipped (nvb_mapper_load_map).
  bool saveLayerCake(const std::string& filename) const { return nvb_mapper_save_map(m_, filename.c_str()) == NVB_OK; }
  bool saveLayerCake(const char* filename) const { return saveLayerCake(std::string(filename)); }
  bool loadMap(const std::string& filename, const BlockMemoryPoolParams = BlockMemoryPoolParams()) {
    return nvb_mapper_load_map(m_, filename.c_str(), nullptr) == NVB_OK;
  }
  bool loadMap(const char* filename, BlockMemoryPoolParams block_memory_pool_params = BlockMemoryPoolParams()) {
    return loadMap(std::string(filename), block_memory_pool_params);
  }
  // Mapper::save*AsPly (mapper.h:676-697)
  bool saveColorMeshAsPly(const std::string& filename) const { return io::outputColorMeshLayerToPly(color_mesh_layer(), filename); }
  bool saveEsdfAsPly(const std::string& filename) const { return io::outputVoxelLayerToPly(esdf_layer(), filename); }
  bool saveTsdfAsPly(const std::string& filename) const { return io::outputVoxelLayerToPly(tsdf_layer(), filename); }
  bool saveFreespaceAsPly(const std::string& filename) const { return io::outputVoxelLayerToPly(freespace_layer(), filename); }
  bool saveOccupancyAsPly(const std::string& filename) const { return io::outputVoxelLayerToPly(occupancy_layer(), filename); }
  // Mapper::updateFreespace(update_time_ms, T_L_C, camera, depth_frame, update_full_layer) (mapper.h:196-214)
  void updateFreespace(Time update_time_ms, const Transform& T_L_C, const Camera& camera,
                       const DepthImageConstView& depth_frame, UpdateFullLayer full = UpdateFullLayer::kNo) {
    b200_detail::check(nvb_mapper_update_freespace(m_, update_time_ms, depth_frame.dataConstPtr(),
                                                   depth_frame.on_device() ? NVB_MEM_DEVICE : NVB_MEM_HOST, depth_frame.rows(),
                                                   depth_frame.cols(), T_L_C.data(), camera.c_abi(),
                                                   full == UpdateFullLayer::kYes ? 1 : 0), "updateFreespace", nvb_last_error());
  }
  void updateFreespace(Time update_time_ms, UpdateFullLayer full = UpdateFullLayer::kNo) {
    b200_detail::check(nvb_mapper_update_freespace(m_, update_time_ms, nullptr, 0, 0, 0, nullptr, nullptr,
                                                   full == UpdateFullLayer::kYes ? 1 : 0), "updateFreespace", nvb_last_error());
  }
  FreespaceLayer freespace_layer() const { return FreespaceLayer(m_, NVB_LAYER_FREESPACE); }
  FreespaceIntegrator freespace_integrator() const { return FreespaceIntegrator(m_); }
  // Decay of the projective layer; deallocated blocks also leave the ESDF layer (mapper.h:218-233).
  void decayTsdfAllVoxels() { decayAll(ProjectiveLayerType::kTsdf); }
  void decayOccupancyAllVoxels() { decayAll(ProjectiveLayerType::kOccupancy); }
  void decayTsdfExcludeLastView() { decayLastView(ProjectiveLayerType::kTsdf); }
  void decayOccupancyExcludeLastView() { decayLastView(ProjectiveLayerType::kOccupancy); }
  // the reference's spelling (mapper/mapper.h:226-233: the sensor type of the last integrated view)
  template <typename SensorType>
  void decayTsdfExcludeLastView() { static_assert(std::is_same<SensorType, Camera>::value, "Camera only"); decayTsdfExcludeLastView(); }
  template <typename SensorType>
  void decayOccupancyExcludeLastView() { static_assert(std::is_same<SensorType, Camera>::value, "Camera only"); decayOccupancyExcludeLastView(); }
  TsdfDecayIntegrator tsdf_decay_integrator() const { return TsdfDecayIntegrator(m_); }
  OccupancyDecayIntegrator occupancy_decay_integrator() const { return OccupancyDecayIntegrator(m_); }
  float voxel_size_m() const { return nvb_mapper_voxel_size(m_); }
  TsdfLayer tsdf_layer() const { return TsdfLayer(m_, NVB_LAYER_TSDF); }
  OccupancyLayer occupancy_layer() const { return OccupancyLayer(m_, NVB_LAYER_OCCUPANCY); }
  EsdfLayer esdf_layer() const { return EsdfLayer(m_, NVB_LAYER_ESDF); }
  ProjectiveLayerType projective_layer_type() const { return projective_layer_type_; }
  ProjectiveOccupancyIntegrator occupancy_integrator() const { return ProjectiveOccupancyIntegrator(m_); }
  ProjectiveTsdfIntegrator tsdf_integrator() const { return ProjectiveTsdfIntegrator(m_); }
  EsdfIntegrator esdf_integrator() const { return EsdfIntegrator(m_); }
  NvbMapper* c_abi() const { return m_; }
 private:
  void requireLayer(ProjectiveLayerType t) const {
    const bool tsdf_like = projective_layer_type_ == ProjectiveLayerType::kTsdf || projective_layer_type_ == ProjectiveLayerType::kTsdfWithFreespace;
    if (!(projective_layer_type_ == t || (t == ProjectiveLayerType::kTsdf && tsdf_like))) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "decay", "the mapper does not hold that projective layer");
  }
  void decayAll(ProjectiveLayerType t) {
    requireLayer(t);
    int32_t n = 0;
    b200_detail::check(nvb_mapper_decay(m_, nullptr, nullptr, 0, 0, 0, nullptr, nullptr, nullptr, 0, &n), "decay", nvb_last_error());
  }
  void decayLastView(ProjectiveLayerType t) {
    requireLayer(t);
    int32_t n = 0;
    b200_detail::check(nvb_mapper_decay_exclude_last_view(m_, nullptr, nullptr, 0, &n), "decay", nvb_last_error());
  }
  NvbMapper* m_ = nullptr;
  ProjectiveLayerType projective_layer_type_;
  std::shared_ptr<CudaStream> cuda_stream_;
};
}  // namespace nvblox
