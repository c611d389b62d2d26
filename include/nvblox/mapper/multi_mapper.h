// nvblox/mapper/multi_mapper.h -- nvblox::MultiMapper (reference: nvblox/include/nvblox/mapper/multi_mapper.h:26-330,
// mapper/internal/impl/multi_mapper_impl.h), the object nvblox_ros actually drives
// (nvblox_ros/src/lib/nvblox_node.cpp:187-204, :781, :1058-1062, :1261-1264), as a facade over one or two Mappers of
// libnvblox_b200.so:
//   kStaticTsdf / kStaticOccupancy : background mapper only (multi_mapper_impl.h:27-29);
//   kDynamic                       : background = TSDF + freespace layer, updated after every depth frame
//                                    (multi_mapper_impl.h:115-119); foreground = occupancy of the dynamic depth pixels. The
//                                    mask comes from DynamicsDetection on the background's freespace layer as the previous
//                                    frame left it, cleaned by the connected-component filter (multi_mapper_impl.h:60-124),
//                                    all on the device; a mask given with setDynamicMask takes precedence over the detection;
//   kHumanWithStatic*              : the mask overload runs the reference's sequence (multi_mapper_impl.h:127-155) on the
//                                    device: the connected-component filter on the mask (remove_small_connected_components),
//                                    the ImageMasker split of the depth frame by the mask seen from the mask camera (T_CM_CD,
//                                    with occlusion), then the background frame into the background mapper and the
//                                    foreground frame into the foreground occupancy mapper. Kept deviation: a call with
//                                    T_CM_CD = identity (within 1e-6) and a mask camera equal to the depth camera (intrinsics, size,
//                                    distortion) integrates as before this path existed, through masked views of the frame
//                                    and without the filter; the split still runs, so the getLastDepthFrame* getters
//                                    describe the frame.
// updateEsdf(): 3-D or 2-D (slice) ESDF of the mappers in use (multi_mapper.cpp updateEsdfOfMapper).
#pragma once
#include <memory>
#include <optional>
#include "nvblox/dynamics/dynamics_detection.h"
#include "nvblox/experimental/ground_plane/ground_plane_estimator.h"
#include "nvblox/mapper/mapper.h"
#include "nvblox/semantics/image_masker.h"
#include "nvblox/sensors/mask_preprocessor.h"
namespace nvblox {

enum class MappingType { kStaticTsdf, kStaticOccupancy, kDynamic, kHumanWithStaticTsdf, kHumanWithStaticOccupancy };
inline bool isHumanMapping(MappingType t) { return t == MappingType::kHumanWithStaticTsdf || t == MappingType::kHumanWithStaticOccupancy; }
inline bool isDynamicMapping(MappingType t) { return t == MappingType::kDynamic; }
inline bool isStaticOccupancy(MappingType t) { return t == MappingType::kStaticOccupancy || t == MappingType::kHumanWithStaticOccupancy; }
inline bool isUsingBothMappers(MappingType t) { return isHumanMapping(t) || isDynamicMapping(t); }

struct MultiMapperParams {
  // kDynamic without setDynamicMask: the detected mask loses its components of fewer than threshold pixels
  int connected_mask_component_size_threshold = 2000;
  bool remove_small_connected_components = true;
  // updateEsdf estimates the ground plane from the background TSDF first; a 2-D ESDF then follows it (multi_mapper.h)
  bool experimental_use_ground_plane_estimation = false;
  GroundPlaneEstimatorParams ground_plane_estimator_params;
};

class MultiMapper {
 public:
  MultiMapper(float voxel_size_m, MappingType mapping_type, EsdfMode esdf_mode, MemoryType memory_type = MemoryType::kDevice,
              std::shared_ptr<CudaStream> cuda_stream = std::make_shared<CudaStreamOwning>())
      : mapping_type_(mapping_type), esdf_mode_(esdf_mode), dynamic_detector_(cuda_stream) {
    // multi_mapper.cpp: background layer type by mapping type; the foreground mapper is always occupancy
    const ProjectiveLayerType bg = isStaticOccupancy(mapping_type)   ? ProjectiveLayerType::kOccupancy
                                   : isDynamicMapping(mapping_type) ? ProjectiveLayerType::kTsdfWithFreespace
                                                                    : ProjectiveLayerType::kTsdf;
    background_mapper_ = std::make_shared<Mapper>(voxel_size_m, BlockMemoryPoolParams(memory_type), bg, cuda_stream);
    if (isUsingBothMappers(mapping_type))
      foreground_mapper_ = std::make_shared<Mapper>(voxel_size_m, BlockMemoryPoolParams(memory_type), ProjectiveLayerType::kOccupancy, cuda_stream);
    image_masker_ = std::make_unique<ImageMasker>(cuda_stream, background_mapper_->c_abi());
  }
  void setMultiMapperParams(const MultiMapperParams& p) {
    params_ = p;
    ground_plane_estimator().setParams(p.ground_plane_estimator_params);  // multi_mapper.cpp:121-128
  }
  const MultiMapperParams& getMultiMapperParams() const { return params_; }
  void setMapperParams(const MapperParams& background_mapper_params,
                       const std::optional<MapperParams>& foreground_mapper_params = std::nullopt) {
    background_mapper_->setMapperParams(background_mapper_params);
    if (foreground_mapper_ && foreground_mapper_params.has_value()) foreground_mapper_->setMapperParams(*foreground_mapper_params);
  }

  // integrateDepth(depth_frame, T_L_CD, depth_sensor, update_time_ms) -- multi_mapper.h:146-151
  template <typename SensorType>
  void integrateDepth(const DepthImage& depth_frame, const Transform& T_L_CD, const SensorType& depth_sensor,
                      const std::optional<Time>& update_time_ms = std::nullopt) {
    background_mapper_->integrateDepth(depth_frame, T_L_CD, depth_sensor);
    if (!isDynamicMapping(mapping_type_)) return;
    if (!update_time_ms.has_value()) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "MultiMapper::integrateDepth", "dynamic mapping needs update_time_ms");
    if (dynamic_mask_.has_value())
      foreground_mapper_->integrateDepth(MaskedDepthImageConstView(depth_frame, *dynamic_mask_), T_L_CD, depth_sensor);
    else
      integrateDetectedDynamics(depth_frame, T_L_CD, depth_sensor);
    background_mapper_->updateFreespace(*update_time_ms, T_L_CD, depth_sensor, DepthImageConstView(depth_frame));
  }
  // The dynamic mask of the depth frames that follow (kDynamic): >0 = dynamic pixel. Once set, it replaces the detection.
  void setDynamicMask(const MonoImageConstView& mask) { dynamic_mask_ = mask; }
  // getLastDynamicFrameMaskOverlay / getLastDynamicPointcloud (multi_mapper.h:296-297): the detector's outputs of the last
  // kDynamic frame (empty while a setDynamicMask mask is in use)
  const ColorImage& getLastDynamicFrameMaskOverlay() { return dynamic_detector_.getDynamicOverlayImage(); }
  const Pointcloud& getLastDynamicPointcloud() { return dynamic_detector_.getDynamicPointcloudDevice(); }

  // integrateDepth(depth_frame, mask, T_L_CD, T_CM_CD, depth_sensor, mask_sensor) -- multi_mapper.h:205-209 (human mapping):
  // the mask (> 0: human) is an image of mask_sensor, whose frame is T_CM_CD * (depth camera frame).
  template <typename SensorType>
  void integrateDepth(const DepthImage& depth_frame, const MonoImage& mask, const Transform& T_L_CD, const Transform& T_CM_CD,
                      const SensorType& depth_sensor, const SensorType& mask_sensor) {
    if (!isHumanMapping(mapping_type_)) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "MultiMapper::integrateDepth", "a mask is only valid for human mapping");
    if (isIdentity(T_CM_CD) && sameCamera(*depth_sensor.c_abi(), *mask_sensor.c_abi())) {
      // the kept deviation (see the top of this file): masked views, no filter; the split only feeds the getters
      image_masker_->split(depth_frame, mask, T_CM_CD, depth_sensor, mask_sensor, true);
      foreground_mapper_->integrateDepth(MaskedDepthImageConstView(depth_frame, MonoImageConstView(mask)), T_L_CD, depth_sensor);
      background_mapper_->integrateDepth(MaskedDepthImageConstView(depth_frame, MonoImageConstView(mask), MaskMode::kInverted), T_L_CD,
                                         depth_sensor);
      return;
    }
    NvbMapper* bg = background_mapper_->c_abi();
    const MonoImage* split_mask = &mask;
    if (params_.remove_small_connected_components) {  // on the background mapper's stream, like the split
      if (cleaned_mask_.rows() != mask.rows() || cleaned_mask_.cols() != mask.cols()) cleaned_mask_ = MonoImage(mask.rows(), mask.cols());
      b200_detail::check(nvb_mapper_remove_small_components(bg, mask.dataConstPtr(), cleaned_mask_.dataPtr(), NVB_MEM_HOST, mask.rows(),
                                                            mask.cols(), params_.connected_mask_component_size_threshold),
                         "removeSmallConnectedComponents", nvb_last_error());
      split_mask = &cleaned_mask_;
    }
    image_masker_->split(depth_frame, *split_mask, T_CM_CD, depth_sensor, mask_sensor, true);
    NvbSplitBuffers b;
    b200_detail::check(nvb_mapper_split_device_buffers(bg, &b), "MultiMapper::integrateDepth", nvb_last_error());
    // The background integration follows the split on the same stream; the foreground's is ordered behind it by an event.
    // Both integrateDepth calls return only when their kernels are done, so the split's buffers are no longer read when
    // the next frame's split overwrites them.
    background_mapper_->integrateDepth(DepthImageConstView(b.background, b.rows, b.cols, MemoryType::kDevice), T_L_CD, depth_sensor);
    b200_detail::check(nvb_mapper_wait_for(foreground_mapper_->c_abi(), bg), "MultiMapper::integrateDepth", nvb_last_error());
    foreground_mapper_->integrateDepth(DepthImageConstView(b.foreground, b.rows, b.cols, MemoryType::kDevice), T_L_CD, depth_sensor);
  }
  // getLastDepthFrameBackground / Foreground / MaskOverlay (multi_mapper.h:290-294): the last human-mapping split, read back
  // from the device (empty before the first)
  const DepthImage& getLastDepthFrameBackground() { return readSplit(NVB_SPLIT_BACKGROUND, &depth_frame_background_); }
  const DepthImage& getLastDepthFrameForeground() { return readSplit(NVB_SPLIT_FOREGROUND, &depth_frame_foreground_); }
  const ColorImage& getLastDepthFrameMaskOverlay() {
    int32_t rows = 0, cols = 0;
    NvbMapper* bg = background_mapper_->c_abi();
    b200_detail::check(nvb_mapper_split_output(bg, NVB_SPLIT_OVERLAY, nullptr, NVB_MEM_HOST, &rows, &cols), "getLastDepthFrameMaskOverlay", nvb_last_error());
    depth_frame_overlay_ = ColorImage(rows, cols, MemoryType::kHost);
    if (rows > 0 && cols > 0)
      b200_detail::check(nvb_mapper_split_output(bg, NVB_SPLIT_OVERLAY, reinterpret_cast<uint8_t*>(depth_frame_overlay_.dataPtr()),
                                                 NVB_MEM_HOST, &rows, &cols),
                         "getLastDepthFrameMaskOverlay", nvb_last_error());
    return depth_frame_overlay_;
  }
  // image_masker() -- the human split's parameters (occlusion threshold, invalid pixel values)
  ImageMasker& image_masker() { return *image_masker_; }

  // integrateColor(color_frame, T_L_C, sensor) -- multi_mapper.h:237-239: colour only goes to the background mapper
  template <typename SensorType>
  void integrateColor(const ColorImage& color_frame, const Transform& T_L_C, const SensorType& sensor) {
    background_mapper_->integrateColor(color_frame, T_L_C, sensor);
  }
  template <typename SensorType>
  void integrateColor(const ColorImage& color_frame, const MonoImage& mask, const Transform& T_L_C, const SensorType& sensor) {
    // human mapping: the pixels that are NOT on a human colour the static map (multi_mapper.h:241-250)
    background_mapper_->integrateColor(MaskedColorImageConstView(color_frame, MonoImageConstView(mask), MaskMode::kInverted), T_L_C, sensor);
  }

  // updateEsdf() -- multi_mapper.h:266, multi_mapper.cpp:159-175: with experimental_use_ground_plane_estimation the plane
  // is computed from the background mapper's TSDF (none on an occupancy background), and a 2-D ESDF of both mappers follows
  // it; without a plane the slice is the constant-z one.
  void updateEsdf() {
    std::optional<Plane> plane;
    if (params_.experimental_use_ground_plane_estimation)
      plane = ground_plane_estimator().computeGroundPlane(background_mapper_->tsdf_layer());
    updateEsdfOfMapper(background_mapper_, plane);
    if (foreground_mapper_) updateEsdfOfMapper(foreground_mapper_, plane);
  }
  // ground_plane_estimator() -- the estimator of the background mapper
  GroundPlaneEstimator ground_plane_estimator() const { return GroundPlaneEstimator(background_mapper_->c_abi()); }

  const Mapper& background_mapper() const { return *background_mapper_; }
  const Mapper& foreground_mapper() const { return *foreground_mapper_; }
  std::shared_ptr<Mapper> background_mapper() { return background_mapper_; }
  std::shared_ptr<Mapper> foreground_mapper() { return foreground_mapper_; }
  MappingType mapping_type() const { return mapping_type_; }
  EsdfMode esdf_mode() const { return esdf_mode_; }

 protected:
  // Steps 2-4 of the reference's kDynamic frame (multi_mapper_impl.h:72-113), in order on the device: the detection on the
  // background's stream (its freespace layer is still the previous frame's: integrateDepth does not touch it), the filter
  // on the same stream, then the foreground's occupancy integration of the staged depth under the mask, ordered behind
  // them by an event. The foreground's integrateDepth returns only when its kernels are done, so the detector's buffers
  // are no longer read when the next frame's detection overwrites them.
  template <typename SensorType>
  void integrateDetectedDynamics(const DepthImage& depth_frame, const Transform& T_L_CD, const SensorType& depth_sensor) {
    NvbMapper* bg = background_mapper_->c_abi();
    dynamic_detector_.computeDynamics(depth_frame, background_mapper_->freespace_layer(), depth_sensor, T_L_CD);
    NvbDynamicsBuffers b;
    b200_detail::check(nvb_mapper_dynamics_device_buffers(bg, &b), "MultiMapper::integrateDepth", nvb_last_error());
    const uint8_t* mask = b.mask;
    if (params_.remove_small_connected_components) {
      b200_detail::check(nvb_mapper_remove_small_components(bg, b.mask, b.cleaned_mask, NVB_MEM_DEVICE, b.rows, b.cols,
                                                            params_.connected_mask_component_size_threshold),
                         "removeSmallConnectedComponents", nvb_last_error());
      mask = b.cleaned_mask;
    }
    b200_detail::check(nvb_mapper_wait_for(foreground_mapper_->c_abi(), bg), "MultiMapper::integrateDepth", nvb_last_error());
    foreground_mapper_->integrateDepth(
        MaskedDepthImageConstView(DepthImageConstView(b.depth, b.rows, b.cols, MemoryType::kDevice),
                                  MonoImageConstView(mask, b.rows, b.cols, MemoryType::kDevice)),
        T_L_CD, depth_sensor);
  }
  static bool isIdentity(const Transform& T) {
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 4; c++)
        if (std::fabs(T(r, c) - (r == c ? 1.0f : 0.0f)) > 1e-6f) return false;
    return true;
  }
  static bool sameCamera(const NvbCamera& a, const NvbCamera& b) {
    const bool same = a.fu == b.fu && a.fv == b.fv && a.cu == b.cu && a.cv == b.cv && a.width == b.width && a.height == b.height &&
                      a.has_distortion == b.has_distortion;
    if (!same || !a.has_distortion) return same;
    return a.k1 == b.k1 && a.k2 == b.k2 && a.k3 == b.k3 && a.k4 == b.k4 && a.k5 == b.k5 && a.k6 == b.k6 && a.p1 == b.p1 && a.p2 == b.p2;
  }
  const DepthImage& readSplit(int which, DepthImage* out) {
    int32_t rows = 0, cols = 0;
    NvbMapper* bg = background_mapper_->c_abi();
    b200_detail::check(nvb_mapper_split_output(bg, which, nullptr, NVB_MEM_HOST, &rows, &cols), "getLastDepthFrame", nvb_last_error());
    *out = DepthImage(rows, cols, MemoryType::kHost);
    if (rows > 0 && cols > 0)
      b200_detail::check(nvb_mapper_split_output(bg, which, out->dataPtr(), NVB_MEM_HOST, &rows, &cols), "getLastDepthFrame", nvb_last_error());
    return *out;
  }
  void updateEsdfOfMapper(const std::shared_ptr<Mapper>& mapper, const std::optional<Plane>& plane) {
    if (esdf_mode_ == EsdfMode::k2D && plane) mapper->updateEsdfSlice(UpdateFullLayer::kNo, *plane);
    else if (esdf_mode_ == EsdfMode::k2D) mapper->updateEsdfSlice();
    else mapper->updateEsdf();
  }
  const MappingType mapping_type_;
  const EsdfMode esdf_mode_;
  MultiMapperParams params_;
  std::shared_ptr<Mapper> background_mapper_, foreground_mapper_;
  std::optional<MonoImageConstView> dynamic_mask_;
  DynamicsDetection dynamic_detector_;
  std::unique_ptr<ImageMasker> image_masker_;
  MonoImage cleaned_mask_{0, 0};
  DepthImage depth_frame_background_{0, 0}, depth_frame_foreground_{0, 0};
  ColorImage depth_frame_overlay_{0, 0};
};
}  // namespace nvblox
