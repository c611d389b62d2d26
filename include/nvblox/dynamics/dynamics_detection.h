// nvblox/dynamics/dynamics_detection.h -- nvblox::DynamicsDetection (reference: nvblox/include/nvblox/dynamics/
// dynamics_detection.h): a depth pixel is dynamic when its surface point falls into a high-confidence freespace voxel.
// computeDynamics runs on the mapper that owns the FreespaceLayer handle (nvb_mapper_compute_dynamics); the outputs live in
// that mapper and stay on the device until a getter reads them. Points come in row-major pixel order.
#pragma once
#include <memory>
#include <type_traits>
#include <vector>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/core/types.h"
#include "nvblox/map/layer.h"
#include "nvblox/sensors/camera.h"
#include "nvblox/sensors/image.h"
#include "nvblox/sensors/pointcloud.h"
#include "nvblox_b200.h"
namespace nvblox {

class DynamicsDetection {
 public:
  DynamicsDetection() = delete;
  explicit DynamicsDetection(std::shared_ptr<CudaStream> cuda_stream) : cuda_stream_(std::move(cuda_stream)) {}
  virtual ~DynamicsDetection() = default;

  // computeDynamics(depth_frame_C, freespace_layer_L, sensor, T_L_C); SensorType = Camera is built.
  template <typename SensorType>
  void computeDynamics(const DepthImage& depth_frame_C, const FreespaceLayer& freespace_layer_L, const SensorType& sensor,
                       const Transform& T_L_C) {
    computeDynamics(DepthImageConstView(depth_frame_C), freespace_layer_L, sensor, T_L_C);
  }
  template <typename SensorType>
  void computeDynamics(const DepthImageConstView& depth_frame_C, const FreespaceLayer& freespace_layer_L,
                       const SensorType& sensor, const Transform& T_L_C) {
    static_assert(std::is_same<SensorType, Camera>::value, "only the Camera sensor model is built on this path");
    m_ = freespace_layer_L.c_abi();
    b200_detail::check(nvb_mapper_compute_dynamics(m_, depth_frame_C.dataConstPtr(),
                                                   depth_frame_C.on_device() ? NVB_MEM_DEVICE : NVB_MEM_HOST,
                                                   depth_frame_C.rows(), depth_frame_C.cols(), T_L_C.data(), sensor.c_abi()),
                       "computeDynamics", nvb_last_error());
  }
  // getDynamicPointsHost(): 3 x N
  Matrix3Xf getDynamicPointsHost() {
    const std::vector<float> xyz = points();
    Matrix3Xf out(3, (int)(xyz.size() / 3));
    for (size_t i = 0; i < xyz.size(); i++) out.data()[i] = xyz[i];
    return out;
  }
  // getDynamicPointcloudDevice(): the points as a Pointcloud (this mirror's Pointcloud keeps them on the host)
  const Pointcloud& getDynamicPointcloudDevice() {
    const std::vector<float> xyz = points();
    std::vector<Vector3f> pts(xyz.size() / 3);
    for (size_t i = 0; i < pts.size(); i++) pts[i] = Vector3f(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    pointcloud_.copyPointsFrom(pts);
    return pointcloud_;
  }
  // getDynamicMaskImage(): 255 dynamic, 0 static (read back from the device)
  const MonoImage& getDynamicMaskImage() const {
    int32_t rows = 0, cols = 0;
    if (m_) b200_detail::check(nvb_mapper_dynamic_mask(m_, nullptr, NVB_MEM_HOST, &rows, &cols), "getDynamicMaskImage", nvb_last_error());
    mask_ = MonoImage(rows, cols, MemoryType::kHost);
    if (rows * cols)
      b200_detail::check(nvb_mapper_dynamic_mask(m_, mask_.dataPtr(), NVB_MEM_HOST, &rows, &cols), "getDynamicMaskImage", nvb_last_error());
    return mask_;
  }
  // getDynamicOverlayImage(): dynamics red, the rest grey by depth, white where nothing was looked up
  const ColorImage& getDynamicOverlayImage() const {
    int32_t rows = 0, cols = 0;
    if (m_) b200_detail::check(nvb_mapper_dynamic_overlay(m_, nullptr, NVB_MEM_HOST, &rows, &cols), "getDynamicOverlayImage", nvb_last_error());
    overlay_ = ColorImage(rows, cols, MemoryType::kHost);
    static_assert(sizeof(Color) == 3, "Color is 3 bytes (RGB)");
    if (rows * cols)
      b200_detail::check(nvb_mapper_dynamic_overlay(m_, reinterpret_cast<uint8_t*>(overlay_.dataPtr()), NVB_MEM_HOST, &rows, &cols),
                         "getDynamicOverlayImage", nvb_last_error());
    return overlay_;
  }

 private:
  std::vector<float> points() {
    int32_t n = 0;
    if (!m_) return {};
    b200_detail::check(nvb_mapper_dynamic_points(m_, nullptr, NVB_MEM_HOST, 0, &n), "getDynamicPoints", nvb_last_error());
    std::vector<float> xyz((size_t)n * 3);
    if (n) b200_detail::check(nvb_mapper_dynamic_points(m_, xyz.data(), NVB_MEM_HOST, n, &n), "getDynamicPoints", nvb_last_error());
    return xyz;
  }
  std::shared_ptr<CudaStream> cuda_stream_;
  NvbMapper* m_ = nullptr;
  Pointcloud pointcloud_;
  mutable MonoImage mask_{0, 0, MemoryType::kHost};
  mutable ColorImage overlay_{0, 0, MemoryType::kHost};
};
}  // namespace nvblox
