// nvblox/rays/sphere_tracer.h -- nvblox::SphereTracer (reference: nvblox/include/nvblox/rays/sphere_tracer.h,
// src/rays/sphere_tracer.cu): depth and RGBD images of a mapper's TSDF (and colour) layer, rendered on the GPU by
// nvb_render_depth / nvb_render_rgbd. Like the reference, every render returns once its images are written.
//
// The layers are views of a mapper's map: the TSDF and colour layers of one RGBD call must belong to the same mapper. A
// view's buffer is device memory (the reference's kDevice) or, for a view of an owning Image, host memory.
#pragma once
#include <memory>
#include <utility>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/core/types.h"
#include "nvblox/map/layer.h"
#include "nvblox/sensors/camera.h"
#include "nvblox/sensors/image.h"
#include "nvblox_b200.h"
namespace nvblox {

class SphereTracer {
 public:
  SphereTracer() : SphereTracer(std::make_shared<CudaStreamOwning>()) {}
  SphereTracer(std::shared_ptr<CudaStream> cuda_stream) : cuda_stream_(std::move(cuda_stream)) {
    nvb_default_sphere_tracer_params(&p_);
  }
  ~SphereTracer() = default;

  struct SubsampledImageSize {
    SubsampledImageSize(int _rows, int _cols) : rows(_rows), cols(_cols) {}
    int rows;
    int cols;
  };

  // Renders into *depth_ptr, reallocating it when its size or memory type differ from the request.
  void renderImageOnGPU(const Camera& camera, const Transform& T_L_C, const TsdfLayer& tsdf_layer,
                        const float truncation_distance_m, DepthImage* depth_ptr,
                        const MemoryType output_image_memory_type = MemoryType::kDevice, const int ray_subsampling_factor = 1) {
    checkRequest(depth_ptr != nullptr, camera, output_image_memory_type, ray_subsampling_factor, "renderImageOnGPU");
    resize(depth_ptr, camera, output_image_memory_type, ray_subsampling_factor);
    DepthImageView depth_view(*depth_ptr);
    renderImageOnGPU(camera, T_L_C, tsdf_layer, truncation_distance_m, &depth_view, output_image_memory_type,
                     ray_subsampling_factor);
  }

  // Renders into a view of (height / f) x (width / f) floats; a view of another size is left alone, as in the reference.
  void renderImageOnGPU(const Camera& camera, const Transform& T_L_C, const TsdfLayer& tsdf_layer,
                        const float truncation_distance_m, DepthImageView* depth_ptr, const MemoryType output_image_memory_type,
                        const int ray_subsampling_factor = 1) {
    checkRequest(depth_ptr != nullptr && depth_ptr->dataPtr() != nullptr, camera, output_image_memory_type,
                 ray_subsampling_factor, "renderImageOnGPU");
    if (!sized(*depth_ptr, camera, ray_subsampling_factor)) return;
    NvbMapper* m = tsdf_layer.mapper_handle();
    b200_detail::check(nvb_render_depth(m, &p_, T_L_C.data(), camera.c_abi(), truncation_distance_m, ray_subsampling_factor,
                                        memoryOf(*depth_ptr), depth_ptr->dataPtr(), cuda_stream_->get()),
                       "renderImageOnGPU", nvb_last_error());
    finish(m, depth_ptr->on_device());
  }

  void renderRgbdImageOnGPU(const Camera& camera, const Transform& T_L_C, const TsdfLayer& tsdf_layer,
                            const ColorLayer& color_layer, const float truncation_distance_m, DepthImage* depth_ptr,
                            ColorImage* color_ptr, const MemoryType output_image_memory_type,
                            const int ray_subsampling_factor = 1) {
    checkRequest(depth_ptr != nullptr && color_ptr != nullptr, camera, output_image_memory_type, ray_subsampling_factor,
                 "renderRgbdImageOnGPU");
    resize(depth_ptr, camera, output_image_memory_type, ray_subsampling_factor);
    resize(color_ptr, camera, output_image_memory_type, ray_subsampling_factor);
    DepthImageView depth_view(*depth_ptr);
    ColorImageView color_view(*color_ptr);
    renderRgbdImageOnGPU(camera, T_L_C, tsdf_layer, color_layer, truncation_distance_m, &depth_view, &color_view,
                         output_image_memory_type, ray_subsampling_factor);
  }

  // Depth and the colour of the colour voxel holding each hit point; black for a miss or a hit without a colour block.
  void renderRgbdImageOnGPU(const Camera& camera, const Transform& T_L_C, const TsdfLayer& tsdf_layer,
                            const ColorLayer& color_layer, const float truncation_distance_m, DepthImageView* depth_ptr,
                            ColorImageView* color_ptr, const MemoryType output_image_memory_type,
                            const int ray_subsampling_factor = 1) {
    checkRequest(depth_ptr != nullptr && color_ptr != nullptr && depth_ptr->dataPtr() != nullptr &&
                     color_ptr->dataPtr() != nullptr,
                 camera, output_image_memory_type, ray_subsampling_factor, "renderRgbdImageOnGPU");
    if (!sized(*depth_ptr, camera, ray_subsampling_factor) || !sized(*color_ptr, camera, ray_subsampling_factor)) return;
    if (depth_ptr->on_device() != color_ptr->on_device())
      b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "renderRgbdImageOnGPU", "the depth and colour views are in different memory");
    NvbMapper* m = tsdf_layer.mapper_handle();
    if (color_layer.mapper_handle() != m)
      b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "renderRgbdImageOnGPU", "the colour layer belongs to another mapper");
    b200_detail::check(nvb_render_rgbd(m, &p_, T_L_C.data(), camera.c_abi(), truncation_distance_m, ray_subsampling_factor,
                                       memoryOf(*depth_ptr), depth_ptr->dataPtr(),
                                       reinterpret_cast<uint8_t*>(color_ptr->dataPtr()), cuda_stream_->get()),
                       "renderRgbdImageOnGPU", nvb_last_error());
    finish(m, depth_ptr->on_device());
  }

  SubsampledImageSize getSubsampledImageSize(const Camera& camera, const int subsampling_factor) const {
    return SubsampledImageSize(camera.height() / subsampling_factor, camera.width() / subsampling_factor);
  }

  int maximum_steps() const { return p_.maximum_steps; }
  float maximum_ray_length_m() const { return p_.maximum_ray_length_m; }
  float surface_distance_epsilon_vox() const { return p_.surface_distance_epsilon_vox; }
  void maximum_steps(int maximum_steps) {
    positive(maximum_steps > 0, "maximum_steps");
    p_.maximum_steps = maximum_steps;
  }
  void maximum_ray_length_m(float maximum_ray_length_m) {
    positive(maximum_ray_length_m > 0.0f, "maximum_ray_length_m");
    p_.maximum_ray_length_m = maximum_ray_length_m;
  }
  void surface_distance_epsilon_vox(float surface_distance_epsilon_vox) {
    positive(surface_distance_epsilon_vox > 0.0f, "surface_distance_epsilon_vox");
    p_.surface_distance_epsilon_vox = surface_distance_epsilon_vox;
  }

 private:
  static void positive(bool ok, const char* what) {  // the setters' CHECK_GT (sphere_tracer.cu:319-333)
    if (!ok) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, what, "must be positive");
  }
  // CHECK_NOTNULL, CHECK_EQ(size % f, 0) and CHECK(memory type != kHost) of the reference's render calls
  static void checkRequest(bool not_null, const Camera& camera, MemoryType mt, int f, const char* what) {
    if (!not_null) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, what, "null output image");
    if (f <= 0 || camera.width() % f != 0 || camera.height() % f != 0)
      b200_detail::check(NVB_ERR_INVALID_ARGUMENT, what, "the ray subsampling factor must divide the image size");
    if (mt == MemoryType::kHost) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, what, "the output memory type is kHost");
  }
  template <typename T>
  void resize(Image<T>* img, const Camera& camera, MemoryType mt, int f) const {
    const SubsampledImageSize s = getSubsampledImageSize(camera, f);
    if (img->rows() != s.rows || img->cols() != s.cols || img->memory_type() != mt) *img = Image<T>(s.rows, s.cols, mt);
  }
  template <typename T>
  bool sized(const MutableImageView<T>& v, const Camera& camera, int f) const {
    const SubsampledImageSize s = getSubsampledImageSize(camera, f);
    return v.rows() == s.rows && v.cols() == s.cols;
  }
  template <typename T>
  static int32_t memoryOf(const MutableImageView<T>& v) {
    return v.on_device() ? NVB_MEM_DEVICE : NVB_MEM_HOST;
  }
  // A device render is ordered behind the mapper's stream: synchronising the mapper returns once the images are written.
  static void finish(NvbMapper* m, bool on_device) {
    if (on_device) b200_detail::check(nvb_mapper_synchronize(m), "SphereTracer", nvb_last_error());
  }

  NvbSphereTracerParams p_{};
  std::shared_ptr<CudaStream> cuda_stream_;
};

}  // namespace nvblox
