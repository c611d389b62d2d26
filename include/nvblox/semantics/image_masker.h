// nvblox/semantics/image_masker.h -- nvblox::ImageMasker (reference: nvblox/include/nvblox/semantics/image_masker.h,
// src/semantics/image_masker.cu), on the GPU (nvb_mapper_split_depth_image, nvb_mapper_split_color_image).
// The depth split sends a depth pixel to the masked output when it lands, unoccluded, on a set pixel of a mask seen from
// another camera (T_CM_CD, mask_camera); the colour split applies a mask lying on top of the image. Both write the
// caller's images. Differences from the reference: a projection exactly on u == width or v == height is a miss (the
// reference reads past the mask's row there); a negative depth has overlay grey 0 (undefined in the reference).
#pragma once
#include <memory>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/core/types.h"
#include "nvblox/sensors/camera.h"
#include "nvblox/sensors/image.h"
#include "nvblox_b200.h"
namespace nvblox {

class ImageMasker {
 public:
  // The split needs a device and scratch: it keeps a small mapper of its own (or runs on `mapper` when one is given, whose
  // split outputs it then overwrites).
  ImageMasker() : ImageMasker(std::make_shared<CudaStreamOwning>()) {}
  explicit ImageMasker(std::shared_ptr<CudaStream> cuda_stream, NvbMapper* mapper = nullptr)
      : cuda_stream_(std::move(cuda_stream)), m_(mapper) {
    nvb_default_image_masker_params(&params_);
    if (!m_) {
      NvbMapperOptions o;
      nvb_default_mapper_options(&o);
      o.tsdf_capacity_blocks = o.esdf_capacity_blocks = 64;
      b200_detail::check(nvb_mapper_create(&o, &owned_), "ImageMasker", nvb_last_error());
      m_ = owned_;
    }
  }
  ~ImageMasker() { if (owned_) nvb_mapper_destroy(owned_); }
  ImageMasker(const ImageMasker&) = delete;
  ImageMasker& operator=(const ImageMasker&) = delete;

  // splitImageOnGPU(input, mask, unmasked_output, masked_output, masked_color_overlay): the mask lies on top of the
  // colour image; the pixels that went to the other output are black.
  void splitImageOnGPU(const ColorImage& input, const MonoImage& mask, ColorImage* unmasked_output, ColorImage* masked_output,
                       ColorImage* masked_color_overlay = nullptr) {
    if (mask.rows() != input.rows() || mask.cols() != input.cols()) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "splitImageOnGPU", "mask/image size mismatch");
    static_assert(sizeof(Color) == 3, "Color is 3 bytes (RGB)");
    allocate(input.rows(), input.cols(), unmasked_output, masked_output, masked_color_overlay);
    b200_detail::check(nvb_mapper_split_color_image(m_, reinterpret_cast<const uint8_t*>(input.dataConstPtr()), mask.dataConstPtr(),
                                                    NVB_MEM_HOST, input.rows(), input.cols(),
                                                    reinterpret_cast<uint8_t*>(unmasked_output->dataPtr()),
                                                    reinterpret_cast<uint8_t*>(masked_output->dataPtr()),
                                                    masked_color_overlay ? reinterpret_cast<uint8_t*>(masked_color_overlay->dataPtr()) : nullptr),
                       "splitImageOnGPU", nvb_last_error());
  }

  // splitImageOnGPU(depth_input, mask, T_CM_CD, depth_camera, mask_camera, unmasked_depth_output, masked_depth_output,
  // masked_depth_overlay): unmasked pixels of the masked output, and masked pixels of the unmasked output, hold the
  // invalid values (-1 by default). Sizes must match the cameras.
  void splitImageOnGPU(const DepthImage& depth_input, const MonoImage& mask, const Transform& T_CM_CD, const Camera& depth_camera,
                       const Camera& mask_camera, DepthImage* unmasked_depth_output, DepthImage* masked_depth_output,
                       ColorImage* masked_depth_overlay = nullptr) {
    split(depth_input, mask, T_CM_CD, depth_camera, mask_camera, masked_depth_overlay != nullptr);
    allocate(depth_input.rows(), depth_input.cols(), unmasked_depth_output, masked_depth_output, masked_depth_overlay);
    int32_t rows = 0, cols = 0;
    b200_detail::check(nvb_mapper_split_output(m_, NVB_SPLIT_BACKGROUND, unmasked_depth_output->dataPtr(), NVB_MEM_HOST, &rows, &cols),
                       "splitImageOnGPU", nvb_last_error());
    b200_detail::check(nvb_mapper_split_output(m_, NVB_SPLIT_FOREGROUND, masked_depth_output->dataPtr(), NVB_MEM_HOST, &rows, &cols),
                       "splitImageOnGPU", nvb_last_error());
    if (masked_depth_overlay)
      b200_detail::check(nvb_mapper_split_output(m_, NVB_SPLIT_OVERLAY, reinterpret_cast<uint8_t*>(masked_depth_overlay->dataPtr()),
                                                 NVB_MEM_HOST, &rows, &cols),
                         "splitImageOnGPU", nvb_last_error());
  }

  float occlusion_threshold_m() const { return params_.occlusion_threshold_m; }
  void occlusion_threshold_m(float occlusion_threshold_m) { params_.occlusion_threshold_m = occlusion_threshold_m; }
  float depth_masked_image_invalid_pixel() const { return params_.depth_masked_image_invalid_pixel; }
  void depth_masked_image_invalid_pixel(float value) { params_.depth_masked_image_invalid_pixel = value; }
  float depth_unmasked_image_invalid_pixel() const { return params_.depth_unmasked_image_invalid_pixel; }
  void depth_unmasked_image_invalid_pixel(float value) { params_.depth_unmasked_image_invalid_pixel = value; }

  // The split alone: its outputs stay in the mapper's device buffers (nvb_mapper_split_device_buffers), enqueued on the
  // mapper's stream without a synchronisation.
  void split(const DepthImage& depth_input, const MonoImage& mask, const Transform& T_CM_CD, const Camera& depth_camera,
             const Camera& mask_camera, bool with_overlay) {
    b200_detail::check(nvb_mapper_split_depth_image(m_, depth_input.dataConstPtr(), depth_input.rows(), depth_input.cols(),
                                                    mask.dataConstPtr(), mask.rows(), mask.cols(), NVB_MEM_HOST, T_CM_CD.data(),
                                                    depth_camera.c_abi(), mask_camera.c_abi(), &params_, with_overlay ? 1 : 0),
                       "splitImageOnGPU", nvb_last_error());
  }
  NvbMapper* c_abi() const { return m_; }

 private:
  template <typename T>
  static void allocate(int rows, int cols, Image<T>* unmasked, Image<T>* masked, ColorImage* overlay) {
    if (!unmasked || !masked) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "splitImageOnGPU", "null output");
    if (unmasked->rows() != rows || unmasked->cols() != cols) *unmasked = Image<T>(rows, cols, unmasked->memory_type());
    if (masked->rows() != rows || masked->cols() != cols) *masked = Image<T>(rows, cols, masked->memory_type());
    if (overlay && (overlay->rows() != rows || overlay->cols() != cols)) *overlay = ColorImage(rows, cols, overlay->memory_type());
  }
  std::shared_ptr<CudaStream> cuda_stream_;
  NvbMapper* m_ = nullptr;
  NvbMapper* owned_ = nullptr;
  NvbImageMaskerParams params_;
};
}  // namespace nvblox
