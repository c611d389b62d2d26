// nvblox/sensors/mask_preprocessor.h -- nvblox::image::MaskPreprocessor (reference: nvblox/include/nvblox/sensors/
// mask_preprocessor.h, src/sensors/mask_preprocessor.cpp:140-183), on the GPU (nvb_mapper_remove_small_components).
// Difference from the reference: mask_out keeps mask_in's size; a trailing odd row or column is 0 (the reference's output
// shrinks to an even size).
#pragma once
#include <memory>
#include "nvblox/core/cuda_stream.h"
#include "nvblox/sensors/image.h"
#include "nvblox_b200.h"
namespace nvblox {
namespace image {

class MaskPreprocessor {
 public:
  static constexpr int kDownScaleFactor = 2;
  // The filter needs a device and scratch: it keeps a small mapper of its own (or runs on `mapper` when one is given).
  explicit MaskPreprocessor(std::shared_ptr<CudaStream> cuda_stream, NvbMapper* mapper = nullptr)
      : cuda_stream_(std::move(cuda_stream)), m_(mapper) {
    if (!m_) {
      NvbMapperOptions o;
      nvb_default_mapper_options(&o);
      o.tsdf_capacity_blocks = o.esdf_capacity_blocks = 64;
      b200_detail::check(nvb_mapper_create(&o, &owned_), "MaskPreprocessor", nvb_last_error());
      m_ = owned_;
    }
  }
  ~MaskPreprocessor() { if (owned_) nvb_mapper_destroy(owned_); }
  MaskPreprocessor(const MaskPreprocessor&) = delete;
  MaskPreprocessor& operator=(const MaskPreprocessor&) = delete;

  // removeSmallConnectedComponents(mask_in, size_threshold, mask_out): components of the 2x-downscaled mask with fewer
  // than size_threshold / 4 pixels are erased; survivors hold 254. size_threshold <= 0 copies the mask.
  void removeSmallConnectedComponents(const MonoImage& mask_in, int size_threshold, MonoImage* mask_out) {
    if (mask_out->rows() != mask_in.rows() || mask_out->cols() != mask_in.cols())
      *mask_out = MonoImage(mask_in.rows(), mask_in.cols(), mask_out->memory_type());
    b200_detail::check(nvb_mapper_remove_small_components(m_, mask_in.dataConstPtr(), mask_out->dataPtr(), NVB_MEM_HOST,
                                                          mask_in.rows(), mask_in.cols(), size_threshold),
                       "removeSmallConnectedComponents", nvb_last_error());
  }

 private:
  std::shared_ptr<CudaStream> cuda_stream_;
  NvbMapper* m_ = nullptr;
  NvbMapper* owned_ = nullptr;
};
}  // namespace image
}  // namespace nvblox
