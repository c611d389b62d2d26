// nvblox/sensors/image.h -- DepthImage / MonoImage / MaskedDepthImageConstView subset
// (reference: nvblox/include/nvblox/sensors/image.h, MaskMode at :383, MaskedImageView :389-438).
#pragma once
#include <optional>
#include <vector>
#include "nvblox/core/types.h"
#include "nvblox/map/voxels.h"
#include "nvblox_b200.h"
namespace nvblox {
enum class MaskMode { kNonInverted, kInverted };
constexpr std::nullopt_t kMaskActiveEverywhere = std::nullopt;

// Owning image. kHost / kUnified keep the pixels in host memory (operator() works); device-resident
// frames are passed as ImageView(ptr, rows, cols, MemoryType::kDevice).
template <typename T>
class Image {
 public:
  Image(int rows, int cols, MemoryType mt = MemoryType::kHost) : rows_(rows), cols_(cols), mt_(mt), px_((size_t)rows * cols) {}
  int rows() const { return rows_; }
  int cols() const { return cols_; }
  int numel() const { return rows_ * cols_; }
  MemoryType memory_type() const { return mt_; }
  T& operator()(int r, int c) { return px_[(size_t)r * cols_ + c]; }
  const T& operator()(int r, int c) const { return px_[(size_t)r * cols_ + c]; }
  T& operator()(int lin) { return px_[lin]; }
  T* dataPtr() { return px_.data(); }
  const T* dataConstPtr() const { return px_.data(); }
 private:
  int rows_, cols_;
  MemoryType mt_;
  std::vector<T> px_;
};
using DepthImage = Image<float>;
using MonoImage = Image<uint8_t>;
using ColorImage = Image<Color>;  // 3 bytes per pixel, RGB (sensors/image.h:442)

template <typename T>
class ImageView {
 public:
  ImageView() = default;
  ImageView(const T* data, int rows, int cols, MemoryType mt) : data_(data), rows_(rows), cols_(cols), mt_(mt) {}
  ImageView(const Image<T>& img) : data_(img.dataConstPtr()), rows_(img.rows()), cols_(img.cols()), mt_(MemoryType::kHost) {}
  const T* dataConstPtr() const { return data_; }
  int rows() const { return rows_; }
  int cols() const { return cols_; }
  bool on_device() const { return mt_ == MemoryType::kDevice; }
 private:
  const T* data_ = nullptr;
  int rows_ = 0, cols_ = 0;
  MemoryType mt_ = MemoryType::kHost;
};
using DepthImageConstView = ImageView<float>;
using MonoImageConstView = ImageView<uint8_t>;
using ColorImageConstView = ImageView<Color>;

// Writable view (the reference's ImageView<float> / ImageView<Color>, sensors/image.h:326-444) of a buffer the caller owns:
// rows x cols pixels on the device unless told otherwise; a view of an owning Image is host memory.
template <typename T>
class MutableImageView {
 public:
  MutableImageView() = default;
  MutableImageView(int rows, int cols, T* data = nullptr, MemoryType mt = MemoryType::kDevice)
      : data_(data), rows_(rows), cols_(cols), mt_(mt) {}
  MutableImageView(Image<T>& img) : data_(img.dataPtr()), rows_(img.rows()), cols_(img.cols()), mt_(MemoryType::kHost) {}
  T* dataPtr() const { return data_; }
  const T* dataConstPtr() const { return data_; }
  int rows() const { return rows_; }
  int cols() const { return cols_; }
  int width() const { return cols_; }
  int height() const { return rows_; }
  bool on_device() const { return mt_ == MemoryType::kDevice; }
 private:
  T* data_ = nullptr;
  int rows_ = 0, cols_ = 0;
  MemoryType mt_ = MemoryType::kDevice;
};
using DepthImageView = MutableImageView<float>;
using ColorImageView = MutableImageView<Color>;

class MaskedDepthImageConstView : public DepthImageConstView {
 public:
  MaskedDepthImageConstView(const DepthImageConstView& image, std::optional<MonoImageConstView> mask = std::nullopt,
                            MaskMode mode = MaskMode::kNonInverted)
      : DepthImageConstView(image), mode_(mode) {
    if (mask.has_value()) {
      if (mask->rows() != image.rows() || mask->cols() != image.cols()) b200_detail::check(-1, "MaskedImageView", "mask/image size mismatch");
      mask_ = *mask;
    }
  }
  MaskedDepthImageConstView(const DepthImage& image, std::nullopt_t) : DepthImageConstView(image) {}
  const MonoImageConstView& mask() const { return mask_; }
  MaskMode mode() const { return mode_; }
 private:
  MonoImageConstView mask_;
  MaskMode mode_ = MaskMode::kNonInverted;
};

// MaskedImageView<const Color> (sensors/image.h:389-438)
class MaskedColorImageConstView : public ColorImageConstView {
 public:
  MaskedColorImageConstView(const ColorImageConstView& image, std::optional<MonoImageConstView> mask = std::nullopt,
                            MaskMode mode = MaskMode::kNonInverted)
      : ColorImageConstView(image), mode_(mode) {
    if (mask.has_value()) {
      if (mask->rows() != image.rows() || mask->cols() != image.cols()) b200_detail::check(-1, "MaskedImageView", "mask/image size mismatch");
      mask_ = *mask;
    }
  }
  MaskedColorImageConstView(const ColorImage& image, std::nullopt_t) : ColorImageConstView(image) {}
  const MonoImageConstView& mask() const { return mask_; }
  MaskMode mode() const { return mode_; }
 private:
  MonoImageConstView mask_;
  MaskMode mode_ = MaskMode::kNonInverted;
};
}  // namespace nvblox
