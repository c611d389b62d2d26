// nvblox/core/types.h -- source-compatible subset of the reference header
// (nvblox/include/nvblox/core/types.h:141-153) for the depth-integration path.
//
// With -DNVBLOX_B200_WITH_EIGEN the real Eigen types are used (what nvblox_ros builds with);
// otherwise a minimal layout-compatible shim provides the members this path touches, so the
// headers compile on a box without Eigen (like this build container).
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#ifdef NVBLOX_B200_WITH_EIGEN
#include <Eigen/Core>
#include <Eigen/Geometry>
namespace nvblox {
using Index3D = Eigen::Vector3i;
using Index2D = Eigen::Vector2i;
using Vector3f = Eigen::Vector3f;
using Vector2f = Eigen::Vector2f;
using Transform = Eigen::Isometry3f;
using Matrix3Xf = Eigen::Matrix3Xf;
}  // namespace nvblox
#else
namespace nvblox {

template <typename T, int N>
struct VecShim {
  T v[N];
  VecShim() { for (int i = 0; i < N; i++) v[i] = T(0); }
  VecShim(T a, T b) { static_assert(N == 2, ""); v[0] = a, v[1] = b; }
  VecShim(T a, T b, T c) { static_assert(N == 3, ""); v[0] = a, v[1] = b, v[2] = c; }
  T& x() { return v[0]; }
  T& y() { return v[1]; }
  T& z() { static_assert(N >= 3, ""); return v[2]; }
  const T& x() const { return v[0]; }
  const T& y() const { return v[1]; }
  const T& z() const { static_assert(N >= 3, ""); return v[2]; }
  T& operator[](int i) { return v[i]; }
  const T& operator[](int i) const { return v[i]; }
  T& operator()(int i) { return v[i]; }
  const T& operator()(int i) const { return v[i]; }
  T* data() { return v; }
  const T* data() const { return v; }
  static VecShim Zero() { return VecShim(); }
  bool operator==(const VecShim& o) const { for (int i = 0; i < N; i++) if (v[i] != o.v[i]) return false; return true; }
  bool operator!=(const VecShim& o) const { return !(*this == o); }
  VecShim operator+(const VecShim& o) const { VecShim r; for (int i = 0; i < N; i++) r.v[i] = v[i] + o.v[i]; return r; }
  VecShim operator-(const VecShim& o) const { VecShim r; for (int i = 0; i < N; i++) r.v[i] = v[i] - o.v[i]; return r; }
};
using Index3D = VecShim<int, 3>;
using Index2D = VecShim<int, 2>;
using Vector3f = VecShim<float, 3>;
using Vector2f = VecShim<float, 2>;

// Eigen::Isometry3f stand-in: 4x4 column-major, data() is what the C-ABI takes.
struct Transform {
  float m[16];
  Transform() { setIdentity(); }
  static Transform Identity() { return Transform(); }
  void setIdentity() { for (int i = 0; i < 16; i++) m[i] = (i % 5 == 0) ? 1.0f : 0.0f; }
  float& operator()(int r, int c) { return m[c * 4 + r]; }
  const float& operator()(int r, int c) const { return m[c * 4 + r]; }
  const float* data() const { return m; }
  float* data() { return m; }
  Vector3f translation() const { return Vector3f(m[12], m[13], m[14]); }
  void setTranslation(const Vector3f& t) { m[12] = t[0], m[13] = t[1], m[14] = t[2]; }
  Vector3f operator*(const Vector3f& p) const {
    Vector3f r;
    for (int i = 0; i < 3; i++) r[i] = m[12 + i] + ((*this)(i, 0) * p[0] + ((*this)(i, 1) * p[1] + (*this)(i, 2) * p[2]));
    return r;
  }
  Transform inverse() const {
    Transform o;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) o(i, j) = (*this)(j, i);
    for (int i = 0; i < 3; i++) o.m[12 + i] = -(o(i, 0) * m[12] + (o(i, 1) * m[13] + o(i, 2) * m[14]));
    return o;
  }
};

// Eigen::Matrix3Xf stand-in (DynamicsDetection::getDynamicPointsHost): 3 x cols, column-major.
struct Matrix3Xf {
  std::vector<float> m;
  Matrix3Xf() = default;
  Matrix3Xf(int rows, int cols) : m((size_t)3 * cols) { (void)rows; }
  int rows() const { return 3; }
  int cols() const { return (int)(m.size() / 3); }
  float& operator()(int r, int c) { return m[(size_t)c * 3 + r]; }
  const float& operator()(int r, int c) const { return m[(size_t)c * 3 + r]; }
  Vector3f col(int c) const { return Vector3f(m[(size_t)c * 3], m[(size_t)c * 3 + 1], m[(size_t)c * 3 + 2]); }
  float* data() { return m.data(); }
  const float* data() const { return m.data(); }
};
}  // namespace nvblox
#endif

namespace nvblox {
// nvblox/include/nvblox/core/types.h MemoryType
enum class MemoryType { kDevice, kUnified, kHost };

namespace b200_detail {
// The reference aborts through glog CHECK on errors (core/internal/error_check.h:28-65).
inline void check(int rc, const char* what, const char* msg) {
  if (rc != 0) {
    std::fprintf(stderr, "nvblox(b200): %s failed (%d): %s\n", what, rc, msg);
    std::abort();
  }
}
}  // namespace b200_detail
}  // namespace nvblox
