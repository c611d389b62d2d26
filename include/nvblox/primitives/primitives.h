// nvblox/primitives/primitives.h -- nvblox::primitives::Primitive and its planes, cubes, spheres and cylinders (reference:
// nvblox/include/nvblox/primitives/primitives.h, src/primitives/primitives.cpp). The distance and ray functions run on the host
// with the arithmetic of the library's kernels (csrc/nvb_scene.cu): float where the reference computes in float, double where
// its literals promote; an unqualified sqrt of a float is the float square root; Eigen's three-term sums are a0 + (a1 + a2).
#pragma once
#include <algorithm>
#include <cmath>
#include <string>
#include "nvblox/core/types.h"
#include "nvblox_b200.h"
namespace nvblox {
namespace primitives {

namespace detail {
inline float dot3(const Vector3f& a, const Vector3f& b) { return a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]); }
template <typename T>
inline T maxStd(T a, T b) { return (a < b) ? b : a; }
}  // namespace detail

/// Base class for primitive objects.
class Primitive {
 public:
  enum class Type { kPlane, kCube, kSphere, kCylinder };
  static std::string toString(const Type& type) {
    switch (type) {
      case Type::kPlane: return "kPlane";
      case Type::kCube: return "kCube";
      case Type::kSphere: return "kSphere";
      case Type::kCylinder: return "kCylinder";
    }
    b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "Primitive::toString", "Primitive type not recognized.");
    return "";
  }
  /// Epsilon for ray intersection and computation.
  static constexpr float kEpsilon = 1e-4;

  Primitive(const Vector3f& center, Type type) : center_(center), type_(type) {}
  virtual ~Primitive() {}
  virtual float getDistanceToPoint(const Vector3f& point) const = 0;
  Type getType() const { return type_; }
  virtual bool getRayIntersection(const Vector3f& ray_origin, const Vector3f& ray_direction, float max_dist,
                                  Vector3f* intersect_point, float* intersect_dist) const = 0;
  const Vector3f& center() const { return center_; }
  // (not in the reference) the primitive as the C ABI's NvbPrimitive, for the scene's GPU calls
  virtual NvbPrimitive c_abi() const = 0;

 protected:
  NvbPrimitive base(int32_t type) const {
    NvbPrimitive p{};
    p.type = type;
    for (int k = 0; k < 3; k++) p.center[k] = center_[k];
    return p;
  }
  static Vector3f pointAt(const Vector3f& o, const Vector3f& u, float t) {
    return Vector3f(o[0] + t * u[0], o[1] + t * u[1], o[2] + t * u[2]);
  }
  Vector3f center_;
  Type type_;
};

/// Primitive sphere, given a center and a radius.
class Sphere : public Primitive {
 public:
  Sphere(const Vector3f& center, float radius) : Primitive(center, Type::kSphere), radius_(radius) {}
  float getDistanceToPoint(const Vector3f& point) const override {
    const Vector3f d = center_ - point;
    return std::sqrt(detail::dot3(d, d)) - radius_;
  }
  bool getRayIntersection(const Vector3f& o, const Vector3f& u, float max_dist, Vector3f* intersect_point,
                          float* intersect_dist) const override {
    const Vector3f oc = o - center_;
    const float b = detail::dot3(u, oc);
    const float disc = (float)(((double)b * (double)b - (double)detail::dot3(oc, oc)) + (double)radius_ * (double)radius_);
    if (disc < 0.0f) return false;
    const float d = -b - std::sqrt(disc);
    if (d < 0.0f || d > max_dist) return false;
    *intersect_point = pointAt(o, u, d);
    *intersect_dist = d;
    return true;
  }
  NvbPrimitive c_abi() const override {
    NvbPrimitive p = base(NVB_PRIM_SPHERE);
    p.params[0] = radius_;
    return p;
  }

 protected:
  float radius_;
};

/// Primitive cube, given a center and an X,Y,Z size (can be a rectangular prism).
class Cube : public Primitive {
 public:
  Cube(const Vector3f& center, const Vector3f& size) : Primitive(center, Type::kCube), size_(size) {}
  float getDistanceToPoint(const Vector3f& p) const override {
    double lo[3], hi[3];
    Vector3f v;
    for (int k = 0; k < 3; k++) {
      lo[k] = ((double)center_[k] - (double)size_[k] / 2.0) - (double)p[k];
      hi[k] = (double)(p[k] - center_[k]) - (double)size_[k] / 2.0;
      v[k] = (float)detail::maxStd(detail::maxStd(lo[k], 0.0), hi[k]);
    }
    float dist = std::sqrt(detail::dot3(v, v));
    if (dist < kEpsilon) {
      for (int k = 0; k < 3; k++) v[k] = (float)detail::maxStd(lo[k], hi[k]);
      dist = detail::maxStd(v[0], detail::maxStd(v[1], v[2]));
    }
    return dist;
  }
  bool getRayIntersection(const Vector3f& o, const Vector3f& u, float max_dist, Vector3f* intersect_point,
                          float* intersect_dist) const override {
    float inv[3], b0[3], b1[3], tlo[3], thi[3];
    for (int k = 0; k < 3; k++) {
      inv[k] = (float)(1.0 / (double)u[k]);
      b0[k] = center_[k] - size_[k] / 2.0f;
      b1[k] = center_[k] + size_[k] / 2.0f;
      const bool neg = inv[k] < 0.0f;
      tlo[k] = ((neg ? b1[k] : b0[k]) - o[k]) * inv[k];
      thi[k] = ((neg ? b0[k] : b1[k]) - o[k]) * inv[k];
    }
    float tmin = tlo[0], tmax = thi[0];
    if ((tmin > thi[1]) || (tlo[1] > tmax)) return false;
    if (tlo[1] > tmin) tmin = tlo[1];
    if (thi[1] < tmax) tmax = thi[1];
    if ((tmin > thi[2]) || (tlo[2] > tmax)) return false;
    if (tlo[2] > tmin) tmin = tlo[2];
    if (thi[2] < tmax) tmax = thi[2];
    float t = tmin;
    if (t < 0.0f) {
      t = tmax;
      if (t < 0.0f) return false;
    }
    if (t > max_dist) return false;
    *intersect_dist = t;
    *intersect_point = pointAt(o, u, t);
    return true;
  }
  NvbPrimitive c_abi() const override {
    NvbPrimitive p = base(NVB_PRIM_CUBE);
    for (int k = 0; k < 3; k++) p.params[k] = size_[k];
    return p;
  }

 protected:
  Vector3f size_;
};

/// Primitive plane, given a center and a normal of unit length (norm 1 +- 1e-3, else the program aborts like CHECK_NEAR).
class Plane : public Primitive {
 public:
  Plane(const Vector3f& center, const Vector3f& normal) : Primitive(center, Type::kPlane), normal_(normal) {
    const double n = std::sqrt(detail::dot3(normal, normal));
    if (!(n <= 1.0 + 1e-3 && n >= 1.0 - 1e-3)) b200_detail::check(NVB_ERR_INVALID_ARGUMENT, "Plane", "the normal is not unit length");
  }
  float getDistanceToPoint(const Vector3f& point) const override {
    const float d = -detail::dot3(normal_, center_);
    const float p = d / std::sqrt(detail::dot3(normal_, normal_));
    return detail::dot3(normal_, point) + p;
  }
  bool getRayIntersection(const Vector3f& o, const Vector3f& u, float max_dist, Vector3f* intersect_point,
                          float* intersect_dist) const override {
    const float den = detail::dot3(u, normal_);
    if (std::fabs(den) < kEpsilon) return false;
    const float d = detail::dot3(center_ - o, normal_) / den;
    if (d < 0.0f || d > max_dist) return false;
    *intersect_point = pointAt(o, u, d);
    *intersect_dist = d;
    return true;
  }
  const Vector3f& normal() const { return normal_; }
  NvbPrimitive c_abi() const override {
    NvbPrimitive p = base(NVB_PRIM_PLANE);
    for (int k = 0; k < 3; k++) p.params[k] = normal_[k];
    return p;
  }

 protected:
  Vector3f normal_;
};

/// Cylinder centered on the XY plane, with a given radius and height (in Z).
class Cylinder : public Primitive {
 public:
  Cylinder(const Vector3f& center, float radius, float height)
      : Primitive(center, Type::kCylinder), radius_(radius), height_(height) {}
  float getDistanceToPoint(const Vector3f& p) const override {
    const float zmin = (float)((double)center_[2] - (double)height_ / 2.0);
    const float zmax = (float)((double)center_[2] + (double)height_ / 2.0);
    const float dx = p[0] - center_[0], dy = p[1] - center_[1];
    const float sq = dx * dx + dy * dy;
    if (p[2] >= zmin && p[2] <= zmax) return std::sqrt(sq) - radius_;
    const float dz = p[2] > zmax ? p[2] - zmax : p[2] - zmin;
    return std::sqrt(detail::maxStd(sq - radius_ * radius_, 0.0f) + dz * dz);
  }
  bool getRayIntersection(const Vector3f& o, const Vector3f& u, float max_dist, Vector3f* intersect_point,
                          float* intersect_dist) const override {
    const float r = radius_, h = height_;
    const Vector3f E = o - center_;
    const float a = u[0] * u[0] + u[1] * u[1];
    const float b = 2.0f * E[0] * u[0] + 2.0f * E[1] * u[1];
    const float cc = (E[0] * E[0] + E[1] * E[1]) - r * r;
    if (std::fabs(a) < kEpsilon) return false;
    const float disc = b * b - 4.0f * a * cc;
    if (disc < 0.0f) return false;
    float t1, t2 = -1.0f;
    if (disc <= kEpsilon) {
      t1 = -b / (2.0f * a);
    } else {
      t1 = (-b + std::sqrt(disc)) / (2.0f * a);
      t2 = (-b - std::sqrt(disc)) / (2.0f * a);
    }
    const double hh = (double)h / 2.0;
    const float z1 = E[2] + t1 * u[2], z2 = E[2] + t2 * u[2];
    const bool v1 = t1 >= 0.0f && (double)z1 >= -hh && (double)z1 <= hh;
    const bool v2 = t2 >= 0.0f && (double)z2 >= -hh && (double)z2 <= hh;
    float t3 = 0.0f, t4 = 0.0f;
    bool v3 = false, v4 = false;
    if (std::fabs(u[2]) > kEpsilon) {
      t3 = (float)((-(double)h / 2.0 - (double)E[2]) / (double)u[2]);
      t4 = (float)(((double)h / 2.0 - (double)E[2]) / (double)u[2]);
      const float q3x = E[0] + t3 * u[0], q3y = E[1] + t3 * u[1], q4x = E[0] + t4 * u[0], q4y = E[1] + t4 * u[1];
      v3 = t3 >= 0.0f && std::sqrt(q3x * q3x + q3y * q3y) < r;
      v4 = t4 >= 0.0f && std::sqrt(q4x * q4x + q4y * q4y) < r;
    }
    if (!(v1 || v2 || v3 || v4)) return false;
    float t = max_dist;
    if (v1 && t1 < t) t = t1;
    if (v2 && t2 < t) t = t2;
    if (v3 && t3 < t) t = t3;
    if (v4 && t4 < t) t = t4;
    if (t >= max_dist) return false;
    *intersect_point = pointAt(o, u, t);
    *intersect_dist = t;
    return true;
  }
  NvbPrimitive c_abi() const override {
    NvbPrimitive p = base(NVB_PRIM_CYLINDER);
    p.params[0] = radius_, p.params[1] = height_;
    return p;
  }

 protected:
  float radius_;
  float height_;
};

}  // namespace primitives
}  // namespace nvblox
