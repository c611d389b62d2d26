// nvblox/geometry/plane.h -- Plane and AxisAlignedBoundingBox subset (reference: nvblox/include/nvblox/geometry/plane.h:25-80,
// internal/impl/plane_impl.h:20-72; AxisAlignedBoundingBox = Eigen::AlignedBox3f in core/types.h).
#pragma once
#include <cmath>
#include "nvblox/core/types.h"
namespace nvblox {
// n . x + d = 0 with a unit normal.
class Plane {
 public:
  Plane() : normal_(1.0f, 0.0f, 0.0f), d_(0.0f) {}
  Plane(const Vector3f& normal, float d) : normal_(normalized(normal)), d_(d) {}
  Plane(const Vector3f& normal, const Vector3f& point) : normal_(normalized(normal)) {
    d_ = -(point[0] * normal_[0] + (point[1] * normal_[1] + point[2] * normal_[2]));
  }
  // The plane with exactly these coefficients, without normalising again (the library's planes are already unit length;
  // the reference hands its Plane objects back by copy).
  static Plane fromCoefficients(const Vector3f& unit_normal, float d) {
    Plane p;
    p.normal_ = unit_normal;
    p.d_ = d;
    return p;
  }
  const Vector3f& normal() const { return normal_; }
  float d() const { return d_; }
  float offset() const { return d_; }
  float signedDistance(const Vector3f& p) const { return normal_[0] * p[0] + (normal_[1] * p[1] + normal_[2] * p[2]) + d_; }
  float getHeightAtXY(const Vector2f& xy) const { return -1.0f * (normal_[0] * xy[0] + normal_[1] * xy[1] + d_) / normal_[2]; }

 private:
  static Vector3f normalized(const Vector3f& v) {
    const float n = std::sqrt(v[0] * v[0] + (v[1] * v[1] + v[2] * v[2]));
    return Vector3f(v[0] / n, v[1] / n, v[2] / n);
  }
  Vector3f normal_;
  float d_;
};

// The subset of Eigen::AlignedBox3f the slicer's and the shape clearer's interfaces need (both builds: the reference's type is
// Eigen::AlignedBox3f, whose arithmetic is restated here in Eigen's order).
class AxisAlignedBoundingBox {
 public:
  AxisAlignedBoundingBox() = default;
  AxisAlignedBoundingBox(const Vector3f& mn, const Vector3f& mx) : min_(mn), max_(mx), empty_(false) {}
  const Vector3f& min() const { return min_; }
  const Vector3f& max() const { return max_; }
  bool isEmpty() const { return empty_ || min_[0] > max_[0] || min_[1] > max_[1] || min_[2] > max_[2]; }
  // Eigen::AlignedBox::merged: the box that encloses both (an empty box contributes nothing)
  AxisAlignedBoundingBox merged(const AxisAlignedBoundingBox& o) const {
    if (isEmpty()) return o;
    if (o.isEmpty()) return *this;
    Vector3f mn, mx;
    for (int a = 0; a < 3; a++) mn[a] = min_[a] < o.min_[a] ? min_[a] : o.min_[a], mx[a] = max_[a] > o.max_[a] ? max_[a] : o.max_[a];
    return AxisAlignedBoundingBox(mn, mx);
  }
  // Eigen::AlignedBox::contains(point) / intersects(box): inclusive on both sides
  bool contains(const Vector3f& p) const {
    return min_[0] <= p[0] && min_[1] <= p[1] && min_[2] <= p[2] && p[0] <= max_[0] && p[1] <= max_[1] && p[2] <= max_[2];
  }
  bool intersects(const AxisAlignedBoundingBox& b) const {
    return min_[0] <= b.max_[0] && min_[1] <= b.max_[1] && min_[2] <= b.max_[2] && b.min_[0] <= max_[0] &&
           b.min_[1] <= max_[1] && b.min_[2] <= max_[2];
  }
  // Eigen::AlignedBox::squaredExteriorDistance / exteriorDistance: the axes accumulate in order from 0
  float squaredExteriorDistance(const Vector3f& p) const {
    float dist2 = 0.0f;
    for (int k = 0; k < 3; k++) {
      if (min_[k] > p[k]) {
        const float aux = min_[k] - p[k];
        dist2 += aux * aux;
      } else if (p[k] > max_[k]) {
        const float aux = p[k] - max_[k];
        dist2 += aux * aux;
      }
    }
    return dist2;
  }
  float exteriorDistance(const Vector3f& p) const { return std::sqrt(squaredExteriorDistance(p)); }

 private:
  Vector3f min_, max_;
  bool empty_ = true;
};
}  // namespace nvblox
