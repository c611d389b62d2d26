// nvb_scene.cu -- primitives::Scene on the GPU: Primitive::getDistanceToPoint / getRayIntersection
// (src/primitives/primitives.cpp), Scene::getSignedDistanceToPoint / getRayIntersection (src/primitives/scene.cpp), and
// Scene::generateDepthImageFromScene / generateLayerFromScene (primitives/internal/impl/scene_impl.h).
//
// The reference runs both generators as host loops, one analytic evaluation per pixel or voxel. Here a thread takes one
// pixel, point or voxel and loops over the primitives, which a CTA stages through shared memory in tiles, so a scene may hold
// any number of them. Layer generation allocates the blocks the AABB touches through the device hash in one launch, then a
// CTA per block (512 threads, one voxel each) writes the voxels inside the AABB.
//
// Precision: the reference mixes float and double through its literals; the same promotions are spelled out here, and
// tests/scene_reference.py restates them in numpy. Two places the source leaves open are read as follows. An unqualified
// `sqrt` of a float is the float square root (std::sqrt(float)). Eigen sums three terms as a0 + (a1 + a2) (its unrolled
// reduction, sum3), for dot products and squared norms alike; two terms are a0 + a1. std::max(a, b) is (a < b) ? b : a, and
// Eigen's maxCoeff of three is max(a0, max(a1, a2)) in that form, so signed zeros come out as in the reference.
#include <algorithm>

#include "nvb_internal.cuh"

namespace nvb {

namespace {

constexpr float kEpsilon = 1e-4f;  // Primitive::kEpsilon (primitives.h)
constexpr int kPrimTile = 256;     // primitives staged in shared memory per pass (8 KiB)

template <typename T>
__device__ __forceinline__ T maxStd(T a, T b) {
  return (a < b) ? b : a;
}

__device__ __forceinline__ float dot3(const float a[3], const float b[3]) { return sum3(a[0] * b[0], a[1] * b[1], a[2] * b[2]); }

// ---------------------------------------------------------------------------
// Primitive::getDistanceToPoint
// ---------------------------------------------------------------------------
__device__ float primitiveDistance(const NvbPrimitive& q, const float p[3]) {
  const float* c = q.center;
  switch (q.type) {
    case NVB_PRIM_PLANE: {  // d = -n.c, p = d / |n|, n.x + p
      const float* n = q.params;
      const float d = -dot3(n, c);
      const float off = d / sqrtf(dot3(n, n));
      return dot3(n, p) + off;
    }
    case NVB_PRIM_CUBE: {  // per axis max(max(c - s / 2.0 - p, 0.0), p - c - s / 2.0) in double, rounded to float
      const float* s = q.params;
      double lo[3], hi[3];
      float v[3];
#pragma unroll
      for (int k = 0; k < 3; k++) {
        lo[k] = ((double)c[k] - (double)s[k] / 2.0) - (double)p[k];
        hi[k] = (double)(p[k] - c[k]) - (double)s[k] / 2.0;
        v[k] = (float)maxStd(maxStd(lo[k], 0.0), hi[k]);
      }
      float dist = sqrtf(dot3(v, v));
      if (dist < kEpsilon) {  // inside: the largest per-axis term
#pragma unroll
        for (int k = 0; k < 3; k++) v[k] = (float)maxStd(lo[k], hi[k]);
        dist = maxStd(v[0], maxStd(v[1], v[2]));
      }
      return dist;
    }
    case NVB_PRIM_SPHERE: {
      const float d[3] = {c[0] - p[0], c[1] - p[1], c[2] - p[2]};
      return sqrtf(dot3(d, d)) - q.params[0];
    }
    default: {  // NVB_PRIM_CYLINDER
      const float r = q.params[0], h = q.params[1];
      const float zmin = (float)((double)c[2] - (double)h / 2.0), zmax = (float)((double)c[2] + (double)h / 2.0);
      const float dx = p[0] - c[0], dy = p[1] - c[1];
      const float sq_xy = dx * dx + dy * dy;
      if (p[2] >= zmin && p[2] <= zmax) return sqrtf(sq_xy) - r;
      const float dz = p[2] > zmax ? p[2] - zmax : p[2] - zmin;
      return sqrtf(maxStd(sq_xy - r * r, 0.0f) + dz * dz);
    }
  }
}

// ---------------------------------------------------------------------------
// Primitive::getRayIntersection: whether the ray o + t * u hits within max_dist, and t. Every primitive's intersection point
// is o + t * u per component, so the scene only keeps t.
// ---------------------------------------------------------------------------
__device__ bool primitiveRay(const NvbPrimitive& q, const float o[3], const float u[3], float max_dist, float& t_out) {
  const float* c = q.center;
  switch (q.type) {
    case NVB_PRIM_PLANE: {
      const float* n = q.params;
      const float den = dot3(u, n);
      if (fabsf(den) < kEpsilon) return false;
      const float co[3] = {c[0] - o[0], c[1] - o[1], c[2] - o[2]};
      const float d = dot3(co, n) / den;
      if (d < 0.0f || d > max_dist) return false;
      t_out = d;
      return true;
    }
    case NVB_PRIM_CUBE: {
      const float* s = q.params;
      float inv[3], b0[3], b1[3];
#pragma unroll
      for (int k = 0; k < 3; k++) {
        inv[k] = (float)(1.0 / (double)u[k]);
        b0[k] = c[k] - s[k] / 2.0f;  // center_ -/+ size_ / 2.0 (the literal becomes a float scalar)
        b1[k] = c[k] + s[k] / 2.0f;
      }
      auto slab = [&](int k, float& tlo, float& thi) {
        const bool neg = inv[k] < 0.0f;
        tlo = ((neg ? b1[k] : b0[k]) - o[k]) * inv[k];
        thi = ((neg ? b0[k] : b1[k]) - o[k]) * inv[k];
      };
      float tmin, tmax, tymin, tymax, tzmin, tzmax;
      slab(0, tmin, tmax);
      slab(1, tymin, tymax);
      if ((tmin > tymax) || (tymin > tmax)) return false;
      if (tymin > tmin) tmin = tymin;
      if (tymax < tmax) tmax = tymax;
      slab(2, tzmin, tzmax);
      if ((tmin > tzmax) || (tzmin > tmax)) return false;
      if (tzmin > tmin) tmin = tzmin;
      if (tzmax < tmax) tmax = tzmax;
      float t = tmin;
      if (t < 0.0f) {  // the ray starts inside: the exit
        t = tmax;
        if (t < 0.0f) return false;
      }
      if (t > max_dist) return false;
      t_out = t;
      return true;
    }
    case NVB_PRIM_SPHERE: {
      const float oc[3] = {o[0] - c[0], o[1] - c[1], o[2] - c[2]};
      const float b = dot3(u, oc);
      const double r = (double)q.params[0];
      // pow(..., 2) - squaredNorm + pow(radius, 2) in double
      const float disc = (float)(((double)b * (double)b - (double)dot3(oc, oc)) + r * r);
      if (disc < 0.0f) return false;
      const float d = -b - sqrtf(disc);
      if (d < 0.0f || d > max_dist) return false;  // a ray that starts inside does not hit
      t_out = d;
      return true;
    }
    default: {  // NVB_PRIM_CYLINDER
      const float r = q.params[0], h = q.params[1];
      const float E[3] = {o[0] - c[0], o[1] - c[1], o[2] - c[2]};
      const float a = u[0] * u[0] + u[1] * u[1];
      const float b = 2.0f * E[0] * u[0] + 2.0f * E[1] * u[1];
      const float cc = (E[0] * E[0] + E[1] * E[1]) - r * r;
      if (fabsf(a) < kEpsilon) return false;  // a vertical ray misses, caps included
      const float disc = b * b - 4.0f * a * cc;
      if (disc < 0.0f) return false;
      float t1, t2 = -1.0f;
      if (disc <= kEpsilon) {
        t1 = -b / (2.0f * a);
      } else {
        t1 = (-b + sqrtf(disc)) / (2.0f * a);
        t2 = (-b - sqrtf(disc)) / (2.0f * a);
      }
      const double hh = (double)h / 2.0;
      const float z1 = E[2] + t1 * u[2], z2 = E[2] + t2 * u[2];
      const bool v1 = t1 >= 0.0f && (double)z1 >= -hh && (double)z1 <= hh;
      const bool v2 = t2 >= 0.0f && (double)z2 >= -hh && (double)z2 <= hh;
      float t3 = 0.0f, t4 = 0.0f;
      bool v3 = false, v4 = false;
      if (fabsf(u[2]) > kEpsilon) {
        t3 = (float)((-(double)h / 2.0 - (double)E[2]) / (double)u[2]);
        t4 = (float)(((double)h / 2.0 - (double)E[2]) / (double)u[2]);
        const float q3x = E[0] + t3 * u[0], q3y = E[1] + t3 * u[1];
        const float q4x = E[0] + t4 * u[0], q4y = E[1] + t4 * u[1];
        v3 = t3 >= 0.0f && sqrtf(q3x * q3x + q3y * q3y) < r;
        v4 = t4 >= 0.0f && sqrtf(q4x * q4x + q4y * q4y) < r;
      }
      if (!(v1 || v2 || v3 || v4)) return false;
      float t = max_dist;  // std::min(t, ti) = (ti < t) ? ti : t
      if (v1 && t1 < t) t = t1;
      if (v2 && t2 < t) t = t2;
      if (v3 && t3 < t) t = t3;
      if (v4 && t4 < t) t = t4;
      if (t >= max_dist) return false;
      t_out = t;
      return true;
    }
  }
}

// Stages primitives [first, first + tile) of the scene into shared memory; every thread of the CTA calls it.
__device__ __forceinline__ void stageTile(NvbPrimitive* s, const NvbPrimitive* g, int first, int tile) {
  __syncthreads();
  for (int i = threadIdx.x + blockDim.x * threadIdx.y; i < tile; i += blockDim.x * blockDim.y) s[i] = g[first + i];
  __syncthreads();
}

// Scene::generateDepthImageFromScene: one thread per pixel. Threads outside the image stay for the tile barriers.
template <bool kDistort>
__global__ void __launch_bounds__(128) sceneDepthKernel(const __grid_constant__ SceneDepthArgs a) {
  __shared__ NvbPrimitive s_prims[kPrimTile];
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y * blockDim.y + threadIdx.y;
  const bool in_image = r < a.rows && c < a.cols;
  float dz;
  Vec3 u3;
  pixelRay<kDistort>(a.cam, a.T_S_C, 1, in_image ? r : 0, in_image ? c : 0, dz, u3);
  const float u[3] = {u3.x, u3.y, u3.z};
  // Scene::getRayIntersection: the first primitive with the smallest t
  bool hit = false;
  float best = a.max_dist;
  for (int first = 0; first < a.scene.num_primitives; first += kPrimTile) {
    const int tile = min(kPrimTile, a.scene.num_primitives - first);
    stageTile(s_prims, a.scene.primitives, first, tile);
    if (!in_image) continue;
    for (int s = 0; s < tile; s++) {
      float t;
      if (primitiveRay(s_prims[s], a.T_S_C.t, u, a.max_dist, t) && (!hit || t < best)) hit = true, best = t;
    }
  }
  if (!in_image) return;
  float depth = a.invalid_depth;
  if (hit) {  // Camera::getDepth(T_C_S * p): the z of the hit in the camera frame
    const Vec3 p{a.T_S_C.t[0] + best * u[0], a.T_S_C.t[1] + best * u[1], a.T_S_C.t[2] + best * u[2]};
    depth = transformPoint(a.T_C_S, p).z;
  }
  a.depth[(size_t)r * a.cols + c] = depth;
}

// Scene::getSignedDistanceToPoint: starts at max_dist, the minimum over the primitives.
__device__ __forceinline__ float sceneDistanceTile(const NvbPrimitive* s_prims, int tile, const float p[3], float d) {
  for (int s = 0; s < tile; s++) {
    const float ds = primitiveDistance(s_prims[s], p);
    if (ds < d) d = ds;
  }
  return d;
}

__global__ void __launch_bounds__(256) sceneDistanceKernel(const NvbScene scene, const float* xyz, long long n, float max_dist,
                                                           float* out) {
  __shared__ NvbPrimitive s_prims[kPrimTile];
  for (long long base = (long long)blockIdx.x * blockDim.x; base < n; base += (long long)gridDim.x * blockDim.x) {
    const long long i = base + threadIdx.x;
    float p[3] = {0.0f, 0.0f, 0.0f};
    if (i < n) p[0] = xyz[3 * i], p[1] = xyz[3 * i + 1], p[2] = xyz[3 * i + 2];
    float d = max_dist;
    for (int first = 0; first < scene.num_primitives; first += kPrimTile) {
      const int tile = min(kPrimTile, scene.num_primitives - first);
      stageTile(s_prims, scene.primitives, first, tile);
      d = sceneDistanceTile(s_prims, tile, p, d);
    }
    if (i < n) out[i] = d;
  }
}

// getBlockIndicesTouchedByBoundingBox + allocateBlockAtIndex: one thread per block of the index box, z fastest.
__global__ void sceneAllocateKernel(const __grid_constant__ SceneLayerArgs a) {
  const long long yz = (long long)a.box_size.y * a.box_size.z;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.cells; i += (long long)gridDim.x * blockDim.x) {
    const int x = a.box_lo.x + (int)(i / yz), y = a.box_lo.y + (int)((i / a.box_size.z) % a.box_size.y),
              z = a.box_lo.z + (int)(i % a.box_size.z);
    bool was_new;
    hashFindOrInsert(a.layer, x, y, z, a.error, &was_new);
  }
}

// callFunctionOnAllVoxels with the generator's lambda: a CTA per block of the layer, a thread per voxel. Voxels whose centre is
// outside the closed AABB keep their values.
__global__ void __launch_bounds__(kVpb) sceneFillKernel(const __grid_constant__ SceneLayerArgs a) {
  __shared__ NvbPrimitive s_prims[kPrimTile];
  const int tid = threadIdx.x;
  const int vidx[3] = {tid >> 6, (tid >> 3) & 7, tid & 7};  // linear voxel offset (x * 8 + y) * 8 + z
  const float voxel_size = a.block_size * (1.0f / kVps), half_voxel_size = a.block_size * (0.5f / kVps);
  const int num = a.scene.num_primitives;
  const bool one_tile = num <= kPrimTile;
  if (one_tile) stageTile(s_prims, a.scene.primitives, 0, num);
  const int n = min(*a.layer.count, a.layer.capacity);
  for (int slot = blockIdx.x; slot < n; slot += gridDim.x) {
    const int bidx[3] = {a.layer.block_index[3 * slot], a.layer.block_index[3 * slot + 1], a.layer.block_index[3 * slot + 2]};
    if (bidx[0] == kDeadSlotX) continue;
    float p[3];  // getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:51-81)
#pragma unroll
    for (int k = 0; k < 3; k++) p[k] = (a.block_size * (float)bidx[k] + voxel_size * (float)vidx[k]) + half_voxel_size;
    const bool inside = a.scene.aabb_min[0] <= p[0] && a.scene.aabb_min[1] <= p[1] && a.scene.aabb_min[2] <= p[2] &&
                        p[0] <= a.scene.aabb_max[0] && p[1] <= a.scene.aabb_max[1] && p[2] <= a.scene.aabb_max[2];
    float sdf = a.max_dist;
    for (int first = 0; first < num; first += kPrimTile) {
      const int tile = min(kPrimTile, num - first);
      if (!one_tile) stageTile(s_prims, a.scene.primitives, first, tile);
      if (inside) sdf = sceneDistanceTile(s_prims, tile, p, sdf);
    }
    if (!inside) continue;
    unsigned char* blk = a.layer.blocks + (size_t)slot * a.layer.block_bytes;
    if (a.layer_id == NVB_LAYER_TSDF) {  // setVoxel<TsdfVoxel>(std::max(distance, -max_dist)), weight 1
      reinterpret_cast<float2*>(blk)[tid] = make_float2(maxStd(sdf, -a.max_dist), 1.0f);
    } else {
      const bool object_inside = sdf <= a.occupied_threshold_m;  // the voxel's half body diagonal
      if (a.layer_id == NVB_LAYER_OCCUPANCY)
        reinterpret_cast<float*>(blk)[tid] = object_inside ? a.occupied_log_odds : a.free_log_odds;
      else  // FreespaceVoxel::is_high_confidence_freespace (byte 16 of the 24-byte voxel) only
        blk[(size_t)tid * kFreespaceVoxelBytes + 16] = object_inside ? 0 : 1;
    }
  }
}

}  // namespace

void launchSceneDepth(const SceneDepthArgs& a, cudaStream_t stream) {
  const dim3 threads(16, 8, 1);
  const dim3 grid((a.cols + threads.x - 1) / threads.x, (a.rows + threads.y - 1) / threads.y, 1);
  if (a.cam.has_distortion)
    sceneDepthKernel<true><<<grid, threads, 0, stream>>>(a);
  else
    sceneDepthKernel<false><<<grid, threads, 0, stream>>>(a);
}

void launchSceneDistance(const NvbScene& scene, const float* xyz, long long n, float max_dist, float* out, int num_sms,
                         cudaStream_t stream) {
  if (n <= 0) return;
  const long long need = (n + 255) / 256;
  const int grid = (int)std::min<long long>(need, 16ll * num_sms);
  sceneDistanceKernel<<<grid, 256, 0, stream>>>(scene, xyz, n, max_dist, out);
}

void launchSceneAllocate(const SceneLayerArgs& a, int num_sms, cudaStream_t stream) {
  if (a.cells <= 0) return;
  const int grid = (int)std::min<long long>((a.cells + 255) / 256, 16ll * num_sms);
  sceneAllocateKernel<<<grid, 256, 0, stream>>>(a);
}

void launchSceneFill(const SceneLayerArgs& a, int num_sms, cudaStream_t stream) {
  sceneFillKernel<<<4 * num_sms, kVpb, 0, stream>>>(a);
}

}  // namespace nvb
