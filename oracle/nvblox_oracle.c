/*
 * nvblox_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (see nvblox_oracle.h).
 *
 * CPU restatement of the reference's depth-integration hot path. Citations are
 * relative to nvblox_ros/nvblox_core/nvblox/ of isaac_ros_nvblox ("C/" in SURVEY.md).
 * Parity: "parity unpinned" against a reference binary -- pinned against the reference's
 * known-answer tests only (the reference itself cannot be built in this environment): see
 * tests/test_oracle_kat.py, tests/test_oracle_color_kat.py, tests/test_oracle_esdf_scenes_kat.py.
 *
 * Build: gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared
 */
#include "nvblox_oracle.h"

#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define VPS 8 /* VoxelBlock::kVoxelsPerSide, include/nvblox/map/blox.h:36 */
#define VPB (VPS * VPS * VPS)

typedef struct {
  float x, y, z;
} v3;
typedef struct {
  int32_t x, y, z;
} i3;

/* ------------------------------------------------------------------------- */
/* Scalar helpers                                                            */
/* ------------------------------------------------------------------------- */

/* float -> int with the CUDA device semantics (cvt.rzi.s32.f32): NaN -> 0,
 * saturating. The reference performs these casts in device code. */
static int32_t f2i(float f) {
  if (f != f) return 0;
  if (f >= 2147483648.0f) return INT32_MAX;
  if (f <= -2147483648.0f) return INT32_MIN;
  return (int32_t)f;
}

/* Eigen fixed-size-3 reduction order: a0 + (a1 + a2)
 * (Eigen/src/Core/Redux.h redux_novec_unroller, Length=3 -> {1, 2}). */
static float sum3(float a0, float a1, float a2) { return a0 + (a1 + a2); }

static int signum(float x) { /* ray_caster_impl.h:22-24 */
  return (x > 0.0f) ? 1 : ((x < 0.0f) ? -1 : 0);
}

/* Transform = Eigen::Isometry3f, 4x4 column-major (core/types.h:141-153). */
static float Rm(const float* T, int i, int j) { return T[j * 4 + i]; }
static float Tt(const float* T, int i) { return T[12 + i]; }

/* Isometry * point: res = translation; res += linear * p (lazy coefficient
 * product; Eigen/src/Geometry/Transform.h transform_right_product_impl). */
static v3 transform_point(const float* T, v3 p) {
  v3 r;
  r.x = Tt(T, 0) + sum3(Rm(T, 0, 0) * p.x, Rm(T, 0, 1) * p.y, Rm(T, 0, 2) * p.z);
  r.y = Tt(T, 1) + sum3(Rm(T, 1, 0) * p.x, Rm(T, 1, 1) * p.y, Rm(T, 1, 2) * p.z);
  r.z = Tt(T, 2) + sum3(Rm(T, 2, 0) * p.x, Rm(T, 2, 1) * p.y, Rm(T, 2, 2) * p.z);
  return r;
}

/* Isometry inverse: R' = R^T, t' = -(R^T t) (Transform::inverse, Isometry). */
static void invert_isometry(const float* T, float* out) {
  memset(out, 0, 16 * sizeof(float));
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) out[j * 4 + i] = Rm(T, j, i);
  for (int i = 0; i < 3; i++) {
    out[12 + i] = -sum3(out[0 * 4 + i] * Tt(T, 0), out[1 * 4 + i] * Tt(T, 1),
                        out[2 * 4 + i] * Tt(T, 2));
  }
  out[15] = 1.0f;
}

/* getBlockIndexFromPositionInLayer (core/internal/impl/indexing_impl.h:31-35). */
static i3 block_index_from_position(float block_size, v3 p) {
  i3 r;
  r.x = f2i(floorf(p.x / block_size));
  r.y = f2i(floorf(p.y / block_size));
  r.z = f2i(floorf(p.z / block_size));
  return r;
}

/* ------------------------------------------------------------------------- */
/* Camera (sensors/internal/impl/camera_impl.h)                              */
/* ------------------------------------------------------------------------- */

/* radialDistortionScale<T> (sensors/internal/impl/distortion_impl.h:24-32). The literal 1.0 is a double, so
 * for T = float the float products are promoted and summed in double, then narrowed to T. */
static float radial_scale_f(float r2, const OrCamera* c) {
  const float r4 = r2 * r2;
  const float r6 = r2 * r4;
  const float numerator = (float)(1.0 + (double)(c->k1 * r2) + (double)(c->k2 * r4) + (double)(c->k3 * r6));
  const float denominator = (float)(1.0 + (double)(c->k4 * r2) + (double)(c->k5 * r4) + (double)(c->k6 * r6));
  return numerator / denominator;
}
static double radial_scale_d(double r2, const OrCamera* c) {
  const double r4 = r2 * r2;
  const double r6 = r2 * r4;
  const double numerator = 1.0 + (double)c->k1 * r2 + (double)c->k2 * r4 + (double)c->k3 * r6;
  const double denominator = 1.0 + (double)c->k4 * r2 + (double)c->k5 * r4 + (double)c->k6 * r6;
  return numerator / denominator;
}

/* applyDistortion (distortion_impl.h:37-60): float in/out, tangential terms evaluated in double
 * (2.0 literals) and narrowed to float. */
static void apply_distortion(const OrCamera* c, float* ux, float* uy) {
  const float x = *ux, y = *uy;
  const float r2 = x * x + y * y;
  const float scale = radial_scale_f(r2, c);
  const float xy = x * y;
  const float tx = (float)(2.0 * (double)c->p1 * (double)xy + (double)c->p2 * ((double)r2 + 2.0 * (double)x * (double)x));
  const float ty = (float)(2.0 * (double)c->p2 * (double)xy + (double)c->p1 * ((double)r2 + 2.0 * (double)y * (double)y));
  *ux = x * scale + tx;
  *uy = y * scale + ty;
}

/* compute_dR_dr2 (distortion_impl.h:62-91). */
static double compute_dR_dr2(double r2, double k1, double k2, double k3, double k4, double k5, double k6) {
  const double q = r2, q2 = q * q, q3 = q2 * q;
  const double k4q = k4 * q, k5q2 = k5 * q2, k6q3 = k6 * q3;
  const double a = k1 + 2. * k2 * q + 3. * k3 * q2;
  const double cc = k4 + 2. * k5 * q + 3. * k6 * q2;
  const double b = k4q + k5q2 + k6q3 + 1.;
  const double d = k1 * q + k2 * q2 + k3 * q3 + 1.;
  return (a * b - cc * d) / (b * b);
}

/* removeDistortion (distortion_impl.h:93-176): Newton-Raphson in double, at most 6 iterations. */
static void remove_distortion(const OrCamera* c, float* ux, float* uy) {
  const double k1 = c->k1, k2 = c->k2, k3 = c->k3, k4 = c->k4, k5 = c->k5, k6 = c->k6, p1 = c->p1, p2 = c->p2;
  const double u_in_x = *ux, u_in_y = *uy;
  double x = u_in_x, y = u_in_y;
  for (int i = 0; i < 6; i++) {
    const double x2 = x * x, y2 = y * y, r2 = x2 + y2;
    const double R = radial_scale_d(r2, c);
    const double xy = x * y;
    const double tan_x = 2.0 * p1 * xy + p2 * (r2 + 2.0 * x * x);
    const double tan_y = 2.0 * p2 * xy + p1 * (r2 + 2.0 * y * y);
    const double x_est = x * R + tan_x, y_est = y * R + tan_y;
    const double error_x = x_est - u_in_x, error_y = y_est - u_in_y;
    const double dR_dr2 = compute_dR_dr2(r2, k1, k2, k3, k4, k5, k6);
    const double dR_dx = 2.0 * x * dR_dr2, dR_dy = 2.0 * y * dR_dr2;
    const double a = R + x * dR_dx + 2 * p1 * y + 6 * p2 * x;
    const double b = x * dR_dy + 2 * p1 * x + 2 * p2 * y;
    const double cc = y * dR_dx + 2 * p2 * y + 2 * p1 * x;
    const double d = R + y * dR_dy + 2 * p2 * x + 6 * p1 * y;
    const double det = a * d - b * cc;
    const double delta_x = (d * error_x - b * error_y) / det;
    const double delta_y = (-cc * error_x + a * error_y) / det;
    if (isfinite(delta_x) && isfinite(delta_y)) {
      x = x - delta_x;
      y = y - delta_y;
    }
    if (delta_x * delta_x + delta_y * delta_y < 1e-20) break;
  }
  *ux = (float)x;
  *uy = (float)y;
}

/* vectorFromImagePlaneCoordinates (camera_impl.h:89-104). */
static v3 cam_vector_from_image_plane(const OrCamera* c, float u, float v) {
  v3 r;
  r.x = (u - c->cu) / c->fu;
  r.y = (v - c->cv) / c->fv;
  if (c->has_distortion) remove_distortion(c, &r.x, &r.y);
  r.z = 1.0f;
  return r;
}

/* vectorFromPixelIndices (camera_impl.h:106-112): pixel centre = index + 0.5. */
static v3 cam_vector_from_pixel(const OrCamera* c, int col, int row) {
  return cam_vector_from_image_plane(c, (float)col + 0.5f, (float)row + 0.5f);
}

/* Camera::project (camera_impl.h:37-63, 65-76), min_depth = 1e-6, viewport
 * check on, distortion applied to the normalised coordinates if present. Returns 0 if rejected. */
static int cam_project(const OrCamera* c, v3 p, float* u, float* v) {
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return 0;
  const float min_depth = 1e-6f;
  if (!(p.z >= min_depth)) return 0;
  float un = p.x / p.z;
  float vn = p.y / p.z;
  if (c->has_distortion) apply_distortion(c, &un, &vn);
  *u = un * c->fu + c->cu;
  *v = vn * c->fv + c->cv;
  if (*u > (float)c->width || *v > (float)c->height || *u < 0.0f || *v < 0.0f)
    return 0;
  return 1;
}

/* Camera::getViewAABB (src/sensors/camera.cpp:31-83): 4 image-corner rays at
 * min and max depth, transformed into the layer frame. */
static void cam_view_aabb(const OrCamera* c, const float* T_L_C, float min_depth,
                          float max_depth, v3* mn, v3* mx) {
  const float w = (float)c->width, h = (float)c->height;
  v3 ray[4];
  ray[0] = cam_vector_from_image_plane(c, 0.0f, 0.0f);
  ray[1] = cam_vector_from_image_plane(c, w, 0.0f);
  ray[2] = cam_vector_from_image_plane(c, w, h);
  ray[3] = cam_vector_from_image_plane(c, 0.0f, h);
  const int order[4] = {2, 1, 0, 3};
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
  float hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int k = 0; k < 8; k++) {
    const float d = (k < 4) ? min_depth : max_depth;
    const v3 r = ray[order[k & 3]];
    v3 corner_C = {d * r.x, d * r.y, d * r.z};
    v3 corner_L = transform_point(T_L_C, corner_C);
    const float cl[3] = {corner_L.x, corner_L.y, corner_L.z};
    for (int i = 0; i < 3; i++) {
      /* std::min(a, b) = (b < a) ? b : a ; std::max(a, b) = (a < b) ? b : a */
      lo[i] = (cl[i] < lo[i]) ? cl[i] : lo[i];
      hi[i] = (hi[i] < cl[i]) ? cl[i] : hi[i];
    }
  }
  mn->x = lo[0], mn->y = lo[1], mn->z = lo[2];
  mx->x = hi[0], mx->y = hi[1], mx->z = hi[2];
}

/* applyWorkspaceBounds (src/geometry/workspace_bounds.cpp:20-61). Returns 0 if
 * the resulting AABB is empty (Eigen AlignedBox::isEmpty = any(min > max)). */
static int apply_workspace_bounds(const OrTsdfParams* p, v3* mn, v3* mx) {
  if (p->workspace_bounds_type == OR_WS_HEIGHT_BOUNDS) {
    mn->z = (mn->z < p->workspace_min[2]) ? p->workspace_min[2] : mn->z;
    mx->z = (p->workspace_max[2] < mx->z) ? p->workspace_max[2] : mx->z;
  } else if (p->workspace_bounds_type == OR_WS_BOUNDING_BOX) {
    /* AlignedBox::intersection = (cwiseMax(mins), cwiseMin(maxs)) with the
     * workspace box as *this. */
    float* a[3] = {&mn->x, &mn->y, &mn->z};
    float* b[3] = {&mx->x, &mx->y, &mx->z};
    for (int i = 0; i < 3; i++) {
      *a[i] = (p->workspace_min[i] < *a[i]) ? *a[i] : p->workspace_min[i];
      *b[i] = (*b[i] < p->workspace_max[i]) ? *b[i] : p->workspace_max[i];
    }
  }
  if (mn->x > mx->x || mn->y > mx->y || mn->z > mx->z) return 0;
  return 1;
}

/* ------------------------------------------------------------------------- */
/* RayCaster (rays/internal/impl/ray_caster_impl.h:26-75)                    */
/* ------------------------------------------------------------------------- */

typedef struct {
  int32_t cur[3];
  int32_t sign[3];
  float t_next[3];
  float t_step[3];
  uint32_t step, length;
} RayCaster;

static void raycaster_init(RayCaster* rc, v3 origin, v3 dest, float scale) {
  const float o[3] = {origin.x / scale, origin.y / scale, origin.z / scale};
  const float e[3] = {dest.x / scale, dest.y / scale, dest.z / scale};
  const i3 ci = block_index_from_position(scale, origin);
  const i3 ei = block_index_from_position(scale, dest);
  rc->cur[0] = ci.x, rc->cur[1] = ci.y, rc->cur[2] = ci.z;
  const int32_t end[3] = {ei.x, ei.y, ei.z};
  rc->step = 0;
  /* diff_index.cwiseAbs().sum(): int arithmetic (wraps like the device). */
  uint32_t len = 0;
  for (int i = 0; i < 3; i++) {
    uint32_t d = (uint32_t)end[i] - (uint32_t)rc->cur[i];
    int32_t di = (int32_t)d;
    uint32_t ad = (di < 0) ? (0u - (uint32_t)di) : (uint32_t)di;
    len += ad;
  }
  rc->length = len;
  for (int i = 0; i < 3; i++) {
    const float ray = e[i] - o[i];
    rc->sign[i] = signum(ray);
    const int corrected = rc->sign[i] > 0 ? rc->sign[i] : 0; /* cwiseMax(0) */
    const float shifted = o[i] - (float)rc->cur[i];
    const float dist = (float)corrected - shifted;
    rc->t_next[i] = dist / ray;                 /* NaN/inf allowed */
    rc->t_step[i] = (float)rc->sign[i] / ray;   /* NaN/inf allowed */
  }
}

/* nextRayIndex (ray_caster_impl.h:56-72): returns steps+1 cells. minCoeff is
 * Eigen's visitor: start at element 0, replace on strict '<'. */
static int raycaster_next(RayCaster* rc, int32_t out[3]) {
  /* current_step_++ > ray_length_in_steps_ compares ints in the reference;
   * lengths are far below 2^31 for finite inputs. */
  if ((int32_t)(rc->step++) > (int32_t)rc->length) return 0;
  out[0] = rc->cur[0], out[1] = rc->cur[1], out[2] = rc->cur[2];
  int k = 0;
  float best = rc->t_next[0];
  if (rc->t_next[1] < best) best = rc->t_next[1], k = 1;
  if (rc->t_next[2] < best) best = rc->t_next[2], k = 2;
  rc->cur[k] = (int32_t)((uint32_t)rc->cur[k] + (uint32_t)rc->sign[k]);
  rc->t_next[k] = rc->t_next[k] + rc->t_step[k];
  return 1;
}

int32_t or_raycast_cells(const float origin[3], const float dest[3], float scale,
                         int32_t* out_xyz, int32_t cap) {
  RayCaster rc;
  v3 o = {origin[0], origin[1], origin[2]}, d = {dest[0], dest[1], dest[2]};
  raycaster_init(&rc, o, d, scale);
  int32_t n = 0, c[3];
  while (raycaster_next(&rc, c)) {
    if (n < cap) out_xyz[3 * n] = c[0], out_xyz[3 * n + 1] = c[1], out_xyz[3 * n + 2] = c[2];
    n++;
  }
  return n;
}

/* ------------------------------------------------------------------------- */
/* Block storage: index -> slot hash + dense block arrays                    */
/* ------------------------------------------------------------------------- */

typedef struct {
  int32_t cap; /* power of two */
  int32_t n;
  i3* keys;
  int32_t* vals; /* -1 = empty */
} Hash;

static uint32_t hash_i3(i3 k) {
  uint64_t h = (uint64_t)(uint32_t)k.x * 0x9E3779B97F4A7C15ull;
  h ^= (uint64_t)(uint32_t)k.y * 0xC2B2AE3D27D4EB4Full;
  h ^= (uint64_t)(uint32_t)k.z * 0x165667B19E3779F9ull;
  h ^= h >> 29;
  h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 32;
  return (uint32_t)h;
}

static void hash_init(Hash* h, int32_t cap) {
  h->cap = cap, h->n = 0;
  h->keys = (i3*)malloc(sizeof(i3) * (size_t)cap);
  h->vals = (int32_t*)malloc(sizeof(int32_t) * (size_t)cap);
  for (int32_t i = 0; i < cap; i++) h->vals[i] = -1;
}
static void hash_free(Hash* h) {
  free(h->keys), free(h->vals);
  h->keys = NULL, h->vals = NULL;
}
static int32_t hash_find(const Hash* h, i3 k) {
  uint32_t m = (uint32_t)h->cap - 1, p = hash_i3(k) & m;
  while (h->vals[p] >= 0) {
    if (h->keys[p].x == k.x && h->keys[p].y == k.y && h->keys[p].z == k.z) return h->vals[p];
    p = (p + 1) & m;
  }
  return -1;
}
static void hash_put_raw(Hash* h, i3 k, int32_t v) {
  uint32_t m = (uint32_t)h->cap - 1, p = hash_i3(k) & m;
  while (h->vals[p] >= 0) p = (p + 1) & m;
  h->keys[p] = k, h->vals[p] = v, h->n++;
}
static void hash_put(Hash* h, i3 k, int32_t v) {
  if ((h->n + 1) * 2 > h->cap) {
    Hash g;
    hash_init(&g, h->cap * 2);
    for (int32_t i = 0; i < h->cap; i++)
      if (h->vals[i] >= 0) hash_put_raw(&g, h->keys[i], h->vals[i]);
    hash_free(h);
    *h = g;
  }
  hash_put_raw(h, k, v);
}

typedef struct {
  Hash hash;
  int32_t n, cap;
  size_t block_bytes;
  i3* index;
  uint8_t* data;
} Layer;

static void layer_init(Layer* l, size_t block_bytes) {
  hash_init(&l->hash, 1024);
  l->n = 0, l->cap = 256, l->block_bytes = block_bytes;
  l->index = (i3*)malloc(sizeof(i3) * (size_t)l->cap);
  l->data = (uint8_t*)malloc(block_bytes * (size_t)l->cap);
}
static void layer_free(Layer* l) {
  hash_free(&l->hash);
  free(l->index), free(l->data);
}
static void layer_clear(Layer* l) {
  size_t bb = l->block_bytes;
  layer_free(l);
  layer_init(l, bb);
}
/* BlockLayer::allocateBlockAtIndex (map/internal/impl/layer_impl.h:106-128):
 * new blocks are zero bytes (map/internal/impl/blox_impl.h:37-45,92-97). */
static int32_t layer_allocate(Layer* l, i3 k) {
  int32_t s = hash_find(&l->hash, k);
  if (s >= 0) return s;
  if (l->n == l->cap) {
    l->cap *= 2;
    l->index = (i3*)realloc(l->index, sizeof(i3) * (size_t)l->cap);
    l->data = (uint8_t*)realloc(l->data, l->block_bytes * (size_t)l->cap);
  }
  s = l->n++;
  l->index[s] = k;
  memset(l->data + l->block_bytes * (size_t)s, 0, l->block_bytes);
  hash_put(&l->hash, k, s);
  return s;
}
static void* layer_block(const Layer* l, int32_t slot) {
  return l->data + l->block_bytes * (size_t)slot;
}
/* BlockLayer::clearBlockAsync (map/internal/impl/layer_impl.h): the listed blocks (those that exist) leave the
 * layer. Slots are an internal detail of this file: the survivors are compacted and the hash is rebuilt. */
static void layer_remove_blocks(Layer* l, const i3* keys, int32_t n) {
  if (n == 0 || l->n == 0) return;
  uint8_t* dead = (uint8_t*)calloc((size_t)l->n, 1);
  int any = 0;
  for (int32_t i = 0; i < n; i++) {
    const int32_t s = hash_find(&l->hash, keys[i]);
    if (s >= 0) dead[s] = 1, any = 1;
  }
  if (any) {
    int32_t w = 0;
    for (int32_t s = 0; s < l->n; s++) {
      if (dead[s]) continue;
      if (w != s) {
        l->index[w] = l->index[s];
        memmove(l->data + l->block_bytes * (size_t)w, l->data + l->block_bytes * (size_t)s, l->block_bytes);
      }
      w++;
    }
    l->n = w;
    const int32_t cap = l->hash.cap;
    hash_free(&l->hash);
    hash_init(&l->hash, cap);
    for (int32_t s = 0; s < l->n; s++) hash_put(&l->hash, l->index[s], s);
  }
  free(dead);
}

/* Growable list of block indices. */
typedef struct {
  i3* v;
  int32_t n, cap;
} List;
static void list_push(List* l, i3 k) {
  if (l->n == l->cap) {
    l->cap = l->cap ? l->cap * 2 : 256;
    l->v = (i3*)realloc(l->v, sizeof(i3) * (size_t)l->cap);
  }
  l->v[l->n++] = k;
}
static void list_free(List* l) {
  free(l->v);
  l->v = NULL, l->n = l->cap = 0;
}
static int cmp_i3(const void* a, const void* b) {
  const i3 *p = (const i3*)a, *q = (const i3*)b;
  if (p->x != q->x) return p->x < q->x ? -1 : 1;
  if (p->y != q->y) return p->y < q->y ? -1 : 1;
  if (p->z != q->z) return p->z < q->z ? -1 : 1;
  return 0;
}
/* sortAndTakeUniqueIndices (src/integrators/esdf_integrator.cu:1282-1321): only
 * the resulting SET matters downstream. */
static void list_sort_unique(List* l) {
  if (l->n == 0) return;
  qsort(l->v, (size_t)l->n, sizeof(i3), cmp_i3);
  int32_t w = 1;
  for (int32_t i = 1; i < l->n; i++)
    if (cmp_i3(&l->v[i], &l->v[w - 1]) != 0) l->v[w++] = l->v[i];
  l->n = w;
}

/* MeshBlock (mesh/mesh_block.h:32-83): vertices, vertex_normals, vertex_appearances (Color), triangles */
typedef struct {
  int32_t nv, nt, nc; /* sizes of vertices (= normals), triangles, colours */
  float* v;
  float* nrm;
  int32_t* tri;
  uint8_t* col; /* rgba */
} MeshBlock;

static void mesh_block_release(MeshBlock* b) {
  free(b->v), free(b->nrm), free(b->tri), free(b->col);
  memset(b, 0, sizeof(*b));
}
static void mesh_layer_release(Layer* l) {
  for (int32_t s = 0; s < l->n; s++) mesh_block_release((MeshBlock*)layer_block(l, s));
}

struct OrMap {
  float voxel_size, block_size;
  Layer tsdf, esdf, occ, freespace, color;
  Layer mesh; /* MeshBlockLayer: one MeshBlock header per slot (the arrays hang off it) */
  int64_t freespace_last_update_time_ms; /* FreespaceIntegrator::last_update_time_ms_ (freespace_integrator.h:171) */
  float slice_min_z, slice_max_z, slice_out_z; /* heights of the last or_esdf_integrate_slice call (for the 2-D clear) */
  /* EsdfIntegrator::cleared_block_indices_device_ (integrators/esdf_integrator.h:389)
   * is a member that is only overwritten when a call has blocks to clear
   * (esdf_integrator.cu:242-257), so its content carries over between calls. */
  List esdf_cleared_persistent;
  int64_t stats[8];
  /* ViewpointCache of the projective integrator's ViewCalculator (integrators/view_calculator.h:196,211-244): up to
   * kMaxCacheSize = 2 (pose, sensor, block list) entries, newest first; cache_last_viewpoint_ defaults to true. */
  int32_t cache_last_viewpoint;
  int32_t view_cache_n;
  float view_cache_T[2][16];
  OrCamera view_cache_cam[2];
  List view_cache_blocks[2];
};

void or_default_tsdf_params(OrTsdfParams* p) {
  /* integrators/projective_integrator_params.h:24-63, view_calculator_params.h:22-25 */
  memset(p, 0, sizeof(*p));
  p->truncation_distance_vox = 4.0f;
  p->max_integration_distance_m = 7.0f;
  p->max_weight = 5.0f;
  p->invalid_depth_decay_factor = -1.0f;
  p->weighting_type = OR_WEIGHT_INVERSE_SQUARE;
  p->raycast_subsampling = 4;
  p->workspace_bounds_type = OR_WS_UNBOUNDED;
}
void or_default_esdf_params(OrEsdfParams* p) {
  /* integrators/esdf_integrator_params.h:22-31 */
  p->max_esdf_distance_m = 2.0f;
  p->max_site_distance_vox = 1.0f;
  p->min_weight = 1e-4f;
  p->occupied_threshold = 0.5f; /* esdf_integrator.h:375 */
}
void or_default_occupancy_params(OrOccupancyParams* p) {
  /* integrators/occupancy_integrator_params.h:21-40 */
  p->free_region_occupancy_probability = 0.3f;
  p->occupied_region_occupancy_probability = 0.7f;
  p->unobserved_region_occupancy_probability = 0.5f;
  p->occupied_region_half_width_m = 0.1f;
}

OrMap* or_map_create(float voxel_size_m) {
  OrMap* m = (OrMap*)calloc(1, sizeof(OrMap));
  m->cache_last_viewpoint = 1;
  m->voxel_size = voxel_size_m;
  m->block_size = voxel_size_m * (float)VPS; /* voxelSizeToBlockSize, indexing_impl.h:22 */
  layer_init(&m->tsdf, sizeof(OrTsdfVoxel) * VPB);
  layer_init(&m->esdf, sizeof(OrEsdfVoxel) * VPB);
  layer_init(&m->occ, sizeof(float) * VPB); /* OccupancyVoxel{float log_odds} (map/voxels.h:92-97) */
  layer_init(&m->freespace, sizeof(OrFreespaceVoxel) * VPB);
  layer_init(&m->color, sizeof(OrColorVoxel) * VPB);
  layer_init(&m->mesh, sizeof(MeshBlock));
  return m;
}
void or_map_destroy(OrMap* m) {
  if (!m) return;
  layer_free(&m->tsdf), layer_free(&m->esdf), layer_free(&m->occ), layer_free(&m->freespace), layer_free(&m->color);
  mesh_layer_release(&m->mesh), layer_free(&m->mesh);
  list_free(&m->esdf_cleared_persistent);
  for (int i = 0; i < m->view_cache_n; i++) list_free(&m->view_cache_blocks[i]);
  free(m);
}
void or_map_clear(OrMap* m) {
  layer_clear(&m->tsdf), layer_clear(&m->esdf), layer_clear(&m->occ), layer_clear(&m->freespace), layer_clear(&m->color);
  mesh_layer_release(&m->mesh), layer_clear(&m->mesh);
  m->esdf_cleared_persistent.n = 0;
  /* (Mapper::clear does not touch the integrators: the viewpoint cache survives) */
}

/* ------------------------------------------------------------------------- */
/* View calculation                                                          */
/* ------------------------------------------------------------------------- */

/* layerIndexToAabbLinearIndex + setIndexUpdated (view_calculator_impl.cuh:30-56):
 * int arithmetic, converted to size_t, guarded only by lin < linear_size. */
static void set_index_updated(i3 idx, i3 mn, i3 sz, uint8_t* grid) {
  const size_t linear_size = (size_t)(int64_t)(int32_t)((uint32_t)sz.x * (uint32_t)sz.y * (uint32_t)sz.z);
  const int32_t sx = (int32_t)((uint32_t)idx.x - (uint32_t)mn.x);
  const int32_t sy = (int32_t)((uint32_t)idx.y - (uint32_t)mn.y);
  const int32_t szz = (int32_t)((uint32_t)idx.z - (uint32_t)mn.z);
  const int32_t lin32 = (int32_t)((uint32_t)sx + (uint32_t)sy * (uint32_t)sz.x +
                                  (uint32_t)szz * (uint32_t)sz.x * (uint32_t)sz.y);
  const size_t lin = (size_t)(int64_t)lin32; /* negative -> huge */
  if (lin < linear_size) __atomic_store_n(&grid[lin], (uint8_t)1, __ATOMIC_RELAXED);
}

/* Returns a malloc'ed list of block indices in x-fastest order. */
static int g_view_not_cacheable; /* set when the last view_raycast returned before the cache store (empty workspace) */
static List view_raycast(const float* depth, int rows, int cols, const float* T_L_C,
                         const OrCamera* cam, float block_size, float trunc_m,
                         const OrTsdfParams* P) {
  List out = {0};
  g_view_not_cacheable = 1;
  const float max_dist = P->max_integration_distance_m;
  const int f = P->raycast_subsampling;
  /* view_calculator_impl.cuh:137-156 */
  v3 mn, mx;
  cam_view_aabb(cam, T_L_C, 0.0f, max_dist, &mn, &mx);
  if (!apply_workspace_bounds(P, &mn, &mx)) return out;
  const i3 min_index = block_index_from_position(block_size, mn);
  const i3 max_index = block_index_from_position(block_size, mx);
  const i3 size = {max_index.x - min_index.x + 1, max_index.y - min_index.y + 1,
                   max_index.z - min_index.z + 1};
  const int64_t lin_size = (int64_t)size.x * size.y * size.z;
  if (lin_size <= 0) return out;
  g_view_not_cacheable = 0; /* from here on the result reaches storeResultInCache (view_calculator_impl.cuh:193-196) */
  uint8_t* grid = (uint8_t*)calloc((size_t)lin_size, 1);

  /* getBlocksByRaycastingPixelsAsync launch shape (view_calculator_impl.cuh:200-233). */
  const int rows_s = (int)ceilf((float)(rows + 1) / (float)f);
  const int cols_s = (int)ceilf((float)(cols + 1) / (float)f);
  const int thr_rows = ((rows_s + 15) / 16) * 16;
  const int thr_cols = ((cols_s + 15) / 16) * 16;
  const v3 origin = {Tt(T_L_C, 0), Tt(T_L_C, 1), Tt(T_L_C, 2)};
  const v3 origin_s = {origin.x / block_size, origin.y / block_size, origin.z / block_size};

  /* combinedBlockIndicesInImageKernel (view_calculator_impl.cuh:62-115). */
#pragma omp parallel for schedule(dynamic, 4)
  for (int rr = 0; rr < thr_rows; rr++) {
    for (int rc_ = 0; rc_ < thr_cols; rc_++) {
      int pixel_row = rr * f, pixel_col = rc_ * f;
      if (pixel_row >= rows + f - 1 || pixel_col >= cols + f - 1) continue;
      if (pixel_row >= rows) pixel_row = rows - 1;
      if (pixel_col >= cols) pixel_col = cols - 1;
      float d = depth[(size_t)pixel_row * cols + pixel_col];
      if (d <= 0.0f) continue; /* NaN passes, as in the reference */
      if (max_dist > 0.0f && d > max_dist) d = max_dist;
      const v3 vec = cam_vector_from_pixel(cam, pixel_col, pixel_row);
      const float s = d + trunc_m;
      const v3 p_C = {s * vec.x, s * vec.y, s * vec.z};
      const v3 p_L = transform_point(T_L_C, p_C);
      set_index_updated(block_index_from_position(block_size, p_L), min_index, size, grid);
      const v3 dest_s = {p_L.x / block_size, p_L.y / block_size, p_L.z / block_size};
      RayCaster rc;
      raycaster_init(&rc, origin_s, dest_s, 1.0f);
      int32_t c[3];
      while (raycaster_next(&rc, c)) {
        i3 ci = {c[0], c[1], c[2]};
        set_index_updated(ci, min_index, size, grid);
      }
    }
  }
  /* convertAabbUpdatedToVector (src/integrators/view_calculator.cu:157-195). */
  for (int64_t lin = 0; lin < lin_size; lin++) {
    if (grid[lin]) {
      i3 k = {(int32_t)(lin % size.x) + min_index.x,
              (int32_t)((lin / size.x) % size.y) + min_index.y,
              (int32_t)(lin / ((int64_t)size.x * size.y)) + min_index.z};
      list_push(&out, k);
    }
  }
  free(grid);
  return out;
}

/* arePosesClose (src/geometry/transforms.cpp:20-36) in binary32: T_B1_B2 = T_A_B1^-1 * T_A_B2, translation norm and the angle of
 * Eigen::AngleAxisf(R) (via the quaternion: 2 atan2(|vec|, |w|), Eigen/src/Geometry/AngleAxis.h). */
static int poses_close(const float* T1, const float* T2, float tol_m, float tol_deg) {
  float inv[16], R[3][3], t[3];
  invert_isometry(T1, inv);
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) R[i][j] = (Rm(inv, i, 0) * Rm(T2, 0, j) + Rm(inv, i, 1) * Rm(T2, 1, j)) + Rm(inv, i, 2) * Rm(T2, 2, j);
    t[i] = ((Rm(inv, i, 0) * Tt(T2, 0) + Rm(inv, i, 1) * Tt(T2, 1)) + Rm(inv, i, 2) * Tt(T2, 2)) + Tt(inv, i);
  }
  if (sqrtf(t[0] * t[0] + (t[1] * t[1] + t[2] * t[2])) > tol_m) return 0;
  /* QuaternionBase::operator=(matrix) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl<Other,3,3>) */
  float w, x, y, z;
  const float tr = R[0][0] + R[1][1] + R[2][2];
  if (tr > 0.0f) {
    float q = sqrtf(tr + 1.0f);
    w = 0.5f * q;
    q = 0.5f / q;
    x = (R[2][1] - R[1][2]) * q, y = (R[0][2] - R[2][0]) * q, z = (R[1][0] - R[0][1]) * q;
  } else {
    int i = 0;
    if (R[1][1] > R[0][0]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    float q = sqrtf(R[i][i] - R[j][j] - R[k][k] + 1.0f);
    float v[3];
    v[i] = 0.5f * q;
    q = 0.5f / q;
    w = (R[k][j] - R[j][k]) * q;
    v[j] = (R[j][i] + R[i][j]) * q;
    v[k] = (R[k][i] + R[i][k]) * q;
    x = v[0], y = v[1], z = v[2];
  }
  const float n = sqrtf(x * x + (y * y + z * z));
  const float angle = n != 0.0f ? 2.0f * atan2f(n, fabsf(w)) : 0.0f;
  const float deg = (float)((double)(angle * 180.0f) / 3.14159265358979323846); /* float * 180.0f / M_PI (double) -> float */
  return !(fabsf(deg) > tol_deg);
}
/* operator==(Camera, Camera) (sensors/internal/impl/camera_impl.h:134-156) */
static int cameras_equal(const OrCamera* a, const OrCamera* b) {
  int same = 1;
  same &= fabs((double)(a->fu - b->fu)) <= 0.1;
  same &= fabs((double)(a->fv - b->fv)) <= 0.1;
  same &= fabs((double)(a->cu - b->cu)) <= 0.1;
  same &= fabs((double)(a->cv - b->cv)) <= 0.1;
  same &= a->width == b->width && a->height == b->height;
  same &= (a->has_distortion != 0) == (b->has_distortion != 0);
  if (a->has_distortion && b->has_distortion)
    same &= a->k1 == b->k1 && a->k2 == b->k2 && a->k3 == b->k3 && a->k4 == b->k4 && a->k5 == b->k5 && a->k6 == b->k6 &&
            a->p1 == b->p1 && a->p2 == b->p2;
  return same;
}
/* getBlocksInImageViewRaycast with its ViewpointCache (view_calculator_impl.cuh:117-197, view_calculator_impl.h:120-174): a
 * hit is keyed on the pose (1 mm, 0.1 degree) and the sensor ONLY -- not on the depth image, not on the distances. */
static List view_raycast_cached(OrMap* map, const float* depth, int rows, int cols, const float* T_L_C, const OrCamera* cam,
                                float block_size, float trunc_m, const OrTsdfParams* P) {
  if (map->cache_last_viewpoint) {
    for (int i = 0; i < map->view_cache_n; i++) {
      if (poses_close(T_L_C, map->view_cache_T[i], 0.001f, 0.1f) && cameras_equal(cam, &map->view_cache_cam[i])) {
        List out = {0};
        for (int32_t q = 0; q < map->view_cache_blocks[i].n; q++) list_push(&out, map->view_cache_blocks[i].v[q]);
        return out;
      }
    }
  }
  List l = view_raycast(depth, rows, cols, T_L_C, cam, block_size, trunc_m, P);
  if (map->cache_last_viewpoint && !g_view_not_cacheable) {
    if (map->view_cache_n == 2) { /* pop_back */
      list_free(&map->view_cache_blocks[1]);
      map->view_cache_n = 1;
    }
    if (map->view_cache_n == 1) { /* push_front */
      memcpy(map->view_cache_T[1], map->view_cache_T[0], sizeof(float) * 16);
      map->view_cache_cam[1] = map->view_cache_cam[0];
      map->view_cache_blocks[1] = map->view_cache_blocks[0];
    }
    memcpy(map->view_cache_T[0], T_L_C, sizeof(float) * 16);
    map->view_cache_cam[0] = *cam;
    List copy = {0};
    for (int32_t q = 0; q < l.n; q++) list_push(&copy, l.v[q]);
    map->view_cache_blocks[0] = copy;
    map->view_cache_n++;
  }
  return l;
}
void or_map_cache_last_viewpoint(OrMap* map, int32_t enable) { map->cache_last_viewpoint = enable; }

/* DepthPreprocessor::dilateInvalidRegionsAsync (src/sensors/depth_preprocessing.cpp:36-58), step by step like the NPP calls
 * it is made of (src/sensors/npp_image_operations.cpp): getInvalidDepthMaskAsync = nppiCompareC_32f_C1R(NPP_CMP_LESS)
 * -> 255 where depth < threshold; num_dilations x nppiDilate3x3Border_8u_C1R(NPP_BORDER_REPLICATE) through a double buffer;
 * maskedSetAsync = nppiSet_32f_C1MR -> value where the mask is non-zero. */
void or_depth_dilate_invalid(const float* depth, int32_t rows, int32_t cols, int32_t num_dilations, float threshold,
                             float value, float* out) {
  const size_t n = (size_t)rows * cols;
  uint8_t* a = (uint8_t*)malloc(n);
  uint8_t* b = (uint8_t*)malloc(n);
  for (size_t i = 0; i < n; i++) a[i] = depth[i] < threshold ? 255 : 0;
  for (int32_t it = 0; it < num_dilations; it++) {
    for (int32_t y = 0; y < rows; y++)
      for (int32_t x = 0; x < cols; x++) {
        uint8_t m = 0;
        for (int32_t dy = -1; dy <= 1; dy++)
          for (int32_t dx = -1; dx <= 1; dx++) {
            int32_t yy = y + dy, xx = x + dx; /* replicated border */
            yy = yy < 0 ? 0 : (yy >= rows ? rows - 1 : yy);
            xx = xx < 0 ? 0 : (xx >= cols ? cols - 1 : xx);
            const uint8_t v = a[(size_t)yy * cols + xx];
            if (v > m) m = v;
          }
        b[(size_t)y * cols + x] = m;
      }
    uint8_t* t = a;
    a = b, b = t;
  }
  for (size_t i = 0; i < n; i++) out[i] = a[i] ? value : depth[i];
  free(a), free(b);
}

static int32_t copy_out(const List* l, int32_t* out_xyz, int32_t cap) {
  for (int32_t i = 0; i < l->n && i < cap; i++)
    out_xyz[3 * i] = l->v[i].x, out_xyz[3 * i + 1] = l->v[i].y, out_xyz[3 * i + 2] = l->v[i].z;
  return l->n;
}

int32_t or_view_raycast(const float* depth, int32_t rows, int32_t cols,
                        const float* T_L_C, const OrCamera* cam, float block_size,
                        float truncation_distance_m, const OrTsdfParams* params,
                        int32_t* out_xyz, int32_t cap) {
  List l = view_raycast(depth, rows, cols, T_L_C, cam, block_size, truncation_distance_m, params);
  int32_t n = copy_out(&l, out_xyz, cap);
  list_free(&l);
  return n;
}

/* ------------------------------------------------------------------------- */
/* TSDF                                                                      */
/* ------------------------------------------------------------------------- */

/* WeightingFunction (integrators/internal/impl/weighting_function_impl.h:20-117). */
static float w_dropoff(float measured, float voxel_depth, float trunc) {
  if (trunc <= 1e-2f) return 0.0f;
  if (voxel_depth > measured) {
    const float behind = voxel_depth - measured;
    if (behind > trunc) return 0.0f;
    return (trunc - behind) / trunc;
  }
  return 1.0f;
}
static float w_inverse_square(float measured, float voxel_depth, float trunc) {
  if (voxel_depth <= 1e-2f) return 1.0f;
  if (voxel_depth - measured >= trunc) return 0.0f;
  return 1.0f / (voxel_depth * voxel_depth);
}
static float w_tsdf_penalty(float measured, float voxel_depth, float trunc) {
  const float d = measured - voxel_depth;
  if (fabsf(d) >= trunc) return 0.1f;
  return 1.0f;
}
static float weighting(int type, float measured, float voxel_depth, float trunc) {
  switch (type) {
    case OR_WEIGHT_CONSTANT:
      return 1.0f;
    case OR_WEIGHT_CONSTANT_DROPOFF:
      return 1.0f * w_dropoff(measured, voxel_depth, trunc);
    case OR_WEIGHT_INVERSE_SQUARE:
      return w_inverse_square(measured, voxel_depth, trunc);
    case OR_WEIGHT_INVERSE_SQUARE_DROPOFF:
      return w_inverse_square(measured, voxel_depth, trunc) * w_dropoff(measured, voxel_depth, trunc);
    case OR_WEIGHT_INVERSE_SQUARE_TSDF_DISTANCE_PENALTY:
      return w_inverse_square(measured, voxel_depth, trunc) * w_tsdf_penalty(measured, voxel_depth, trunc);
    case OR_WEIGHT_LINEAR_WITH_MAX:
      return (voxel_depth > 1.0f) ? 1.0f / voxel_depth : 1.0f;
    default:
      abort();
  }
}

/* WeightingFunction::operator(), exposed for the known-answer tests (tests/test_weighting_function.cpp). */
float or_weighting(int32_t type, float measured, float voxel_depth, float trunc) { return weighting(type, measured, voxel_depth, trunc); }

/* UpdateTsdfVoxelFunctor::operator() (integrators/internal/cuda/impl/
 * projective_tsdf_integrator_impl.cuh:30-90). */
static void tsdf_update_voxel(float surface_depth, float voxel_depth, int is_active,
                              float trunc, float max_weight, float decay, int wtype,
                              OrTsdfVoxel* v) {
  if (surface_depth <= 0.0f) {
    if (decay >= 0.0f) v->weight = v->weight * decay;
    return;
  }
  const float sdf = surface_depth - voxel_depth;
  if (sdf < -trunc) return;
  if (!is_active && sdf < trunc) return;
  const float dist_cur = v->distance, w_cur = v->weight;
  const float w = weighting(wtype, surface_depth, voxel_depth, trunc);
  float fused = (sdf * w + dist_cur * w_cur) / (w + w_cur);
  if (fused > 0.0f) {
    fused = fminf(trunc, fused);
  } else {
    fused = fmaxf(-trunc, fused);
  }
  const float weight = fminf(w + w_cur, max_weight);
  v->distance = fused;
  v->weight = weight;
}

/* integrateBlocksKernel for one block (integrators/internal/cuda/impl/
 * projective_integrator_impl.cuh:59-114, projective_integrators_common_impl.cuh:21-55,
 * interpolation/internal/impl/interpolation_2d_impl.h:99-150,
 * sensors/internal/impl/image_impl.h:250-259). */
typedef struct {
  float free_lo, occ_lo, unobs_lo, half_width, min_lo, max_lo;
} OccFunctor;

/* logOddsFromProbability (core/log_odds.h:23-30); evaluated on the host in the reference as well. */
static float log_odds_from_probability(float p) {
  p = fmaxf(1e-3f, fminf(p, 1.0f - 1e-3f));
  return logf(p / (1.0f - p));
}

/* UpdateOccupancyVoxelFunctor::operator() (integrators/internal/cuda/impl/projective_occupancy_integrator_impl.cuh:27-73). */
static void occupancy_update_voxel(float surface_depth, float voxel_depth, int is_active, const OccFunctor* f,
                                   float* log_odds) {
  if (surface_depth <= 0.0f) return;
  float upd;
  if (!is_active || voxel_depth > surface_depth + f->half_width) {
    upd = f->unobs_lo;
  } else if (voxel_depth > surface_depth - f->half_width) {
    upd = f->occ_lo;
  } else {
    upd = f->free_lo;
  }
  const float updated = *log_odds + upd;
  *log_odds = fmaxf(f->min_lo, fminf(updated, f->max_lo));
}

/* `blk` is OrTsdfVoxel[512] when occ == NULL, float[512] otherwise. */
static void projective_integrate_block(void* blk_any, const OccFunctor* occ, i3 bi, const float* depth,
                                 const uint8_t* mask, int mask_mode, int rows, int cols,
                                 const float* T_C_L, const OrCamera* cam, float block_size,
                                 float trunc, const OrTsdfParams* P) {
  OrTsdfVoxel* blk = (OrTsdfVoxel*)blk_any;
  const float voxel_size = block_size * (1.0f / VPS);      /* indexing_impl.h:26-29 */
  const float half_voxel = block_size * (0.5f / VPS);      /* indexing_impl.h:75-77 */
  const float max_depth = P->max_integration_distance_m;
  for (int vx = 0; vx < VPS; vx++)
    for (int vy = 0; vy < VPS; vy++)
      for (int vz = 0; vz < VPS; vz++) {
        /* getCenterPositionFromBlockIndexAndVoxelIndex (indexing_impl.h:51-81) */
        v3 p_L;
        p_L.x = (block_size * (float)bi.x + voxel_size * (float)vx) + half_voxel;
        p_L.y = (block_size * (float)bi.y + voxel_size * (float)vy) + half_voxel;
        p_L.z = (block_size * (float)bi.z + voxel_size * (float)vz) + half_voxel;
        const v3 p_C = transform_point(T_C_L, p_L);
        float u, v;
        if (!cam_project(cam, p_C, &u, &v)) continue;
        const float voxel_depth = p_C.z;
        if (max_depth > 0.0f && voxel_depth > max_depth) continue;
        /* interpolate2DClosest<float, PixelAlwaysValid> */
        const int ux = f2i(floorf(u)), uy = f2i(floorf(v));
        if (ux < 0 || uy < 0 || ux >= cols || uy >= rows) continue;
        float d = depth[(size_t)uy * cols + ux];
        /* PixelIsValidDepth (interpolation_2d_impl.h:99-104) */
        if (!(isfinite(d) && d > 1e-6f)) d = 0.0f;
        /* MaskedImageView::isMasked (image_impl.h:250-259) */
        int is_active = 1;
        if (mask != NULL) {
          const uint8_t mv = mask[(size_t)uy * cols + ux];
          is_active = (mask_mode == OR_MASK_NON_INVERTED) ? (mv != 0) : (mv == 0);
        }
        if (occ == NULL) {
          tsdf_update_voxel(d, voxel_depth, is_active, trunc, P->max_weight,
                            P->invalid_depth_decay_factor, P->weighting_type,
                            &blk[(vx * VPS + vy) * VPS + vz]);
        } else {
          occupancy_update_voxel(d, voxel_depth, is_active, occ, &((float*)blk_any)[(vx * VPS + vy) * VPS + vz]);
        }
      }
}

static void projective_integrate_list(OrMap* map, Layer* layer, const OccFunctor* occ, const List* blocks,
                                const float* depth,
                                const uint8_t* mask, int mask_mode, int rows, int cols,
                                const float* T_L_C, const OrCamera* cam,
                                const OrTsdfParams* P) {
  const float trunc = P->truncation_distance_vox * map->voxel_size;
  /* allocateBlocksWhereRequired (integrators/internal/impl/integrators_common_impl.h:52-58) */
  int32_t* slots = (int32_t*)malloc(sizeof(int32_t) * (size_t)(blocks->n + 1));
  for (int32_t i = 0; i < blocks->n; i++) slots[i] = layer_allocate(layer, blocks->v[i]);
  float T_C_L[16];
  invert_isometry(T_L_C, T_C_L); /* projective_integrator_impl.cuh:268 */
#pragma omp parallel for schedule(static)
  for (int32_t i = 0; i < blocks->n; i++) {
    projective_integrate_block(layer_block(layer, slots[i]), occ, blocks->v[i], depth,
                         mask, mask_mode, rows, cols, T_C_L, cam, map->block_size, trunc, P);
  }
  free(slots);
}
static void tsdf_integrate_list(OrMap* map, const List* blocks, const float* depth, const uint8_t* mask,
                                int mask_mode, int rows, int cols, const float* T_L_C, const OrCamera* cam,
                                const OrTsdfParams* P) {
  projective_integrate_list(map, &map->tsdf, NULL, blocks, depth, mask, mask_mode, rows, cols, T_L_C, cam, P);
}

/* ProjectiveIntegrator::integrateFrameTemplate (projective_integrator_impl.cuh:211-275). */
int32_t or_tsdf_integrate(OrMap* map, const float* depth, const uint8_t* mask,
                          int32_t mask_mode, int32_t rows, int32_t cols,
                          const float* T_L_C, const OrCamera* cam,
                          const OrTsdfParams* P, int32_t* out_xyz, int32_t cap) {
  const float trunc = P->truncation_distance_vox * map->voxel_size;
  List blocks = view_raycast_cached(map, depth, rows, cols, T_L_C, cam, map->block_size, trunc, P);
  if (blocks.n == 0) {
    list_free(&blocks);
    return 0;
  }
  tsdf_integrate_list(map, &blocks, depth, mask, mask_mode, rows, cols, T_L_C, cam, P);
  int32_t n = copy_out(&blocks, out_xyz, cap);
  list_free(&blocks);
  return n;
}

/* ProjectiveOccupancyIntegrator::integrateFrame (projective_occupancy_integrator_impl.cuh:75-86) +
 * setFunctorParameters (src/integrators/projective_occupancy_integrator.cu:42-65). */
int32_t or_occupancy_integrate(OrMap* map, const float* depth, const uint8_t* mask, int32_t mask_mode,
                               int32_t rows, int32_t cols, const float* T_L_C, const OrCamera* cam,
                               OrTsdfParams* P, const OrOccupancyParams* O, int32_t* out_xyz, int32_t cap) {
  OccFunctor f;
  f.free_lo = log_odds_from_probability(O->free_region_occupancy_probability);
  f.occ_lo = log_odds_from_probability(O->occupied_region_occupancy_probability);
  f.unobs_lo = log_odds_from_probability(O->unobserved_region_occupancy_probability);
  f.half_width = O->occupied_region_half_width_m;
  f.max_lo = log_odds_from_probability(0.99f);
  f.min_lo = log_odds_from_probability(0.01f);
  if (P->truncation_distance_vox * map->voxel_size < f.half_width)
    P->truncation_distance_vox = f.half_width / map->voxel_size; /* persists, like the setter call */
  const float trunc = P->truncation_distance_vox * map->voxel_size;
  List blocks = view_raycast_cached(map, depth, rows, cols, T_L_C, cam, map->block_size, trunc, P);
  if (blocks.n == 0) {
    list_free(&blocks);
    return 0;
  }
  projective_integrate_list(map, &map->occ, &f, &blocks, depth, mask, mask_mode, rows, cols, T_L_C, cam, P);
  int32_t n = copy_out(&blocks, out_xyz, cap);
  list_free(&blocks);
  return n;
}

void or_tsdf_integrate_blocks(OrMap* map, const float* depth, const uint8_t* mask,
                              int32_t mask_mode, int32_t rows, int32_t cols,
                              const float* T_L_C, const OrCamera* cam,
                              const OrTsdfParams* P, const int32_t* blocks_xyz,
                              int32_t num_blocks) {
  List l = {0};
  for (int32_t i = 0; i < num_blocks; i++) {
    i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    list_push(&l, k);
  }
  tsdf_integrate_list(map, &l, depth, mask, mask_mode, rows, cols, T_L_C, cam, P);
  list_free(&l);
}

/* ------------------------------------------------------------------------- */
/* ESDF (src/integrators/esdf_integrator.cu)                                 */
/* ------------------------------------------------------------------------- */

#define EV(blk, x, y, z) (&(blk)[((x) * VPS + (y)) * VPS + (z)])

static void esdf_clear_voxel(OrEsdfVoxel* v, float max_sq) { /* :152-157 */
  v->parent_direction[0] = v->parent_direction[1] = v->parent_direction[2] = 0;
  v->squared_distance_vox = max_sq;
  v->is_site = 0;
}

/* updateEsdfVoxelToChanges with TsdfSiteFunctor (:113-138, :401-458). */
static void esdf_apply_observation(int is_observed, int is_inside, int near_surface, float max_sq,
                                   OrEsdfVoxel* e, int* cleared, int* updated);

static void esdf_update_voxel_to_changes(const OrTsdfVoxel* t, int is_freespace, float min_weight,
                                         float max_site_distance_m, float max_sq,
                                         OrEsdfVoxel* e, int* cleared, int* updated) {
  /* TsdfSiteFunctor (:113-138); "voxels being freespace can not be inside an object" (:413-415) */
  esdf_apply_observation(t->weight >= min_weight, (t->distance <= 0.0f) & !is_freespace,
                         fabsf(t->distance) <= max_site_distance_m, max_sq, e, cleared, updated);
}

/* OccupancySiteFunctor (:140-170): observed <=> |log_odds - 0| > 1e-4; inside <=> log_odds > threshold;
 * every inside voxel is near the surface. */
static void esdf_update_voxel_to_changes_occ(float log_odds, float threshold_log_odds, float max_sq, OrEsdfVoxel* e,
                                             int* cleared, int* updated) {
  esdf_apply_observation(fabsf(log_odds - 0.0f) > 1e-4f, log_odds > threshold_log_odds, 1, max_sq, e, cleared, updated);
}

/* updateEsdfVoxelToChanges (:401-458), no freespace layer. */
static void esdf_apply_observation(int is_observed, int is_inside_in, int near_surface, float max_sq,
                                   OrEsdfVoxel* e, int* cleared, int* updated) {
  if (is_observed) {
    const int is_inside = is_inside_in;
    const int is_site = is_inside && near_surface;
    if (e->is_inside && !is_inside) {
      esdf_clear_voxel(e, max_sq);
      *cleared = 1;
    }
    e->is_inside = (uint8_t)is_inside;
    if (is_site) {
      if (e->is_site) {
        *updated = 1;
      } else {
        e->is_site = 1;
        e->squared_distance_vox = 0.0f;
        e->parent_direction[0] = e->parent_direction[1] = e->parent_direction[2] = 0;
        *updated = 1;
      }
    } else {
      if (e->is_site) {
        esdf_clear_voxel(e, max_sq);
        *cleared = 1;
      } else if (!e->observed) {
        esdf_clear_voxel(e, max_sq);
      } else if ((double)e->squared_distance_vox <= 1e-4) { /* double literal, as in :447 */
        esdf_clear_voxel(e, max_sq);
        *cleared = 1;
      }
    }
    e->observed = 1;
  } else {
    esdf_clear_voxel(e, max_sq);
    *cleared = 1;
    e->observed = 0;
  }
}

/* sweepSingleBand (:542-600): forward then backward pass along one line. */
static void esdf_sweep_line(OrEsdfVoxel* blk, int vi[3], int axis, float max_sq) {
  for (int pass = 0; pass < 2; pass++) {
    int last_site[3] = {0, 0, 0};
    int site_found = 0;
    const int direction = pass ? -1 : 1;
    const int start = pass ? VPS - 1 : 0;
    const int end = pass ? -1 : VPS;
    for (vi[axis] = start; vi[axis] != end; vi[axis] += direction) {
      OrEsdfVoxel* e = EV(blk, vi[0], vi[1], vi[2]);
      if (!e->observed) continue;
      if (e->is_site) {
        last_site[0] = vi[0], last_site[1] = vi[1], last_site[2] = vi[2];
        site_found = 1;
      } else if (!site_found) {
        if (e->squared_distance_vox < max_sq) {
          site_found = 1;
          for (int k = 0; k < 3; k++) last_site[k] = e->parent_direction[k] + vi[k];
        }
      } else {
        int pd[3];
        for (int k = 0; k < 3; k++) pd[k] = last_site[k] - vi[k];
        /* Vector3i::squaredNorm() -> int, then converted to float. */
        const float pdist = (float)(pd[0] * pd[0] + (pd[1] * pd[1] + pd[2] * pd[2]));
        if (e->squared_distance_vox > pdist) {
          for (int k = 0; k < 3; k++) e->parent_direction[k] = pd[k];
          e->squared_distance_vox = pdist;
        } else if (e->squared_distance_vox < max_sq) {
          for (int k = 0; k < 3; k++) last_site[k] = e->parent_direction[k] + vi[k];
        }
      }
    }
  }
}

/* sweepBlockBandKernel (:1390-1431): x lines, then y lines, then z lines. */
static void esdf_sweep_block(OrEsdfVoxel* blk, float max_sq) {
  for (int axis = 0; axis < 3; axis++)
    for (int a = 0; a < VPS; a++)
      for (int b = 0; b < VPS; b++) {
        int vi[3];
        if (axis == 0) vi[0] = 0, vi[1] = a, vi[2] = b;
        else if (axis == 1) vi[0] = a, vi[1] = 0, vi[2] = b;
        else vi[0] = a, vi[1] = b, vi[2] = 0;
        esdf_sweep_line(blk, vi, axis, max_sq);
      }
}

static void esdf_sweep_list(OrMap* map, const List* l, float max_sq) {
#pragma omp parallel for schedule(static)
  for (int32_t i = 0; i < l->n; i++) {
    const int32_t s = hash_find(&map->esdf.hash, l->v[i]);
    if (s < 0) continue;
    esdf_sweep_block((OrEsdfVoxel*)layer_block(&map->esdf, s), max_sq);
  }
  map->stats[5] += l->n;
}

/* updateSingleNeighbor (:602-633). */
static int esdf_update_single_neighbor(const OrEsdfVoxel* e, OrEsdfVoxel* n, int axis,
                                       int direction, float max_sq) {
  if (!e->observed || !n->observed || n->is_site || e->squared_distance_vox >= max_sq) return 0;
  int pd[3] = {e->parent_direction[0], e->parent_direction[1], e->parent_direction[2]};
  pd[axis] -= direction;
  const float pdist = (float)(pd[0] * pd[0] + (pd[1] * pd[1] + pd[2] * pd[2]));
  if (n->squared_distance_vox > pdist) {
    n->parent_direction[0] = pd[0], n->parent_direction[1] = pd[1], n->parent_direction[2] = pd[2];
    n->squared_distance_vox = pdist;
    return 1;
  }
  return 0;
}

/* updateNeighborBands (:1323-1386): six sequential passes over the whole list
 * (+x,-x,+y,-y,+z,-z; getDirectionAndVoxelIndicesFromThread :1062-1091), each
 * seeing the writes of the previous ones; then sort-unique of the touched
 * neighbours. */
static List esdf_update_neighbor_bands(OrMap* map, const List* l, float max_sq) {
  List out = {0};
  uint8_t* flag = (uint8_t*)malloc((size_t)l->n + 1);
  for (int i = 0; i < 6; i++) {
    const int axis = i / 2, direction = (i % 2) ? -1 : 1;
    memset(flag, 0, (size_t)l->n + 1);
#pragma omp parallel for schedule(static)
    for (int32_t b = 0; b < l->n; b++) {
      const int32_t s = hash_find(&map->esdf.hash, l->v[b]);
      i3 nk = l->v[b];
      if (axis == 0) nk.x += direction;
      else if (axis == 1) nk.y += direction;
      else nk.z += direction;
      const int32_t ns = hash_find(&map->esdf.hash, nk);
      if (s < 0 || ns < 0) continue;
      const OrEsdfVoxel* blk = (const OrEsdfVoxel*)layer_block(&map->esdf, s);
      OrEsdfVoxel* nblk = (OrEsdfVoxel*)layer_block(&map->esdf, ns);
      int any = 0;
      for (int tx = 0; tx < VPS; tx++)
        for (int ty = 0; ty < VPS; ty++) {
          int vi[3], ni[3];
          if (axis == 0) vi[0] = 0, vi[1] = tx, vi[2] = ty;
          else if (axis == 1) vi[0] = tx, vi[1] = 0, vi[2] = ty;
          else vi[0] = tx, vi[1] = ty, vi[2] = 0;
          ni[0] = vi[0], ni[1] = vi[1], ni[2] = vi[2];
          if (direction < 0) vi[axis] = 0, ni[axis] = VPS - 1;
          else vi[axis] = VPS - 1, ni[axis] = 0;
          any |= esdf_update_single_neighbor(EV(blk, vi[0], vi[1], vi[2]),
                                             EV(nblk, ni[0], ni[1], ni[2]), axis, direction, max_sq);
        }
      flag[b] = (uint8_t)any;
    }
    for (int32_t b = 0; b < l->n; b++)
      if (flag[b]) {
        i3 nk = l->v[b];
        if (axis == 0) nk.x += direction;
        else if (axis == 1) nk.y += direction;
        else nk.z += direction;
        list_push(&out, nk);
      }
    map->stats[6] += l->n;
  }
  free(flag);
  list_sort_unique(&out);
  return out;
}

/* Debug aid (not part of the algorithm): when set, every ring's ESDF slot list is appended to this file. */
static FILE* g_ring_dump = NULL;
void or_debug_ring_dump(const char* path) {
  if (g_ring_dump) fclose(g_ring_dump);
  g_ring_dump = path ? fopen(path, "w") : NULL;
}
static void dump_ring(const OrMap* map, const List* l, const char* tag) {
  if (!g_ring_dump) return;
  fprintf(g_ring_dump, "%s %d", tag, l->n);
  for (int32_t i = 0; i < l->n; i++) fprintf(g_ring_dump, " %d", hash_find(&map->esdf.hash, l->v[i]));
  fprintf(g_ring_dump, "\n");
}

/* computeEsdf (:1465-1496). */
static void esdf_compute(OrMap* map, const List* blocks_with_sites, float max_sq) {
  if (blocks_with_sites->n == 0) return;
  List cur = {0};
  for (int32_t i = 0; i < blocks_with_sites->n; i++) list_push(&cur, blocks_with_sites->v[i]);
  dump_ring(map, &cur, "init");
  esdf_sweep_list(map, &cur, max_sq);
  while (cur.n > 0) {
    List upd = esdf_update_neighbor_bands(map, &cur, max_sq);
    dump_ring(map, &upd, "ring");
    esdf_sweep_list(map, &upd, max_sq);
    list_free(&cur);
    cur = upd;
    map->stats[7]++;
  }
  list_free(&cur);
}

/* getBlockAndVoxelIndexFromOffset (:1498-1520): C++ '/' and '%' truncate. */
static void block_and_voxel_from_offset(i3 bi, const int vi[3], const int32_t off[3],
                                        i3* nb, int nv[3]) {
  int32_t b[3] = {bi.x, bi.y, bi.z};
  for (int i = 0; i < 3; i++) {
    b[i] = b[i] + off[i] / VPS;
    nv[i] = vi[i] + off[i] % VPS;
    if (nv[i] >= VPS) {
      nv[i] -= VPS;
      b[i]++;
    } else if (nv[i] < 0) {
      nv[i] += VPS;
      b[i]--;
    }
  }
  nb->x = b[0], nb->y = b[1], nb->z = b[2];
}

/* clearAllInvalid + clearAllInvalidKernel (:1522-1647); candidate selection by
 * getBlocksWithinRadiusOfAABB (src/geometry/bounding_spheres.cpp:76-91),
 * getAABBOfBlocks (src/geometry/bounding_boxes.cpp:20-27). */
static void esdf_clear_all_invalid(OrMap* map, const List* to_clear, float max_esdf_distance_m,
                                   float max_sq, List* cleared_out) {
  if (to_clear->n == 0) return;
  const float bs = map->block_size;
  /* Merged AABB of the to-clear blocks. */
  float amin[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, amax[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int32_t i = 0; i < to_clear->n; i++) {
    const int32_t k[3] = {to_clear->v[i].x, to_clear->v[i].y, to_clear->v[i].z};
    for (int a = 0; a < 3; a++) {
      const float lo = (float)k[a] * bs, hi = ((float)k[a] + 1.0f) * bs;
      amin[a] = (lo < amin[a]) ? lo : amin[a];
      amax[a] = (amax[a] < hi) ? hi : amax[a];
    }
  }
  cleared_out->n = 0; /* resizeAsync + overwrite */
  const int32_t nb = map->esdf.n;
  uint8_t* flag = (uint8_t*)calloc((size_t)nb + 1, 1);
  int64_t candidates = 0;
#pragma omp parallel for schedule(static) reduction(+ : candidates)
  for (int32_t s = 0; s < nb; s++) {
    const i3 bi = map->esdf.index[s];
    const int32_t k[3] = {bi.x, bi.y, bi.z};
    /* AlignedBox::exteriorDistance = sqrt(squaredExteriorDistance) */
    float d2 = 0.0f;
    for (int a = 0; a < 3; a++) {
      const float lo = (float)k[a] * bs, hi = ((float)k[a] + 1.0f) * bs;
      if (amin[a] > hi) {
        const float aux = amin[a] - hi;
        d2 += aux * aux;
      } else if (lo > amax[a]) {
        const float aux = lo - amax[a];
        d2 += aux * aux;
      }
    }
    if (sqrtf(d2) > max_esdf_distance_m) continue;
    candidates++;
    OrEsdfVoxel* blk = (OrEsdfVoxel*)layer_block(&map->esdf, s);
    int any = 0;
    for (int x = 0; x < VPS; x++)
      for (int y = 0; y < VPS; y++)
        for (int z = 0; z < VPS; z++) {
          OrEsdfVoxel* e = EV(blk, x, y, z);
          const int32_t* pd = e->parent_direction;
          if (e->observed && !e->is_site && (pd[0] != 0 || pd[1] != 0 || pd[2] != 0)) {
            const int vi[3] = {x, y, z};
            i3 nbk;
            int nv[3];
            block_and_voxel_from_offset(bi, vi, pd, &nbk, nv);
            const OrEsdfVoxel* parent = NULL;
            if (nbk.x == bi.x && nbk.y == bi.y && nbk.z == bi.z) {
              parent = EV(blk, nv[0], nv[1], nv[2]);
            } else {
              const int32_t ps = hash_find(&map->esdf.hash, nbk);
              if (ps >= 0) parent = EV((const OrEsdfVoxel*)layer_block(&map->esdf, ps), nv[0], nv[1], nv[2]);
            }
            /* is_site is never written by this kernel, so reading it from another
             * block while that block is being processed is race-free. */
            if (parent == NULL || !parent->is_site) {
              e->parent_direction[0] = e->parent_direction[1] = e->parent_direction[2] = 0;
              e->squared_distance_vox = max_sq;
              any = 1;
            }
          }
        }
    flag[s] = (uint8_t)any;
  }
  for (int32_t s = 0; s < nb; s++)
    if (flag[s]) list_push(cleared_out, map->esdf.index[s]);
  free(flag);
  map->stats[3] += candidates;
}

/* EsdfIntegrator::integrateBlocksTemplate<TsdfLayer> (:220-260) with
 * markAllSites (:678-747) / markAllSitesKernel (:467-540). */
static void esdf_integrate_from(OrMap* map, int from_occupancy, int use_freespace, const int32_t* blocks_xyz,
                                int32_t num_blocks, const OrEsdfParams* P);
void or_esdf_integrate(OrMap* map, const int32_t* blocks_xyz, int32_t num_blocks, const OrEsdfParams* P) {
  esdf_integrate_from(map, 0, 0, blocks_xyz, num_blocks, P);
}
void or_esdf_integrate_occupancy(OrMap* map, const int32_t* blocks_xyz, int32_t num_blocks, const OrEsdfParams* P) {
  esdf_integrate_from(map, 1, 0, blocks_xyz, num_blocks, P);
}
/* EsdfIntegrator::integrateBlocks(tsdf_layer, freespace_layer, blocks, esdf_layer) (esdf_integrator.h:64-70, .cu:266-275). */
void or_esdf_integrate_with_freespace(OrMap* map, const int32_t* blocks_xyz, int32_t num_blocks, const OrEsdfParams* P) {
  esdf_integrate_from(map, 0, 1, blocks_xyz, num_blocks, P);
}
static void esdf_integrate_from(OrMap* map, int from_occupancy, int use_freespace, const int32_t* blocks_xyz,
                                int32_t num_blocks, const OrEsdfParams* P) {
  memset(map->stats, 0, sizeof(map->stats));
  if (num_blocks == 0) return;
  /* allocateBlocksOnCPU (:391-397) */
  List blocks = {0};
  for (int32_t i = 0; i < num_blocks; i++) {
    i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    list_push(&blocks, k);
    layer_allocate(&map->esdf, k);
  }
  /* Real callers pass a set (Mapper::getBlocksToUpdate, src/mapper/mapper.cpp:523-537);
   * a duplicated entry would make two CTAs race on one block in the reference. */
  list_sort_unique(&blocks);
  num_blocks = blocks.n;
  /* :693-696 */
  const float max_esdf_distance_vox = P->max_esdf_distance_m / map->voxel_size;
  const float max_sq = max_esdf_distance_vox * max_esdf_distance_vox;
  const float max_site_distance_m = P->max_site_distance_vox * map->voxel_size; /* :672-676 */
  const float occupied_threshold_log_odds = log_odds_from_probability(P->occupied_threshold); /* :71-75 */

  uint8_t* upd = (uint8_t*)calloc((size_t)num_blocks, 1);
  uint8_t* clr = (uint8_t*)calloc((size_t)num_blocks, 1);
#pragma omp parallel for schedule(static)
  for (int32_t i = 0; i < num_blocks; i++) {
    const Layer* src = from_occupancy ? &map->occ : &map->tsdf;
    const int32_t ts = hash_find(&src->hash, blocks.v[i]);
    const int32_t es = hash_find(&map->esdf.hash, blocks.v[i]);
    if (ts < 0 || es < 0) continue;
    OrEsdfVoxel* e = (OrEsdfVoxel*)layer_block(&map->esdf, es);
    int cleared = 0, updated = 0;
    if (from_occupancy) {
      const float* lo = (const float*)layer_block(src, ts);
      for (int v = 0; v < VPB; v++)
        esdf_update_voxel_to_changes_occ(lo[v], occupied_threshold_log_odds, max_sq, &e[v], &cleared, &updated);
    } else {
      const OrTsdfVoxel* t = (const OrTsdfVoxel*)layer_block(src, ts);
      /* isVoxelFreespace (:101-111): no freespace block -> not freespace */
      const int32_t fs = use_freespace ? hash_find(&map->freespace.hash, blocks.v[i]) : -1;
      const OrFreespaceVoxel* f = fs >= 0 ? (const OrFreespaceVoxel*)layer_block(&map->freespace, fs) : NULL;
      for (int v = 0; v < VPB; v++)
        esdf_update_voxel_to_changes(&t[v], f ? f[v].is_high_confidence_freespace != 0 : 0, P->min_weight,
                                     max_site_distance_m, max_sq, &e[v], &cleared, &updated);
    }
    upd[i] = (uint8_t)updated, clr[i] = (uint8_t)cleared;
  }
  List updated = {0}, to_clear = {0};
  for (int32_t i = 0; i < num_blocks; i++) {
    if (upd[i]) list_push(&updated, blocks.v[i]);
    if (clr[i]) list_push(&to_clear, blocks.v[i]);
  }
  free(upd), free(clr);
  map->stats[0] = num_blocks, map->stats[1] = updated.n, map->stats[2] = to_clear.n;

  if (to_clear.n > 0) {
    esdf_clear_all_invalid(map, &to_clear, P->max_esdf_distance_m, max_sq,
                           &map->esdf_cleared_persistent);
  }
  map->stats[4] = map->esdf_cleared_persistent.n;
  esdf_compute(map, &updated, max_sq);
  if (map->esdf_cleared_persistent.n > 0) esdf_compute(map, &map->esdf_cleared_persistent, max_sq);
  list_free(&blocks), list_free(&updated), list_free(&to_clear);
}

/* getBlockAndVoxelIndexFrom1DPositionInLayer (core/internal/impl/indexing_impl.h:105-115). */
static void block_and_voxel_from_1d(float block_size, float p, int* block_idx, int* voxel_idx) {
  const float voxel_size_inv = (float)(1.0 / (double)(block_size * (1.0f / VPS)));
  const int b = f2i(floorf(p / block_size));
  int v = f2i((p - block_size * (float)b) * voxel_size_inv);
  if (v > VPS - 1) v = VPS - 1;
  *block_idx = b, *voxel_idx = v;
}

/* EsdfIntegrator::integrateSlice with a ConstantZSliceDescription (src/integrators/esdf_integrator.cu:283-347,
 * markSitesInSlice + markSitesInSliceKernel :754-1055): the band z_min..z_max of the projective layer is squashed
 * onto the x/y voxels of ONE layer of ESDF blocks (min TSDF distance / max log odds of the observed, non-freespace
 * voxels of each column), those voxels go through updateEsdfVoxelToChanges, and the usual clear + computeEsdf
 * follow on the slice's blocks. */
static void esdf_integrate_slice_impl(OrMap* map, int32_t from_occupancy, int32_t use_freespace, const int32_t* blocks_xyz,
                                      int32_t num_blocks, const OrEsdfParams* P, float z_min_m, float z_max_m, float z_output_m,
                                      const float* plane, float above_plane_m, float thickness_m);
void or_esdf_integrate_slice(OrMap* map, int32_t from_occupancy, int32_t use_freespace, const int32_t* blocks_xyz,
                             int32_t num_blocks, const OrEsdfParams* P, float z_min_m, float z_max_m, float z_output_m) {
  map->slice_min_z = z_min_m, map->slice_max_z = z_max_m, map->slice_out_z = z_output_m;
  esdf_integrate_slice_impl(map, from_occupancy, use_freespace, blocks_xyz, num_blocks, P, z_min_m, z_max_m, z_output_m, NULL, 0.0f,
                            0.0f);
}
/* integrateSlice with a PlanarSliceDescription (esdf_integrator.cu:349-390; PlanarSliceColumnBoundsGetter,
 * esdf_integrator_slicing_impl.cuh:90-130): the band starts `above_plane_m` above the ground plane
 * n . p + d = 0 (plane = nx, ny, nz, d with a unit normal) and is `thickness_m` thick, per voxel column. */
void or_esdf_integrate_slice_planar(OrMap* map, int32_t from_occupancy, int32_t use_freespace, const int32_t* blocks_xyz,
                                    int32_t num_blocks, const OrEsdfParams* P, const float plane[4], float above_plane_m,
                                    float thickness_m, float z_output_m) {
  float pl[4] = {plane[0], plane[1], plane[2], plane[3]};
  if (fabsf(pl[2]) < 1e-4f) pl[0] = 0.0f, pl[1] = 0.0f, pl[2] = 1.0f, pl[3] = 0.0f; /* checkForVerticalPlane (:208-216) */
  esdf_integrate_slice_impl(map, from_occupancy, use_freespace, blocks_xyz, num_blocks, P, 0.0f, 0.0f, z_output_m, pl, above_plane_m,
                            thickness_m);
}
/* PlanarSliceColumnBoundsGetter::getColumnBounds (esdf_integrator_slicing_impl.cuh:103-130): out = min block z, min voxel z,
 * max block z, max voxel z of the band over the voxel column (block x/y, voxel x/y). */
void or_planar_column_bounds(float block_size, const float plane[4], float above_plane_m, float thickness_m, int32_t bx, int32_t by,
                             int32_t vx, int32_t vy, int32_t out[4]) {
  const float vs = block_size * (1.0f / VPS), half = block_size * (0.5f / VPS);
  const float px = (block_size * (float)bx + vs * (float)vx) + half;
  const float py = (block_size * (float)by + vs * (float)vy) + half;
  const float plane_h = -1.0f * (plane[0] * px + plane[1] * py + plane[3]) / plane[2]; /* Plane::getHeightAtXY */
  const float lo_h = plane_h + above_plane_m, hi_h = lo_h + thickness_m;
  int b0, v0, b1, v1;
  block_and_voxel_from_1d(block_size, lo_h, &b0, &v0);
  block_and_voxel_from_1d(block_size, hi_h, &b1, &v1);
  out[0] = b0, out[1] = v0, out[2] = b1, out[3] = v1;
}
/* PlanarSliceColumnBoundsGetter::num_blocks_in_vertical_column (:84-101) */
int32_t or_planar_num_blocks_in_column(float block_size, float thickness_m) { return f2i(ceilf(thickness_m / block_size)) + 1; }
/* getBlockAndVoxelIndexFrom1DPositionInLayer, exposed for the known-answer tests */
void or_block_and_voxel_from_1d(float block_size, float p, int32_t out[2]) {
  int b, v;
  block_and_voxel_from_1d(block_size, p, &b, &v);
  out[0] = b, out[1] = v;
}
static void esdf_integrate_slice_impl(OrMap* map, int32_t from_occupancy, int32_t use_freespace, const int32_t* blocks_xyz,
                                      int32_t num_blocks, const OrEsdfParams* P, float z_min_m, float z_max_m, float z_output_m,
                                      const float* plane, float above_plane_m, float thickness_m) {
  memset(map->stats, 0, sizeof(map->stats));
  if (num_blocks == 0) return;
  const float max_esdf_distance_vox = P->max_esdf_distance_m / map->voxel_size;
  const float max_sq = max_esdf_distance_vox * max_esdf_distance_vox;
  const float max_site_distance_m = P->max_site_distance_vox * map->voxel_size;
  const float occupied_threshold_log_odds = log_odds_from_probability(P->occupied_threshold);
  int out_bz, out_vz, cmin_bz, cmin_vz, cmax_bz, cmax_vz;
  block_and_voxel_from_1d(map->block_size, z_output_m, &out_bz, &out_vz);
  block_and_voxel_from_1d(map->block_size, z_min_m, &cmin_bz, &cmin_vz); /* ConstantZColumnBoundsGetter (:76-88 of the impl) */
  block_and_voxel_from_1d(map->block_size, z_max_m, &cmax_bz, &cmax_vz);
  /* one output block per vertical column (Index3DSet, :968-973) */
  List blocks = {0};
  {
    Hash seen;
    int32_t hc = 16;
    while (hc < 4 * num_blocks) hc *= 2;
    hash_init(&seen, hc);
    for (int32_t i = 0; i < num_blocks; i++) {
      i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], out_bz};
      if (hash_find(&seen, k) >= 0) continue;
      hash_put(&seen, k, i);
      list_push(&blocks, k);
      layer_allocate(&map->esdf, k);
    }
    hash_free(&seen);
  }
  const Layer* src = from_occupancy ? &map->occ : &map->tsdf;
  uint8_t* upd = (uint8_t*)calloc((size_t)blocks.n, 1);
  uint8_t* clr = (uint8_t*)calloc((size_t)blocks.n, 1);
#pragma omp parallel for schedule(static)
  for (int32_t i = 0; i < blocks.n; i++) {
    const i3 ob = blocks.v[i];
    OrEsdfVoxel* e = (OrEsdfVoxel*)layer_block(&map->esdf, hash_find(&map->esdf.hash, ob));
    int cleared = 0, updated = 0;
    for (int vx = 0; vx < VPS; vx++)
      for (int vy = 0; vy < VPS; vy++) {
        int observed = 0;
        float squashed = from_occupancy ? 0.0f : 2.0f * max_sq; /* :792-799 */
        int min_bz = cmin_bz, min_vz = cmin_vz, max_bz = cmax_bz, max_vz = cmax_vz;
        if (plane) {
          int cb[4];
          or_planar_column_bounds(map->block_size, plane, above_plane_m, thickness_m, ob.x, ob.y, vx, vy, cb);
          min_bz = cb[0], min_vz = cb[1], max_bz = cb[2], max_vz = cb[3];
        }
        for (int bz = min_bz; bz <= max_bz; bz++) {
          const i3 k = {ob.x, ob.y, bz};
          const int32_t ss = hash_find(&src->hash, k);
          if (ss < 0) continue;
          const int32_t fs = use_freespace ? hash_find(&map->freespace.hash, k) : -1;
          const OrFreespaceVoxel* f = fs >= 0 ? (const OrFreespaceVoxel*)layer_block(&map->freespace, fs) : NULL;
          const int z0 = bz == min_bz ? min_vz : 0, z1 = bz == max_bz ? max_vz : VPS - 1; /* getMinAndMaxVoxelZIndex */
          for (int vz = z0; vz <= z1; vz++) {
            const int v = (vx * VPS + vy) * VPS + vz;
            const int is_fs = f ? f[v].is_high_confidence_freespace != 0 : 0;
            if (from_occupancy) {
              const float lo = ((const float*)layer_block(src, ss))[v];
              if (fabsf(lo - 0.0f) > 1e-4f) {
                observed = 1;
                if (!is_fs) squashed = fmaxf(squashed, lo); /* atomicMaxFloat */
              }
            } else {
              const OrTsdfVoxel* t = (const OrTsdfVoxel*)layer_block(src, ss) + v;
              if (t->weight >= P->min_weight) {
                observed = 1;
                if (!is_fs) squashed = fminf(squashed, t->distance); /* atomicMinFloat */
              }
            }
          }
        }
        OrEsdfVoxel* ev = &e[(vx * VPS + vy) * VPS + out_vz];
        if (from_occupancy)
          esdf_apply_observation(observed, squashed > occupied_threshold_log_odds, 1, max_sq, ev, &cleared, &updated);
        else
          esdf_apply_observation(observed, squashed <= 0.0f, fabsf(squashed) <= max_site_distance_m, max_sq, ev, &cleared,
                                 &updated);
      }
    upd[i] = (uint8_t)updated, clr[i] = (uint8_t)cleared;
  }
  List updated = {0}, to_clear = {0};
  for (int32_t i = 0; i < blocks.n; i++) {
    if (upd[i]) list_push(&updated, blocks.v[i]);
    if (clr[i]) list_push(&to_clear, blocks.v[i]);
  }
  free(upd), free(clr);
  map->stats[0] = blocks.n, map->stats[1] = updated.n, map->stats[2] = to_clear.n;
  if (to_clear.n > 0) esdf_clear_all_invalid(map, &to_clear, P->max_esdf_distance_m, max_sq, &map->esdf_cleared_persistent);
  map->stats[4] = map->esdf_cleared_persistent.n;
  esdf_compute(map, &updated, max_sq);
  if (map->esdf_cleared_persistent.n > 0) esdf_compute(map, &map->esdf_cleared_persistent, max_sq);
  list_free(&blocks), list_free(&updated), list_free(&to_clear);
}

/* EsdfSlicer::getAabbOfLayerAtHeight (src/integrators/esdf_slicer.cu:112-147): the blocks at the slice's z index. Returns 0 and
 * leaves aabb_out alone if there is none (an empty AlignedBox in the reference). */
int32_t or_esdf_slice_aabb(const OrMap* map, float slice_height, float aabb_out[6]) {
  const float bs = map->block_size;
  const int zb = f2i(floorf(slice_height / bs));
  int have = 0;
  int32_t mnx = 0, mny = 0, mxx = 0, mxy = 0;
  for (int32_t s = 0; s < map->esdf.n; s++) {
    const i3 k = map->esdf.index[s];
    if (k.z != zb) continue;
    if (!have) mnx = mxx = k.x, mny = mxy = k.y, have = 1;
    if (k.x < mnx) mnx = k.x;
    if (k.x > mxx) mxx = k.x;
    if (k.y < mny) mny = k.y;
    if (k.y > mxy) mxy = k.y;
  }
  if (!have) return 0;
  /* getAABBOfBlock: [index * block_size, (index + 1) * block_size] */
  aabb_out[0] = (float)mnx * bs, aabb_out[1] = (float)mny * bs, aabb_out[2] = (float)zb * bs;
  aabb_out[3] = ((float)mxx + 1.0f) * bs, aabb_out[4] = ((float)mxy + 1.0f) * bs, aabb_out[5] = ((float)zb + 1.0f) * bs;
  return 1;
}

/* EsdfSlicer::sliceLayerToDistanceImage(layer, slice_height, unobserved_value, aabb, image) (:169-199) on a GIVEN box +
 * populateSliceFromLayerKernel (:25-67) + occupancyGridFromSliceImageKernel (:78-110). Returns rows * cols; writes up to cap
 * pixels of the image / grid (either may be NULL). */
int32_t or_esdf_slice_image_in_aabb(const OrMap* map, float slice_height, float unobserved_value, const float aabb[6],
                                    float* image_out, int8_t* grid_out, int32_t cap, int32_t* rows_out, int32_t* cols_out) {
  const float bs = map->block_size;
  const float* amin = aabb;
  const float* amax = aabb + 3;
  const float voxel_size = bs / (float)VPS;
  const int cols = f2i(ceilf((amax[0] - amin[0]) / voxel_size)), rows = f2i(ceilf((amax[1] - amin[1]) / voxel_size));
  *rows_out = rows, *cols_out = cols;
  const float inv = (float)(1.0 / (double)(bs * (1.0f / VPS)));
  for (int r = 0; r < rows; r++)
    for (int cidx = 0; cidx < cols; cidx++) {
      const size_t pix = (size_t)r * cols + cidx;
      if ((int64_t)pix >= cap) continue;
      const float p[3] = {amin[0] + voxel_size / 2.0f + voxel_size * (float)cidx, amin[1] + voxel_size / 2.0f + voxel_size * (float)r,
                          slice_height};
      i3 b;
      int v[3];
      int bb[3];
      for (int a = 0; a < 3; a++) { /* getBlockAndVoxelIndexFromPositionInLayer (indexing_impl.h:37-49) */
        bb[a] = f2i(floorf(p[a] / bs));
        v[a] = f2i((p[a] - bs * (float)bb[a]) * inv);
        if (v[a] > VPS - 1) v[a] = VPS - 1;
      }
      b.x = bb[0], b.y = bb[1], b.z = bb[2];
      float d = unobserved_value;
      const int32_t sl = hash_find(&map->esdf.hash, b);
      if (sl >= 0) {
        const OrEsdfVoxel* e = (const OrEsdfVoxel*)layer_block(&map->esdf, sl) + (v[0] * VPS + v[1]) * VPS + v[2];
        if (e->observed) {
          d = voxel_size * sqrtf(e->squared_distance_vox);
          if (e->is_inside) d = -d;
        }
      }
      if (image_out) image_out[pix] = d;
      if (grid_out) {
        int8_t g = (int8_t)((d < 1e-2f) * 100);
        if (fabsf(d - unobserved_value) < 1e-2f) g = -1;
        grid_out[pix] = g;
      }
    }
  return rows * cols;
}

/* EsdfSlicer::sliceLayerToDistanceImage(layer, slice_height, unobserved_value, &aabb, image) (:157-167): the layer's own box.
 * Returns rows * cols (0 if the layer has no block at that height). */
int32_t or_esdf_slice_image(const OrMap* map, float slice_height, float unobserved_value, float aabb_out[6],
                            float* image_out, int8_t* grid_out, int32_t cap, int32_t* rows_out, int32_t* cols_out) {
  *rows_out = *cols_out = 0;
  float box[6];
  if (!or_esdf_slice_aabb(map, slice_height, box)) return 0;
  for (int a = 0; a < 6; a++) aabb_out[a] = box[a];
  return or_esdf_slice_image_in_aabb(map, slice_height, unobserved_value, box, image_out, grid_out, cap, rows_out, cols_out);
}

void or_esdf_last_stats(const OrMap* map, int64_t out[8]) { memcpy(out, map->stats, sizeof(map->stats)); }

/* ------------------------------------------------------------------------- */
/* Read-back                                                                 */
/* ------------------------------------------------------------------------- */

int32_t or_tsdf_num_blocks(const OrMap* m) { return m->tsdf.n; }
int32_t or_esdf_num_blocks(const OrMap* m) { return m->esdf.n; }
static int32_t layer_indices(const Layer* l, int32_t* out, int32_t cap) {
  for (int32_t i = 0; i < l->n && i < cap; i++)
    out[3 * i] = l->index[i].x, out[3 * i + 1] = l->index[i].y, out[3 * i + 2] = l->index[i].z;
  return l->n;
}
int32_t or_tsdf_block_indices(const OrMap* m, int32_t* out, int32_t cap) { return layer_indices(&m->tsdf, out, cap); }
int32_t or_esdf_block_indices(const OrMap* m, int32_t* out, int32_t cap) { return layer_indices(&m->esdf, out, cap); }
int32_t or_occupancy_num_blocks(const OrMap* m) { return m->occ.n; }
int32_t or_occupancy_block_indices(const OrMap* m, int32_t* out, int32_t cap) { return layer_indices(&m->occ, out, cap); }
int32_t or_freespace_block_indices(const OrMap* m, int32_t* out, int32_t cap) { return layer_indices(&m->freespace, out, cap); }
int32_t or_occupancy_get_block(const OrMap* m, const int32_t xyz[3], float* out) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = hash_find(&m->occ.hash, k);
  if (s < 0) return 0;
  memcpy(out, layer_block(&m->occ, s), m->occ.block_bytes);
  return 1;
}
int32_t or_tsdf_get_block(const OrMap* m, const int32_t xyz[3], OrTsdfVoxel* out) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = hash_find(&m->tsdf.hash, k);
  if (s < 0) return 0;
  memcpy(out, layer_block(&m->tsdf, s), m->tsdf.block_bytes);
  return 1;
}
int32_t or_esdf_get_block(const OrMap* m, const int32_t xyz[3], OrEsdfVoxel* out) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = hash_find(&m->esdf.hash, k);
  if (s < 0) return 0;
  memcpy(out, layer_block(&m->esdf, s), m->esdf.block_bytes);
  return 1;
}

/* ProjectiveIntegrator::markUnobservedFreeInsideRadiusTemplate (projective_integrator_impl.cuh:408-462) behind
 * Mapper::markUnobservedTsdfFreeInsideRadius (src/mapper/mapper.cpp:494-507): every block whose box is closer than `radius`
 * to `center` (getBlocksWithinRadius, src/geometry/bounding_spheres.cpp:24-67; Eigen AlignedBox::exteriorDistance) is
 * allocated, and its unobserved voxels become "slightly observed free": TSDF (truncation distance, weight 0.1) where
 * weight < 1e-3; occupancy log odds -2e-4 where |log odds| < 1e-4 (setUnobservedVoxel, :377-392). Returns the block count. */
int32_t or_mark_unobserved_free_inside_radius(OrMap* map, int32_t occupancy, const float center[3], float radius,
                                              float truncation_distance_m, int32_t* out_xyz, int32_t cap) {
  const v3 mn = {center[0] - radius, center[1] - radius, center[2] - radius};
  const v3 mx = {center[0] + radius, center[1] + radius, center[2] + radius};
  const i3 lo = block_index_from_position(map->block_size, mn), hi = block_index_from_position(map->block_size, mx);
  List blocks = {0};
  for (int x = lo.x; x <= hi.x; x++)
    for (int y = lo.y; y <= hi.y; y++)
      for (int z = lo.z; z <= hi.z; z++) {
        const int idx[3] = {x, y, z};
        float dist2 = 0.0f;
        for (int k = 0; k < 3; k++) { /* AlignedBox::squaredExteriorDistance of getAABBOfBlock */
          const float bmin = (float)idx[k] * map->block_size, bmax = ((float)idx[k] + 1.0f) * map->block_size;
          if (bmin > center[k]) {
            const float aux = bmin - center[k];
            dist2 += aux * aux;
          } else if (center[k] > bmax) {
            const float aux = center[k] - bmax;
            dist2 += aux * aux;
          }
        }
        if (!(sqrtf(dist2) < radius)) continue;
        const i3 k3 = {x, y, z};
        list_push(&blocks, k3);
        if (occupancy) {
          float* lo_v = (float*)layer_block(&map->occ, layer_allocate(&map->occ, k3));
          for (int v = 0; v < VPB; v++)
            if (fabsf(lo_v[v] - 0.0f) < 1e-4f) lo_v[v] = -2e-4f;
        } else {
          OrTsdfVoxel* t = (OrTsdfVoxel*)layer_block(&map->tsdf, layer_allocate(&map->tsdf, k3));
          for (int v = 0; v < VPB; v++)
            if (t[v].weight < 0.001f) t[v].distance = truncation_distance_m, t[v].weight = 0.1f;
        }
      }
  const int32_t n = copy_out(&blocks, out_xyz, cap);
  list_free(&blocks);
  return n;
}

/* ------------------------------------------------------------------------- */
/* Colour integration (src/integrators/projective_appearance_integrator.cu,  */
/* src/rays/sphere_tracer.cu)                                                */
/* ------------------------------------------------------------------------- */
void or_default_color_params(OrColorParams* p) {
  memset(p, 0, sizeof(*p));
  /* integrators/projective_integrator_params.h:24-75, projective_appearance_integrator.h:164, rays/sphere_tracer.h:216-218 */
  p->max_integration_distance_m = 7.0f;
  p->truncation_distance_vox = 4.0f;
  p->max_weight = 5.0f;
  p->measurement_weight = 0.8f;
  p->sphere_tracing_ray_subsampling_factor = 4;
  p->sphere_tracer_maximum_steps = 100;
  p->sphere_tracer_maximum_ray_length_m = 7.0f; /* set from max_integration_distance_m_ in the constructor only (:61) */
  p->sphere_tracer_surface_distance_epsilon_vox = 0.1f;
  p->workspace_bounds_type = OR_WS_UNBOUNDED;
}

/* binary32 -> binary16 -> binary32 (__float2half then the implicit __half -> float), round to nearest even. */
static float round_through_half(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  const uint32_t sign = x & 0x80000000u;
  const uint32_t ax = x & 0x7fffffffu;
  uint32_t out;
  if (ax >= 0x7f800000u) {
    out = ax; /* inf / nan: unchanged (weights never get here) */
  } else if (ax >= 0x477ff000u) {
    out = 0x7f800000u; /* >= 65520 rounds to inf */
  } else if (ax < 0x38800000u) { /* below the smallest normal half 2^-14: the result is a multiple of 2^-24 */
    const float a = fabsf(f);
    const float q = nearbyintf(a * 16777216.0f); /* exact scaling; default rounding mode = nearest even */
    float r = q * (1.0f / 16777216.0f);
    memcpy(&out, &r, 4);
  } else {
    const uint32_t lsb = (ax >> 13) & 1u;
    out = (ax + 0x0fffu + lsb) & 0xffffe000u;
  }
  out |= sign;
  float r;
  memcpy(&r, &out, 4);
  return r;
}
float or_round_through_half(float f) { return round_through_half(f); }

/* getBlockAndVoxelIndexFromPositionInLayer (core/internal/impl/indexing_impl.h:37-49) */
static void block_and_voxel_from_position(float block_size, v3 p, i3* b, int v[3]) {
  const float inv = (float)(1.0 / (double)(block_size * (1.0f / VPS)));
  const float pp[3] = {p.x, p.y, p.z};
  int bb[3];
  for (int a = 0; a < 3; a++) {
    bb[a] = f2i(floorf(pp[a] / block_size));
    v[a] = f2i((pp[a] - block_size * (float)bb[a]) * inv);
    if (v[a] > VPS - 1) v[a] = VPS - 1;
  }
  b->x = bb[0], b->y = bb[1], b->z = bb[2];
}

/* cast (src/rays/sphere_tracer.cu:31-100): march along the ray by the TSDF distance of the voxel under the point. */
static int sphere_trace_cast(const OrMap* map, v3 origin, v3 dir, float truncation_distance_m, int maximum_steps,
                             float maximum_ray_length_m, float surface_distance_epsilon_m, float* t_out) {
  int first = 0; /* 0 not yet known, 1 positive, 2 negative */
  float t = 0.0f;
  for (int i = 0; (i < maximum_steps) && (t < maximum_ray_length_m); i++) {
    const v3 p_L = {origin.x + t * dir.x, origin.y + t * dir.y, origin.z + t * dir.z};
    float step;
    i3 b;
    int v[3];
    block_and_voxel_from_position(map->block_size, p_L, &b, v);
    const int32_t slot = hash_find(&map->tsdf.hash, b);
    const OrTsdfVoxel* vox = slot >= 0 ? (const OrTsdfVoxel*)layer_block(&map->tsdf, slot) + (v[0] * VPS + v[1]) * VPS + v[2] : NULL;
    if (!vox || !(vox->weight > 1e-4f)) { /* isTsdfVoxelValid (:26-29) */
      if (first == 0) {
        step = truncation_distance_m;
      } else {
        *t_out = t;
        return 0;
      }
    } else {
      if (first == 0) first = (vox->distance >= 0.0f) ? 1 : 2;
      if (first == 1) {
        if (vox->distance < surface_distance_epsilon_m) {
          *t_out = t + vox->distance;
          return 1;
        }
        step = vox->distance;
      } else {
        if (vox->distance > -surface_distance_epsilon_m) {
          *t_out = t - vox->distance;
          return 1;
        }
        step = -vox->distance;
      }
    }
    t += step;
  }
  *t_out = t;
  return 0;
}

/* SphereTracer::castOnGPU(ray, ...) (src/rays/sphere_tracer.cu:341-387): one ray, direction already normalised. */
int32_t or_sphere_trace_ray(const OrMap* map, const float origin[3], const float direction[3], float truncation_distance_m,
                            int32_t maximum_steps, float maximum_ray_length_m, float surface_distance_epsilon_m, float* t_out) {
  const v3 o = {origin[0], origin[1], origin[2]}, d = {direction[0], direction[1], direction[2]};
  return sphere_trace_cast(map, o, d, truncation_distance_m, maximum_steps, maximum_ray_length_m, surface_distance_epsilon_m,
                           t_out);
}

/* SphereTracer::renderImageOnGPU + sphereTracingKernel (src/rays/sphere_tracer.cu:134-173, 422-485):
 * out is (rows / f) x (cols / f), -1 where the ray found no surface. */
void or_sphere_trace_image(const OrMap* map, const float* T_L_C, const OrCamera* cam, float truncation_distance_m,
                           int32_t maximum_steps, float maximum_ray_length_m, float surface_distance_epsilon_m,
                           int32_t ray_subsampling_factor, float* out) {
  const int f = ray_subsampling_factor;
  const int ray_rows = cam->height / f, ray_cols = cam->width / f;
  const v3 origin = {Tt(T_L_C, 0), Tt(T_L_C, 1), Tt(T_L_C, 2)};
#pragma omp parallel for schedule(dynamic, 4)
  for (int r = 0; r < ray_rows; r++)
    for (int c = 0; c < ray_cols; c++) {
      const float half = 0.5f * (float)f;
      const float px = (float)(c * f) + half * 1.0f, py = (float)(r * f) + half * 1.0f;
      v3 d = cam_vector_from_image_plane(cam, px, py);
      const float n = sqrtf(sum3(d.x * d.x, d.y * d.y, d.z * d.z)); /* Eigen normalized() */
      d.x = d.x / n, d.y = d.y / n, d.z = d.z / n;
      v3 dir;
      dir.x = sum3(Rm(T_L_C, 0, 0) * d.x, Rm(T_L_C, 0, 1) * d.y, Rm(T_L_C, 0, 2) * d.z);
      dir.y = sum3(Rm(T_L_C, 1, 0) * d.x, Rm(T_L_C, 1, 1) * d.y, Rm(T_L_C, 1, 2) * d.z);
      dir.z = sum3(Rm(T_L_C, 2, 0) * d.x, Rm(T_L_C, 2, 1) * d.y, Rm(T_L_C, 2, 2) * d.z);
      float t;
      const int ok = sphere_trace_cast(map, origin, dir, truncation_distance_m, maximum_steps, maximum_ray_length_m,
                                       surface_distance_epsilon_m, &t);
      out[(size_t)r * ray_cols + c] = ok ? t * d.z : -1.0f;
    }
}

/* ViewCalculator::getBlocksInImageViewProjection (view_calculator_impl.h:29-78) + getVisibleBlocksByProjection<Camera>
 * (src/integrators/view_calculator.cu:380-417), then reduceBlocksToThoseInTruncationBand
 * (projective_appearance_integrator.cu:378-481). */
static List view_projection_blocks(float block_size, const float* T_L_C, const OrCamera* cam, float max_distance,
                                   int32_t workspace_bounds_type, const float* workspace_min, const float* workspace_max) {
  List out = {0};
  v3 mn, mx;
  cam_view_aabb(cam, T_L_C, 1e-6f, max_distance, &mn, &mx);
  OrTsdfParams ws;
  memset(&ws, 0, sizeof(ws));
  ws.workspace_bounds_type = workspace_bounds_type;
  for (int a = 0; a < 3; a++) ws.workspace_min[a] = workspace_min[a], ws.workspace_max[a] = workspace_max[a];
  if (!apply_workspace_bounds(&ws, &mn, &mx)) return out;
  const i3 lo = block_index_from_position(block_size, mn), hi = block_index_from_position(block_size, mx);
  float T_C_L[16];
  invert_isometry(T_L_C, T_C_L);
  /* Camera::getNormalizedViewport(getViewportMargin(height)) (src/sensors/camera.cpp:85-96, view_calculator_impl.h:81-83) */
  const float margin = (float)cam->height / 20.0f;
  const v3 vmin = cam_vector_from_image_plane(cam, -margin, -margin);
  const v3 vmax = cam_vector_from_image_plane(cam, (float)cam->width + margin, (float)cam->height + margin);
  for (int x = lo.x; x <= hi.x; x++)
    for (int y = lo.y; y <= hi.y; y++)
      for (int z = lo.z; z <= hi.z; z++) { /* getBlockIndicesTouchedByBoundingBox order (bounding_boxes_impl.h:28-53) */
        const i3 k = {x, y, z};
        const v3 c_L = {block_size * ((float)x + 0.5f), block_size * ((float)y + 0.5f),
                        block_size * ((float)z + 0.5f)}; /* getCenterPositionFromBlockIndex */
        const v3 p = transform_point(T_C_L, c_L);
        if (!(p.z > 1e-6f)) continue;
        if (!(p.z >= 1e-6f)) continue; /* projectToNormalizedCoordinates (camera_impl.h:65-75) */
        const float un = p.x / p.z, vn = p.y / p.z;
        /* Eigen::AlignedBox::contains: (min <= p).all() && (p <= max).all() */
        if (!(vmin.x <= un && vmin.y <= vn && un <= vmax.x && vn <= vmax.y)) continue;
        list_push(&out, k);
      }
  return out;
}
/* ViewCalculator::getBlocksInImageViewProjection, exposed for the known-answer tests. */
int32_t or_view_projection_blocks(float block_size, const float* T_L_C, const OrCamera* cam, float max_distance,
                                  int32_t* out_xyz, int32_t cap) {
  const float zero[3] = {0.0f, 0.0f, 0.0f};
  List l = view_projection_blocks(block_size, T_L_C, cam, max_distance, OR_WS_UNBOUNDED, zero, zero);
  const int32_t n = copy_out(&l, out_xyz, cap);
  list_free(&l);
  return n;
}
static List color_blocks_in_view_and_band(const OrMap* map, const float* T_L_C, const OrCamera* cam, const OrColorParams* P,
                                          float truncation_distance_m) {
  List in_view = view_projection_blocks(map->block_size, T_L_C, cam, P->max_integration_distance_m + truncation_distance_m,
                                        P->workspace_bounds_type, P->workspace_min, P->workspace_max);
  List out = {0};
  for (int32_t i = 0; i < in_view.n; i++) {
    const i3 k = in_view.v[i];
    const int32_t slot = hash_find(&map->tsdf.hash, k);
    if (slot < 0) continue;
    const OrTsdfVoxel* t = (const OrTsdfVoxel*)layer_block(&map->tsdf, slot);
    int in_band = 0;
    for (int v = 0; v < VPB && !in_band; v++)
      if (t[v].weight > 0.0f && fabsf(t[v].distance) < truncation_distance_m) in_band = 1; /* checkBlocksInTruncationBand */
    if (in_band) list_push(&out, k);
  }
  list_free(&in_view);
  return out;
}

/* interpolatePixels<float> (interpolation_2d_impl.h:26-36) */
static float interpolate_pixels_f(float x, float y, float f00, float f01, float f10, float f11) {
  const float dx = f10 - f00;
  return f00 + x * dx + y * (f01 - f00) + x * y * (f11 - f01 - dx);
}

static int32_t color_layer_allocate(Layer* l, i3 k) {
  const int32_t before = l->n;
  const int32_t slot = layer_allocate(l, k);
  if (l->n != before) { /* ColorVoxel() : color(Color::Gray()), weight(0) (map/voxels.h:77-83) */
    OrColorVoxel* v = (OrColorVoxel*)layer_block(l, slot);
    for (int i = 0; i < VPB; i++) v[i].r = v[i].g = v[i].b = 127, v[i].pad = 0, v[i].weight = 0.0f;
  }
  return slot;
}

/* ProjectiveAppearanceIntegrator<ColorLayer>::integrateFrame (projective_appearance_integrator.cu:68-165): blocks in view and in
 * the truncation band, a sphere-traced synthetic depth image for the occlusion test, then integrateBlocksKernel for
 * appearance voxels (projective_integrator_impl.cuh:117-185) with UpdateAppearanceVoxelFunctor (:312-348).
 * color = rows x cols x 3 bytes (RGB). Returns the number of updated blocks (copied to out_xyz up to cap). */
int32_t or_color_integrate(OrMap* map, const uint8_t* color, const uint8_t* mask, int32_t mask_mode, int32_t rows, int32_t cols,
                           const float* T_L_C, const OrCamera* cam, const OrColorParams* P, int32_t* out_xyz, int32_t cap) {
  const float trunc = P->truncation_distance_vox * map->voxel_size;
  List blocks = color_blocks_in_view_and_band(map, T_L_C, cam, P, trunc);
  if (blocks.n == 0) {
    list_free(&blocks);
    return 0;
  }
  int32_t* slots = (int32_t*)malloc(sizeof(int32_t) * (size_t)blocks.n);
  for (int32_t i = 0; i < blocks.n; i++) slots[i] = color_layer_allocate(&map->color, blocks.v[i]);
  const int f = P->sphere_tracing_ray_subsampling_factor;
  const int drows = cam->height / f, dcols = cam->width / f;
  float* synth = (float*)malloc(sizeof(float) * (size_t)drows * dcols);
  or_sphere_trace_image(map, T_L_C, cam, trunc, P->sphere_tracer_maximum_steps, P->sphere_tracer_maximum_ray_length_m,
                        P->sphere_tracer_surface_distance_epsilon_vox * map->voxel_size, f, synth);
  float T_C_L[16];
  invert_isometry(T_L_C, T_C_L);
  const int depth_subsample = rows / drows; /* projective_integrator_impl.cuh:320 */
  const float voxel_size = map->block_size * (1.0f / VPS), half_voxel = map->block_size * (0.5f / VPS);
  const float max_depth = P->max_integration_distance_m;
  /* blendTwoArrays' weights (:287-306) are the same for every voxel */
  float w_old = 1.0f - P->measurement_weight, w_new = P->measurement_weight;
  const float total = w_old + w_new;
  w_old /= total, w_new /= total;
  const float w_old_h = round_through_half(w_old), w_new_h = round_through_half(w_new);
#pragma omp parallel for schedule(static)
  for (int32_t i = 0; i < blocks.n; i++) {
    OrColorVoxel* blk = (OrColorVoxel*)layer_block(&map->color, slots[i]);
    const i3 bi = blocks.v[i];
    for (int vx = 0; vx < VPS; vx++)
      for (int vy = 0; vy < VPS; vy++)
        for (int vz = 0; vz < VPS; vz++) {
          v3 p_L;
          p_L.x = (map->block_size * (float)bi.x + voxel_size * (float)vx) + half_voxel;
          p_L.y = (map->block_size * (float)bi.y + voxel_size * (float)vy) + half_voxel;
          p_L.z = (map->block_size * (float)bi.z + voxel_size * (float)vz) + half_voxel;
          const v3 p_C = transform_point(T_C_L, p_L);
          float u, v;
          if (!cam_project(cam, p_C, &u, &v)) continue;
          const float voxel_depth = p_C.z;
          if (max_depth > 0.0f && voxel_depth > max_depth) continue;
          /* occlusion test against the synthetic depth (interpolate2DClosest on the subsampled image) */
          const float ud = u / (float)depth_subsample, vd = v / (float)depth_subsample;
          const int dx = f2i(floorf(ud)), dy = f2i(floorf(vd));
          if (dx < 0 || dy < 0 || dx >= dcols || dy >= drows) continue;
          const float surface_depth = synth[(size_t)dy * dcols + dx];
          if (!(isfinite(surface_depth) && surface_depth > 1e-6f)) continue; /* PixelIsValidDepth */
          if (fabsf(surface_depth - voxel_depth) > trunc) continue;
          /* interpolate2DLinear<Color> (interpolation_2d_impl.h:152-199) */
          const float ucx = u - 0.5f, ucy = v - 0.5f;
          const int lx = f2i(floorf(ucx)), ly = f2i(floorf(ucy));
          if (lx < 0 || ly < 0 || (lx + 1) > (cols - 1) || (ly + 1) > (rows - 1)) continue;
          const float ox = ucx - (float)lx, oy = ucy - (float)ly;
          const uint8_t* c00 = color + ((size_t)ly * cols + lx) * 3;
          const uint8_t* c01 = color + ((size_t)(ly + 1) * cols + lx) * 3;
          const uint8_t* c10 = color + ((size_t)ly * cols + lx + 1) * 3;
          const uint8_t* c11 = color + ((size_t)(ly + 1) * cols + lx + 1) * 3;
          uint8_t meas[3];
          for (int ch = 0; ch < 3; ch++)
            meas[ch] = (uint8_t)roundf(interpolate_pixels_f(ox, oy, (float)c00[ch], (float)c01[ch], (float)c10[ch], (float)c11[ch]));
          /* isMasked(u_px.y(), u_px.x()): the float coordinates convert to int by truncation */
          int is_active = 1;
          if (mask != NULL) {
            const uint8_t mv = mask[(size_t)(int)v * cols + (int)u];
            is_active = (mask_mode == OR_MASK_NON_INVERTED) ? (mv != 0) : (mv == 0);
          }
          if (!is_active) continue;
          OrColorVoxel* cv = &blk[(vx * VPS + vy) * VPS + vz];
          const float weight_current = cv->weight;
          if (round_through_half(cv->weight) == 0.0f) {
            cv->r = meas[0], cv->g = meas[1], cv->b = meas[2];
          } else {
            uint8_t* cur[3] = {&cv->r, &cv->g, &cv->b};
            for (int ch = 0; ch < 3; ch++) /* weightedSum(uint8_t, float, uint8_t, float) (:277-285) */
              *cur[ch] = (uint8_t)roundf((float)*cur[ch] * w_old_h + (float)meas[ch] * w_new_h);
          }
          cv->weight = fminf(P->measurement_weight + weight_current, P->max_weight);
        }
  }
  free(synth), free(slots);
  const int32_t n = copy_out(&blocks, out_xyz, cap);
  list_free(&blocks);
  return n;
}
int32_t or_color_num_blocks(const OrMap* m) { return m->color.n; }
int32_t or_color_block_indices(const OrMap* m, int32_t* out, int32_t cap) { return layer_indices(&m->color, out, cap); }
int32_t or_color_get_block(const OrMap* m, const int32_t xyz[3], OrColorVoxel* out) {
  const i3 k = {xyz[0], xyz[1], xyz[2]};
  const int32_t s = hash_find(&m->color.hash, k);
  if (s < 0) return 0;
  memcpy(out, layer_block(&m->color, s), sizeof(OrColorVoxel) * VPB);
  return 1;
}

/* ------------------------------------------------------------------------- */
/* Decay (integrators/internal/cuda/impl/decayer_impl.cuh)                   */
/* ------------------------------------------------------------------------- */

/* doesVoxelHaveDepthMeasurement (integrators/internal/cuda/impl/projective_integrators_common_impl.cuh:58-101). */
static int voxel_has_depth_measurement(i3 bi, int vx, int vy, int vz, const float* depth, int rows, int cols,
                                       const float* T_C_L, const OrCamera* cam, float block_size, float max_distance,
                                       float truncation_distance) {
  const float voxel_size = block_size * (1.0f / VPS);
  const float half_voxel = block_size * (0.5f / VPS);
  v3 p_L;
  p_L.x = (block_size * (float)bi.x + voxel_size * (float)vx) + half_voxel;
  p_L.y = (block_size * (float)bi.y + voxel_size * (float)vy) + half_voxel;
  p_L.z = (block_size * (float)bi.z + voxel_size * (float)vz) + half_voxel;
  const v3 p_C = transform_point(T_C_L, p_L);
  float u, v;
  if (!cam_project(cam, p_C, &u, &v)) return 0;
  const float voxel_depth = p_C.z;
  if (max_distance > 0.0f && voxel_depth > max_distance) return 0;
  const int ux = f2i(floorf(u)), uy = f2i(floorf(v));
  if (ux < 0 || uy < 0 || ux >= cols || uy >= rows) return 0;
  const float d = depth[(size_t)uy * cols + ux];
  if (!(isfinite(d) && d > 1e-6f)) return 0; /* invalid depth: not in view */
  if (d - voxel_depth < -truncation_distance) return 0; /* occluded */
  return 1;
}

/* getBlockIndicesToDecay (decayer_impl.cuh:38-80): 1 = decay this block. */
static int decay_block_selected(const OrMap* map, i3 k, const Hash* excluded, const OrDecayExclusion* X) {
  if (excluded && hash_find(excluded, k) >= 0) return 0;
  if (X && X->has_exclusion_sphere && X->exclusion_radius_m * X->exclusion_radius_m > 0.0f) {
    /* getPositionFromBlockIndex (indexing_impl.h): block origin = block_size * index */
    const float px = map->block_size * (float)k.x, py = map->block_size * (float)k.y, pz = map->block_size * (float)k.z;
    const float dx = px - X->exclusion_center[0], dy = py - X->exclusion_center[1], dz = pz - X->exclusion_center[2];
    const float d2 = sum3(dx * dx, dy * dy, dz * dz);
    return d2 > X->exclusion_radius_m * X->exclusion_radius_m;
  }
  return 1;
}

/* TsdfDecayFunctor (integrators/internal/cuda/impl/tsdf_decay_integrator_impl.cuh:25-75). */
static int tsdf_is_fully_decayed(const OrTsdfVoxel* v, float thr) { return v->weight < (thr + 1e-6f); }
static void tsdf_decay_voxel(OrTsdfVoxel* v, const OrTsdfDecayParams* P, float free_distance_m) {
  float weight = v->weight;
  if (weight < (P->decayed_weight_threshold - 1e-6f)) return;
  weight *= P->decay_factor;
  weight = fmaxf(weight, P->decayed_weight_threshold);
  v->weight = weight;
  if (P->set_free_distance_on_decayed && tsdf_is_fully_decayed(v, P->decayed_weight_threshold)) v->distance = free_distance_m;
}

/* OccupancyDecayFunctor (integrators/internal/cuda/impl/occupancy_decay_integrator_impl.cuh:26-70). */
typedef struct {
  float free_lo, occ_lo, to_lo;
} OccDecay;
static int occ_is_fully_decayed(float lo, const OccDecay* f) {
  if (lo >= f->to_lo) return lo + f->occ_lo < f->to_lo;
  return lo + f->free_lo >= f->to_lo;
}
static void occ_decay_voxel(float* lo, const OccDecay* f) {
  if (occ_is_fully_decayed(*lo, f)) {
    *lo = f->to_lo;
    return;
  }
  if (*lo >= 0) *lo += f->occ_lo;
  else *lo += f->free_lo;
}

/* VoxelDecayer::decay (decayer_impl.cuh:150-262) followed by Mapper::clearBlocksInLayers for the removed blocks
 * (src/mapper/mapper.cpp:546-575) when `clear_esdf` is set. */
static int32_t decay_layer(OrMap* map, int occupancy, const void* params, const OrDecayExclusion* X, const float* depth,
                           int32_t rows, int32_t cols, const float* T_L_C, const OrCamera* cam, float max_view_distance_m,
                           float truncation_distance_m, int32_t deallocate, int32_t clear_esdf, int32_t* out_xyz,
                           int32_t cap) {
  Layer* L = occupancy ? &map->occ : &map->tsdf;
  if (L->n == 0) return 0;
  Hash excl;
  Hash* exclp = NULL;
  if (X && X->num_excluded_blocks > 0) {
    int32_t hc = 16;
    while (hc < 4 * X->num_excluded_blocks) hc *= 2;
    hash_init(&excl, hc);
    for (int32_t i = 0; i < X->num_excluded_blocks; i++) {
      i3 k = {X->excluded_blocks_xyz[3 * i], X->excluded_blocks_xyz[3 * i + 1], X->excluded_blocks_xyz[3 * i + 2]};
      if (hash_find(&excl, k) < 0) hash_put(&excl, k, i);
    }
    exclp = &excl;
  }
  float T_C_L[16];
  if (depth) invert_isometry(T_L_C, T_C_L);
  const OrTsdfDecayParams* TP = (const OrTsdfDecayParams*)params;
  const OrOccupancyDecayParams* OP = (const OrOccupancyDecayParams*)params;
  OccDecay of = {0, 0, 0};
  float free_distance_m = 0.0f;
  if (occupancy) {
    of.free_lo = log_odds_from_probability(OP->free_region_decay_probability);
    of.occ_lo = log_odds_from_probability(OP->occupied_region_decay_probability);
    of.to_lo = log_odds_from_probability(OP->decay_to_probability);
  } else {
    free_distance_m = TP->free_distance_vox * map->voxel_size;
  }
  uint8_t* fully = (uint8_t*)calloc((size_t)L->n, 1);
  uint8_t* selected = (uint8_t*)calloc((size_t)L->n, 1);
#pragma omp parallel for schedule(static)
  for (int32_t s = 0; s < L->n; s++) {
    const i3 k = L->index[s];
    if (!decay_block_selected(map, k, exclp, X)) continue;
    selected[s] = 1;
    int all = 1;
    for (int vx = 0; vx < VPS; vx++)
      for (int vy = 0; vy < VPS; vy++)
        for (int vz = 0; vz < VPS; vz++) {
          const int v = (vx * VPS + vy) * VPS + vz;
          const int do_decay = depth ? !voxel_has_depth_measurement(k, vx, vy, vz, depth, rows, cols, T_C_L, cam, map->block_size,
                                                                    max_view_distance_m, truncation_distance_m)
                                     : 1;
          if (occupancy) {
            float* lo = (float*)layer_block(L, s) + v;
            if (do_decay) occ_decay_voxel(lo, &of);
            if (!occ_is_fully_decayed(*lo, &of)) all = 0;
          } else {
            OrTsdfVoxel* tv = (OrTsdfVoxel*)layer_block(L, s) + v;
            if (do_decay) tsdf_decay_voxel(tv, TP, free_distance_m);
            if (!tsdf_is_fully_decayed(tv, TP->decayed_weight_threshold)) all = 0;
          }
        }
    fully[s] = (uint8_t)all;
  }
  int32_t n_removed = 0;
  if (deallocate) {
    List rm = {0};
    for (int32_t s = 0; s < L->n; s++)
      if (selected[s] && fully[s]) list_push(&rm, L->index[s]);
    n_removed = copy_out(&rm, out_xyz, cap);
    layer_remove_blocks(L, rm.v, rm.n);
    if (clear_esdf == 1) layer_remove_blocks(&map->esdf, rm.v, rm.n);
    if (clear_esdf) layer_remove_blocks(&map->freespace, rm.v, rm.n), layer_remove_blocks(&map->color, rm.v, rm.n);
    if (clear_esdf && !occupancy) { /* ColorMeshLayer::clearBlocksAsync (src/mapper/mapper.cpp:552-557): TSDF mappers only */
      for (int32_t i = 0; i < rm.n; i++) {
        const int32_t ms = hash_find(&map->mesh.hash, rm.v[i]);
        if (ms >= 0) mesh_block_release((MeshBlock*)layer_block(&map->mesh, ms));
      }
      layer_remove_blocks(&map->mesh, rm.v, rm.n);
    }
    if (clear_esdf == 2) {
      /* 2-D ESDF (src/mapper/mapper.cpp:569-626): a column's slice block goes when no projective block is left in the
       * vertical column within the slice bounds (the projective blocks were removed above) */
      List er = {0};
      const int min_bz = f2i(floorf(map->slice_min_z / map->block_size)), max_bz = f2i(floorf(map->slice_max_z / map->block_size)),
                out_bz = f2i(floorf(map->slice_out_z / map->block_size));
      for (int32_t i = 0; i < rm.n; i++) {
        const i3 ek = {rm.v[i].x, rm.v[i].y, out_bz};
        if (hash_find(&map->esdf.hash, ek) < 0) continue;
        int has = 0;
        for (int bz = min_bz; bz <= max_bz && !has; bz++) {
          const i3 pk = {rm.v[i].x, rm.v[i].y, bz};
          has = hash_find(&L->hash, pk) >= 0;
        }
        if (!has) list_push(&er, ek);
      }
      layer_remove_blocks(&map->esdf, er.v, er.n);
      list_free(&er);
    }
    list_free(&rm);
  }
  free(fully), free(selected);
  if (exclp) hash_free(exclp);
  return n_removed;
}


/* ------------------------------------------------------------------------- */
/* Freespace (integrators/internal/cuda/impl/freespace_integrator_impl.cuh)  */
/* ------------------------------------------------------------------------- */
void or_default_freespace_params(OrFreespaceParams* p) {
  /* integrators/freespace_integrator_params.h:22-58 */
  p->max_tsdf_distance_for_occupancy_m = 0.15f;
  p->max_unobserved_to_keep_consecutive_occupancy_ms = 200;
  p->min_duration_since_occupied_for_freespace_ms = 1000;
  p->min_consecutive_occupancy_duration_for_reset_ms = 2000;
  p->check_neighborhood = 1;
  p->initialize_to_high_confidence_freespace = 0;
}

/* FreespaceIntegrator::updateFreespaceLayer (:324-383) + updateFreespaceLayerKernel (:99-246). */
void or_freespace_update(OrMap* map, const int32_t* blocks_xyz, int32_t num_blocks, int64_t update_time_ms,
                         const OrFreespaceParams* P, const float* depth, int32_t rows, int32_t cols, const float* T_L_C,
                         const OrCamera* cam, float max_view_distance_m, float truncation_distance_m) {
  if (num_blocks == 0) return;
  float T_C_L[16];
  if (depth) invert_isometry(T_L_C, T_C_L);
  const int64_t last_update = map->freespace_last_update_time_ms;
  for (int32_t i = 0; i < num_blocks; i++) { /* allocateBlocksAtIndices */
    i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    layer_allocate(&map->freespace, k);
  }
#pragma omp parallel for schedule(static)
  for (int32_t i = 0; i < num_blocks; i++) {
    const i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    const int32_t fsl = hash_find(&map->freespace.hash, k);
    const int32_t ts = hash_find(&map->tsdf.hash, k);
    if (fsl < 0 || ts < 0) continue; /* the reference hands the kernel a TSDF pointer for every block to update */
    OrFreespaceVoxel* fv = (OrFreespaceVoxel*)layer_block(&map->freespace, fsl);
    const OrTsdfVoxel* tv = (const OrTsdfVoxel*)layer_block(&map->tsdf, ts);
    uint8_t is_free_blk[VPB];
    uint8_t update_voxel[VPB], init_voxel[VPB];
    memset(is_free_blk, 0, sizeof(is_free_blk));
    for (int vx = 0; vx < VPS; vx++)
      for (int vy = 0; vy < VPS; vy++)
        for (int vz = 0; vz < VPS; vz++) {
          const int v = (vx * VPS + vy) * VPS + vz;
          OrFreespaceVoxel f = fv[v];
          int upd = 1;
          if (depth && !voxel_has_depth_measurement(k, vx, vy, vz, depth, rows, cols, T_C_L, cam, map->block_size,
                                                    max_view_distance_m, truncation_distance_m))
            upd = 0;
          const int init = f.last_occupied_timestamp_ms == 0;
          if (init) {
            f.last_occupied_timestamp_ms = update_time_ms;
            f.consecutive_occupancy_duration_ms = 0;
            f.is_high_confidence_freespace = (uint8_t)(P->initialize_to_high_confidence_freespace != 0);
          }
          if (upd && !init) {
            if (update_time_ms - f.last_occupied_timestamp_ms <= P->max_unobserved_to_keep_consecutive_occupancy_ms)
              f.consecutive_occupancy_duration_ms += update_time_ms - last_update;
            else
              f.consecutive_occupancy_duration_ms = 0;
            if (tv[v].distance <= P->max_tsdf_distance_for_occupancy_m) f.last_occupied_timestamp_ms = update_time_ms;
            /* isVoxelFree (:36-44): `weight > 1e-6` compares the float with a double literal */
            is_free_blk[v] = (uint8_t)((double)tv[v].weight > 1e-6 && f.last_occupied_timestamp_ms != 0 &&
                                       f.last_occupied_timestamp_ms <= update_time_ms - P->min_duration_since_occupied_for_freespace_ms);
          }
          update_voxel[v] = (uint8_t)upd, init_voxel[v] = (uint8_t)init;
          if (upd || init) fv[v] = f; /* written back below as well; intermediate state is per voxel */
        }
    for (int vx = 0; vx < VPS; vx++)
      for (int vy = 0; vy < VPS; vy++)
        for (int vz = 0; vz < VPS; vz++) {
          const int v = (vx * VPS + vy) * VPS + vz;
          if (!(update_voxel[v] && !init_voxel[v])) continue;
          OrFreespaceVoxel f = fv[v];
          int is_free = is_free_blk[v];
          if (P->check_neighborhood && is_free) { /* isVoxelNeighborhoodFree (:46-83), inside the block only */
            for (int u = -1; u <= 1; u++)
              for (int w = -1; w <= 1; w++)
                for (int q = -1; q <= 1; q++) {
                  const int x = vx + u, y = vy + w, z = vz + q;
                  if (u == 0 && w == 0 && q == 0) continue;
                  if (x < 0 || x >= VPS || y < 0 || y >= VPS || z < 0 || z >= VPS) continue;
                  is_free &= is_free_blk[(x * VPS + y) * VPS + z];
                }
          }
          if (f.consecutive_occupancy_duration_ms >= P->min_consecutive_occupancy_duration_for_reset_ms)
            f.is_high_confidence_freespace = 0;
          else
            f.is_high_confidence_freespace = (uint8_t)(f.is_high_confidence_freespace || is_free);
          fv[v] = f;
        }
  }
  map->freespace_last_update_time_ms = update_time_ms;
}
int32_t or_freespace_num_blocks(const OrMap* m) { return m->freespace.n; }
int32_t or_freespace_block_indices(const OrMap* m, int32_t* out, int32_t cap);
int32_t or_freespace_get_block(const OrMap* m, const int32_t xyz[3], OrFreespaceVoxel* out) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = hash_find(&m->freespace.hash, k);
  if (s < 0) return 0;
  memcpy(out, layer_block(&m->freespace, s), m->freespace.block_bytes);
  return 1;
}

void or_default_tsdf_decay_params(OrTsdfDecayParams* p) {
  p->decay_factor = 0.95f;
  p->decayed_weight_threshold = 1e-3f;
  p->set_free_distance_on_decayed = 0;
  p->free_distance_vox = 4.0f;
  p->deallocate_decayed_blocks = 1;
}
void or_default_occupancy_decay_params(OrOccupancyDecayParams* p) {
  p->free_region_decay_probability = 0.55f;
  p->occupied_region_decay_probability = 0.4f;
  p->decay_to_probability = 0.5f;
  p->deallocate_decayed_blocks = 1;
}
int32_t or_tsdf_decay(OrMap* map, const OrTsdfDecayParams* P, const OrDecayExclusion* X, const float* depth, int32_t rows,
                      int32_t cols, const float* T_L_C, const OrCamera* cam, float max_view_distance_m,
                      float truncation_distance_m, int32_t clear_esdf, int32_t* out_xyz, int32_t cap) {
  return decay_layer(map, 0, P, X, depth, rows, cols, T_L_C, cam, max_view_distance_m, truncation_distance_m,
                     P->deallocate_decayed_blocks, clear_esdf, out_xyz, cap);
}
int32_t or_occupancy_decay(OrMap* map, const OrOccupancyDecayParams* P, const OrDecayExclusion* X, const float* depth,
                           int32_t rows, int32_t cols, const float* T_L_C, const OrCamera* cam, float max_view_distance_m,
                           float truncation_distance_m, int32_t clear_esdf, int32_t* out_xyz, int32_t cap) {
  return decay_layer(map, 1, P, X, depth, rows, cols, T_L_C, cam, max_view_distance_m, truncation_distance_m,
                     P->deallocate_decayed_blocks, clear_esdf, out_xyz, cap);
}

void or_tsdf_set_block(OrMap* m, const int32_t xyz[3], const OrTsdfVoxel* in) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = layer_allocate(&m->tsdf, k);
  memcpy(layer_block(&m->tsdf, s), in, m->tsdf.block_bytes);
}

/* Test hook (no reference counterpart): place an EsdfBlock with given voxel contents, to start the wavefront from a state that
 * was written down by hand (tests/test_oracle_esdf_order_kat.py). */
void or_esdf_set_block(OrMap* m, const int32_t xyz[3], const OrEsdfVoxel* in) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = layer_allocate(&m->esdf, k);
  memcpy(layer_block(&m->esdf, s), in, m->esdf.block_bytes);
}

void or_freespace_set_block(OrMap* m, const int32_t xyz[3], const OrFreespaceVoxel* in) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = layer_allocate(&m->freespace, k);
  memcpy(layer_block(&m->freespace, s), in, m->freespace.block_bytes);
}

void or_occupancy_set_block(OrMap* m, const int32_t xyz[3], const float* in) {
  i3 k = {xyz[0], xyz[1], xyz[2]};
  int32_t s = layer_allocate(&m->occ, k);
  memcpy(layer_block(&m->occ, s), in, m->occ.block_bytes);
}

int32_t or_camera_project(const OrCamera* cam, const float p_C[3], float uv[2]) {
  v3 p = {p_C[0], p_C[1], p_C[2]};
  return cam_project(cam, p, &uv[0], &uv[1]);
}
void or_camera_vector_from_image_plane(const OrCamera* cam, float u, float v, float out[3]) {
  v3 r = cam_vector_from_image_plane(cam, u, v);
  out[0] = r.x, out[1] = r.y, out[2] = r.z;
}

/* ------------------------------------------------------------------------- */
/* Mesh integrator (src/mesh/mesh_integrator.cu, mesh_integrator_appearance.cu) */
/* ------------------------------------------------------------------------- */
#include "mc_table.h"

static int mc_hex(char c) { return c <= '9' ? c - '0' : c - 'a' + 10; }

/* One voxel of meshBlocksCalculateTableIndicesKernel (mesh_integrator.cu:335-452): the 8 corner samples of the cube whose
 * minimum corner is voxel (vx, vy, vz) of `blk`; nb[] = the block and its 7 upper neighbours in
 * neighborIndexFromDirection order (x << 2 | y << 1 | z, marching_cubes_impl.h:17-19). Returns the table index, or -1
 * if a corner is missing / unobserved. */
static int mesh_cube(const OrTsdfVoxel* const nb[8], i3 bidx, float block_size, float voxel_size, float min_weight, int vx,
                     int vy, int vz, float sdf[8], float pos[8][3]) {
  const int v[3] = {vx, vy, vz};
  /* getPositionFromBlockIndex (core/internal/impl/indexing_impl.h): block_size * index */
  const float bp[3] = {block_size * (float)bidx.x, block_size * (float)bidx.y, block_size * (float)bidx.z};
  for (int i = 0; i < 8; i++) {
    int c[3], off[3] = {0, 0, 0};
    for (int j = 0; j < 3; j++) {
      c[j] = v[j] + kMcCornerOffsets[i][j];
      if (c[j] >= VPS) c[j] -= VPS, off[j] = 1;
    }
    const OrTsdfVoxel* b = nb[(off[0] << 2) | (off[1] << 1) | off[2]];
    if (!b) return -1;
    const OrTsdfVoxel* vox = b + (c[0] * VPS + c[1]) * VPS + c[2];
    if (vox->weight < min_weight) return -1;
    sdf[i] = vox->distance;
    /* block_positions[block] + voxel_size * (corner_index + 0.5 + 8 * block_offset)  (:423-426) */
    for (int j = 0; j < 3; j++) pos[i][j] = bp[j] + voxel_size * (((float)c[j] + 0.5f) + (float)(VPS * off[j]));
  }
  int idx = 0; /* calculateVertexConfiguration (marching_cubes_impl.h:6-15) */
  for (int i = 0; i < 8; i++)
    if (sdf[i] < 0) idx |= 1 << i;
  return idx;
}

/* interpolateVertex (marching_cubes_impl.h:28-43) */
static void mc_interpolate(const float a[3], const float b[3], float sa, float sb, float out[3]) {
  const float diff = sa - sb;
  if (fabsf(diff) >= 1e-4f) {
    const float t = sa / diff;
    for (int j = 0; j < 3; j++) out[j] = a[j] + t * (b[j] - a[j]);
  } else {
    for (int j = 0; j < 3; j++) out[j] = 0.5f * (a[j] + b[j]);
  }
}

/* calculateVertices (internal/impl/cuda/marching_cubes_impl.cuh:31-70): the triangles of one cube, appended at `next`. */
static int mc_emit(int table_index, const float sdf[8], float pos[8][3], float* V, float* N, int32_t* T, int next) {
  const char* row = kMcTriangles[table_index];
  if (!row[0]) return next;
  float edge[12][3];
  memset(edge, 0, sizeof(edge));
  for (int e = 0; e < 12; e++) { /* interpolateEdgeVertices (marching_cubes_impl.h:45-64) */
    const int c0 = kMcEdgeCorners[e][0], c1 = kMcEdgeCorners[e][1];
    if ((sdf[c0] < 0 && sdf[c1] >= 0) || (sdf[c0] >= 0 && sdf[c1] < 0)) mc_interpolate(pos[c0], pos[c1], sdf[c0], sdf[c1], edge[e]);
  }
  for (int c = 0; row[c]; c += 3) {
    const float* p0 = edge[mc_hex(row[c + 2])];
    const float* p1 = edge[mc_hex(row[c + 1])];
    const float* p2 = edge[mc_hex(row[c])];
    memcpy(V + 3 * next, p0, 12), memcpy(V + 3 * (next + 1), p1, 12), memcpy(V + 3 * (next + 2), p2, 12);
    T[next] = next, T[next + 1] = next + 1, T[next + 2] = next + 2;
    const float px[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
    const float py[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
    /* Eigen cross + normalized(): v / sqrt(squaredNorm) if squaredNorm > 0 */
    float n[3] = {px[1] * py[2] - px[2] * py[1], px[2] * py[0] - px[0] * py[2], px[0] * py[1] - px[1] * py[0]};
    const float sq = (n[0] * n[0] + n[1] * n[1]) + n[2] * n[2];
    if (sq > 0.0f) {
      const float len = sqrtf(sq);
      n[0] /= len, n[1] /= len, n[2] /= len;
    }
    for (int k = 0; k < 3; k++) memcpy(N + 3 * (next + k), n, 12);
    next += 3;
  }
  return next;
}

typedef struct {
  uint64_t key;
  int32_t idx;
} WeldKey;
static int weld_cmp(const void* a, const void* b) {
  const WeldKey* x = (const WeldKey*)a;
  const WeldKey* y = (const WeldKey*)b;
  if (x->key != y->key) return x->key < y->key ? -1 : 1;
  return x->idx < y->idx ? -1 : (x->idx > y->idx ? 1 : 0); /* the radix sort is stable */
}

/* Index3D(v * kValueScale) in weldVerticesCubKernel (mesh_integrator.cu:755-757) converts on the device: cvt.rzi.s32.f32,
 * which truncates, saturates out-of-range values to INT32_MIN / INT32_MAX and maps NaN to 0 (PTX ISA, cvt). A plain C cast
 * is undefined there, and x86's cvttss2si gives INT32_MIN for both overflows -- wrong for vertices past +2147483.647 m. */
static int32_t weld_key_coord(float v) {
  const float s = v * 1000.0f;
  if (s != s) return 0;
  if (s >= 2147483648.0f) return INT32_MAX;
  if (s < -2147483648.0f) return INT32_MIN;
  return (int32_t)s;
}

/* weldVerticesCubKernel<128, 20> (mesh_integrator.cu:691-803). */
static void mesh_weld(MeshBlock* b) {
  const int n = b->nv;
  if (n <= 0 || n >= 128 * 20) return; /* too many vertices: the block keeps them all */
  WeldKey* k = (WeldKey*)malloc(sizeof(WeldKey) * (size_t)n);
  for (int i = 0; i < n; i++) {
    /* Index3DHash(Index3D(x * 1000, y * 1000, z * 1000)) (core/hash.h:32-40): float products truncated to int, then
     * x + y * 17191 + z * 17191^2 in size_t arithmetic */
    const int32_t x = weld_key_coord(b->v[3 * i]), y = weld_key_coord(b->v[3 * i + 1]), z = weld_key_coord(b->v[3 * i + 2]);
    const uint64_t sl = 17191ull;
    k[i].key = (uint64_t)(int64_t)x + (uint64_t)(int64_t)y * sl + (uint64_t)(int64_t)z * (sl * sl);
    k[i].idx = b->tri[i];
  }
  qsort(k, (size_t)n, sizeof(WeldKey), weld_cmp);
  float* V = (float*)malloc(12 * (size_t)n);
  float* N = (float*)malloc(12 * (size_t)n);
  int heads = 0;
  for (int i = 0; i < n; i++) {
    if (i == 0 || k[i].key != k[i - 1].key) { /* FlagHeads + InclusiveSum */
      memcpy(V + 3 * heads, b->v + 3 * k[i].idx, 12), memcpy(N + 3 * heads, b->nrm + 3 * k[i].idx, 12);
      heads++;
    }
    b->tri[k[i].idx] = heads - 1;
  }
  memcpy(b->v, V, 12 * (size_t)heads), memcpy(b->nrm, N, 12 * (size_t)heads);
  b->nv = heads; /* vertices / normals shrink; `triangles` keeps its pre-weld length (:668-686) */
  free(V), free(N), free(k);
}

void or_default_mesh_params(OrMeshParams* p) {
  p->min_weight = 1e-4f;          /* mesh_integrator_params.h:22-24 */
  p->weld_vertices = 1;           /* mesh_integrator_params.h:25-27 */
  p->cutoff_distance_vox = 5.0f;  /* mesh_integrator.h:129 */
}

/* MeshIntegrator::integrateBlocksGPU (mesh_integrator.cu:66-108) with the per-voxel output order made deterministic: the
 * reference hands out vertex ranges with an atomicAdd per voxel (calculateOutputIndex, marching_cubes_impl.cuh:11-29), so the
 * order of a block's triangles differs from run to run there; here voxels emit in x-major linear order (the CPU path's
 * order, :200-233). */
void or_mesh_integrate_blocks(OrMap* map, const int32_t* blocks_xyz, int32_t num_blocks, const OrMeshParams* P) {
  const float block_size = map->block_size, voxel_size = map->voxel_size;
  /* getIndicesInLayer + "clear all blocks if they exist" (:53-87) */
  for (int32_t i = 0; i < num_blocks; i++) {
    const i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    if (hash_find(&map->tsdf.hash, k) < 0) continue;
    const int32_t ms = hash_find(&map->mesh.hash, k);
    if (ms >= 0) {
      MeshBlock* mb = (MeshBlock*)layer_block(&map->mesh, ms);
      mb->nv = mb->nt = mb->nc = 0; /* MeshBlock::clear */
    }
  }
  const float cutoff = P->cutoff_distance_vox * voxel_size;
  float* V = (float*)malloc(12 * (size_t)VPB * 15);
  float* N = (float*)malloc(12 * (size_t)VPB * 15);
  int32_t* T = (int32_t*)malloc(4 * (size_t)VPB * 15);
  for (int32_t i = 0; i < num_blocks; i++) {
    const i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    const int32_t ts = hash_find(&map->tsdf.hash, k);
    if (ts < 0) continue;
    const OrTsdfVoxel* blk = (const OrTsdfVoxel*)layer_block(&map->tsdf, ts);
    int meshable = 0; /* isBlockMeshableKernel (:313-328) */
    for (int q = 0; q < VPB && !meshable; q++) meshable = fabsf(blk[q].distance) <= cutoff && blk[q].weight >= P->min_weight;
    if (!meshable) continue;
    const OrTsdfVoxel* nb[8];
    for (int j = 0; j < 8; j++) {
      const i3 nk = {k.x + ((j >> 2) & 1), k.y + ((j >> 1) & 1), k.z + (j & 1)};
      const int32_t s = hash_find(&map->tsdf.hash, nk);
      nb[j] = s >= 0 ? (const OrTsdfVoxel*)layer_block(&map->tsdf, s) : NULL;
    }
    int next = 0;
    for (int vx = 0; vx < VPS; vx++)
      for (int vy = 0; vy < VPS; vy++)
        for (int vz = 0; vz < VPS; vz++) {
          float sdf[8], pos[8][3];
          const int idx = mesh_cube(nb, k, block_size, voxel_size, P->min_weight, vx, vy, vz, sdf, pos);
          if (idx < 0) continue;
          next = mc_emit(idx, sdf, pos, V, N, T, next);
        }
    if (next == 0) continue; /* mesh blocks are only allocated for num_vertices > 0 (:603-611) */
    const int32_t ms = layer_allocate(&map->mesh, k);
    MeshBlock* mb = (MeshBlock*)layer_block(&map->mesh, ms);
    free(mb->v), free(mb->nrm), free(mb->tri);
    mb->v = (float*)malloc(12 * (size_t)next), mb->nrm = (float*)malloc(12 * (size_t)next), mb->tri = (int32_t*)malloc(4 * (size_t)next);
    memcpy(mb->v, V, 12 * (size_t)next), memcpy(mb->nrm, N, 12 * (size_t)next), memcpy(mb->tri, T, 4 * (size_t)next);
    mb->nv = next, mb->nt = next, mb->nc = 0;
    if (P->weld_vertices) mesh_weld(mb);
  }
  free(V), free(N), free(T);
}

/* MeshIntegrator::updateAppearanceGPU (mesh_integrator_appearance.cu:281-380) for ColorVoxel: every requested block that has
 * a mesh block gets one colour per vertex -- the colour voxel the vertex falls into in the CO-LOCATED colour block
 * (updateAppearanceBlockByClosestVoxel, :98-147), or Color::Gray() (127, 127, 127, core/color.h:59) if there is none. */
void or_mesh_update_color(OrMap* map, const int32_t* blocks_xyz, int32_t num_blocks) {
  const float block_size = map->block_size, voxel_size = map->voxel_size;
  for (int32_t i = 0; i < num_blocks; i++) {
    const i3 k = {blocks_xyz[3 * i], blocks_xyz[3 * i + 1], blocks_xyz[3 * i + 2]};
    const int32_t ms = hash_find(&map->mesh.hash, k);
    if (ms < 0) continue;
    MeshBlock* mb = (MeshBlock*)layer_block(&map->mesh, ms);
    free(mb->col);
    mb->col = (uint8_t*)malloc(4 * (size_t)(mb->nv > 0 ? mb->nv : 1)); /* expandAppearanceToMatchVertices */
    mb->nc = mb->nv;
    const int32_t cs = hash_find(&map->color.hash, k);
    const OrColorVoxel* cb = cs >= 0 ? (const OrColorVoxel*)layer_block(&map->color, cs) : NULL;
    const float bp[3] = {block_size * (float)k.x, block_size * (float)k.y, block_size * (float)k.z};
    for (int32_t q = 0; q < mb->nv; q++) {
      uint8_t* c = mb->col + 4 * q;
      if (!cb) {
        c[0] = c[1] = c[2] = 127, c[3] = 255;
        continue;
      }
      int vi[3];
      for (int j = 0; j < 3; j++) {
        vi[j] = (int)((mb->v[3 * q + j] - bp[j]) / voxel_size);
        vi[j] = vi[j] > VPS - 1 ? VPS - 1 : vi[j];
        vi[j] = vi[j] < 0 ? 0 : vi[j];
      }
      const OrColorVoxel* cv = cb + (vi[0] * VPS + vi[1]) * VPS + vi[2];
      c[0] = cv->r, c[1] = cv->g, c[2] = cv->b, c[3] = 255;
    }
  }
}

int32_t or_mesh_num_blocks(const OrMap* m) { return m->mesh.n; }
int32_t or_mesh_block_indices(const OrMap* m, int32_t* out, int32_t cap) { return layer_indices(&m->mesh, out, cap); }
int32_t or_mesh_block_sizes(const OrMap* m, const int32_t xyz[3], int32_t out[3]) {
  const i3 k = {xyz[0], xyz[1], xyz[2]};
  const int32_t s = hash_find(&m->mesh.hash, k);
  if (s < 0) return 0;
  const MeshBlock* b = (const MeshBlock*)layer_block(&m->mesh, s);
  out[0] = b->nv, out[1] = b->nt, out[2] = b->nc;
  return 1;
}
int32_t or_mesh_get_block(const OrMap* m, const int32_t xyz[3], float* vertices, float* normals, int32_t* triangles, uint8_t* colors) {
  const i3 k = {xyz[0], xyz[1], xyz[2]};
  const int32_t s = hash_find(&m->mesh.hash, k);
  if (s < 0) return 0;
  const MeshBlock* b = (const MeshBlock*)layer_block(&m->mesh, s);
  if (vertices) memcpy(vertices, b->v, 12 * (size_t)b->nv);
  if (normals) memcpy(normals, b->nrm, 12 * (size_t)b->nv);
  if (triangles) memcpy(triangles, b->tri, 4 * (size_t)b->nt);
  if (colors) memcpy(colors, b->col, 4 * (size_t)b->nc);
  return 1;
}

int32_t or_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
void or_set_num_threads(int32_t n) {
#ifdef _OPENMP
  omp_set_num_threads(n);
#else
  (void)n;
#endif
}
