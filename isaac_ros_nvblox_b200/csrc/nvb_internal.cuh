// nvb_internal.cuh -- shared declarations of the H100-native depth-integration core.
//
// Everything in csrc/ is compiled for sm_90a with -fmad=false: one IEEE
// rounding per floating-point operation, so that block-index sets are
// reproducible bit-for-bit and do not depend on the compiler's contraction
// choices (the reference's nvcc build contracts at the compiler's discretion,
// nvblox_core/cmake/nvblox_targets.cmake:120-171 -- see DESIGN.md "Numerics").
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include <cuda_runtime.h>
#include <stdint.h>

#include "nvblox_b200.h"

namespace nvb {

constexpr int kVps = 8;                 // VoxelBlock::kVoxelsPerSide (map/blox.h:36)
constexpr int kVpb = kVps * kVps * kVps;
constexpr int kTsdfBlockBytes = kVpb * 8;   // 4096
constexpr int kEsdfBlockBytes = kVpb * (16 + 4);  // 10240: a plane of 16-byte cells and a plane of flag words (nvb_esdf_block.cuh)
constexpr int kColorBlockBytes = kVpb * 8;  // ColorVoxel{Color (3 bytes) + 1 pad, float weight} (map/voxels.h:77-83)
constexpr int kOccBlockBytes = kVpb * 4;    // OccupancyVoxel{float log_odds} (map/voxels.h:92-97)
constexpr int kHelperCtas = 132;            // grid of the small grid-stride helper kernels: one CTA per H100 SM

struct Vec3 {
  float x, y, z;
};

// Rigid transform handed to kernels by value (12 floats; Eigen Isometry3f without
// the constant bottom row).
struct Rigid {
  float r[3][3];
  float t[3];
};

// ---------------------------------------------------------------------------
// Arithmetic with the evaluation order of the reference's Eigen expressions.
// ---------------------------------------------------------------------------

// Fixed-size-3 reductions in Eigen evaluate a0 + (a1 + a2).
__host__ __device__ __forceinline__ float sum3(float a0, float a1, float a2) { return a0 + (a1 + a2); }

// Isometry3f * Vector3f : translation + linear * p.
__host__ __device__ __forceinline__ Vec3 transformPoint(const Rigid& T, const Vec3& p) {
  Vec3 o;
  o.x = T.t[0] + sum3(T.r[0][0] * p.x, T.r[0][1] * p.y, T.r[0][2] * p.z);
  o.y = T.t[1] + sum3(T.r[1][0] * p.x, T.r[1][1] * p.y, T.r[1][2] * p.z);
  o.z = T.t[2] + sum3(T.r[2][0] * p.x, T.r[2][1] * p.y, T.r[2][2] * p.z);
  return o;
}

// float -> int with device semantics on both host and device (NaN -> 0, saturating).
__host__ __device__ __forceinline__ int floatToIntRz(float f) {
#ifdef __CUDA_ARCH__
  return __float2int_rz(f);
#else
  if (f != f) return 0;
  if (f >= 2147483648.0f) return INT32_MAX;
  if (f <= -2147483648.0f) return INT32_MIN;
  return (int)f;
#endif
}

// getBlockIndexFromPositionInLayer (core/internal/impl/indexing_impl.h:31-35).
__host__ __device__ __forceinline__ int3 blockIndexFromPosition(float block_size, const Vec3& p) {
  return make_int3(floatToIntRz(floorf(p.x / block_size)), floatToIntRz(floorf(p.y / block_size)),
                   floatToIntRz(floorf(p.z / block_size)));
}

// 1 / blockSizeToVoxelSize(block_size), evaluated in double and rounded to float (core/internal/impl/indexing_impl.h:41).
__host__ __device__ __forceinline__ float voxelSizeInv(float block_size) {
  return (float)(1.0 / (double)(block_size * (1.0f / kVps)));
}

// getBlockAndVoxelIndexFromPositionInLayer (core/internal/impl/indexing_impl.h:37-49): the block index is floor(p / block_size),
// the voxel index (p - block_size * b) * voxel_size_inv truncated toward zero and clamped to kVps - 1.
__host__ __device__ __forceinline__ void blockAndVoxelIndexFromPosition(float block_size, float voxel_size_inv, const Vec3& p,
                                                                        int3& b, int3& v) {
  b = blockIndexFromPosition(block_size, p);
  v.x = min(floatToIntRz((p.x - block_size * (float)b.x) * voxel_size_inv), kVps - 1);
  v.y = min(floatToIntRz((p.y - block_size * (float)b.y) * voxel_size_inv), kVps - 1);
  v.z = min(floatToIntRz((p.z - block_size * (float)b.z) * voxel_size_inv), kVps - 1);
}

// AlignedBox::exteriorDistance(c) of getAABBOfBlock(block_size, idx) (geometry/internal/impl/bounding_boxes_impl.h:55-60,
// src/geometry/bounding_spheres.cpp:23-31): Eigen's squaredExteriorDistance accumulates the axes in order from 0.
__host__ __device__ __forceinline__ float blockExteriorDistance(const int idx[3], float block_size, const float c[3]) {
  float dist2 = 0.0f;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const float bmin = (float)idx[k] * block_size, bmax = ((float)idx[k] + 1.0f) * block_size;
    if (bmin > c[k]) {
      const float aux = bmin - c[k];
      dist2 += aux * aux;
    } else if (c[k] > bmax) {
      const float aux = c[k] - bmax;
      dist2 += aux * aux;
    }
  }
  return sqrtf(dist2);
}

// ---------------------------------------------------------------------------
// Radial-tangential lens distortion (sensors/internal/impl/distortion_impl.h). The reference mixes
// float and double through its `1.0` / `2.0` literals; the same promotions are spelled out here.
// ---------------------------------------------------------------------------
__host__ __device__ __forceinline__ float radialScaleF(float r2, const NvbCamera& c) {  // :24-32, T = float
  const float r4 = r2 * r2;
  const float r6 = r2 * r4;
  const float numerator = (float)(1.0 + (double)(c.k1 * r2) + (double)(c.k2 * r4) + (double)(c.k3 * r6));
  const float denominator = (float)(1.0 + (double)(c.k4 * r2) + (double)(c.k5 * r4) + (double)(c.k6 * r6));
  return numerator / denominator;
}
__host__ __device__ __forceinline__ double radialScaleD(double r2, const NvbCamera& c) {  // T = double
  const double r4 = r2 * r2;
  const double r6 = r2 * r4;
  const double numerator = 1.0 + (double)c.k1 * r2 + (double)c.k2 * r4 + (double)c.k3 * r6;
  const double denominator = 1.0 + (double)c.k4 * r2 + (double)c.k5 * r4 + (double)c.k6 * r6;
  return numerator / denominator;
}
// applyDistortion (:37-60)
__host__ __device__ __forceinline__ void applyDistortion(const NvbCamera& c, float& ux, float& uy) {
  const float x = ux, y = uy;
  const float r2 = x * x + y * y;
  const float scale = radialScaleF(r2, c);
  const float xy = x * y;
  const float tx = (float)(2.0 * (double)c.p1 * (double)xy + (double)c.p2 * ((double)r2 + 2.0 * (double)x * (double)x));
  const float ty = (float)(2.0 * (double)c.p2 * (double)xy + (double)c.p1 * ((double)r2 + 2.0 * (double)y * (double)y));
  ux = x * scale + tx;
  uy = y * scale + ty;
}
// removeDistortion (:93-176): Newton-Raphson in double, at most 6 iterations; compute_dR_dr2 (:62-91).
__host__ __device__ inline void removeDistortion(const NvbCamera& c, float& ux, float& uy) {
  const double k1 = c.k1, k2 = c.k2, k3 = c.k3, k4 = c.k4, k5 = c.k5, k6 = c.k6, p1 = c.p1, p2 = c.p2;
  const double u_in_x = ux, u_in_y = uy;
  double x = u_in_x, y = u_in_y;
  for (int i = 0; i < 6; i++) {
    const double x2 = x * x, y2 = y * y, r2 = x2 + y2;
    const double R = radialScaleD(r2, c);
    const double xy = x * y;
    const double tan_x = 2.0 * p1 * xy + p2 * (r2 + 2.0 * x * x);
    const double tan_y = 2.0 * p2 * xy + p1 * (r2 + 2.0 * y * y);
    const double x_est = x * R + tan_x, y_est = y * R + tan_y;
    const double error_x = x_est - u_in_x, error_y = y_est - u_in_y;
    const double q = r2, q2 = q * q, q3 = q2 * q;
    const double ja = k1 + 2. * k2 * q + 3. * k3 * q2;
    const double jc = k4 + 2. * k5 * q + 3. * k6 * q2;
    const double jb = k4 * q + k5 * q2 + k6 * q3 + 1.;
    const double jd = k1 * q + k2 * q2 + k3 * q3 + 1.;
    const double dR_dr2 = (ja * jb - jc * jd) / (jb * jb);
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
  ux = (float)x;
  uy = (float)y;
}

#ifdef __CUDACC__
// The ray of pixel (r, c) of the f-subsampled image goes through the image-plane point f * (c, r) + f / 2
// (SphereTracer's sphereTracingKernel, src/rays/sphere_tracer.cu:134-173). dz is the camera-frame direction's z, u the
// layer-frame direction. With f = 1 this is Camera::vectorFromPixelIndices(u).normalized() rotated by T's linear part, the
// ray of Scene::generateDepthImageFromScene (nvb_scene.cu).
template <bool kDistort>
__device__ __forceinline__ void pixelRay(const NvbCamera& cam, const Rigid& T, int f, int r, int c, float& dz, Vec3& u) {
  const float half = 0.5f * (float)f;
  const float px = (float)(c * f) + half * 1.0f, py = (float)(r * f) + half * 1.0f;
  // Camera::vectorFromImagePlaneCoordinates (camera_impl.h:89-104), then Eigen normalized()
  float nx = (px - cam.cu) / cam.fu, ny = (py - cam.cv) / cam.fv;
  if (kDistort) removeDistortion(cam, nx, ny);
  const float norm = sqrtf(sum3(nx * nx, ny * ny, 1.0f * 1.0f));
  const float dx = nx / norm, dy = ny / norm;
  dz = 1.0f / norm;
  u.x = sum3(T.r[0][0] * dx, T.r[0][1] * dy, T.r[0][2] * dz);
  u.y = sum3(T.r[1][0] * dx, T.r[1][1] * dy, T.r[1][2] * dz);
  u.z = sum3(T.r[2][0] * dx, T.r[2][1] * dy, T.r[2][2] * dz);
}
#endif  // __CUDACC__

// ---------------------------------------------------------------------------
// Device-resident block hash: packed Index3D -> slot in the layer's slab.
// Open addressing, linear probing, 64-bit keys (3 x 21 bit, biased).
// Replaces the host unordered_map + stdgpu mirror of the reference
// (map/layer.h:48-217, gpu_hash/gpu_layer_view.h:48-141).
// ---------------------------------------------------------------------------

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int kIndexBias = 1 << 20;

__host__ __device__ __forceinline__ bool indexInRange(int x, int y, int z) {
  return x >= -kIndexBias && x < kIndexBias && y >= -kIndexBias && y < kIndexBias && z >= -kIndexBias &&
         z < kIndexBias;
}

__host__ __device__ __forceinline__ unsigned long long packIndex(int x, int y, int z) {
  return ((unsigned long long)(unsigned)(x + kIndexBias) << 42) |
         ((unsigned long long)(unsigned)(y + kIndexBias) << 21) | (unsigned long long)(unsigned)(z + kIndexBias);
}

__host__ __device__ __forceinline__ unsigned int hashKey(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (unsigned int)k;
}

struct DevHash {
  unsigned long long* keys;
  int* vals;
  unsigned int mask;  // capacity - 1 (capacity is a power of two)
};

// One layer = one contiguous slab of fixed-size blocks + the hash + the reverse map.
struct DevLayer {
  unsigned char* blocks;  // capacity * block_bytes, zero-initialised
  int* block_index;       // 3 ints per slot (Index3D of the block living in that slot); x == kDeadSlotX: slot is free
  int* count;             // device counter: slots handed out so far (high-water mark; freed slots are below it)
  int* free_slots;        // stack of deallocated slots (their blocks are zero again), reused before the slab grows
  int* free_count;
  int capacity;
  int block_bytes;
  DevHash hash;
};
constexpr int kDeadSlotX = INT32_MIN;  // block_index[3 * slot] of a deallocated slot

#ifdef __CUDACC__
__device__ __forceinline__ int hashFind(const DevHash& h, int x, int y, int z) {
  if (!indexInRange(x, y, z)) return -1;
  const unsigned long long key = packIndex(x, y, z);
  unsigned int p = hashKey(key) & h.mask;
  while (true) {
    const unsigned long long k = h.keys[p];
    if (k == key) return h.vals[p];
    if (k == kEmptyKey) return -1;
    p = (p + 1) & h.mask;
  }
}

// Find-or-insert. Keys inserted by one kernel launch must be unique within that
// launch (callers guarantee it), so a key that is already present was inserted
// by an earlier launch and its value is visible. Returns the slot, or -1 when
// the slab is exhausted / the index does not fit (flagged in *error).
__device__ __forceinline__ int hashFindOrInsert(const DevLayer& L, int x, int y, int z, int* error, bool* was_new) {
  *was_new = false;
  if (!indexInRange(x, y, z)) {
    atomicOr(error, 2);
    return -1;
  }
  const unsigned long long key = packIndex(x, y, z);
  unsigned int p = hashKey(key) & L.hash.mask;
  while (true) {
    const unsigned long long k = L.hash.keys[p];
    if (k == key) return L.hash.vals[p];
    if (k == kEmptyKey) {
      const unsigned long long old = atomicCAS(&L.hash.keys[p], kEmptyKey, key);
      if (old == kEmptyKey) {
        // a deallocated slot first (decay integrators), else the next fresh one
        int slot = -1;
        if (*(volatile int*)L.free_count > 0) {
          const int f = atomicSub(L.free_count, 1) - 1;
          if (f >= 0) slot = L.free_slots[f];
          else atomicAdd(L.free_count, 1);
        }
        if (slot < 0) slot = atomicAdd(L.count, 1);
        if (slot >= L.capacity) {
          atomicOr(error, 1);
          L.hash.vals[p] = -1;
          return -1;
        }
        L.hash.vals[p] = slot;
        L.block_index[3 * slot + 0] = x;
        L.block_index[3 * slot + 1] = y;
        L.block_index[3 * slot + 2] = z;
        *was_new = true;
        return slot;
      }
      if (old == key) return L.hash.vals[p];
    }
    p = (p + 1) & L.hash.mask;
  }
}
#endif  // __CUDACC__

// ---------------------------------------------------------------------------
// Per-frame view description computed on the host (ViewCalculator setup,
// view_calculator_impl.cuh:137-156).
// ---------------------------------------------------------------------------
struct ViewGrid {
  int3 min_index;
  int3 size;
  int linear_size;  // size.x * size.y * size.z
  int num_words;    // bitset words
};

struct TsdfKernelParams {
  float block_size;
  float voxel_size;       // block_size * (1/8)
  float half_voxel_size;  // block_size * (0.5/8)
  float truncation_distance_m;
  float max_integration_distance_m;
  float max_weight;
  float invalid_depth_decay_factor;
  int weighting_type;
};

// UpdateOccupancyVoxelFunctor's parameters (projective_occupancy_integrator_impl.cuh:58-72), log odds computed
// on the host like in the reference.
struct OccKernelParams {
  float free_log_odds, occupied_log_odds, unobserved_log_odds;
  float occupied_half_width_m;
  float min_log_odds, max_log_odds;
};

// The block-update tracker on the device (BlocksToUpdateTracker, map/blocks_to_update_tracker.h). A consumer's pending
// blocks: a dirty word per projective slot and the list of the slots whose word is set; a null `dirty`: not told.
enum BlocksToUpdateType { kEsdfBlocks, kFreespaceBlocks, kColorMeshBlocks, kNumBlocksToUpdateTypes };
struct TrackerList { int *dirty, *slots, *count; };
struct TrackerLists { TrackerList list[kNumBlocksToUpdateTypes]; };  // by BlocksToUpdateType
#ifdef __CUDACC__
// addBlocksToUpdate (map/blocks_to_update_tracker.cpp:33-63): unique append of `slot` to every consumer that is told.
__device__ __forceinline__ void trackerAdd(const TrackerLists& t, int slot) {
#pragma unroll
  for (const TrackerList& l : t.list)
    if (l.dirty != nullptr && atomicExch(l.dirty + slot, 1) == 0) l.slots[atomicAdd(l.count, 1)] = slot;
}
#endif

// ---------------------------------------------------------------------------
// Kernel launchers (implemented in the .cu files; all enqueue on `stream`).
// ---------------------------------------------------------------------------

// nvb_view.cu
void launchViewRaycast(const float* depth, int rows, int cols, const Rigid& T_L_C, const NvbCamera& cam,
                       float block_size, float trunc_m, float max_dist, int subsample, const ViewGrid& grid,
                       unsigned int* bits, cudaStream_t stream);
// Ordered compaction of the bitset into the frame list (+ optional allocation in `layer`
// and tracker update). frame_blocks: int4 {x,y,z,slot}. Clears the bitset words it reads.
struct CompactArgs {
  unsigned int* bits;
  ViewGrid grid;
  int4* frame_blocks;
  int* frame_count;
  unsigned long long* tile_state;  // chained-scan state, one per tile
  unsigned int* ticket;            // monotonically increasing ticket counter
  unsigned int ticket_base;
  unsigned int epoch;
  int allocate;                    // 1: find-or-insert into layer
  DevLayer layer;
  int* error;
  TrackerLists tracker;            // told about every block found or inserted (allocate only)
};
int compactNumTiles(const ViewGrid& grid);
bool compactUsesTickets(const ViewGrid& grid);
// The compaction leaves the bitset set; it is zeroed by the TSDF kernel's prologue or, on the
// view-only path, by this launch.
void launchClearBits(unsigned int* bits, int num_words, cudaStream_t stream);
void launchMarkList(const int* xyz_dev, int n, const ViewGrid& grid, unsigned int* bits, cudaStream_t stream);
void launchUnpackList(const int4* in, const int* count, int* out, int cap, cudaStream_t stream);
void launchCompactAllocate(const CompactArgs& args, cudaStream_t stream);

// nvb_tsdf.cu
void launchTsdfIntegrate(const int4* frame_blocks, const int* frame_count, unsigned char* tsdf_blocks,
                         const float* depth, const unsigned char* mask, int mask_mode, int rows, int cols,
                         const Rigid& T_C_L, const NvbCamera& cam, const TsdfKernelParams& p, int num_sms,
                         unsigned int* bits_to_clear, int num_words, cudaStream_t stream);

void launchOccupancyIntegrate(const int4* frame_blocks, const int* frame_count, unsigned char* occ_blocks,
                              const float* depth, const unsigned char* mask, int mask_mode, int rows, int cols,
                              const Rigid& T_C_L, const NvbCamera& cam, const TsdfKernelParams& p,
                              const OccKernelParams& op, int num_sms, unsigned int* bits_to_clear, int num_words,
                              cudaStream_t stream);

// nvb_esdf.cu
struct EsdfCtx {
  DevLayer tsdf;
  DevLayer esdf;
  DevLayer freespace;  // FreespaceLayer of a TSDF-with-freespace mapper (use_freespace)
  int use_freespace;
  // work list of this update: {esdf_slot, tsdf_slot, is_new, 0}
  int4* work;
  int* work_count;
  // lists of ESDF slots
  int* upd_list;
  int* upd_count;
  int* clr_list;   // to-clear blocks
  int* clr_count;
  int* clr_aabb;   // 6 ints: min xyz, max xyz (block indices) of the to-clear blocks
  int* cleared_list;  // persistent across calls, like EsdfIntegrator::cleared_block_indices_device_
  int* cleared_count;
  int* ring_a;
  int* ring_b;
  int* ring_count;     // 2 ints
  int* tail_state;     // 2 ints: rings advanced / final member count of a single-CTA tail episode
  int* stamp_a;        // per ESDF slot
  int* stamp_b;
  int* ring_id;        // device: monotonically increasing ring id
  // Ownership-based wavefront (persistent kernel): no lists, every CTA scans the slots it owns.
  int* nbr;           // 6 ints per ESDF slot: slot of the +x,-x,+y,-y,+z,-z neighbour, -1 none, < -1 unknown
  int* nbr27;         // 27 ints per ESDF slot: slot of the block at offset (dx,dy,dz), entry (dx+1)*9+(dy+1)*3+(dz+1);
                      // -1 none, < -1 unknown (never linked)
  unsigned char* shadow;  // second ESDF slab (same slot indexing): results of a ring wait here until all reads are done
  unsigned char* xslab;   // exchange-slab wavefront: two slabs (ring parity) of per-slot block faces, members' faces as their
                          // neighbours' owners read them (esdfWaveXSlabBytes)
  int* xtail;             // exchange-slab wavefront: 4 ints, hand-over of a single-CTA tail episode (rings advanced, K, M)
  int* xrec;              // exchange-slab wavefront: candidate records {slot, 27 neighbour slots, pad}, 32 ints; per ring parity one
                          // segment of `xseg` records per CTA
  int xseg;
  int xsplit_min_k;       // exchange-slab wavefront: grid rings with at least this many candidates fetch the own block split
  int* xcounts;          // exchange-slab wavefront: barrier flags, per barrier parity and CTA {generation, registrations, changed blocks}
  int slice_mode;  // the ESDF layer is a 2-D slice (EsdfMode::k2D)
  // constant-z slice (2-D ESDF): block / voxel z of the band's bottom and top and of the output layer
  int slice_min_bz, slice_min_vz, slice_max_bz, slice_max_vz, slice_out_bz, slice_out_vz;
  // planar slice (PlanarSliceDescription): per-column bounds from the ground plane n . p + d = 0
  int slice_planar;
  float plane_nx, plane_ny, plane_nz, plane_d, slice_above_plane_m, slice_thickness_m;
  unsigned long long* colset_keys;  // set of (x, y) columns of this slice update (open addressing, keys only)
  unsigned int colset_mask;
  int* cols;                // unique columns: x, y pairs
  int* cols_count;
  int* dead_cleared_xyz;    // indices of deallocated blocks that were on the persistent cleared list (3 ints each) ...
  int* dead_cleared_count;  // ... they rejoin it if a block with that index is allocated again while the list persists
  int* cand_a;        // candidate lists of the gather-emulate-sweep rings (ping-pong by ring parity)
  int* cand_b;
  int ges_switch;     // rings with more members than this run as four-phase rings
  int* cand_stamp;    // per slot: == ring  <=> registered as a candidate (neighbour of a member) of that ring
  int* ges_counts;    // 4 ints: candidate count [2], member count [2] (ping-pong by ring parity)
  unsigned int* psum; // two words per slot (the two halves of the block, x < 4 and x >= 4): 0 = no voxel has a parent; bit 31 set: box of the BLOCK OFFSETS the voxels' parents
                      // point into, 5 bits per bound (lo x, hi x, lo y, hi y, lo z, hi z, each + 16); 0xffffffff = unknown.
                      // An upper bound kept by the exchange-slab wavefront (the only writer of non-zero parents in that mode).
  unsigned int* clr_bits;  // bitmap of the to-clear blocks over their AABB (2048 words), built by the mark kernel's last CTA
  int prune;          // clear pass: skip candidates whose parent box holds no to-clear block (exact: a voxel is cleared iff its
                      // parent voxel lost its site flag, and sites are only lost in to-clear blocks)
  int* seed_upd;      // per slot: == update_seq  <=> block has sites in this update (computeEsdf #1 seeds)
  int* seed_clr;      // per slot: == *cleared_seq <=> member of the persistent cleared list (computeEsdf #2 seeds)
  int* cleared_seq;   // device: update_seq of the last update whose clear pass ran
  int update_seq;     // host: sequence number of this update (monotone, starts at 1)
  // tracker (BlocksToUpdateTracker::markBlocksAsUpdated fused into the ESDF kernels); null on explicit lists
  int* tracker_dirty;
  int* tracker_todo_count;
  unsigned int* barrier;  // grid barrier counter
  unsigned long long* phase_max;  // debug, kPhaseMaxEntries: per-phase max-over-CTAs work time in the first 1000
  long long* stats;    // kNumEsdfStats counters, by EsdfStat
  int* error;
  float max_sq;
  float max_esdf_distance_m;
  float max_site_distance_m;
  float min_weight;
  float block_size;
  int from_occupancy;               // the projective layer (`tsdf` above) holds OccupancyVoxels
  float occupied_threshold_log_odds;
};
void launchEsdfSliceAllocateAndMark(const EsdfCtx& c, const int* in_xyz, const int* in_slots, const int* in_count_dev,
                                    int in_count_upper, int num_sms, cudaStream_t stream);
void launchEsdfAllocate(const EsdfCtx& c, const int* in_xyz, const int* in_slots, const int* in_count_dev,
                        int in_count_upper, cudaStream_t stream);
void launchEsdfMark(const EsdfCtx& c, int count_upper, int num_sms, cudaStream_t stream);
void launchEsdfClear(const EsdfCtx& c, int esdf_count_upper, int num_sms, cudaStream_t stream);
// Whole wavefront (both computeEsdf calls) in one cooperative launch. Returns cudaError.
cudaError_t launchEsdfComputeGes(const EsdfCtx& c, int num_sms, cudaStream_t stream, int* launches);
cudaError_t launchEsdfComputePersistent(const EsdfCtx& c, int num_sms, cudaStream_t stream, int* launches);
cudaError_t launchEsdfComputeX(const EsdfCtx& c, int num_sms, int reserved_sms, cudaStream_t stream, int* launches);  // nvb_esdf_wavex.cu
int esdfWaveXGrid(int num_sms, int reserved_sms);  // CTAs of an exchange-slab launch
size_t esdfWaveXFlagBytes();
size_t esdfWaveXSlabBytes(int capacity);  // both exchange slabs: 2 x capacity x 7.5 KiB
int esdfWaveXSplitMinK();  // kSplitMinK, or NVB_WAVEX_SPLIT_MIN_K (read at mapper creation)
// Reference-like driver: one launch per phase, host reads the ring counter.
cudaError_t runEsdfComputeHostLoop(const EsdfCtx& c, int num_sms, cudaStream_t stream, int* launches);
int esdfPersistentMaxCtas(int num_sms);

// The clear pass's parent-box word of half an ESDF block (EsdfCtx::psum) from the bounds of the block offsets its voxels'
// parents point into: 0 without parents, the six bounds + 16 in 5 bits each under bit 31, or 0xffffffff when a bound
// leaves [-16, 15].
__host__ __device__ __forceinline__ unsigned int parentBoxWord(int lo0, int hi0, int lo1, int hi1, int lo2, int hi2) {
  if (lo0 > hi0) return 0u;
  const bool fits = lo0 >= -16 && lo1 >= -16 && lo2 >= -16 && hi0 <= 15 && hi1 <= 15 && hi2 <= 15;
  return fits ? ((1u << 31) | (unsigned)(lo0 + 16) | ((unsigned)(hi0 + 16) << 5) | ((unsigned)(lo1 + 16) << 10) |
                 ((unsigned)(hi1 + 16) << 15) | ((unsigned)(lo2 + 16) << 20) | ((unsigned)(hi2 + 16) << 25))
              : 0xffffffffu;
}

constexpr int kFreespaceVoxelBytes = 24;
constexpr int kFreespaceBlockBytes = 512 * kFreespaceVoxelBytes;  // 12 288
#ifdef __CUDACC__
// FreespaceVoxel::is_high_confidence_freespace (byte 16 of the 24-byte voxel) of voxel v of the freespace block in `slot`;
// false if there is no block (slot < 0), like isVoxelFreespace (esdf_integrator.cu:101-111).
__device__ __forceinline__ bool isVoxelFreespace(const DevLayer& layer, int slot, int v) {
  return slot >= 0 && layer.blocks[(size_t)slot * kFreespaceBlockBytes + (size_t)v * kFreespaceVoxelBytes + 16] != 0;
}
#endif
// nvb_tsdf.cu: freespace (FreespaceIntegrator, integrators/internal/cuda/impl/freespace_integrator_impl.cuh)
struct FreespaceArgs {
  DevLayer tsdf, fs;
  // blocks to update: TSDF slots from the tracker (its dirty words are cleared for the consumed slots), or explicit indices
  TrackerList todo;
  const int* in_xyz;
  int n_explicit;
  int4* work;          // {tsdf slot, freespace slot, -, -}
  int* work_count;
  int* error;
  // parameters
  float max_tsdf_distance_for_occupancy_m;
  long long max_unobserved_ms, min_free_ms, min_reset_ms;
  int check_neighborhood, init_high_confidence;
  long long last_update_ms, now_ms;
  // DepthObservationSpace (null depth: every voxel is updated)
  const float* depth;
  int rows, cols;
  Rigid T_C_L;
  NvbCamera cam;
  TsdfKernelParams p;
};
void launchFreespaceUpdate(const FreespaceArgs& a, int upper, int num_sms, cudaStream_t stream);

// nvb_tsdf.cu: decay (VoxelDecayer::decay, integrators/internal/cuda/impl/decayer_impl.cuh)
// Mapper::markUnobservedTsdfFreeInsideRadius (nvb_tsdf.cu)
struct MarkFreeArgs {
  DevLayer layer;  // the projective layer
  int occupancy;
  int3 lo, size;   // block-index box of center +- radius
  int cells;
  float cx, cy, cz, radius, block_size, trunc_m;
  int4* out;       // {x, y, z, slot} of the blocks inside the radius
  int* out_count;
  int* error;
  TrackerLists tracker;
};
void launchMarkFreeSphere(const MarkFreeArgs& a, int num_sms, cudaStream_t stream);

// Colour integration (nvb_color.cu): one frame's arguments.
struct ColorArgs {
  DevLayer tsdf, color;
  Rigid T_C_L, T_L_C;
  NvbCamera cam;
  int3 aabb_lo, aabb_hi;                   // block-index range of the view AABB
  float vmin_x, vmin_y, vmax_x, vmax_y;    // Camera::getNormalizedViewport(getViewportMargin(height))
  float block_size, voxel_size, half_voxel_size, voxel_size_inv;
  float trunc_m, max_integration_distance_m, max_weight, measurement_weight;
  float w_old_h, w_new_h;                  // blendTwoArrays' normalised weights, rounded through binary16 on the host
  int4* work;                              // {x, y, z, colour slot} of the blocks in view and in the truncation band
  int* work_count;
  int* error;
  float* synth;                            // sphere-traced depth, drows x dcols
  int drows, dcols, subsample, depth_subsample;
  int max_steps;
  float max_ray_len, eps_m;
  const unsigned char* color_image;        // rows x cols x 3 (RGB)
  const unsigned char* mask;
  int mask_mode;
  int rows, cols;
};
void launchColorSelect(const ColorArgs& a, int num_sms, cudaStream_t stream);
void launchSphereTrace(const ColorArgs& a, cudaStream_t stream);
void launchColorIntegrate(const ColorArgs& a, int num_sms, cudaStream_t stream);
// SphereTracer::renderImageOnGPU / renderRgbdImageOnGPU (nvb_color.cu): one image of drows x dcols rays.
struct RenderArgs {
  DevLayer tsdf, color;  // color.blocks == nullptr: the mapper has no colour layer (every hit is black)
  Rigid T_L_C;
  NvbCamera cam;
  float block_size, voxel_size_inv, trunc_m, max_ray_len, eps_m;
  int max_steps, subsample, drows, dcols;
  float* depth;          // drows x dcols
  unsigned char* rgb;    // drows x dcols x 3 (RGB), or nullptr: depth only
};
void launchRender(const RenderArgs& a, cudaStream_t stream);

// primitives::Scene (nvb_scene.cu). The scene's primitives are in device memory here.
struct SceneDepthArgs {  // Scene::generateDepthImageFromScene
  NvbScene scene;
  NvbCamera cam;
  Rigid T_S_C, T_C_S;
  float max_dist, invalid_depth;
  int rows, cols;
  float* depth;  // rows x cols
};
void launchSceneDepth(const SceneDepthArgs& a, cudaStream_t stream);
// Scene::getSignedDistanceToPoint of n points (xyz) into out
void launchSceneDistance(const NvbScene& scene, const float* xyz, long long n, float max_dist, float* out, int num_sms,
                         cudaStream_t stream);
struct SceneLayerArgs {  // Scene::generateLayerFromScene
  NvbScene scene;
  DevLayer layer;
  int layer_id;                  // NVB_LAYER_TSDF, _OCCUPANCY or _FREESPACE
  int3 box_lo, box_size;         // getBlockIndicesTouchedByBoundingBox: the block-index box of the AABB ...
  long long cells;               // ... and its number of blocks
  float block_size, max_dist;
  float occupied_threshold_m;    // sqrt(3) * voxel_size / 2: an object is inside the voxel at or below it
  float occupied_log_odds, free_log_odds;  // logOddsFromProbability(1), (0), computed on the host
  int* error;
};
void launchSceneAllocate(const SceneLayerArgs& a, int num_sms, cudaStream_t stream);
void launchSceneFill(const SceneLayerArgs& a, int num_sms, cudaStream_t stream);

struct DecayArgs {
  DevLayer layer;  // the projective layer (TsdfVoxel or OccupancyVoxel blocks)
  int occupancy;
  // TsdfDecayFunctor / OccupancyDecayFunctor
  float decay_factor, weight_threshold, free_distance_m;
  int set_free_distance;
  float free_log_odds, occupied_log_odds, to_log_odds;
  int deallocate;
  // DecayBlockExclusionOptions
  const int* skip_stamp;  // per slot: == skip_seq -> spared
  int skip_seq;
  int has_sphere;
  float cx, cy, cz, r2;
  // DepthObservationSpace (null depth: every voxel decays)
  const float* depth;
  int rows, cols;
  Rigid T_C_L;
  NvbCamera cam;
  TsdfKernelParams p;  // block/voxel sizes, max view distance (max_integration_distance_m), truncation
  // outputs
  int4* dead;  // {slot, x, y, z} of deallocated blocks
  int* dead_count;
};
void launchDecay(const DecayArgs& a, int num_sms, cudaStream_t stream);
void launchMarkSkipped(const DevLayer& layer, const int* xyz_dev, int n, int* skip_stamp, int skip_seq, cudaStream_t stream);
// nvb_esdf.cu: ESDF side of a deallocation (Mapper::clearBlocksInLayers)
void launchEsdfRemoveBlocks(const EsdfCtx& c, const int4* dead, const int* dead_count, int upper, cudaStream_t stream);

// nvb_merge.cu: device-resident merge of the ranks' block lists (multi-GPU)
void launchAppendFrame(const int4* frame, const int* frame_count, int* seg, int cap, int* error, cudaStream_t stream);
void launchUnionSegments(const int* segs, int num_segments, int stride, int cap, int* state, unsigned int* bits, long long cap_bits,
                         int* out_xyz, int out_cap, int* out_count, cudaStream_t stream);

// nvb_mesh.cu
// Header of one mesh block in the mesh layer's slab (32 bytes): where its vertices / normals / triangle indices / colours
// live in the arena. cap = the arena entries reserved for it (its pre-weld vertex count).
struct MeshHeader {
  int offset, nv, nt, cap, nc, pad[3];
};
constexpr int kMeshHeaderBytes = 32;
static_assert(sizeof(MeshHeader) == kMeshHeaderBytes, "MeshHeader layout");
enum { kArenaUsed = 0, kArenaGarbage = 1, kArenaLastBase = 2, kArenaLastTotal = 3, kArenaInts = 4 };
struct MeshCtx {
  DevLayer tsdf, color, mesh;  // color.blocks == nullptr: the mapper has no colour layer (yet)
  float* vertices;
  float* normals;
  int* triangles;
  unsigned char* colors_raw;
  uchar4* colors;
  int* arena_state;  // kArena* ints
  int* counts;       // per list entry: pre-weld vertex count
  int* offsets;      // per list entry: arena offset
  const int* in_xyz;       // explicit list (device, in_count_host entries) or ...
  TrackerList todo;        // ... TSDF slots from the tracker
  int in_count_host;
  float block_size, voxel_size, min_weight, cutoff_distance_m;
  int weld;
  int* error;
};
size_t meshWeldSmemBytes();
void launchMeshCount(const MeshCtx& c, int upper, int num_sms, cudaStream_t stream);
void launchMeshScan(const MeshCtx& c, cudaStream_t stream);
void launchMeshEmit(const MeshCtx& c, int upper, int num_sms, cudaStream_t stream);
void launchMeshColor(const MeshCtx& c, int upper, int num_sms, cudaStream_t stream);
void launchMeshHeaders(const MeshCtx& c, const int* xyz_dev, int n, int* out4, cudaStream_t stream);
void launchMeshPack(const MeshCtx& c, const int* src4, const int* dst3, int n, float* v_out, float* n_out, int* t_out,
                    unsigned char* c_out, int num_sms, cudaStream_t stream);
void launchMeshCompactSizes(const MeshCtx& c, int nslots, int* sizes, cudaStream_t stream);
void launchMeshCompactMove(const MeshCtx& c, int nslots, const int* new_offsets, float* v2, float* n2, int* t2,
                           unsigned char* c2, int num_sms, cudaStream_t stream);

// nvb_util.cu
// `esdf`: the ESDF layer, whose blocks are copied out as / in from the reference's EsdfVoxel records (nvb_esdf_block.cuh)
void launchGatherBlocks(const DevLayer& layer, bool esdf, const int* xyz_dev, int n, unsigned char* out, unsigned char* found,
                        cudaStream_t stream);
void launchScatterBlocks(const DevLayer& layer, bool esdf, const int* xyz_dev, int n, const unsigned char* in, int* error,
                         cudaStream_t stream);
void launchFillU64(unsigned long long* p, unsigned long long v, size_t n, cudaStream_t stream);
// DepthPreprocessor::dilateInvalidRegionsAsync (src/sensors/depth_preprocessing.cpp); out must not alias in
void launchDilateInvalid(const float* in, float* out, int rows, int cols, int num_dilations, float threshold,
                         float invalid_value, cudaStream_t stream);
void launchRehash(const DevLayer& layer, int count, cudaStream_t stream);
// EsdfSlicer (integrators/esdf_slicer.h): AABB of the ESDF blocks at block height zb (min x, min y, max x, max y; int[4]
// preset to INT_MAX / INT_MIN), and the distance image / occupancy grid over an AABB.
void launchSliceAabb(const DevLayer& esdf, int zb, int* out4, cudaStream_t stream);
void launchSliceImage(const DevLayer& esdf, float block_size, float min_x, float min_y, float slice_height, float unobserved_value,
                      int rows, int cols, float* image, signed char* grid, cudaStream_t stream);
// the ESDF's signed distances (metres) on the voxel grid (min_vox, dims), z fastest; default_value where unknown
void launchEsdfDenseGrid(const DevLayer& esdf, int3 min_vox, int3 dims, float voxel_size, float default_value, float* out,
                         cudaStream_t stream);
void launchRemoveBlocks(const DevLayer& layer, const int4* dead, const int* dead_count, int upper, cudaStream_t stream);
void launchTodoAll(const DevLayer& tsdf, const TrackerList& t, cudaStream_t stream);
// Drops the slots that are dead in `layer` from a list of its slots (*count entries), keeping the order of the others.
void launchDropDeadSlots(const DevLayer& layer, int* list, int* count, cudaStream_t stream);

// nvb_clear.cu: map clearing (Mapper::clearOutsideRadius, ShapeClearer)
// Blocks of `layer` whose box is farther than `radius` from the centre -> dead {slot, x, y, z} (*dead_count zeroed before).
void launchSelectOutsideRadius(const DevLayer& layer, const float center[3], float radius, float block_size, int4* dead,
                               int* dead_count, cudaStream_t stream);
// BlocksToUpdateTracker::removeClearedBlocksFromTracking: zero the dirty words of the dead slots (null arrays skipped); the
// todo lists then lose them through launchDropDeadSlots.
void launchTrackerDropDead(const int4* dead, const int* dead_count, int upper, const TrackerLists& t, cudaStream_t stream);
struct ShapeClearArgs {
  DevLayer layer;
  int voxel_kind;                    // 0 TsdfVoxel, 1 OccupancyVoxel, 2 ColorVoxel
  const NvbBoundingShape* shapes;    // device
  int num_shapes;
  float block_size;
  int4* sel;                         // {slot, x, y, z} of the blocks a shape touches
  int* sel_count;
  TrackerLists tracker;
};
void launchShapeSelect(const ShapeClearArgs& a, cudaStream_t stream);
void launchShapeClear(const ShapeClearArgs& a, int num_sms, cudaStream_t stream);

// nvb_ground.cu: the ground-plane estimator (GroundPlaneEstimator, src/experimental/ground_plane/)
struct GroundExtractArgs {
  DevLayer tsdf;
  const int* slots;   // the TSDF slots below the high-water mark in (x, y, z) block-index order, free slots (-1) last
  int num_blocks;
  int2* counts;       // per listed block: {crossings, candidates}, then their exclusive prefix sums
  int* totals;        // 2 ints: all crossings, all candidates
  float3* crossings;  // emit: the crossings, in list order then voxel (x, y, z) order
  float4* candidates; // emit: the crossings with min_z <= z <= max_z (finite), {x, y, z, 0}, same order
  float block_size, voxel_size, min_tsdf_weight, min_z, max_z;
};
// keys[0, hw) / slots[0, hw): the slots below the high-water mark with their packIndex keys; sorted into keys[hw, 2 hw)
// / slots[hw, 2 hw) (a stable radix sort, cub). temp: groundSortTempBytes(hw) bytes.
size_t groundSortTempBytes(int n);
cudaError_t launchGroundSortBlocks(const DevLayer& tsdf, int hw, unsigned long long* keys, int* slots, void* temp,
                                   size_t temp_bytes, cudaStream_t stream);
void launchGroundCount(const GroundExtractArgs& a, cudaStream_t stream);  // counts + scan + totals
void launchGroundEmit(const GroundExtractArgs& a, cudaStream_t stream);
// Exclusive prefix sums of n int2 counts in place, one CTA; the two totals -> totals[0..1].
void launchExclusiveScanInt2(int2* counts, int n, int* totals, cudaStream_t stream);
void launchPackPoints(const float* xyz, int n, float4* out, cudaStream_t stream);
size_t ransacStateBytes();  // one XORWOW state
// curand_init(1234, i, 0) for the iterations first <= i < n
void launchRansacInit(void* states, int first, int n, cudaStream_t stream);
// MSAC over n >= 1 points (float4, w unused) -> out5 = {nx, ny, nz, d, found (int)}
void launchRansacFit(const float4* pts, int n, int iterations, float threshold, const void* states, float* costs,
                     float4* planes, float* out5, cudaStream_t stream);

// nvb_dynamics.cu: DynamicsDetection::computeDynamics and MaskPreprocessor::removeSmallConnectedComponents
struct DynamicsArgs {
  const float* depth;  // rows x cols, device
  int rows, cols;
  Rigid T_L_C;
  NvbCamera cam;
  DevLayer fs;          // the FreespaceLayer
  float block_size, voxel_size_inv;
  unsigned char* mask;     // rows x cols: 255 dynamic, 0 not
  unsigned char* overlay;  // rows x cols x 3 (RGB)
  int2* counts;            // per 256-pixel tile: dynamic pixels, then their exclusive prefix sums
  float* points;           // xyz of the dynamic pixels' points, in row-major pixel order
};
int dynamicsNumTiles(int pixels);
// detect + scan + emit; the number of points -> totals[0] (totals[1] is 0)
void launchDynamicsDetect(const DynamicsArgs& a, int* totals, cudaStream_t stream);
struct CcArgs {
  const unsigned char* in;  // rows x cols
  unsigned char* out;       // rows x cols (may alias `in`: the input is only read by the first pass)
  int rows, cols;
  int drows, dcols;         // rows / 2, cols / 2
  int min_size;             // components of fewer downscaled pixels are erased
  int* labels;              // drows x dcols
  int* sizes;               // drows x dcols
};
void launchRemoveSmallComponents(const CcArgs& a, int num_sms, cudaStream_t stream);

// nvb_masker.cu: ImageMasker::splitImageOnGPU (depth, with occlusion, and colour)
struct MaskerArgs {
  const float* depth;         // rows x cols, device
  int rows, cols;             // the depth camera's size
  const unsigned char* mask;  // mrows x mcols, device
  int mrows, mcols;           // the mask camera's size
  Rigid T_CM_CD;
  NvbCamera depth_cam, mask_cam;
  float occlusion_threshold_m, masked_invalid, unmasked_invalid;
  float* min_depth;           // mrows x mcols scratch
  float* unmasked;            // rows x cols: the background
  float* masked;              // rows x cols: the foreground
  unsigned char* overlay;     // rows x cols x 3 (RGB), or nullptr
};
// fill + min depth + split: three launches
void launchSplitDepth(const MaskerArgs& a, int num_sms, cudaStream_t stream);
struct ColorSplitArgs {
  const unsigned char* rgb;   // pixels x 3
  const unsigned char* mask;  // pixels
  long long pixels;
  unsigned char* unmasked;    // pixels x 3
  unsigned char* masked;      // pixels x 3
  unsigned char* overlay;     // pixels x 3, or nullptr
};
void launchSplitColor(const ColorSplitArgs& a, cudaStream_t stream);

// nvb_query.cu: point queries (VoxelBlockLayer::getVoxels, interpolation::interpolateOnCPU, nvblox_torch's sdf_query.cu)
struct QueryLayer {
  DevLayer layer;
  float block_size, voxel_size, voxel_size_inv;
};
constexpr int kMaxQueryMappers = 16;
// The mappers of one query, passed by value in the kernel's parameter space: nothing to allocate, free or keep alive while
// the launch is pending.
struct QueryLayers {
  QueryLayer l[kMaxQueryMappers];
  int n;
};
enum QueryInterpKind { kInterpTsdf = 0, kInterpEsdf = 1, kInterpOccupancy = 2 };
// out: n voxels of voxel_bytes (a multiple of 4) each, written only where found[i] = 1 (ESDF voxels as EsdfVoxel records)
void launchQueryVoxels(const QueryLayer& q, int voxel_bytes, bool esdf, const float* xyz, long long n, void* out, unsigned char* found,
                       int num_sms, cudaStream_t stream);
void launchInterpolate(const QueryLayer& q, int kind, const float* xyz, long long n, float* out, unsigned char* success,
                       int num_sms, cudaStream_t stream);
// q.n == 1 without `multi`: the single-mapper rules
void launchQueryEsdf(const QueryLayers& q, bool multi, const float* spheres_xyzr, long long n, bool with_gradient, float* out,
                     int num_sms, cudaStream_t stream);
void launchQueryTsdf(const QueryLayers& q, bool multi, const float* xyz, long long n, float* out, int num_sms,
                     cudaStream_t stream);
void launchQueryOccupancy(const QueryLayers& q, bool multi, float initial_log_odds, const float* xyz, long long n, float* out,
                          int num_sms, cudaStream_t stream);

// nvb_map_io.cu: map files (the reference's .nvblx SQLite layer cake) and the voxel-layer point export
constexpr int kMapFileLayers = 6;  // tables by NvbLayer id: tsdf, esdf, occupancy, freespace, color, then feature_layer
const char* mapFileTableName(int k);
// One layer to write: the blocks of slab slots order[0, n), xyz (3 ints) and voxels (block_bytes) indexed by slot.
struct MapFileLayerOut {
  const int* xyz;
  const unsigned char* voxels;
  const int* order;
  int n;
  int block_bytes;
};
struct PinnedFree {
  void operator()(void* p) const { cudaFreeHost(p); }
};
// One layer read: present = the file has its tables; n blocks in (x, y, z) order, their voxels in pinned memory.
struct MapFileLayerIn {
  bool present = false;
  float block_size = 0.0f;
  int n = 0;
  std::vector<int> xyz;
  std::unique_ptr<unsigned char, PinnedFree> voxels;
};
// Truncates `path` and writes the six layers' tables, one transaction per layer. NVB_OK or NVB_ERR_IO (*err says why).
int writeMapFile(const char* path, const MapFileLayerOut layers[kMapFileLayers], float block_size, std::string* err);
// Reads and validates `path`: every present layer has a positive block_size and they agree, tsdf_layer is present, and the
// tables with want[k] hold unique in-range indices with blobs of nvb_layer_block_bytes(k). Only those are read.
int readMapFile(const char* path, const bool want[kMapFileLayers], MapFileLayerIn in[kMapFileLayers], std::string* err);
// psum words of ESDF slots [0, n) from their voxels
void launchEsdfParentBoxes(const DevLayer& esdf, int n, unsigned int* psum, cudaStream_t stream);
struct ExportPointsArgs {
  DevLayer layer;
  int layer_id;       // NVB_LAYER_TSDF, _OCCUPANCY, _FREESPACE or _ESDF
  const int* slots;   // num_blocks slots in (x, y, z) block-index order, free slots (-1) last
  int num_blocks;
  int2* counts;       // per listed block: kept voxels, then their exclusive prefix sums
  int* totals;        // 2 ints: all kept voxels, 0
  float4* out;        // {x, y, z, intensity} per kept voxel
  float block_size, voxel_size;
};
void launchExportCount(const ExportPointsArgs& a, cudaStream_t stream);  // counts + scan + totals
void launchExportEmit(const ExportPointsArgs& a, cudaStream_t stream);

// nvb_esdf*.cu: the slots of EsdfCtx::stats, the last update's statistics, by what the kernels store in them. Two slots
// depend on the wavefront driver: slot 9 is CTA 0's axis-pass time in the persistent wavefront and its work time in the
// gather-replay and exchange-slab ones; slot 10 is the persistent wavefront's sweep time, 0 in the gather-replay one, and
// the exchange-slab one's single-CTA tail rings.
enum EsdfStat {
  kStatWork,                 // the update's work items
  kStatWithSites,            // blocks with sites
  kStatToClear,              // to-clear blocks
  kStatClearCandidates,      // the clear pass's candidate blocks
  kStatCleared,              // blocks on the cleared list
  kStatSwept,                // ring members swept
  kStatFaces,                // face passes
  kStatRings,
  kStatBarrierNs,            // CTA 0's wait in grid barriers
  kStatAxisNs = 9,           // persistent wavefront
  kStatWorkNs = 9,           // gather-replay and exchange-slab wavefronts
  kStatSweepNs = 10,         // persistent wavefront
  kStatTailRings = 10,       // exchange-slab wavefront
  kStatBarriers,
  kStatSlowestCtaWorkNs,     // sum over barrier phases of the slowest CTA's work time
  kStatClearBlocksRead,      // blocks the clear pass read
  kStatSplitCandidates,      // exchange-slab wavefront: candidates that fetched their own block split ...
  kStatRestFetches,          // ... and those that then fetched the rest of it
  kNumEsdfStats
};
constexpr int kPhaseMaxEntries = 4000;  // EsdfCtx::phase_max: the wavefront's per-phase debug words

// nvb_merge.cu: the state words of a merge of segments. launchUnionSegments takes them as `int* state`: declared with this
// type, nvcc's code for an unrelated ESDF kernel (nvb_esdf_wave.cu) was no longer the same from one build to the next.
struct UnionState {
  int aabb_min[3], aabb_max[3];  // the union's AABB; INT32_MAX / INT32_MIN while it is empty
  int error;                     // 1: the AABB does not fit the bitset
  int words;                     // bitset words in use
};
static_assert(sizeof(UnionState) == 8 * sizeof(int), "UnionState layout");

}  // namespace nvb
