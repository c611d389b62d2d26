// nvb_esdf_common.cuh -- small device helpers shared by the ESDF kernels.
#pragma once
#include "nvb_esdf_block.cuh"

namespace nvb {
namespace {

constexpr int kThreads = 256;
constexpr int kGroups = kThreads / 64;  // 64-thread groups, one ESDF block each
constexpr int kBlockWords = kEsdfBlockBytes / 4;  // 2560

__device__ __forceinline__ unsigned int* esdfBlockPtr(const DevLayer& L, int slot) {
  return reinterpret_cast<unsigned int*>(L.blocks + (size_t)slot * kEsdfBlockBytes);
}

// A voxel's flag word (nvb_esdf_block.cuh): byte0 is_inside, byte1 observed, byte2 is_site -- map/voxels.h:55-74.
__device__ __forceinline__ bool flagInside(unsigned int f) { return (f & 0xffu) != 0; }
__device__ __forceinline__ bool flagObserved(unsigned int f) { return (f & 0xff00u) != 0; }
__device__ __forceinline__ bool flagSite(unsigned int f) { return (f & 0xff0000u) != 0; }

__device__ __forceinline__ void loadBlockGroup(unsigned int* sm, const unsigned int* g, int lane64) {
  const uint4* src = reinterpret_cast<const uint4*>(g);
  uint4* dst = reinterpret_cast<uint4*>(sm);
#pragma unroll
  for (int k = 0; k < kBlockWords / 4 / 64; k++) dst[lane64 + k * 64] = __ldcg(src + lane64 + k * 64);
}
__device__ __forceinline__ void storeBlockGroup(unsigned int* g, const unsigned int* sm, int lane64) {
  uint4* dst = reinterpret_cast<uint4*>(g);
  const uint4* src = reinterpret_cast<const uint4*>(sm);
#pragma unroll
  for (int k = 0; k < kBlockWords / 4 / 64; k++) __stcg(dst + lane64 + k * 64, src[lane64 + k * 64]);
}

struct VoxelRegs {
  float sq;
  int p0, p1, p2;
  unsigned int fl;
};
// voxel v of a block in the layer
__device__ __forceinline__ VoxelRegs loadVoxel(const unsigned int* blk, int v) {
  const uint4 q = __ldcg(reinterpret_cast<const uint4*>(esdfCell(blk, v)));
  VoxelRegs r;
  r.sq = __uint_as_float(q.x);
  r.p0 = (int)q.y, r.p1 = (int)q.z, r.p2 = (int)q.w;
  r.fl = __ldcg(esdfFlag(blk, v));
  return r;
}
// updateSingleNeighbor (:602-633): src -> dst (voxel v_nb of the block blk_nb) across a face; `direction` is the
// block direction from src to dst along `axis`.
__device__ __forceinline__ bool updateSingleNeighbor(const VoxelRegs& e, VoxelRegs& nb, unsigned int* blk_nb, int v_nb, int axis,
                                                     int direction, float max_sq) {
  if (!flagObserved(e.fl) || !flagObserved(nb.fl) || flagSite(nb.fl) || e.sq >= max_sq) return false;
  int d0 = e.p0, d1 = e.p1, d2 = e.p2;
  if (axis == 0) d0 -= direction;
  else if (axis == 1) d1 -= direction;
  else d2 -= direction;
  const float pdist = (float)(d0 * d0 + (d1 * d1 + d2 * d2));
  if (nb.sq > pdist) {
    nb.p0 = d0, nb.p1 = d1, nb.p2 = d2, nb.sq = pdist;
    __stcg(reinterpret_cast<uint4*>(esdfCell(blk_nb, v_nb)), make_uint4(__float_as_uint(pdist), (unsigned)d0, (unsigned)d1, (unsigned)d2));
    return true;
  }
  return false;
}

// A newly allocated ESDF block is linked with its neighbours in both directions: the six face neighbours
// (c.nbr) and the whole 3x3x3 neighbourhood (c.nbr27). Replaces the per-ring getBlockPtr hash lookups
// (esdf_integrator.cu:1100-1131). Threads 0..26 of the calling CTA take one offset each.
__device__ __forceinline__ void linkNewBlock(const EsdfCtx& c, int slot, int tid) {
  if (tid >= 27) return;
  const int dx = tid / 9 - 1, dy = (tid / 3) % 3 - 1, dz = tid % 3 - 1;
  const int* bi = c.esdf.block_index + 3 * slot;
  const int other = (tid == 13) ? slot : hashFind(c.esdf.hash, bi[0] + dx, bi[1] + dy, bi[2] + dz);
  c.nbr27[27 * slot + tid] = other;
  if (other >= 0) c.nbr27[27 * other + (26 - tid)] = slot;
  // face neighbours: c.nbr order is +x,-x,+y,-y,+z,-z
  const int nz = (dx != 0) + (dy != 0) + (dz != 0);
  if (nz == 1) {
    const int axis = dx ? 0 : (dy ? 1 : 2);
    const int neg = (dx + dy + dz) < 0 ? 1 : 0;
    c.nbr[6 * slot + axis * 2 + neg] = other;
    if (other >= 0) c.nbr[6 * other + axis * 2 + (neg ^ 1)] = slot;
  }
}

__device__ __forceinline__ long long globalTimerNs() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)::"memory");
  return t;
}

__device__ __forceinline__ void gridBarrier(unsigned int* bar, unsigned int& generation, unsigned int nctas) {
  __syncthreads();
  if (threadIdx.x == 0) {
    generation++;
    const unsigned int target = generation * nctas;
    __threadfence();
    atomicAdd(bar, 1u);
    while (*(volatile unsigned int*)bar < target) {
    }
    __threadfence();
  }
  __syncthreads();
}


}  // namespace
}  // namespace nvb
