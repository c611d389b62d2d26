// nvb_esdf.cu -- incremental ESDF update from the TSDF layer.
//
// Replaces EsdfIntegrator::integrateBlocks(TsdfLayer, blocks, EsdfLayer*)
// (nvblox/src/integrators/esdf_integrator.cu:220-266) and its kernels
// markAllSitesKernel (:467-540), clearAllInvalidKernel (:1522-1585),
// sweepBlockBandKernel (:1390-1431), getBlockPtr/updateNeighborBandsKernel
// (:1100-1183) and sortUniqueKernel (:1187-1280).
//
// The reference's result depends on the ORDER of its passes (in-block x->y->z
// sweeps; face propagation +x,-x,+y,-y,+z,-z, each pass seeing the previous
// ones; repeat until no block changes), so that order is kept. What changes:
//   * everything is driven from device-side lists and counters: no host hash,
//     no D2H of counters per ring, no host scan of all block indices;
//   * blocks move through shared memory with 128-bit coalesced accesses (the
//     reference walks 20-byte AoS voxels straight in global memory);
//   * the +dir / -dir passes of one axis are fused per block INTERFACE: the two
//     operations on an interface only touch that interface's two faces and keep
//     their relative order inside one thread, so the six passes need three
//     grid-wide phases instead of six launches;
//   * the "updated blocks" list of a ring is built unique with a per-slot stamp
//     (atomicExch), which replaces the sort + unique launch;
//   * the whole wavefront (both computeEsdf calls) runs in ONE cooperative
//     persistent launch with a grid barrier between phases.
#include "nvb_esdf_common.cuh"
#include "nvb_tma.cuh"

#include <cstdlib>

namespace nvb {

namespace {

// To-clear bitmap for the clear pass's pruning (esdfClearKernel): 64 x 32 columns x 32 layers of block indices, folded
// (x mod 64, y mod 32, z mod 32): no origin to agree on, so every mark CTA sets the bits of its own to-clear blocks while it
// runs; two blocks that alias (25.6 m x 12.8 m x 12.8 m apart at 5 cm voxels) only cost an unnecessary read. Zeroed by the
// allocate kernel of the update.
constexpr int kClearBitWords = 2048;
__device__ __forceinline__ int clearBitWord(int x, int y) { return ((x & 63) << 5) | (y & 31); }

// Per-update reset of the counters, the statistics and the to-clear bitmap, over the grid of an allocate kernel
// (n = the update's work items).
__device__ __forceinline__ void resetEsdfUpdate(const EsdfCtx& c, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    *c.work_count = n;
    *c.upd_count = 0;
    *c.clr_count = 0;
    c.clr_aabb[0] = c.clr_aabb[1] = c.clr_aabb[2] = INT32_MAX;
    c.clr_aabb[3] = c.clr_aabb[4] = c.clr_aabb[5] = INT32_MIN;
    c.ring_count[0] = c.ring_count[1] = 0;
    c.ring_count[2] = 0;  // mark-kernel "CTAs done" counter
    c.ges_counts[0] = c.ges_counts[1] = c.ges_counts[2] = c.ges_counts[3] = 0;
    *c.barrier = 0;
    for (int k = 0; k < kNumEsdfStats; k++) c.stats[k] = 0;
    c.stats[kStatWork] = n;
  }
  for (int q = i; q < kPhaseMaxEntries; q += gridDim.x * blockDim.x) c.phase_max[q] = 0ull;
  if (c.clr_bits)
    for (int q = i; q < kClearBitWords; q += gridDim.x * blockDim.x) c.clr_bits[q] = 0u;
}

// ---------------------------------------------------------------------------
// Allocation of the ESDF blocks + per-update counter reset
// (EsdfIntegrator::allocateBlocksOnCPU, esdf_integrator.cu:391-397).
// ---------------------------------------------------------------------------
__global__ void esdfAllocateKernel(EsdfCtx c, const int* in_xyz, const int* in_slots, const int* in_count_dev,
                                   int in_count_host) {
  const int n = in_count_dev ? *in_count_dev : in_count_host;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  resetEsdfUpdate(c, n);
  if (i >= n) return;
  int x, y, z, tslot;
  if (in_slots) {
    tslot = in_slots[i];
    if (c.tracker_dirty) c.tracker_dirty[tslot] = 0;  // this block's pending update is being consumed
    x = c.tsdf.block_index[3 * tslot], y = c.tsdf.block_index[3 * tslot + 1], z = c.tsdf.block_index[3 * tslot + 2];
  } else {
    x = in_xyz[3 * i], y = in_xyz[3 * i + 1], z = in_xyz[3 * i + 2];
    tslot = hashFind(c.tsdf.hash, x, y, z);
  }
  bool was_new;
  const int eslot = hashFindOrInsert(c.esdf, x, y, z, c.error, &was_new);
  // isVoxelFreespace (:101-111): the freespace twin, if the mapper has a freespace layer and the block exists there
  const int fslot = c.use_freespace ? hashFind(c.freespace.hash, x, y, z) : -1;
  c.work[i] = make_int4(eslot, tslot, was_new ? 1 : 0, fslot);
}

// Per-CTA bookkeeping of the mark kernels: which of this CTA's blocks have sites / lost sites, and the AABB of the
// latter. Kept in shared memory and published once per CTA (two atomicAdds + six atomicMin/Max per CTA instead of
// per block: the returning atomics are dependent L2 round trips on thread 0's critical path).
constexpr int kMarkLocalMax = 64;
struct MarkLocal {
  int upd[kMarkLocalMax];
  int clr[kMarkLocalMax];
  int nu, nc;
  int aabb[6];
};
__device__ __forceinline__ void markLocalInit(MarkLocal& ml) {
  ml.nu = ml.nc = 0;
  ml.aabb[0] = ml.aabb[1] = ml.aabb[2] = INT32_MAX;
  ml.aabb[3] = ml.aabb[4] = ml.aabb[5] = INT32_MIN;
}
// thread 0 only
__device__ __forceinline__ void markLocalFlush(const EsdfCtx& c, MarkLocal& ml) {
  if (ml.nu) {
    const int base = atomicAdd(c.upd_count, ml.nu);
    for (int i = 0; i < ml.nu; i++) c.upd_list[base + i] = ml.upd[i];
  }
  if (ml.nc) {
    const int base = atomicAdd(c.clr_count, ml.nc);
    for (int i = 0; i < ml.nc; i++) c.clr_list[base + i] = ml.clr[i];
    atomicMin(c.clr_aabb + 0, ml.aabb[0]), atomicMin(c.clr_aabb + 1, ml.aabb[1]), atomicMin(c.clr_aabb + 2, ml.aabb[2]);
    atomicMax(c.clr_aabb + 3, ml.aabb[3]), atomicMax(c.clr_aabb + 4, ml.aabb[4]), atomicMax(c.clr_aabb + 5, ml.aabb[5]);
  }
  markLocalInit(ml);
}
// thread 0 only; bi = the block's index if the caller already has it, else nullptr
__device__ __forceinline__ void markLocalRecord(const EsdfCtx& c, MarkLocal& ml, int slot, bool updated, bool cleared,
                                                const int* bi_known = nullptr) {
  if (updated) {
    if (ml.nu == kMarkLocalMax) markLocalFlush(c, ml);
    ml.upd[ml.nu++] = slot;
    c.seed_upd[slot] = c.update_seq;
  }
  if (cleared) {
    if (ml.nc == kMarkLocalMax) markLocalFlush(c, ml);
    ml.clr[ml.nc++] = slot;
    const int* bi = bi_known ? bi_known : c.esdf.block_index + 3 * slot;
    const int x = bi[0], y = bi[1], z = bi[2];
    ml.aabb[0] = min(ml.aabb[0], x), ml.aabb[1] = min(ml.aabb[1], y), ml.aabb[2] = min(ml.aabb[2], z);
    ml.aabb[3] = max(ml.aabb[3], x), ml.aabb[4] = max(ml.aabb[4], y), ml.aabb[5] = max(ml.aabb[5], z);
    if (c.clr_bits) atomicOr(c.clr_bits + clearBitWord(x, y), 1u << (z & 31));
  }
}

// The persistent cleared list at the end of the mark pass (last CTA, one thread). If this update has blocks to
// clear the list is about to be rewritten (clearAllInvalid resizes it, :1620); otherwise it keeps the previous
// call's content (:242-257). The reference keeps block INDICES, so an entry whose block was deallocated (decay
// integrators) and allocated again counts again: such indices wait in dead_cleared_xyz and rejoin here.
__device__ __forceinline__ void updatePersistentClearedList(const EsdfCtx& c, int nclr) {
  if (nclr > 0) {
    *c.cleared_count = 0;
    *c.cleared_seq = c.update_seq;
    if (c.dead_cleared_count) *c.dead_cleared_count = 0;
    return;
  }
  if (!c.dead_cleared_count) return;
  int nd = *c.dead_cleared_count;
  for (int i = 0; i < nd;) {
    const int slot = hashFind(c.esdf.hash, c.dead_cleared_xyz[3 * i], c.dead_cleared_xyz[3 * i + 1], c.dead_cleared_xyz[3 * i + 2]);
    if (slot >= 0) {
      c.cleared_list[(*c.cleared_count)++] = slot;
      c.seed_clr[slot] = *c.cleared_seq;
      nd--;
      c.dead_cleared_xyz[3 * i] = c.dead_cleared_xyz[3 * nd], c.dead_cleared_xyz[3 * i + 1] = c.dead_cleared_xyz[3 * nd + 1],
                          c.dead_cleared_xyz[3 * i + 2] = c.dead_cleared_xyz[3 * nd + 2];
    } else {
      i++;
    }
  }
  *c.dead_cleared_count = nd;
}

// Start of a mark kernel: thread 0 empties the CTA's lists, CTA 0 marks the tracker's to-do list consumed (the allocate
// kernel has read it). Returns the number of work items.
__device__ __forceinline__ int markBegin(const EsdfCtx& c, MarkLocal& ml) {
  if (threadIdx.x == 0) markLocalInit(ml);
  const int n = *c.work_count;
  if (blockIdx.x == 0 && threadIdx.x == 0 && c.tracker_todo_count) *c.tracker_todo_count = 0;
  return n;
}

// End of a mark kernel (thread 0, after the CTA's last write-back): publish the CTA's lists; the last CTA out updates the
// persistent cleared list and writes the update's block counts.
__device__ __forceinline__ void markFinish(const EsdfCtx& c, MarkLocal& ml) {
  markLocalFlush(c, ml);
  __threadfence();
  if (atomicAdd(c.ring_count + 2, 1) == (int)gridDim.x - 1) {
    __threadfence();
    const int nclr = *(volatile int*)c.clr_count;
    const int nupd = *(volatile int*)c.upd_count;
    updatePersistentClearedList(c, nclr);
    c.stats[kStatWithSites] = nupd, c.stats[kStatToClear] = nclr;
  }
}

// ---------------------------------------------------------------------------
// updateEsdfVoxelToChanges (esdf_integrator.cu:401-460) on voxel v of an ESDF block, in shared or global memory.
// Sets `updated` if the voxel is a site and `cleared` if it lost its site or inside status (or is unobserved); returns
// whether a word changed.
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool updateVoxelToChanges(unsigned int* blk, int v, bool is_observed, bool is_inside, bool is_site,
                                                     float max_sq, bool& updated, bool& cleared) {
  unsigned int* e = esdfCell(blk, v);
  unsigned int* f = esdfFlag(blk, v);
  float sq = __uint_as_float(e[0]);
  int p0 = (int)e[1], p1 = (int)e[2], p2 = (int)e[3];
  const unsigned int fl = *f;
  bool e_inside = flagInside(fl), e_observed = flagObserved(fl), e_site = flagSite(fl);
  if (is_observed) {
    if (e_inside && !is_inside) {
      p0 = p1 = p2 = 0, sq = max_sq, e_site = false;
      cleared = true;
    }
    e_inside = is_inside;
    if (is_site) {
      if (!e_site) e_site = true, sq = 0.0f, p0 = p1 = p2 = 0;
      updated = true;
    } else if (e_site) {
      p0 = p1 = p2 = 0, sq = max_sq, e_site = false;
      cleared = true;
    } else if (!e_observed) {
      p0 = p1 = p2 = 0, sq = max_sq, e_site = false;
    } else if ((double)sq <= 1e-4) {
      p0 = p1 = p2 = 0, sq = max_sq, e_site = false;
      cleared = true;
    }
    e_observed = true;
  } else {
    p0 = p1 = p2 = 0, sq = max_sq, e_site = false;
    cleared = true;
    e_observed = false;
  }
  const unsigned int nfl = (fl & 0xff000000u) | (e_inside ? 1u : 0u) | (e_observed ? 0x100u : 0u) | (e_site ? 0x10000u : 0u);
  const unsigned int nsq = __float_as_uint(sq);
  if (nsq == e[0] && (unsigned)p0 == e[1] && (unsigned)p1 == e[2] && (unsigned)p2 == e[3] && nfl == fl) return false;
  e[0] = nsq, e[1] = (unsigned)p0, e[2] = (unsigned)p1, e[3] = (unsigned)p2, *f = nfl;
  return true;
}

// The site functors (TsdfSiteFunctor / OccupancySiteFunctor, :113-168): which projective voxels are observed, inside an
// object and near the surface, and how the slice squashes a voxel column (initial value :792-799, extremum
// updateSquashedExtremumAtomic). `inside` and `nearSurface` take the voxel's value, so the slice applies them to the
// squashed one.
struct TsdfSite {
  using Voxel = float2;  // {distance, weight}
  static constexpr int kBlockBytes = kTsdfBlockBytes;
  float min_weight, max_site_distance_m;
  __device__ static TsdfSite of(const EsdfCtx& c) { return {c.min_weight, c.max_site_distance_m}; }
  __device__ static float value(float2 t) { return t.x; }
  __device__ bool observed(float2 t) const { return t.y >= min_weight; }
  __device__ bool inside(float d) const { return d <= 0.0f; }
  __device__ bool nearSurface(float d) const { return fabsf(d) <= max_site_distance_m; }
  __device__ float squashInit(float max_sq) const { return 2.0f * max_sq; }
  __device__ float squash(float acc, float d) const { return fminf(acc, d); }
};
struct OccupancySite {
  using Voxel = float;  // log odds
  static constexpr int kBlockBytes = kOccBlockBytes;
  float occupied_threshold_log_odds;
  __device__ static OccupancySite of(const EsdfCtx& c) { return {c.occupied_threshold_log_odds}; }
  __device__ static float value(float lo) { return lo; }
  __device__ bool observed(float lo) const { return fabsf(lo - 0.0f) > 1e-4f; }
  __device__ bool inside(float lo) const { return lo > occupied_threshold_log_odds; }
  __device__ bool nearSurface(float) const { return true; }  // every inside voxel is a site
  __device__ float squashInit(float) const { return 0.0f; }
  __device__ float squash(float acc, float lo) const { return fmaxf(acc, lo); }
};

// One voxel of markAllSitesKernel (:467-540): "voxels being freespace can not be inside an object" (:413-415).
template <class Site>
__device__ __forceinline__ bool markVoxel(const Site& site, unsigned int* blk, int v, typename Site::Voxel t, bool is_freespace,
                                          float max_sq, bool& updated, bool& cleared) {
  const float d = Site::value(t);
  const bool is_inside = site.inside(d) & !is_freespace;
  return updateVoxelToChanges(blk, v, site.observed(t), is_inside, is_inside && site.nearSurface(d), max_sq, updated, cleared);
}

// ---------------------------------------------------------------------------
// markAllSitesKernel (:467-540) with plain staging: a CTA copies the ESDF block into shared memory, marks it there and
// writes it back if a voxel changed. Occupancy, and TSDF with a freespace layer (the TMA ring below stages the ESDF and
// TSDF blocks only).
// ---------------------------------------------------------------------------
template <class Site>
__device__ __forceinline__ void markStaged(const EsdfCtx& c, const Site site) {
  using V = typename Site::Voxel;
  __shared__ __align__(16) unsigned int s[kBlockWords];
  __shared__ int s_flags[3];  // updated, cleared, changed
  __shared__ MarkLocal ml;
  const int tid = threadIdx.x;
  const int n = markBegin(c, ml);
  for (int item = blockIdx.x; item < n; item += gridDim.x) {
    const int4 w = c.work[item];
    if (w.x >= 0 && w.z) linkNewBlock(c, w.x, tid);  // newly allocated ESDF block
    if (w.x < 0 || w.y < 0) continue;  // block_ptr == nullptr || esdf_block == nullptr (:513-517)
    if (tid < 3) s_flags[tid] = 0;
    uint4* gblk = reinterpret_cast<uint4*>(esdfBlockPtr(c.esdf, w.x));
    for (int k = tid; k < kBlockWords / 4; k += kThreads) reinterpret_cast<uint4*>(s)[k] = gblk[k];
    const V* src = reinterpret_cast<const V*>(c.tsdf.blocks + (size_t)w.y * Site::kBlockBytes);
    const V t0 = src[tid], t1 = src[tid + kThreads];
    // w.w: the block's freespace twin (-1 if there is none or the mapper has no freespace layer)
    const bool fs0 = isVoxelFreespace(c.freespace, w.w, tid), fs1 = isVoxelFreespace(c.freespace, w.w, tid + kThreads);
    __syncthreads();
    bool updated = false, cleared = false, changed = false;
#pragma unroll
    for (int h = 0; h < 2; h++)
      changed |= markVoxel(site, s, tid + h * kThreads, h ? t1 : t0, h ? fs1 : fs0, c.max_sq, updated,
                           cleared);
    if (updated) s_flags[0] = 1;
    if (cleared) s_flags[1] = 1;
    if (changed) s_flags[2] = 1;
    __syncthreads();
    if (s_flags[2]) {
      for (int k = tid; k < kBlockWords / 4; k += kThreads) gblk[k] = reinterpret_cast<uint4*>(s)[k];
    }
    if (tid == 0) markLocalRecord(c, ml, w.x, s_flags[0] != 0, s_flags[1] != 0);
    __syncthreads();
  }
  if (tid == 0) markFinish(c, ml);
}
// Five resident CTAs per SM, i.e. at most 48 registers: without the bound ptxas gives these two 60-64 and one CTA less.
__global__ void __launch_bounds__(kThreads, 5) esdfMarkKernel(EsdfCtx c) { markStaged(c, TsdfSite::of(c)); }
__global__ void __launch_bounds__(kThreads, 5) esdfMarkOccupancyKernel(EsdfCtx c) { markStaged(c, OccupancySite::of(c)); }

// ---------------------------------------------------------------------------
// markAllSites with TMA staging, for TSDF without freespace. Same voxel rule as esdfMarkKernel; what
// changes is how blocks move: one elected thread issues cp.async.bulk copies (SASS UBLKCP)
// of the 10 KiB ESDF block and the 4 KiB TSDF block into a 3-stage shared-memory ring,
// completion is tracked by an mbarrier per stage (expect_tx = 14 336 B), the block is updated
// in place in shared memory and goes back with one bulk store. Loads of the next two work
// items are in flight while the current one is processed, so a persistent CTA keeps
// ~28 KiB outstanding without spending registers or LSU slots on it.
// The rule is written out in this kernel instead of calling markVoxel: with the call, ptxas
// allocates the kernel differently (32 registers instead of 46), and the C2 bench's mark stage
// took ~3 us per frame longer (one H100 SXM, 400 W power limit: 40.3 - 41.6 against
// 37.2 - 38.2 us). Any change to updateVoxelToChanges has to be made here too; the parity
// tests pin both to the oracle.
// ---------------------------------------------------------------------------
constexpr int kMarkStages = 3;
struct __align__(128) MarkStage {
  unsigned int esdf[kBlockWords];     // 10 240 B
  float2 tsdf[kVpb];                  //  4 096 B
};
constexpr unsigned int kMarkStageTxBytes = kEsdfBlockBytes + kTsdfBlockBytes;

__global__ void __launch_bounds__(kThreads) esdfMarkTmaKernel(EsdfCtx c) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  MarkStage* st = reinterpret_cast<MarkStage*>(smem_raw);
  __shared__ __align__(8) uint64_t s_bar[kMarkStages];
  __shared__ int4 s_work[kMarkStages];
  __shared__ int s_flags[3];  // updated, cleared, changed
  __shared__ int s_bi[3];
  __shared__ MarkLocal ml;
  const int tid = threadIdx.x;
  const int n = markBegin(c, ml);
  const int my_count = (n > (int)blockIdx.x) ? (n - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  if (tid == 0) {
    for (int s = 0; s < kMarkStages; s++) tma::mbarInit(&s_bar[s], 1);
    tma::fenceBarrierInit();
  }
  __syncthreads();
  // producer (thread 0): stage the blocks of this CTA's j-th work item
  auto issue = [&](int j) {
    const int s = j % kMarkStages;
    const int4 w = c.work[blockIdx.x + j * gridDim.x];
    s_work[s] = w;
    if (w.x >= 0 && w.y >= 0) {
      tma::mbarArriveExpectTx(&s_bar[s], kMarkStageTxBytes);
      tma::bulkLoad(st[s].esdf, c.esdf.blocks + (size_t)w.x * kEsdfBlockBytes, kEsdfBlockBytes, &s_bar[s]);
      tma::bulkLoad(st[s].tsdf, c.tsdf.blocks + (size_t)w.y * kTsdfBlockBytes, kTsdfBlockBytes, &s_bar[s]);
    } else {
      tma::mbarArrive(&s_bar[s]);  // nothing to load: complete the phase
    }
  };
  if (tid == 0) {
    for (int j = 0; j < kMarkStages - 1 && j < my_count; j++) issue(j);
  }
  __syncthreads();
  for (int j = 0; j < my_count; j++) {
    const int s = j % kMarkStages;
    if (tid == 0 && j + kMarkStages - 1 < my_count) {
      // stage (j-1) % S is about to be refilled: its bulk store must have finished reading it
      tma::bulkWaitRead<0>();
      issue(j + kMarkStages - 1);
    }
    tma::mbarWait(&s_bar[s], (unsigned int)((j / kMarkStages) & 1));
    const int4 w = s_work[s];
    // the block's index, for the to-clear AABB: fetched now so that thread 0 does not wait for it at the end of the item
    if (tid >= 32 && tid < 35 && w.x >= 0) s_bi[tid - 32] = c.esdf.block_index[3 * w.x + (tid - 32)];
    if (w.x >= 0 && w.z) linkNewBlock(c, w.x, tid);  // newly allocated ESDF block
    const bool valid = (w.x >= 0 && w.y >= 0);  // block_ptr == nullptr || esdf_block == nullptr (:513-517)
    if (tid < 3) s_flags[tid] = 0;
    __syncthreads();
    if (valid) {
      unsigned int* sblk = st[s].esdf;
      bool updated = false, cleared = false, changed = false;
      // updateVoxelToChanges with TsdfSite, written out: see above
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const float2 t = st[s].tsdf[tid + h * kThreads];
        unsigned int* e = esdfCell(sblk, tid + h * kThreads);
        unsigned int* f = esdfFlag(sblk, tid + h * kThreads);
        float sq = __uint_as_float(e[0]);
        int p0 = (int)e[1], p1 = (int)e[2], p2 = (int)e[3];
        const unsigned int fl = *f;
        bool e_inside = flagInside(fl), e_observed = flagObserved(fl), e_site = flagSite(fl);
        const bool is_observed = t.y >= c.min_weight;
        if (is_observed) {
          const bool is_inside = t.x <= 0.0f;
          const bool is_site = is_inside && (fabsf(t.x) <= c.max_site_distance_m);
          if (e_inside && !is_inside) {
            p0 = p1 = p2 = 0, sq = c.max_sq, e_site = false;
            cleared = true;
          }
          e_inside = is_inside;
          if (is_site) {
            if (!e_site) {
              e_site = true, sq = 0.0f, p0 = p1 = p2 = 0;
            }
            updated = true;
          } else {
            if (e_site) {
              p0 = p1 = p2 = 0, sq = c.max_sq, e_site = false;
              cleared = true;
            } else if (!e_observed) {
              p0 = p1 = p2 = 0, sq = c.max_sq, e_site = false;
            } else if ((double)sq <= 1e-4) {
              p0 = p1 = p2 = 0, sq = c.max_sq, e_site = false;
              cleared = true;
            }
          }
          e_observed = true;
        } else {
          p0 = p1 = p2 = 0, sq = c.max_sq, e_site = false;
          cleared = true;
          e_observed = false;
        }
        const unsigned int nfl = (fl & 0xff000000u) | (e_inside ? 1u : 0u) | (e_observed ? 0x100u : 0u) |
                                 (e_site ? 0x10000u : 0u);
        const unsigned int nsq = __float_as_uint(sq);
        if (nsq != e[0] || (unsigned)p0 != e[1] || (unsigned)p1 != e[2] || (unsigned)p2 != e[3] || nfl != fl) {
          e[0] = nsq, e[1] = (unsigned)p0, e[2] = (unsigned)p1, e[3] = (unsigned)p2, *f = nfl;
          changed = true;
        }
      }
      if (updated) s_flags[0] = 1;
      if (cleared) s_flags[1] = 1;
      if (changed) s_flags[2] = 1;
      tma::fenceProxyAsyncShared();  // this thread's smem writes -> visible to the bulk store
    }
    __syncthreads();
    if (valid && tid == 0) {
      if (s_flags[2]) {
        tma::bulkStore(c.esdf.blocks + (size_t)w.x * kEsdfBlockBytes, st[s].esdf, kEsdfBlockBytes);
        tma::bulkCommit();
      }
      markLocalRecord(c, ml, w.x, s_flags[0] != 0, s_flags[1] != 0, s_bi);
    }
    __syncthreads();
  }
  if (tid == 0) {
    tma::bulkWait<0>();  // all write-backs performed before this CTA reports "done"
    markFinish(c, ml);
  }
}

// ---------------------------------------------------------------------------
// clearAllInvalid (:1587-1647): candidate = every ESDF block whose box is within
// max_esdf_distance of the AABB of the to-clear blocks
// (geometry/bounding_spheres.cpp:76-91, bounding_boxes.cpp:20-27);
// clearAllInvalidKernel (:1522-1585) per candidate.
// ---------------------------------------------------------------------------
constexpr int kClearMaxCand = 256;  // candidates of one CTA per selection round
__device__ __forceinline__ void clearPrefetch(const EsdfCtx& c, unsigned int* sblk, int* snb, int slot, int tid) {
  const unsigned char* g = c.esdf.blocks + (size_t)slot * kEsdfBlockBytes;
  for (int k = tid; k < kBlockWords / 4; k += kThreads) {
    const unsigned int d = (unsigned int)__cvta_generic_to_shared(sblk + 4 * k);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(g + 16 * k) : "memory");
  }
  if (tid < 27) {  // the 3x3x3 block neighbourhood (most parents live there): one row of the neighbour table
    const unsigned int d = (unsigned int)__cvta_generic_to_shared(snb + tid);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(c.nbr27 + 27 * slot + tid) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// Selection and candidate processing in one kernel: a CTA reads the candidates among its own slots (their number per CTA is
// Poisson-distributed, ~2 on average and 7-8 on the unluckiest of 1184 CTAs, which sets the kernel's time).
// Five resident CTAs per SM, i.e. at most 48 registers: without the bound ptxas gives this kernel 64 and one CTA less.
__global__ void __launch_bounds__(kThreads, 5) esdfClearKernel(EsdfCtx c) {
  __shared__ __align__(16) unsigned int s_blk[2][kBlockWords];
  __shared__ int s_nb[2][32];
  __shared__ int s_cand[kClearMaxCand];
  __shared__ int s_done[kClearMaxCand];
  __shared__ int s_ncand, s_ndone, s_any;
  const int nclr = *c.clr_count;
  if (nclr == 0) return;
  const int tid = threadIdx.x, lane = tid & 31;
  const int nblocks = *c.esdf.count < c.esdf.capacity ? *c.esdf.count : c.esdf.capacity;
  const float bs = c.block_size;
  float amin[3], amax[3];
  int ia[3], ib[3];  // the to-clear AABB in block indices
#pragma unroll
  for (int a = 0; a < 3; a++) {
    ia[a] = c.clr_aabb[a], ib[a] = c.clr_aabb[3 + a];
    amin[a] = (float)ia[a] * bs;
    amax[a] = ((float)ib[a] + 1.0f) * bs;
  }
  // Pruning (c.prune): a voxel is cleared iff its parent voxel is no longer a site, and sites are only lost in the to-clear
  // blocks; c.psum[slot] bounds the block offsets the parents of the block's voxels point into. A candidate is only READ if that
  // box (clipped to the to-clear AABB) contains a to-clear block: tested against the folded bitmap the mark kernel filled.
  const bool use_bits = c.prune && c.clr_bits != nullptr;
  long long ncand_total = 0, nread_total = 0;
  // Slots are dealt round-robin over the CTAs (recently allocated = high slots are the likely candidates);
  // one selection round tests 256 of this CTA's slots at once, one thread per slot.
  for (long long first = (long long)blockIdx.x; first < (long long)nblocks; first += (long long)gridDim.x * kThreads) {
    if (tid == 0) s_ncand = 0, s_ndone = 0;
    __syncthreads();
    const long long slot_ll = first + (long long)tid * gridDim.x;
    bool is_cand = false, ref_cand = false;
    if (slot_ll < nblocks && c.esdf.block_index[3 * slot_ll] != kDeadSlotX) {
      const int* bi = c.esdf.block_index + 3 * slot_ll;
      const int b3[3] = {bi[0], bi[1], bi[2]};
      // AlignedBox::exteriorDistance(box) > radius -> skip
      float d2 = 0.0f;
#pragma unroll
      for (int a = 0; a < 3; a++) {
        const float lo = (float)b3[a] * bs, hi = ((float)b3[a] + 1.0f) * bs;
        if (amin[a] > hi) {
          const float aux = amin[a] - hi;
          d2 += aux * aux;
        } else if (lo > amax[a]) {
          const float aux = lo - amax[a];
          d2 += aux * aux;
        }
      }
      is_cand = !(sqrtf(d2) > c.max_esdf_distance_m);
      if (is_cand && c.prune) {
        // union of the two half-block boxes (one word per warp of the storing group)
        const uint2 pw = __ldg(reinterpret_cast<const uint2*>(c.psum) + slot_ll);
        if (pw.x == 0u && pw.y == 0u) {
          is_cand = false, ref_cand = true;  // no voxel of the block has a parent
        } else if (pw.x != 0xffffffffu && pw.y != 0xffffffffu) {
          ref_cand = true;
          int lo[3], hi[3];
          bool hit = true;
#pragma unroll
          for (int a = 0; a < 3; a++) {
            int l = 99, h = -99;
            if (pw.x) l = (int)((pw.x >> (10 * a)) & 31u) - 16, h = (int)((pw.x >> (10 * a + 5)) & 31u) - 16;
            if (pw.y) l = min(l, (int)((pw.y >> (10 * a)) & 31u) - 16), h = max(h, (int)((pw.y >> (10 * a + 5)) & 31u) - 16);
            lo[a] = b3[a] + l, hi[a] = b3[a] + h;
            lo[a] = lo[a] > ia[a] ? lo[a] : ia[a], hi[a] = hi[a] < ib[a] ? hi[a] : ib[a];
            hit = hit && lo[a] <= hi[a];
          }
          if (hit && use_bits) {
            unsigned int zmask = 0xffffffffu;  // z layers lo..hi, folded mod 32
            if (hi[2] - lo[2] < 31) {
              const unsigned int m = (1u << (hi[2] - lo[2] + 1)) - 1u;
              const int sh = lo[2] & 31;
              zmask = (m << sh) | (sh ? (m >> (32 - sh)) : 0u);
            }
            hit = false;
            for (int x = lo[0]; x <= hi[0] && !hit; x++)
              for (int y = lo[1]; y <= hi[1]; y++)
                if (__ldg(c.clr_bits + clearBitWord(x, y)) & zmask) {
                  hit = true;
                  break;
                }
          }
          is_cand = hit;
        }
      }
      ref_cand = ref_cand || is_cand;
    }
    // (the statistics count the reference's candidates; `is_cand` decides what is read)
    const unsigned int ref_ballot = __ballot_sync(0xffffffffu, ref_cand);
    const unsigned int ballot = __ballot_sync(0xffffffffu, is_cand);
    int wbase = 0;
    if (lane == 0 && ballot) wbase = atomicAdd(&s_ncand, __popc(ballot));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (is_cand) s_cand[wbase + __popc(ballot & ((1u << lane) - 1u))] = (int)slot_ll;
    if (lane == 0) ncand_total += __popc(ref_ballot);
    __syncthreads();
    const int ncand = s_ncand;
    if (tid == 0) nread_total += ncand;
    // Candidates one after the other; the next one's block and neighbour row are already on their way.
    if (ncand > 0) clearPrefetch(c, s_blk[0], s_nb[0], s_cand[0], tid);
    for (int i = 0; i < ncand; i++) {
      const int buf = i & 1;
      const int slot = s_cand[i];
      if (i + 1 < ncand) {
        clearPrefetch(c, s_blk[buf ^ 1], s_nb[buf ^ 1], s_cand[i + 1], tid);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      if (tid == 0) s_any = 0;
      __syncthreads();
      const unsigned int* s = s_blk[buf];
      const int* nbrow = s_nb[buf];
      unsigned int* gw = esdfBlockPtr(c.esdf, slot);
      const int bx = c.esdf.block_index[3 * slot], by = c.esdf.block_index[3 * slot + 1], bz = c.esdf.block_index[3 * slot + 2];
      bool any = false;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int v = tid + h * kThreads;
        const unsigned int* e = esdfCell(s, v);
        const unsigned int fl = *esdfFlag(s, v);
        const int p[3] = {(int)e[1], (int)e[2], (int)e[3]};
        if (flagObserved(fl) && !flagSite(fl) && (p[0] != 0 || p[1] != 0 || p[2] != 0)) {
          // getBlockAndVoxelIndexFromOffset (:1498-1520): C++ '/' and '%' truncate toward zero.
          const int vi[3] = {v >> 6, (v >> 3) & 7, v & 7};
          // The reference splits p with truncating '/' and '%' and then carries nv back into [0, 8): the result is the floor
          // division of vi + p by 8 (8 nb + nv = vi + p with 0 <= nv < 8 has one solution), i.e. a shift and a mask.
          int nb[3], nv[3];
#pragma unroll
          for (int a = 0; a < 3; a++) {
            const int q = vi[a] + p[a];
            nb[a] = q >> 3;  // block offset (relative)
            nv[a] = q & (kVps - 1);
          }
          const int pv = (nv[0] * kVps + nv[1]) * kVps + nv[2];
          bool parent_is_site = false;
          if (nb[0] == 0 && nb[1] == 0 && nb[2] == 0) {
            parent_is_site = flagSite(*esdfFlag(s, pv));
          } else {
            int ps = -2;
            if (nb[0] >= -1 && nb[0] <= 1 && nb[1] >= -1 && nb[1] <= 1 && nb[2] >= -1 && nb[2] <= 1)
              ps = nbrow[(nb[0] + 1) * 9 + (nb[1] + 1) * 3 + (nb[2] + 1)];
            if (ps < -1) ps = hashFind(c.esdf.hash, bx + nb[0], by + nb[1], bz + nb[2]);  // far parent / row never linked
            // is_site is never written by this kernel: reading it from a block another
            // CTA is processing is race-free.
            if (ps >= 0) parent_is_site = flagSite(__ldcg(esdfFlag(esdfBlockPtr(c.esdf, ps), pv)));
          }
          if (!parent_is_site) {
            unsigned int* g = esdfCell(gw, v);
            g[0] = __float_as_uint(c.max_sq), g[1] = 0u, g[2] = 0u, g[3] = 0u;
            any = true;
          }
        }
      }
      if (any) s_any = 1;
      __syncthreads();
      if (tid == 0 && s_any) {
        s_done[s_ndone++] = slot;
        c.seed_clr[slot] = c.update_seq;
      }
      // (the next iteration's __syncthreads orders s_any / the buffers)
    }
    __syncthreads();
    // publish this round's cleared blocks: one atomicAdd per CTA
    if (s_ndone > 0) {
      __shared__ int s_base;
      if (tid == 0) s_base = atomicAdd(c.cleared_count, s_ndone);
      __syncthreads();
      for (int i = tid; i < s_ndone; i += kThreads) c.cleared_list[s_base + i] = s_done[i];
    }
    __syncthreads();
  }
  if (lane == 0 && ncand_total) atomicAdd((unsigned long long*)&c.stats[kStatClearCandidates], (unsigned long long)ncand_total);
  if (tid == 0 && nread_total) atomicAdd((unsigned long long*)&c.stats[kStatClearBlocksRead], (unsigned long long)nread_total);
}

// ---------------------------------------------------------------------------
// Phases of computeEsdf (:1465-1496), written as device functions over
// (cta, num_ctas) so the persistent kernel and the per-phase kernels share them.
// ---------------------------------------------------------------------------

// sweepSingleBand (:542-600): forward then backward along one line of 8 voxels.
__device__ __forceinline__ bool sweepLine(unsigned int* s, int c0, int c1, int c2, int axis, float max_sq) {
  const int stride = (axis == 0) ? 64 : ((axis == 1) ? 8 : 1);
  const int basev = c0 * 64 + c1 * 8 + c2;  // coordinate along `axis` is 0 on entry
  bool changed = false;
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
    int l0 = 0, l1 = 0, l2 = 0;
    bool found = false;
#pragma unroll
    for (int k = 0; k < kVps; k++) {
      const int cc = pass ? (kVps - 1 - k) : k;
      unsigned int* e = esdfCell(s, basev + cc * stride);
      const unsigned int fl = *esdfFlag(s, basev + cc * stride);
      if (!flagObserved(fl)) continue;
      const int v0 = (axis == 0) ? cc : c0, v1 = (axis == 1) ? cc : c1, v2 = (axis == 2) ? cc : c2;
      if (flagSite(fl)) {
        l0 = v0, l1 = v1, l2 = v2;
        found = true;
      } else if (!found) {
        if (__uint_as_float(e[0]) < max_sq) {
          found = true;
          l0 = (int)e[1] + v0, l1 = (int)e[2] + v1, l2 = (int)e[3] + v2;
        }
      } else {
        const int d0 = l0 - v0, d1 = l1 - v1, d2 = l2 - v2;
        const float pdist = (float)(d0 * d0 + (d1 * d1 + d2 * d2));
        const float sq = __uint_as_float(e[0]);
        if (sq > pdist) {
          e[1] = (unsigned)d0, e[2] = (unsigned)d1, e[3] = (unsigned)d2;
          e[0] = __float_as_uint(pdist);
          changed = true;
        } else if (sq < max_sq) {
          l0 = (int)e[1] + v0, l1 = (int)e[2] + v1, l2 = (int)e[3] + v2;
        }
      }
    }
  }
  return changed;
}

// sweepBlockBandKernel (:1390-1431) for up to kGroups blocks per CTA iteration.
// If `src` is non-null this is the initial sweep of a computeEsdf call: the source
// list is also copied into `list` and stamped as the members of ring `ring`.
__device__ void phaseSweep(const EsdfCtx& c, const int* src, int* list, int n, int* stamp, int ring,
                           unsigned int* smem, int* s_changed, int cta, int nctas) {
  const int tid = threadIdx.x, group = tid >> 6, lane64 = tid & 63;
  unsigned int* sm = smem + group * kBlockWords;
  const int a = lane64 >> 3, b = lane64 & 7;
  for (int base = cta * kGroups; base < n; base += nctas * kGroups) {
    const int item = base + group;
    int slot = -1;
    if (item < n) {
      slot = src ? __ldcg(src + item) : __ldcg(list + item);
      if (src && lane64 == 0) {
        list[item] = slot;
        stamp[slot] = ring;
      }
    }
    if (lane64 == 0) s_changed[group] = 0;
    if (slot >= 0) loadBlockGroup(sm, esdfBlockPtr(c.esdf, slot), lane64);
    __syncthreads();
    bool ch = false;
    if (slot >= 0) ch |= sweepLine(sm, 0, a, b, 0, c.max_sq);
    __syncthreads();
    if (slot >= 0) ch |= sweepLine(sm, a, 0, b, 1, c.max_sq);
    __syncthreads();
    if (slot >= 0) ch |= sweepLine(sm, a, b, 0, 2, c.max_sq);
    if (ch) s_changed[group] = 1;
    __syncthreads();
    if (slot >= 0 && s_changed[group]) storeBlockGroup(esdfBlockPtr(c.esdf, slot), sm, lane64);
    __syncthreads();
  }
}

__device__ __forceinline__ void appendUnique(int slot, int* nxt, int* nxt_count, int* stamp_nxt, int ring_next) {
  if (atomicExch(stamp_nxt + slot, ring_next) != ring_next) nxt[atomicAdd(nxt_count, 1)] = slot;
}

// The two passes of one axis of updateNeighborBands (:1323-1386,
// getDirectionAndVoxelIndicesFromThread :1062-1091), fused per interface.
// For a list member b:
//   group "hi": interface (b, b+d): P = b -> b+d (pass +dir); then, if b+d is a
//               list member too, Q = b+d -> b (pass -dir).
//   group "lo": interface (b-d, b), only when b-d is NOT a list member (otherwise
//               b-d's "hi" group owns it): Q = b -> b-d.
// P precedes Q on every interface, different interfaces touch disjoint faces, so
// this equals running pass +dir over the whole list and then pass -dir.
__device__ void phaseNeighbors(const EsdfCtx& c, int axis, const int* cur, int n, const int* stamp_cur, int ring,
                               int* nxt, int* nxt_count, int* stamp_nxt, int* s_slot, int* s_upd, int cta,
                               int nctas) {
  const int tid = threadIdx.x, group = tid >> 6, lane64 = tid & 63;
  const int entry_in_cta = group >> 1, side = group & 1;  // side 0 = hi, 1 = lo
  const int u = lane64 >> 3, w = lane64 & 7;
  // voxel offset of this thread's face voxel at coordinate `cc` along `axis`
  const int strideA = (axis == 0) ? 64 : ((axis == 1) ? 8 : 1);
  const int faceBase = (axis == 0) ? (u * 8 + w) : ((axis == 1) ? (u * 64 + w) : (u * 64 + w * 8));
  const int vHi = faceBase + (kVps - 1) * strideA, vLo = faceBase;
  for (int base = cta * (kGroups / 2); base < n; base += nctas * (kGroups / 2)) {
    const int item = base + entry_in_cta;
    if (lane64 == 0) {
      int other = -1;
      int mine = -1;
      if (item < n) {
        mine = __ldcg(cur + item);
        const int* bi = c.esdf.block_index + 3 * mine;
        int x = bi[0], y = bi[1], z = bi[2];
        const int d = side ? -1 : 1;
        if (axis == 0) x += d;
        else if (axis == 1) y += d;
        else z += d;
        other = hashFind(c.esdf.hash, x, y, z);
      }
      s_slot[group * 2] = mine;
      s_slot[group * 2 + 1] = other;
      s_upd[group * 2] = 0;
      s_upd[group * 2 + 1] = 0;
    }
    __syncthreads();
    const int mine = s_slot[group * 2], other = s_slot[group * 2 + 1];
    if (mine >= 0 && other >= 0) {
      const bool other_member = (__ldcg(stamp_cur + other) == ring);
      if (side == 0) {
        // interface (A = mine, B = other = mine + d)
        unsigned int* gA = esdfBlockPtr(c.esdf, mine);
        unsigned int* gB = esdfBlockPtr(c.esdf, other);
        VoxelRegs A = loadVoxel(gA, vHi), B = loadVoxel(gB, vLo);
        if (updateSingleNeighbor(A, B, gB, vLo, axis, +1, c.max_sq)) s_upd[group * 2 + 1] = 1;  // B updated
        if (other_member) {
          if (updateSingleNeighbor(B, A, gA, vHi, axis, -1, c.max_sq)) s_upd[group * 2] = 1;  // A updated
        }
      } else if (!other_member) {
        // interface (A = other = mine - d, B = mine): only Q = B -> A
        unsigned int* gA = esdfBlockPtr(c.esdf, other);
        unsigned int* gB = esdfBlockPtr(c.esdf, mine);
        VoxelRegs A = loadVoxel(gA, vHi), B = loadVoxel(gB, vLo);
        if (updateSingleNeighbor(B, A, gA, vHi, axis, -1, c.max_sq)) s_upd[group * 2 + 1] = 1;  // A (= other) updated
      }
    }
    __syncthreads();
    if (lane64 == 0 && mine >= 0 && other >= 0) {
      if (s_upd[group * 2]) appendUnique(mine, nxt, nxt_count, stamp_nxt, ring + 1);
      if (s_upd[group * 2 + 1]) appendUnique(other, nxt, nxt_count, stamp_nxt, ring + 1);
    }
    __syncthreads();
  }
}

// Grid-wide barrier for the cooperative launch: monotonically increasing arrival
// counter in L2 (reset by esdfAllocateKernel before every update).
// Per-phase kernels for the host-driven loop (reference-like orchestration).
__global__ void __launch_bounds__(kThreads) esdfSweepKernel(EsdfCtx c, const int* src, int* list, const int* n_dev,
                                                            int* stamp, int ring) {
  extern __shared__ __align__(16) unsigned int smem[];
  __shared__ int s_changed[kGroups];
  phaseSweep(c, src, list, *n_dev, stamp, ring, smem, s_changed, blockIdx.x, gridDim.x);
}
__global__ void __launch_bounds__(kThreads) esdfNeighborKernel(EsdfCtx c, int axis, const int* cur, const int* n_dev,
                                                               const int* stamp_cur, int ring, int* nxt,
                                                               int* nxt_count, int* stamp_nxt) {
  __shared__ int s_slot[kGroups * 2];
  __shared__ int s_upd[kGroups * 2];
  phaseNeighbors(c, axis, cur, *n_dev, stamp_cur, ring, nxt, nxt_count, stamp_nxt, s_slot, s_upd, blockIdx.x,
                 gridDim.x);
}
__global__ void esdfSetIntKernel(int* p, int v) { *p = v; }

constexpr size_t kSweepSmemBytes = (size_t)kGroups * kEsdfBlockBytes;  // 40 KiB

// ---------------------------------------------------------------------------
// Mapper::clearBlocksInLayers (src/mapper/mapper.cpp:546-575) for the ESDF layer: the blocks the decay integrator
// deallocated leave the ESDF layer too. One CTA per block: unlink it from its neighbours' tables, zero its bytes
// (slab invariant), give the slot back. The host rebuilds the hash afterwards.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) esdfRemoveBlocksKernel(EsdfCtx c, const int4* dead, const int* dead_count) {
  const int tid = threadIdx.x;
  const int n = *dead_count;
  __shared__ int s_slot;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    int4 d = dead[i];
    if (c.slice_mode) {
      // 2-D ESDF (src/mapper/mapper.cpp:569-626): the column's slice block goes only when no projective block is left
      // in the vertical column within the slice bounds; several dead blocks of one column elect one remover.
      d.w = c.slice_out_bz;
      if (tid == 0) {
        int es = hashFind(c.esdf.hash, d.y, d.z, d.w);
        if (es >= 0) {
          bool has_block = false;
          for (int bz = c.slice_min_bz; bz <= c.slice_max_bz && !has_block; bz++) {
            const int ps = hashFind(c.tsdf.hash, d.y, d.z, bz);  // the hash still lists the dead blocks: check the slot
            has_block = ps >= 0 && c.tsdf.block_index[3 * ps] != kDeadSlotX;
          }
          if (has_block || atomicExch(&c.esdf.block_index[3 * es], kDeadSlotX) == kDeadSlotX) es = -1;
        }
        s_slot = es;
      }
    } else if (tid == 0) {
      s_slot = hashFind(c.esdf.hash, d.y, d.z, d.w);
    }
    __syncthreads();
    const int slot = s_slot;
    if (slot >= 0) {
      if (tid < 27 && tid != 13) {
        int nb = c.nbr27[27 * slot + tid];
        const int dx = tid / 9 - 1, dy = (tid / 3) % 3 - 1, dz = tid % 3 - 1;
        if (nb < -1) nb = hashFind(c.esdf.hash, d.y + dx, d.z + dy, d.w + dz);  // row never linked
        if (nb >= 0) {
          c.nbr27[27 * nb + (26 - tid)] = -1;
          if ((dx != 0) + (dy != 0) + (dz != 0) == 1) {
            const int axis = dx ? 0 : (dy ? 1 : 2);
            const int neg = (dx + dy + dz) < 0 ? 1 : 0;
            c.nbr[6 * nb + axis * 2 + (neg ^ 1)] = -1;
          }
        }
      }
      __syncthreads();
      if (tid < 27) c.nbr27[27 * slot + tid] = (int)0xFEFEFEFE;
      if (tid < 6) c.nbr[6 * slot + tid] = (int)0xFEFEFEFE;
      uint4* g = reinterpret_cast<uint4*>(esdfBlockPtr(c.esdf, slot));
      for (int k = tid; k < kBlockWords / 4; k += kThreads) g[k] = make_uint4(0, 0, 0, 0);
      if (tid == 0) {
        if (*c.cleared_count > 0 && c.seed_clr[slot] == *c.cleared_seq) {
          const int q = atomicAdd(c.dead_cleared_count, 1);
          c.dead_cleared_xyz[3 * q] = d.y, c.dead_cleared_xyz[3 * q + 1] = d.z, c.dead_cleared_xyz[3 * q + 2] = d.w;
        }
        c.seed_clr[slot] = 0, c.seed_upd[slot] = 0;
        c.esdf.block_index[3 * slot] = kDeadSlotX;
        c.esdf.free_slots[atomicAdd(c.esdf.free_count, 1)] = slot;
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// 2-D ESDF: EsdfIntegrator::markSitesInSlice with a ConstantZSliceDescription (esdf_integrator.cu:754-1055).
// (1) the blocks to update are reduced to their (x, y) columns (the reference builds an Index3DSet on the host),
// (2) the ESDF blocks of the output layer are allocated, (3) one CTA per column block squashes the band of the
// projective layer onto the slice voxels (min TSDF distance / max log odds over the observed, non-freespace voxels:
// order-independent, so no atomics are needed when one thread walks its own voxel column) and runs
// updateEsdfVoxelToChanges on them.
// ---------------------------------------------------------------------------
__global__ void esdfSliceColumnsKernel(EsdfCtx c, const int* in_xyz, const int* in_slots, const int* in_count_dev,
                                       int in_count_host) {
  const int n = in_count_dev ? *in_count_dev : in_count_host;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x, y;
  if (in_slots) {
    const int tslot = in_slots[i];
    if (c.tracker_dirty) c.tracker_dirty[tslot] = 0;
    x = c.tsdf.block_index[3 * tslot], y = c.tsdf.block_index[3 * tslot + 1];
  } else {
    x = in_xyz[3 * i], y = in_xyz[3 * i + 1];
  }
  if (!indexInRange(x, y, c.slice_out_bz)) {
    atomicOr(c.error, 2);
    return;
  }
  const unsigned long long key = packIndex(x, y, c.slice_out_bz);
  unsigned int p = hashKey(key) & c.colset_mask;
  while (true) {
    const unsigned long long old = atomicCAS(&c.colset_keys[p], kEmptyKey, key);
    if (old == kEmptyKey) {
      const int q = atomicAdd(c.cols_count, 1);
      c.cols[2 * q] = x, c.cols[2 * q + 1] = y;
      return;
    }
    if (old == key) return;
    p = (p + 1) & c.colset_mask;
  }
}

__global__ void esdfSliceAllocateKernel(EsdfCtx c) {
  const int n = *c.cols_count;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  resetEsdfUpdate(c, n);
  const int stride = gridDim.x * blockDim.x;
  for (int k = i; k < n; k += stride) {
    const int x = c.cols[2 * k], y = c.cols[2 * k + 1];
    bool was_new;
    const int eslot = hashFindOrInsert(c.esdf, x, y, c.slice_out_bz, c.error, &was_new);
    c.work[k] = make_int4(eslot, x, y, was_new ? 1 : 0);
  }
}

// getBlockAndVoxelIndexFrom1DPositionInLayer (core/internal/impl/indexing_impl.h:105-115)
__device__ __forceinline__ void blockAndVoxelFrom1D(float block_size, float p, int& b, int& v) {
  const float inv = (float)(1.0 / (double)(block_size * (1.0f / kVps)));
  b = floatToIntRz(floorf(p / block_size));
  v = floatToIntRz((p - block_size * (float)b) * inv);
  if (v > kVps - 1) v = kVps - 1;
}

template <class Site>
__global__ void __launch_bounds__(64) esdfMarkSliceKernel(EsdfCtx c) {
  using V = typename Site::Voxel;
  __shared__ int s_src[16], s_fs[16];
  __shared__ int s_flags[2];  // updated, cleared
  __shared__ int s_range[2];  // block range of the CTA's columns (planar slices: the union over the 64 voxel columns)
  __shared__ MarkLocal ml;
  const Site site = Site::of(c);
  const int tid = threadIdx.x;
  const int n = markBegin(c, ml);
  const int vx = tid >> 3, vy = tid & 7;
  const int nb_col = c.slice_max_bz - c.slice_min_bz + 1;
  for (int item = blockIdx.x; item < n; item += gridDim.x) {
    const int4 w = c.work[item];
    if (w.x >= 0 && w.w) linkNewBlock(c, w.x, tid);
    if (tid < 2) s_flags[tid] = 0;
    __syncthreads();
    if (w.x < 0) continue;
    bool observed = false;
    float squashed = site.squashInit(c.max_sq);
    // ColumnBounds of this thread's voxel column: the constant-z slice's, or from the ground plane
    // (PlanarSliceColumnBoundsGetter::getColumnBounds, esdf_integrator_slicing_impl.cuh:100-130)
    int min_bz = c.slice_min_bz, min_vz = c.slice_min_vz, max_bz = c.slice_max_bz, max_vz = c.slice_max_vz;
    int first_bz = c.slice_min_bz, ncol = nb_col;
    if (c.slice_planar) {
      const float vs = c.block_size * (1.0f / kVps), half = c.block_size * (0.5f / kVps);
      const float px = (c.block_size * (float)w.y + vs * (float)vx) + half;
      const float py = (c.block_size * (float)w.z + vs * (float)vy) + half;
      const float plane_h = -1.0f * (c.plane_nx * px + c.plane_ny * py + c.plane_d) / c.plane_nz;
      const float lo_h = plane_h + c.slice_above_plane_m, hi_h = lo_h + c.slice_thickness_m;
      blockAndVoxelFrom1D(c.block_size, lo_h, min_bz, min_vz);
      blockAndVoxelFrom1D(c.block_size, hi_h, max_bz, max_vz);
      if (tid == 0) s_range[0] = INT32_MAX, s_range[1] = INT32_MIN;
      __syncthreads();
      atomicMin(&s_range[0], min_bz), atomicMax(&s_range[1], max_bz);
      __syncthreads();
      first_bz = s_range[0];
      ncol = s_range[1] - s_range[0] + 1;
      __syncthreads();
    }
    for (int b0 = 0; b0 < ncol; b0 += 16) {
      if (tid < 16 && b0 + tid < ncol) {
        s_src[tid] = hashFind(c.tsdf.hash, w.y, w.z, first_bz + b0 + tid);
        s_fs[tid] = c.use_freespace ? hashFind(c.freespace.hash, w.y, w.z, first_bz + b0 + tid) : -1;
      }
      __syncthreads();
      for (int q = 0; q < 16 && b0 + q < ncol; q++) {
        const int ss = s_src[q];
        if (ss < 0) continue;
        const int bz = first_bz + b0 + q;
        if (bz < min_bz || bz > max_bz) continue;  // isBlockIdxInRange
        const int z0 = bz == min_bz ? min_vz : 0, z1 = bz == max_bz ? max_vz : kVps - 1;
        const V* src = reinterpret_cast<const V*>(c.tsdf.blocks + (size_t)ss * Site::kBlockBytes);
        const int fs = s_fs[q];
        for (int vz = z0; vz <= z1; vz++) {
          const int v = (vx * kVps + vy) * kVps + vz;
          const V t = src[v];
          if (site.observed(t)) {
            observed = true;
            if (!isVoxelFreespace(c.freespace, fs, v)) squashed = site.squash(squashed, Site::value(t));  // freespace is skipped
          }
        }
      }
      __syncthreads();
    }
    // updateEsdfVoxelToChanges on the slice voxel, with the squashed value in place of a projective voxel's
    bool updated = false, cleared = false;
    const bool is_inside = site.inside(squashed);
    updateVoxelToChanges(esdfBlockPtr(c.esdf, w.x), (vx * kVps + vy) * kVps + c.slice_out_vz, observed,
                         is_inside, is_inside && site.nearSurface(squashed), c.max_sq, updated, cleared);
    if (updated) s_flags[0] = 1;
    if (cleared) s_flags[1] = 1;
    __syncthreads();
    if (tid == 0) markLocalRecord(c, ml, w.x, s_flags[0] != 0, s_flags[1] != 0);
    __syncthreads();
  }
  if (tid == 0) markFinish(c, ml);
}

}  // namespace

void launchEsdfAllocate(const EsdfCtx& c, const int* in_xyz, const int* in_slots, const int* in_count_dev,
                        int in_count_upper, cudaStream_t stream) {
  const int threads = 256;
  const int blocks = (in_count_upper + threads - 1) / threads;
  esdfAllocateKernel<<<blocks < 1 ? 1 : blocks, threads, 0, stream>>>(c, in_xyz, in_slots, in_count_dev,
                                                                       in_count_upper);
}

void launchEsdfRemoveBlocks(const EsdfCtx& c, const int4* dead, const int* dead_count, int upper, cudaStream_t stream) {
  int grid = upper < 1184 ? (upper < 1 ? 1 : upper) : 1184;
  esdfRemoveBlocksKernel<<<grid, kThreads, 0, stream>>>(c, dead, dead_count);
  launchDropDeadSlots(c.esdf, c.cleared_list, c.cleared_count, stream);  // off the persistent cleared list
}

void launchEsdfSliceAllocateAndMark(const EsdfCtx& c, const int* in_xyz, const int* in_slots, const int* in_count_dev,
                                    int in_count_upper, int num_sms, cudaStream_t stream) {
  if (in_count_upper < 1) in_count_upper = 1;
  cudaMemsetAsync(c.colset_keys, 0xFF, ((size_t)c.colset_mask + 1) * sizeof(unsigned long long), stream);
  cudaMemsetAsync(c.cols_count, 0, sizeof(int), stream);
  esdfSliceColumnsKernel<<<(in_count_upper + 255) / 256, 256, 0, stream>>>(c, in_xyz, in_slots, in_count_dev, in_count_upper);
  esdfSliceAllocateKernel<<<(in_count_upper + 255) / 256, 256, 0, stream>>>(c);
  int grid = num_sms * 16;
  if (in_count_upper < grid) grid = in_count_upper;
  if (c.from_occupancy)
    esdfMarkSliceKernel<OccupancySite><<<grid, 64, 0, stream>>>(c);
  else
    esdfMarkSliceKernel<TsdfSite><<<grid, 64, 0, stream>>>(c);
}

// Test hook: NVB_ESDF_GRID_CAP=<n> caps the grids of the mark and clear kernels so that small maps exercise their
// multi-round paths (per-CTA list flushes, several selection rounds).
static int esdfGridCap() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("NVB_ESDF_GRID_CAP");
    v = e ? atoi(e) : 0;
    if (v < 0) v = 0;
  }
  return v;
}
// Grid of a mark or clear kernel: `per_sm` CTAs per SM, at most one per work item (`upper` bounds their number) and at
// least one, then capped by the test hook.
static int esdfGrid(int num_sms, int per_sm, int upper) {
  int grid = num_sms * per_sm;
  if (upper < grid) grid = upper;
  if (grid < 1) grid = 1;
  const int cap = esdfGridCap();
  return (cap > 0 && grid > cap) ? cap : grid;
}

void launchEsdfMark(const EsdfCtx& c, int count_upper, int num_sms, cudaStream_t stream) {
  if (c.from_occupancy) {
    esdfMarkOccupancyKernel<<<esdfGrid(num_sms, 8, count_upper), kThreads, 0, stream>>>(c);
  } else if (c.use_freespace) {  // the TMA ring stages the ESDF + TSDF blocks only
    // 8 CTAs per SM, 5 of them resident (10 KiB smem, 256 threads, 48 registers each)
    esdfMarkKernel<<<esdfGrid(num_sms, 8, count_upper), kThreads, 0, stream>>>(c);
  } else {
    static const cudaError_t smem_attr = cudaFuncSetAttribute(
        esdfMarkTmaKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMarkStages * sizeof(MarkStage)));
    (void)smem_attr;
    // 4 x 43 KiB of staging per SM; ~3000 items -> ~5 per CTA, 2 loads in flight each
    esdfMarkTmaKernel<<<esdfGrid(num_sms, 4, count_upper), kThreads, kMarkStages * sizeof(MarkStage), stream>>>(c);
  }
}

// One fused launch: on the 80-frame C2 bench (one H100 SXM, 400 W power limit) it took 28.5 - 29.9 us per frame over eight
// runs against 30.6 us for selection and processing as two kernels with a balanced candidate list in between -- the
// imbalance of the per-CTA candidate counts costs less than the second launch (DESIGN.md section 9).
void launchEsdfClear(const EsdfCtx& c, int esdf_count_upper, int num_sms, cudaStream_t stream) {
  esdfClearKernel<<<esdfGrid(num_sms, 8, esdf_count_upper), kThreads, 0, stream>>>(c);
}

// One launch per phase; the host reads the ring's block count after every ring,
// like the reference does (sortAndTakeUniqueIndices, :1296-1297).
cudaError_t runEsdfComputeHostLoop(const EsdfCtx& c, int num_sms, cudaStream_t stream, int* launches) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(esdfSweepKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSweepSmemBytes);
    attr_set = true;
  }
  int h_ring = 0, h_counts[2] = {0, 0}, h_work = 0;
  cudaError_t e;
  if ((e = cudaMemcpyAsync(&h_ring, c.ring_id, sizeof(int), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
  if ((e = cudaMemcpyAsync(&h_work, c.work_count, sizeof(int), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
  if (h_work == 0) return cudaSuccess;  // empty block list: nothing to do (:226-228)
  int ring = h_ring;
  int* lists[2] = {c.ring_a, c.ring_b};
  int* stamps[2] = {c.stamp_a, c.stamp_b};
  long long swept = 0, faces = 0, rings = 0;
  const int grid = num_sms * 2;
  for (int pass = 0; pass < 2; pass++) {
    const int* src = pass ? c.cleared_list : c.upd_list;
    const int* src_count = pass ? c.cleared_count : c.upd_count;
    int n = 0;
    if ((e = cudaMemcpyAsync(&n, src_count, sizeof(int), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    if (n == 0) continue;
    int ci = ring & 1;
    esdfSweepKernel<<<grid, kThreads, kSweepSmemBytes, stream>>>(c, src, lists[ci], src_count, stamps[ci], ring);
    esdfSetIntKernel<<<1, 1, 0, stream>>>(c.ring_count + ci, n);
    esdfSetIntKernel<<<1, 1, 0, stream>>>(c.ring_count + (ci ^ 1), 0);
    (*launches) += 3;
    swept += n;
    while (n > 0) {
      const int ni = ci ^ 1;
      for (int axis = 0; axis < 3; axis++) {
        esdfNeighborKernel<<<grid, kThreads, 0, stream>>>(c, axis, lists[ci], c.ring_count + ci, stamps[ci], ring,
                                                          lists[ni], c.ring_count + ni, stamps[ni]);
      }
      esdfSweepKernel<<<grid, kThreads, kSweepSmemBytes, stream>>>(c, nullptr, lists[ni], c.ring_count + ni, nullptr,
                                                                   0);
      (*launches) += 4;
      faces += 6ll * n;
      if ((e = cudaMemcpyAsync(h_counts, c.ring_count, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream)) !=
          cudaSuccess)
        return e;
      if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
      const int n_next = h_counts[ni];
      esdfSetIntKernel<<<1, 1, 0, stream>>>(c.ring_count + ci, 0);
      (*launches)++;
      swept += n_next;
      rings++;
      ring++;
      ci = ni;
      n = n_next;
    }
    ring++;
  }
  ring++;
  long long h_stats[3] = {swept, faces, rings};
  int h_cleared = 0;
  if ((e = cudaMemcpyAsync(&h_cleared, c.cleared_count, sizeof(int), cudaMemcpyDeviceToHost, stream)) != cudaSuccess)
    return e;
  if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
  long long h_cl = h_cleared;
  cudaMemcpyAsync(c.stats + kStatCleared, &h_cl, sizeof(long long), cudaMemcpyHostToDevice, stream);
  cudaMemcpyAsync(c.stats + kStatSwept, h_stats, 3 * sizeof(long long), cudaMemcpyHostToDevice, stream);
  cudaMemcpyAsync(c.ring_id, &ring, sizeof(int), cudaMemcpyHostToDevice, stream);
  return cudaStreamSynchronize(stream);
}

}  // namespace nvb
