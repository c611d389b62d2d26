// nvb_esdf_wave_common.cuh -- device helpers shared by the ESDF wavefront kernels (nvb_esdf_wave.cu: four-phase and
// gather-replay wavefronts with 256-thread CTAs; nvb_esdf_wavex.cu: the exchange-slab wavefront). Everything that depends
// on the CTA size is a template on WT (threads per CTA, a multiple of 64: one 64-thread group per ESDF block).
#pragma once
#include "nvb_esdf_common.cuh"
#include "nvb_tma.cuh"

namespace nvb {
namespace {

#ifndef NVB_WAVE_INLINE
#define NVB_WAVE_INLINE 1
#endif
#if NVB_WAVE_INLINE
#define NVB_WAVE_FN __forceinline__
#else
#define NVB_WAVE_FN __noinline__
#endif
constexpr int kWaveMaxMembers = 1024;   // owned candidates scanned per round
constexpr int kPendMax = 1024;         // pending "updated block" records per CTA per ring before a forced flush
constexpr int kNbrCache = 128;          // members whose neighbour slots are cached in smem
constexpr int kSweepBlockWords = kBlockWords;  // unpadded: a bank-conflict-free padded image needs scalar smem stores (design reasoning, not measured on the H100)
template <int WT>
constexpr size_t waveSmemBytes() { return (size_t)(WT / 64) * kSweepBlockWords * sizeof(unsigned int); }  // sweep buffers

__device__ __forceinline__ int resolveNeighbor(const EsdfCtx& c, int slot, int dir) {
  int v = __ldcg(c.nbr + 6 * slot + dir);
  if (v < -1) {  // unknown (block created outside the ESDF update path): resolve through the hash once
    const int* bi = c.esdf.block_index + 3 * slot;
    int x = bi[0], y = bi[1], z = bi[2];
    const int d = (dir & 1) ? -1 : 1;
    if ((dir >> 1) == 0) x += d;
    else if ((dir >> 1) == 1) y += d;
    else z += d;
    v = hashFind(c.esdf.hash, x, y, z);
    c.nbr[6 * slot + dir] = v;
  }
  return v;
}

template <int WT>
struct WaveShared {
  int members[kWaveMaxMembers];
  int nbr[kNbrCache * 6];
  int scan[WT / 32];
  int count;
  int changed[(WT / 64)];
  int slot[(WT / 64) * 2];
  int upd[(WT / 64) * 2];
  int npend;
  int pend[kPendMax];  // blocks updated by this CTA's face operations in the current ring (with duplicates)
};

// Members of a ring are dealt round-robin over the CTAs from the ring's global list: CTA c takes entries
// c, c+G, c+2G, ... so every CTA gets ceil(n/G) or floor(n/G) blocks (the static slot-ownership scheme this
// replaces was far from balanced, and the slowest CTA is what a phase costs). Entries [first, first+cap) of this
// CTA's share are cached in shared memory. Optionally stamps them (initial list of a computeEsdf call).
// `have` leading entries are already in sh.members (fetched speculatively with the ring's count).
template <int WT>
__device__ NVB_WAVE_FN int loadMembers(WaveShared<WT>& sh, const int* list, int n, int cta, int nctas, int first,
                                       int* stamp_out, int stamp_value, int have = 0) {
  const int tid = threadIdx.x;
  const int mine = (n > cta) ? (n - cta + nctas - 1) / nctas : 0;  // entries of this CTA
  int k = mine - first;
  k = k < 0 ? 0 : (k > kWaveMaxMembers ? kWaveMaxMembers : k);
  for (int j = tid; j < k; j += WT) {
    const int slot = j < have ? sh.members[j] : __ldcg(list + cta + (first + j) * nctas);
    sh.members[j] = slot;
    if (stamp_out) stamp_out[slot] = stamp_value;
  }
  __syncthreads();
  return k;
}

// Neighbour slots of the first kNbrCache members -> shared memory (one thread per (member, dir)).
template <int WT>
__device__ __forceinline__ void prefetchNeighbors(const EsdfCtx& c, WaveShared<WT>& sh, int k) {
  const int tid = threadIdx.x;
  const int kc = k < kNbrCache ? k : kNbrCache;
  for (int q = tid; q < kc * 6; q += WT) sh.nbr[q] = resolveNeighbor(c, sh.members[q / 6], q % 6);
}

// sweepSingleBand (:542-600) on registers, written for a SHORT DEPENDENT CHAIN: one block's sweep is
// 3 axes x 16 sequential steps on two warps, so its latency is (instructions on the chain) x (ALU
// latency), not throughput. Per step the only loop-carried state is the candidate site (l0,l1,l2) and
// `found`; everything that does not depend on it is hoisted:
//   * squared distances are exact integers (or max_sq), so "sq > |d|^2" is evaluated as the integer test
//     ceil(sq) > |d|^2 -- no int->float conversion on the chain; "sq < max_sq" becomes a bit mask;
//   * each voxel's own parent position (parent + voxel) is precomputed;
//   * the four cases of the reference (unobserved / site / first valid voxel / candidate vs own) are
//     folded into branch-free selects.
// The line's 8 voxels are loaded once, walked forward, the register image is reversed and walked again
// (= the backward pass); changed voxels are written back. `axis` and `pass` are run-time values so that
// ONE copy of the 8-step body serves all six passes.
// `sm` is a split image in shared memory (a block: nvb_esdf_block.cuh, or a gather region): voxel u's cell at words
// [4 u, 4 u + 4), its flag word at flag_w + u. v0 is the line's first voxel, stride the voxel stride along the line;
// (c0,c1,c2) are the voxel coordinates at position 0.
__device__ __forceinline__ bool sweepLineRegs(unsigned int* sm, int flag_w, int v0, int stride, int c0, int c1, int c2,
                                              int axis, float max_sq) {
  int T[kVps];  // ceil(squared distance): sq > n  <=>  T > n for every integer n
  int p0[kVps], p1[kVps], p2[kVps];
  unsigned int obs = 0, site = 0, valid = 0, dirty = 0;
#pragma unroll
  for (int i = 0; i < kVps; i++) {
    const uint4 e = *reinterpret_cast<const uint4*>(sm + kEsdfCellWords * (v0 + i * stride));
    const float sq = __uint_as_float(e.x);
    T[i] = __float2int_ru(sq);
    p0[i] = (int)e.y, p1[i] = (int)e.z, p2[i] = (int)e.w;
    const unsigned int fl = sm[flag_w + v0 + i * stride];
    if (flagObserved(fl)) obs |= 1u << i;
    if (flagSite(fl)) site |= 1u << i;
    if (sq < max_sq) valid |= 1u << i;
  }
  const int a0 = (axis == 0), a1 = (axis == 1), a2 = (axis == 2);
#pragma unroll 1
  for (int pass = 0; pass < 2; pass++) {
    int l0 = 0, l1 = 0, l2 = 0;
    bool found = false;
#pragma unroll
    for (int k = 0; k < kVps; k++) {
      // register slot k holds line position pos = k (pass 0) or 7 - k (pass 1, image reversed)
      const int pos = pass ? (kVps - 1 - k) : k;
      const int x0 = c0 + a0 * pos, x1 = c1 + a1 * pos, x2 = c2 + a2 * pos;  // voxel coordinates
      const bool o = (obs >> k) & 1u, st = (site >> k) & 1u, vl = (valid >> k) & 1u;
      const int own0 = p0[k] + x0, own1 = p1[k] + x1, own2 = p2[k] + x2;    // off the chain
      const int d0 = l0 - x0, d1 = l1 - x1, d2 = l2 - x2;
      const int pd = d0 * d0 + (d1 * d1 + d2 * d2);
      const bool better = found && o && !st && (T[k] > pd);  // candidate site is closer than the voxel's value
      const bool take_site = o && st;
      const bool take_own = o && !st && !better && vl;       // voxel's own parent becomes the running site
      if (better) {
        p0[k] = d0, p1[k] = d1, p2[k] = d2, T[k] = pd;
        dirty |= 1u << k;
        valid |= 1u << k;  // pd < old sq <= max_sq
      }
      l0 = take_site ? x0 : (take_own ? own0 : l0);
      l1 = take_site ? x1 : (take_own ? own1 : l1);
      l2 = take_site ? x2 : (take_own ? own2 : l2);
      found = found || take_site || take_own;
    }
    // reverse the register image (and the bit masks) for the other direction / back to line order
#pragma unroll
    for (int k = 0; k < kVps / 2; k++) {
      const int r = kVps - 1 - k;
      int ti = T[k]; T[k] = T[r]; T[r] = ti;
      ti = p0[k]; p0[k] = p0[r]; p0[r] = ti;
      ti = p1[k]; p1[k] = p1[r]; p1[r] = ti;
      ti = p2[k]; p2[k] = p2[r]; p2[r] = ti;
    }
    obs = __brev(obs) >> 24, site = __brev(site) >> 24, dirty = __brev(dirty) >> 24, valid = __brev(valid) >> 24;
  }
  // after two reversals slot i is line position i again
#pragma unroll
  for (int i = 0; i < kVps; i++) {
    if ((dirty >> i) & 1u) {
      *reinterpret_cast<uint4*>(sm + kEsdfCellWords * (v0 + i * stride)) =
          make_uint4(__float_as_uint((float)T[i]), (unsigned)p0[i], (unsigned)p1[i], (unsigned)p2[i]);
    }
  }
  return dirty != 0;
}

// sweepBlockBandKernel (:1390-1431) for the cached members, (WT / 64) blocks at a time.
template <int WT>
__device__ NVB_WAVE_FN void sweepMembers(const EsdfCtx& c, WaveShared<WT>& sh, int k, unsigned int* smem,
                                         bool prefetch_nbr) {
  const int tid = threadIdx.x, group = tid >> 6, lane64 = tid & 63;
  unsigned int* sm = smem + group * kSweepBlockWords;
  const int a = lane64 >> 3, b = lane64 & 7;
  for (int base = 0; base < k; base += (WT / 64)) {
    const int item = base + group;
    const int slot = item < k ? sh.members[item] : -1;
    if (lane64 == 0) sh.changed[group] = 0;
    if (slot >= 0) loadBlockGroup(sm, esdfBlockPtr(c.esdf, slot), lane64);
    // neighbour slots for the coming axis phases: issued behind the block loads, not in front of them
    if (prefetch_nbr && base == 0) prefetchNeighbors(c, sh, k);
    __syncthreads();
    bool ch = false;
#pragma unroll 1
    for (int axis = 0; axis < 3; axis++) {
      // x lines: (x, a, b); y lines: (a, y, b); z lines: (a, b, z)
      const int v0 = (axis == 0) ? (a * 8 + b) : ((axis == 1) ? (a * 64 + b) : (a * 64 + b * 8));
      const int stride = (axis == 0) ? 64 : ((axis == 1) ? 8 : 1);
      const int c0 = (axis == 0) ? 0 : a;
      const int c1 = (axis == 0) ? a : ((axis == 1) ? 0 : b);
      const int c2 = (axis == 2) ? 0 : b;
      if (slot >= 0)
        ch |= sweepLineRegs(sm, kEsdfFlagWord0, v0, stride, c0, c1, c2, axis, c.max_sq);
      __syncthreads();
    }
    if (ch) sh.changed[group] = 1;
    __syncthreads();
    if (slot >= 0 && sh.changed[group]) storeBlockGroup(esdfBlockPtr(c.esdf, slot), sm, lane64);
    __syncthreads();
  }
}

// The +dir and -dir passes of one axis of updateNeighborBands (:1323-1386), fused per block
// interface (see nvb_esdf.cu phaseNeighbors for the ownership rule and why it is exact):
//   group side 0 ("hi"): interface (b, b+d): P = b -> b+d, then Q = b+d -> b if b+d is a member;
//   group side 1 ("lo"): interface (b-d, b) only when b-d is NOT a member: Q = b -> b-d.
// Destination blocks are stamped for ring+1 with a plain store.
template <int WT>
__device__ NVB_WAVE_FN void axisMembers(const EsdfCtx& c, WaveShared<WT>& sh, int axis, int k, const int* stamp_cur, int ring,
                                        int* stamp_nxt, int* list_nxt, int* count_nxt) {
  // One warp per (member, side) interface, two face voxels per lane: WT/32 interfaces = WT/64 members per
  // iteration, so the handful of members a CTA owns are all in flight at once (one L2 round trip per phase).
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int kWarps = WT / 32;
  const int entry_in_cta = warp >> 1, side = warp & 1;
  const int strideA = (axis == 0) ? 64 : ((axis == 1) ? 8 : 1);
  for (int base = 0; base < k; base += kWarps / 2) {
    const int item = base + entry_in_cta;
    int mine = -1, other = -1;
    if (item < k) {
      mine = sh.members[item];
      other = item < kNbrCache ? sh.nbr[item * 6 + axis * 2 + side] : resolveNeighbor(c, mine, axis * 2 + side);
    }
    bool updA = false, updB = false;  // A = low block's hi face, B = high block's lo face
    if (mine >= 0 && other >= 0) {
      // membership of the neighbour and the face voxels are fetched in the same round trip
      const int other_stamp = __ldcg(stamp_cur + other);
      unsigned int* blkA = esdfBlockPtr(c.esdf, side == 0 ? mine : other);
      unsigned int* blkB = esdfBlockPtr(c.esdf, side == 0 ? other : mine);
      VoxelRegs A[2], B[2];
      int vHi[2], vLo[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int f = lane + 32 * h, u = f >> 3, w = f & 7;
        const int faceBase = (axis == 0) ? (u * 8 + w) : ((axis == 1) ? (u * 64 + w) : (u * 64 + w * 8));
        vHi[h] = faceBase + (kVps - 1) * strideA;
        vLo[h] = faceBase;
        A[h] = loadVoxel(blkA, vHi[h]);
        B[h] = loadVoxel(blkB, vLo[h]);
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (side == 0) {
          updB |= updateSingleNeighbor(A[h], B[h], blkB, vLo[h], axis, +1, c.max_sq);  // P: mine -> mine + d
          if (other_stamp == ring) updA |= updateSingleNeighbor(B[h], A[h], blkA, vHi[h], axis, -1, c.max_sq);  // Q
        } else if (other_stamp != ring) {
          updA |= updateSingleNeighbor(B[h], A[h], blkA, vHi[h], axis, -1, c.max_sq);  // Q: mine -> mine - d
        }
      }
    }
    updA = __any_sync(0xffffffffu, updA);
    updB = __any_sync(0xffffffffu, updB);
    if (lane == 0 && mine >= 0 && other >= 0) {
      const int slotA = side == 0 ? mine : other, slotB = side == 0 ? other : mine;
      // Record the updated blocks; they are appended to ring+1 once per ring (flushPending), so the two
      // dependent L2 atomics of the unique append are paid once instead of in each of the three axis phases.
      if (updA) {
        const int q = atomicAdd(&sh.npend, 1);
        if (q < kPendMax) sh.pend[q] = slotA;
        else if (atomicExch(stamp_nxt + slotA, ring + 1) != ring + 1) list_nxt[atomicAdd(count_nxt, 1)] = slotA;
      }
      if (updB) {
        const int q = atomicAdd(&sh.npend, 1);
        if (q < kPendMax) sh.pend[q] = slotB;
        else if (atomicExch(stamp_nxt + slotB, ring + 1) != ring + 1) list_nxt[atomicAdd(count_nxt, 1)] = slotB;
      }
    }
  }
}

// 96 registers x 512 threads = 3/4 of the register file: the wavefront runs on a side stream and must
// leave room for the next frame's raycast / compaction / TSDF CTAs on the same SM.
// Unique append of the recorded blocks to ring+1: the stamp (atomicExch) dedupes across CTAs and doubles as the
// membership flag of ring+1; each warp reserves its range of the list with one atomicAdd.
template <int WT>
__device__ NVB_WAVE_FN void flushPending(WaveShared<WT>& sh, int* stamp_nxt, int ring, int* list_nxt, int* count_nxt) {
  __syncthreads();
  const int tid = threadIdx.x, lane = tid & 31;
  const int np = sh.npend < kPendMax ? sh.npend : kPendMax;
  for (int base = 0; base < np; base += WT) {
    const int q = base + tid;
    int slot = -1;
    bool fresh = false;
    if (q < np) {
      slot = sh.pend[q];
      fresh = atomicExch(stamp_nxt + slot, ring + 1) != ring + 1;
    }
    const unsigned int ballot = __ballot_sync(0xffffffffu, fresh);
    if (ballot) {
      int basepos = 0;
      if (lane == 0) basepos = atomicAdd(count_nxt, __popc(ballot));
      basepos = __shfl_sync(0xffffffffu, basepos, 0);
      if (fresh) list_nxt[basepos + __popc(ballot & ((1u << lane) - 1u))] = slot;
    }
  }
  __syncthreads();
  if (tid == 0) sh.npend = 0;
  __syncthreads();
}

#ifndef NVB_WAVE_MAXREG
#define NVB_WAVE_MAXREG 128
#endif
#ifndef NVB_WAVE_TAIL
#define NVB_WAVE_TAIL 4  // rings with at most this many members (= one sweep round of a CTA) are run by CTA 0 alone; 0 disables (not re-tuned on the H100)
#endif
constexpr int kTail = NVB_WAVE_TAIL;
constexpr int kSpec = 8;  // list entries per CTA fetched speculatively together with the ring's member count

// Unique hand-over of the recorded blocks to the next ring when ONE CTA runs the ring (tail mode): duplicates are
// found by comparing the (<= 12 per member) records in shared memory; no atomics, no L2 round trip.
// Next ring's members end up in sh.members[0..n), their stamps and the global list are written with plain stores
// (the list is only read if the ring outgrows the tail mode).
template <int WT>
__device__ NVB_WAVE_FN int flushLocal(WaveShared<WT>& sh, int* stamp_nxt, int ring, int* list_nxt) {
  const int tid = threadIdx.x;
  if (tid == 0) sh.count = 0;
  __syncthreads();
  const int np = sh.npend;
  for (int q = tid; q < np; q += WT) {
    const int slot = sh.pend[q];
    bool fresh = true;
    for (int j = 0; j < q; j++) fresh = fresh && (sh.pend[j] != slot);
    if (fresh) {
      const int pos = atomicAdd(&sh.count, 1);
      sh.members[pos] = slot;
      stamp_nxt[slot] = ring + 1;
      list_nxt[pos] = slot;
    }
  }
  __syncthreads();
  const int n = sh.count;
  if (tid == 0) sh.npend = 0;
  __syncthreads();
  return n;
}

// =====================================================================================================
// Gather-emulate-sweep wavefront ("GES"): the same computeEsdf, two grid barriers per ring instead of four.
//
// A ring's six face passes only move information across block boundaries by ONE voxel, so what they do to a
// block B is a function of B and its one-voxel halo (10x10x10 voxels, taken from the 3x3x3 block neighbourhood)
// as they were at the start of the ring, plus which of those 27 blocks are members (sources) of the ring: every
// voxel pair of every pass that touches the region has both voxels inside it. So the CTA that owns a CANDIDATE
// block (= neighbour of a member) gathers the region into shared memory, replays the six passes there in the
// reference's order (halo results are thrown away: their owners compute the same values), and if B changed --
// i.e. B is a member of the next ring -- sweeps it straight away in shared memory. No communication between
// the passes, no unique-append of "updated" blocks (a candidate has exactly one owner). Results are parked in a
// shadow slab until every CTA has finished reading the old state (barrier), then copied over the layer while
// the next ring's candidates and their neighbour rows are fetched (barrier).
// =====================================================================================================
// Region layout: split like a block (nvb_esdf_block.cuh), a plane of 16-byte cells then a plane of flag words, over 1 000
// region voxels: "core" = the 10 x 10 z-rows zr = rx * 10 + ry of the 8 voxels rz = 1..8 (voxel zr * 8 + rz - 1), so a
// z-row's cells (128 bytes) and flags (32 bytes) are contiguous here as in their source block; then the two z-halo planes
// rz = 0 and rz = 9 (voxels 800 + zr and 900 + zr).
constexpr int kZLoVox = 800;
constexpr int kZHiVox = 900;
constexpr int kRegionFlagWord0 = 1000 * kEsdfCellWords;  // word offset of the flag plane
constexpr int kRegionWords = kRegionFlagWord0 + 1000;   // 5000
constexpr int kGesMaxCand = 32;                 // candidates of one CTA per chunk
constexpr int kGesDoneMax = 64;                 // changed blocks remembered per 64-thread group and ring
template <int WT>
constexpr size_t gesSmemBytes() { return (size_t)(WT / 64) * kRegionWords * sizeof(unsigned int); }

template <int WT>
struct GesShared {
  // per-lane constants of the gather and of the pass replay (the same for every candidate): packed descriptors
  unsigned int tz[4][64];  // z-halo voxel copies:  d27 | hi << 5 | zr << 6 | src voxel << 13 | valid << 27
  unsigned int tc[4][64];  // core row copies:      d27 | zr << 6 | src z-row << 13 | valid << 27
  unsigned int te[6][4][64];  // boundary pairs per pass: src voxel | dst voxel << 13 | d27 << 26 | inner << 31; 0 = none
  int cand[kGesMaxCand];
  int rows[kGesMaxCand * 27];
  int done_slots[(WT / 64)][kGesDoneMax];
  int done_n[(WT / 64)];
  int overflow;
  unsigned int mask[(WT / 64)];
  int changed[(WT / 64)];
};

__device__ __forceinline__ void groupSync(int group) { asm volatile("bar.sync %0, 64;" ::"r"(group + 1) : "memory"); }
__device__ __forceinline__ void cpAsync16(unsigned int* smem_dst, const void* gsrc, bool valid) {
  const unsigned int d = (unsigned int)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 16 : 0;  // src-size 0: nothing is read, the 16 bytes are zero-filled (block not allocated)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cpAsyncWaitAll() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ int regionVox(int rx, int ry, int rz) {
  const int zr = rx * 10 + ry;
  return rz == 0 ? (kZLoVox + zr) : (rz == 9 ? (kZHiVox + zr) : (zr * 8 + rz - 1));
}
// region coordinate (0..9) -> block offset (-1, 0, +1) and voxel coordinate inside that block
__device__ __forceinline__ int regOff(int r) { return r == 0 ? -1 : (r == 9 ? 1 : 0); }
__device__ __forceinline__ int regLoc(int r) { return r == 0 ? 7 : (r == 9 ? 0 : r - 1); }

// Region of a candidate block <- the 27 blocks of `row` (slots; < 0 = not allocated -> zeros = unobserved voxels).
// All bulk traffic is 16-byte cp.async.cg (L2 -> shared, no L1, no registers). Core: a z-row is 8 cells (128 bytes) and 8
// flag words (32 bytes), contiguous and 16-byte aligned on both sides; two neighbouring lanes take alternate chunks of one
// row, and the row is decoded once per five copies. z-halo planes: per voxel one cell plus one flag word.
template <int WT>
__device__ __forceinline__ void gesInitTables(GesShared<WT>& gs, int tid) {
  if (tid < 64) {
    for (int j = 0; j < 4; j++) {
      {
        const int t = tid + 64 * j;
        unsigned int v = 0;
        if (t < 200) {
          const int zr = t >> 1, hi = t & 1;  // hi: rz = 9 <- block +z, voxel z = 0; lo: rz = 0 <- block -z, voxel z = 7
          const int rx = zr / 10, ry = zr % 10;
          const int d = (regOff(rx) + 1) * 9 + (regOff(ry) + 1) * 3 + (hi ? 2 : 0);
          const int off = (regLoc(rx) * 8 + regLoc(ry)) * 8 + (hi ? 0 : 7);  // source voxel
          v = (unsigned)d | ((unsigned)hi << 5) | ((unsigned)zr << 6) | ((unsigned)off << 13) | (1u << 27);
        }
        gs.tz[j][tid] = v;
      }
      {
        const int zr = j * 32 + (tid >> 1);
        unsigned int v = 0;
        if (zr < 100) {
          const int rx = zr / 10, ry = zr % 10;
          const int d = (regOff(rx) + 1) * 9 + (regOff(ry) + 1) * 3 + 1;
          const int off = regLoc(rx) * 8 + regLoc(ry);  // source z-row
          v = (unsigned)d | ((unsigned)zr << 6) | ((unsigned)off << 13) | (1u << 27);
        }
        gs.tc[j][tid] = v;
      }
      for (int pass = 0; pass < 6; pass++) {
        const int t = tid + 64 * j;
        unsigned int v = 0;
        if (t < 200) {
          const int axis = pass >> 1, dir = (pass & 1) ? -1 : 1;
          const int A = axis == 0 ? 9 : (axis == 1 ? 3 : 1), U = axis == 0 ? 3 : 9, W = axis == 2 ? 3 : 1;
          const int p = t / 100, u = (t % 100) / 10, w = t % 10;
          const int sa = dir > 0 ? (p ? 8 : 0) : (p ? 9 : 1);  // source coordinate along the axis
          const int so = dir > 0 ? (p ? 0 : -1) : (p ? 1 : 0);   // block offset of the source along the axis
          const int da = sa + dir;
          const int d = 13 + so * A + regOff(u) * U + regOff(w) * W;
          const int inner = da >= 1 && da <= 8 && u >= 1 && u <= 8 && w >= 1 && w <= 8;
          const int sw = axis == 0 ? regionVox(sa, u, w) : (axis == 1 ? regionVox(u, sa, w) : regionVox(u, w, sa));
          const int dw = axis == 0 ? regionVox(da, u, w) : (axis == 1 ? regionVox(u, da, w) : regionVox(u, w, da));
          v = (unsigned)sw | ((unsigned)dw << 13) | ((unsigned)d << 26) | ((unsigned)inner << 31);
        }
        gs.te[pass][j][tid] = v;
      }
    }
  }
}

template <int WT>
__device__ __forceinline__ void gesGather(const EsdfCtx& c, const GesShared<WT>& gs, unsigned int* R, const int* row,
                                          int lane64) {
  unsigned int zw[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const unsigned int t = gs.tz[j][lane64];
    zw[j] = 0;
    if (t >> 27) {
      const int slot = row[t & 31u], hi = (t >> 5) & 1u, zr = (t >> 6) & 127u, v = (t >> 13) & 511u;
      const unsigned int* blk = esdfBlockPtr(c.esdf, slot < 0 ? 0 : slot);
      cpAsync16(esdfCell(R, (hi ? kZHiVox : kZLoVox) + zr), esdfCell(blk, v), slot >= 0);
      if (slot >= 0) zw[j] = __ldcg(esdfFlag(blk, v));
    }
  }
  const int half = lane64 & 1;
#pragma unroll
  for (int it = 0; it < 4; it++) {
    const unsigned int t = gs.tc[it][lane64];
    if (t >> 27) {
      const int slot = row[t & 31u], zr = (t >> 6) & 127u, r = (t >> 13) & 63u;
      const unsigned int* blk = esdfBlockPtr(c.esdf, slot < 0 ? 0 : slot);
      // chunks 2 j + half of the row: cells 0..7, then the two 16-byte halves of its flag words
#pragma unroll
      for (int j = 0; j < 4; j++) cpAsync16(esdfCell(R, zr * 8 + 2 * j + half), esdfCell(blk, r * 8 + 2 * j + half), slot >= 0);
      cpAsync16(R + kRegionFlagWord0 + zr * 8 + 4 * half, esdfFlag(blk, r * 8 + 4 * half), slot >= 0);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const unsigned int t = gs.tz[j][lane64];
    if (t >> 27) {
      const int hi = (t >> 5) & 1u, zr = (t >> 6) & 127u;
      R[kRegionFlagWord0 + (hi ? kZHiVox : kZLoVox) + zr] = zw[j];
    }
  }
  cpAsyncWaitAll();
}

// updateSingleNeighbor (:602-633) on two voxels in shared memory, split into an operand fetch and the update so
// that the fetches of a thread's (up to three) pairs of a plane are in flight together.
struct PairOps {
  unsigned int e0, e1, e2, e3, e4, n0, n4;
  unsigned int* nb;
  bool act;
};
__device__ __forceinline__ PairOps pairLoad(unsigned int* R, unsigned int desc, bool act) {
  PairOps q;
  q.act = act;
  const int sv = desc & 8191u, dv = (desc >> 13) & 8191u;
  q.nb = esdfCell(R, dv);
  // unconditional fetch (the addresses of an inactive descriptor are valid voxels of the region): no branch, so the
  // operands of the lane's four pairs are in flight together
  const unsigned int* e = esdfCell(R, sv);
  q.e0 = e[0], q.e1 = e[1], q.e2 = e[2], q.e3 = e[3], q.e4 = R[kRegionFlagWord0 + sv];
  q.n0 = q.nb[0], q.n4 = R[kRegionFlagWord0 + dv];
  return q;
}
__device__ __forceinline__ bool pairApply(const PairOps& q, int axis, int direction, float max_sq) {
  const bool ok = q.act && flagObserved(q.e4) && flagObserved(q.n4) && !flagSite(q.n4) && !(__uint_as_float(q.e0) >= max_sq);
  const int d0 = (int)q.e1 - (axis == 0 ? direction : 0), d1 = (int)q.e2 - (axis == 1 ? direction : 0),
            d2 = (int)q.e3 - (axis == 2 ? direction : 0);
  const float pdist = (float)(d0 * d0 + (d1 * d1 + d2 * d2));
  if (ok && __uint_as_float(q.n0) > pdist) {
    q.nb[1] = (unsigned)d0, q.nb[2] = (unsigned)d1, q.nb[3] = (unsigned)d2;
    q.nb[0] = __float_as_uint(pdist);
    return true;
  }
  return false;
}

// The six passes of updateLocalNeighborBands (:1323-1386) restricted to the region: +x, -x, +y, -y, +z, -z, each
// seeing the previous ones. A pass along `axis` has two boundary planes (block -1|0 and block 0|+1) of 10 x 10
// voxel pairs; a pair is processed iff its SOURCE block is a member of the ring (bit in `mask`). Inside one pass
// sources and destinations are disjoint planes, so its 200 pairs are independent: each lane owns (up to) four of
// them -- the same for every candidate, so their shared-memory addresses and source-block indices come from a
// table built once per launch (the replay is instruction-bound, not latency-bound) -- fetches the operands of the
// active ones together and then applies them.
template <int WT>
__device__ __forceinline__ bool gesEmulate(const GesShared<WT>& gs, unsigned int* R, unsigned int mask, int lane64, int group,
                                           float max_sq) {
  bool changed = false;
#pragma unroll 1
  for (int pass = 0; pass < 6; pass++) {
    const int axis = pass >> 1, dir = (pass & 1) ? -1 : 1;
    const int A = axis == 0 ? 9 : (axis == 1 ? 3 : 1);
    // source blocks of this pass: offset along the axis in {-1, 0} (dir +) or {0, +1} (dir -)
    const unsigned int lo = axis == 0 ? 0x000001ffu : (axis == 1 ? 0x001c0e07u : 0x01249249u);  // offset -1 along the axis
    const unsigned int src_blocks = dir > 0 ? (lo | (lo << A)) : ((lo << A) | (lo << (2 * A)));
    if (!(mask & src_blocks)) continue;  // group-uniform
    unsigned int desc[4];
    PairOps q[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      desc[j] = gs.te[pass][j][lane64];
      q[j] = pairLoad(R, desc[j], desc[j] != 0u && ((mask >> ((desc[j] >> 26) & 31u)) & 1u));
    }
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (pairApply(q[j], axis, dir, max_sq)) changed = changed || (desc[j] >> 31);
    groupSync(group);
  }
  return changed;
}

__device__ __forceinline__ void copyShadowToLayer(const EsdfCtx& c, int slot, int lane64) {
  const uint4* src = reinterpret_cast<const uint4*>(c.shadow + (size_t)slot * kEsdfBlockBytes);
  uint4* dst = reinterpret_cast<uint4*>(c.esdf.blocks + (size_t)slot * kEsdfBlockBytes);
  uint4 q[kBlockWords / 4 / 64];
#pragma unroll
  for (int k = 0; k < kBlockWords / 4 / 64; k++) q[k] = __ldcg(src + lane64 + k * 64);
#pragma unroll
  for (int k = 0; k < kBlockWords / 4 / 64; k++) __stcg(dst + lane64 + k * 64, q[k]);
}

}  // namespace
}  // namespace nvb
