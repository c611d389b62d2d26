// nvb_esdf_wavex.cu -- the ESDF wavefront (computeEsdf, nvblox/src/integrators/esdf_integrator.cu:1465-1496) with ONE
// grid barrier per ring and no contended atomics: "exchange-slab" wavefront, esdf_persistent = 3.
//
// The four-phase wavefront (nvb_esdf_wave.cu) pays four grid barriers per ring whatever the ring's size (~18 rings per frame)
// plus the dependent L2 round trips between them. What a ring costs is its dependent chain, so this
// kernel shortens the chain:
//
//   * A ring's six face passes (+x,-x,+y,-y,+z,-z, each seeing the previous ones, :1323-1386) move information across block
//     boundaries by one voxel. Their effect on a block B is a function of B, of the one-voxel halo around it (10x10x10 voxels
//     out of the 3x3x3 block neighbourhood) as it was at the START of the ring, and of which of those 27 blocks are members
//     (sources) of the ring. The owner of a CANDIDATE block (a face neighbour of a member) gathers that region into shared
//     memory, replays the passes there in the reference's order, and -- if B changed, i.e. B is a member of ring+1 -- sweeps
//     it at once (sweepBlockBandKernel, :1390-1431). No communication inside a ring.
//   * Sources are always MEMBERS. Every member's state at the start of the ring is published in an exchange slab indexed by
//     slot, X[ring & 1]: the owner of a block that changes in ring r writes the new block to the layer (read by the block's
//     next owner only) and its six faces to X[(r+1) & 1] (read by its neighbours' owners during ring r+1, who only ever read
//     boundary voxels) while ring r's readers read X[r & 1]. Two slabs by ring parity, one barrier per ring, no version words,
//     no copy-back phase. A slot is face-major and in the region's split form (kXSlotBytes: 6 x 64 16-byte cells, then
//     6 x 64 flag words, 7.5 KiB), so a halo voxel is one 16-byte and one 4-byte copy and a face 1 KiB + 256 contiguous bytes.
//   * Only what can matter is fetched and replayed. A pass-p pair (source voxel -> destination voxel) matters iff its source
//     block is a member and its destination block is B or a member that can still influence B through the LATER passes: the
//     blocks whose state after pass p matters are D6 = {B}, D5 = D6 + {B+z}, D4 = D5 + {B-z}, D3 = D4 + (D4 + y),
//     D2 = D3 + (D3 - y), D1 = D2 + (D2 + x) (backwards through -z,+z,-y,+y,-x,+x). With one to three member neighbours --
//     the usual case -- one or two of the six passes are live and a few per cent of the 1 200 pair slots; halo voxels of
//     blocks that are in no live pair are not fetched (they would miss L2: nobody wrote them lately). The halo travels by
//     cp.async from the exchange slab straight into the region planes, so no registers are held across its round trip.
//   * Region layout in shared memory: a plane of 16-byte cells {squared distance, parent} and a plane of flag words, voxel
//     index rx*110 + ry*11 + rz, the split the layer's blocks (nvb_esdf_block.cuh) and the exchange slab use too. Every line
//     of the three sweeps and every pair of the replay is ONE conflict-free 128-bit access per voxel (a 20-byte array-of-
//     structures layout costs five 32-bit accesses with up to 8-way bank conflicts on z lines; with eight groups per SM the
//     kernel is bound by shared-memory instructions, not by latency), and the own block moves between the layer and the
//     region in aligned 16-byte cells and flag words, with no reshuffling.
//   * The sweep keeps, per line, the running site as (offset along the line, squared perpendicular offset, the two
//     perpendicular components): the loop-carried chain per voxel is one subtract, one multiply-add, one compare, one select.
//   * No hot words. Candidates of ring r+1 are registered by the owners of the blocks that changed in ring r (unique by an
//     atomicExch on a per-slot stamp) as RECORDS {slot, its 27 neighbour slots} in a per-CTA segment of the ring's list,
//     positions from a shared-memory counter; each CTA publishes its two counts (registrations, changed blocks) with a plain
//     store before the barrier, and after it every CTA reads the per-CTA pairs, scans them and deals the ring's candidates
//     round-robin (CTA, then 64-thread group). Same-address global atomics serialise in L2: hundreds of registrations per
//     ring on one counter would sit on the critical path.
//   * Rings with at most one candidate per 64-thread group of ONE CTA are run by CTA 0 alone with block-level barriers (half
//     of a frame's rings); everybody else waits at one grid barrier.
//   * 512-thread CTAs = 8 groups per SM x 132 SMs of an H100: 1 056 candidates in flight at once (176 KB of regions per CTA,
//     within the 227 KB of shared memory a Hopper block may use).
#include "nvb_esdf_wave_common.cuh"

#include <cstdlib>

namespace nvb {

namespace {

#ifndef NVB_WAVEX_THREADS
#define NVB_WAVEX_THREADS 512
#endif
#ifndef NVB_WAVEX_MAXREG
#define NVB_WAVEX_MAXREG 96  // 512 x 96 = 3/4 of the register file: the next frame's raycast / compaction / TSDF CTAs co-reside
#endif
#ifndef NVB_WAVEX_TAIL
#define NVB_WAVEX_TAIL 1
#endif
#ifndef NVB_WAVEX_PROF
#define NVB_WAVEX_PROF 0  // 1: per-phase times and per-stage cycle counters of CTA 0 / group 0 (nvb_mapper_debug_phase_max,
                          // tools/wavex_profile.py); the timers spill at 96 registers, so quote its shares, not its times
#endif
#if NVB_WAVEX_PROF
#define X_PROF_BEGIN() long long tq = clock64();
#define X_PROF(i) \
  if (lane64 == 0) xs.prof[group][i] += clock64() - tq; \
  tq = clock64();
#define X_PROF_COUNT(i) \
  if (lane64 == 0) xs.prof[group][i]++;
// stage i, also binned by the ring's candidate count K (bins K <= 256, <= 1 040, > 1 040 at index j, j + 1, j + 2; the
// candidates per bin at j + 3 ..): the own-block fetch of all of a ring's candidates leaves at once after the barrier
#define X_PROF_BIN(i, j, K)                                                  \
  if (lane64 == 0) {                                                         \
    const int kb = (K) <= 256 ? 0 : ((K) <= 1040 ? 1 : 2);                   \
    const long long dt = clock64() - tq;                                     \
    xs.prof[group][i] += dt, xs.prof[group][(j) + kb] += dt, xs.prof[group][(j) + 3 + kb]++; \
  }                                                                          \
  tq = clock64();
// stage i, also binned by K at index j + bin (the candidates per bin are counted by X_PROF_BIN)
#define X_PROF_KBIN(i, j, K)                                \
  if (lane64 == 0) {                                        \
    const int kb = (K) <= 256 ? 0 : ((K) <= 1040 ? 1 : 2);  \
    const long long dt = clock64() - tq;                    \
    xs.prof[group][i] += dt, xs.prof[group][(j) + kb] += dt; \
  }                                                         \
  tq = clock64();
#else
#define X_PROF_BEGIN()
#define X_PROF(i)
#define X_PROF_COUNT(i)
#define X_PROF_BIN(i, j, K)
#define X_PROF_KBIN(i, j, K)
#endif
constexpr int kXT = NVB_WAVEX_THREADS;
constexpr int kXG = kXT / 64;
constexpr int kRecInts = 32;      // candidate record: [0] slot, [1..27] its 3x3x3 neighbour slots, [28..31] unused (128-byte records)
constexpr int kMaxCtas = 192;     // per-CTA flags
constexpr int kRX = 110, kRY = 11;  // region voxel index = rx * 110 + ry * 11 + rz, rx, ry, rz in 0..9 (block voxel + 1)
constexpr int kRegionVox = 1100;
constexpr int kFlagBase = 4 * kRegionVox;        // word offset of the flag plane
constexpr int kXRegionWords = (kEsdfCellWords + 1) * kRegionVox;  // the two planes: 5 500 words = 22 000 bytes per group
constexpr size_t kXSmemBytes = (size_t)kXG * kXRegionWords * sizeof(unsigned int);
// Exchange-slab slot: the block's six faces (+x,-x,+y,-y,+z,-z), 64 voxels each in the order of the halo batches (face f, voxel
// (c1, c2) of the two other axes in axis order at index f * 64 + c1 * 8 + c2), as a plane of 16-byte cells {squared distance,
// parent} followed by a plane of flag words: 7.5 KiB instead of the layer's 10 KiB block, and the interior, which no halo
// reads, is not written at all.
constexpr int kXFaceCells = 6 * 64;
constexpr int kXFlagOff = kXFaceCells * 16;           // byte offset of the flag plane in a slot
constexpr int kXSlotBytes = kXFaceCells * (16 + 4);  // 7 680
#if NVB_WAVEX_PROF
constexpr int kXProfWords = 24;  // counters per group, copied to phase_max[kXProfBase ..] (tools/wavex_profile.py)
constexpr int kXProfBase = kPhaseMaxEntries - kXProfWords;
#endif

struct XTables {
  unsigned int halo[8][64];     // halo voxel copies: dst voxel | src cell in its block's exchange-slab slot << 11 | d27 << 20 | valid << 25
  unsigned int pair[6][4][64];  // boundary pairs per pass: src voxel | dst voxel << 11 | d27 of the source block << 22 | inner << 27 | valid << 28
};

struct XShared {
  int rec[kXG][kRecInts];  // the record of the candidate each group is working on
  int nb[kXG][8];          // face neighbours (+x,-x,+y,-y,+z,-z) of the block being registered from
  int pos[kXG][8];         // position won for that neighbour in this CTA's segment, -1: somebody else registered it
  unsigned int mask[kXG];
  int changed[kXG];
  unsigned int live[kXG][8];  // per pass: source blocks whose pairs are replayed (liveMasks)
  int seg[kXG][2];         // where the group's entry lives: registering CTA, index in its segment
  int pre[kMaxCtas + 1];   // exclusive scan of the per-CTA registration counts of the current ring
  int warp_tot[2][8];
  int ncand, nchanged;     // this CTA's registrations / changed blocks in the ring it is processing
  int next;                // next unclaimed entry of this CTA's share of the ring (groups pull work: a changed candidate costs
                           // twice an unchanged one, a static deal left groups with two changed ones on the critical path)
  int cur[kXG];
  int seeds[kXG];  // length of the seed list being processed (per group: written and read across the group's barriers)
  int bcast[4];
  // Per-launch state kept here rather than in registers: processCandidate / processSeed are real calls, and whatever the
  // kernel keeps live across them is saved to the stack at every call.
  unsigned int generation;  // grid-barrier generation (thread 0)
  int n_bar;                // grid barriers passed in this launch
  int ring;                 // the ring being processed (written by thread 0 between two CTA barriers)
  int swept, faces, rings, n_tail;  // statistics (thread 0)
  int n_split, n_rest;              // statistics: candidates fetched split, rest-of-block fetches (lane 0 of each group)
#if NVB_WAVEX_PROF
  // per group, cycles: [0] record, [1] stamps (+ own block when not split; + speculative faces), [2] halo (+ the own block's
  // live planes when split), [3] replay, [4] sweep (+ registration), [5] stores; [6] candidates, [7] changed; [8] rest of
  // the block (issue + registerBegin + wait; changed candidates); [9..11] [1] by K bin, [12..14] candidates by K bin,
  // [15..17] [2] by K bin, [18..20] [5] by K bin
  long long prof[kXG][kXProfWords];
#endif
};

// What the per-candidate functions need of the kernel parameter, in shared memory: they are real calls (one copy of the code for
// the grid rings and the single-CTA tail), and a reference to a kernel parameter would be copied to the stack at every call.
struct XCtx {
  unsigned char* blocks;  // the ESDF layer's slab
  int* block_index;
  DevHash hash;
  int* nbr;
  int* nbr27;
  int* cand_stamp;
  unsigned int* psum;     // per slot: box of the block offsets the voxels' parents point into (clear-pass pruning)
  int* stamp[2];          // member stamps by ring parity
  unsigned char* X[2];    // exchange slabs by ring parity
  int* recs[2];           // candidate records by ring parity: one segment of `seg` records per CTA
  int seg;
  int split_min_k;        // grid rings with at least this many candidates fetch the own block split (processCandidate)
  int* error;             // bit 8: a registration did not fit its CTA's segment (dropped, the launch's result is invalid)
  float max_sq;
  __device__ __forceinline__ int* segment(int p, int cta) const { return recs[p] + (size_t)cta * seg * kRecInts; }
};

// The kernel's shared state lives at namespace scope: the per-candidate functions address it directly (32-bit shared
// addresses folded into the instructions) instead of receiving generic pointers that would occupy registers for the whole call.
__shared__ XTables x_tab;
__shared__ XShared x_xs;
__shared__ XCtx x_ctx;
extern __shared__ __align__(16) unsigned int x_smem[];  // kXG regions of kXRegionWords

__device__ __forceinline__ int rvox(int rx, int ry, int rz) { return rx * kRX + ry * kRY + rz; }
__device__ __forceinline__ int faceEntry(int f) {  // +x,-x,+y,-y,+z,-z -> index into a 3x3x3 row
  return f == 0 ? 22 : (f == 1 ? 4 : (f == 2 ? 16 : (f == 3 ? 10 : (f == 4 ? 14 : 12))));
}
__device__ __forceinline__ int boundaryOff(int r) { return r == 0 ? -1 : (r == 9 ? 1 : 0); }   // region coordinate -> block offset
__device__ __forceinline__ int boundaryLoc(int r) { return r == 0 ? 7 : (r == 9 ? 0 : r - 1); }  // ... and voxel coordinate in that block

// nbr27 entry of `slot` towards offset d (0..26), resolving "never linked" entries (blocks created outside the ESDF
// update path) through the hash once.
__device__ __forceinline__ int neighbor27(const XCtx& c, int slot, int d) {
  int v = __ldcg(c.nbr27 + 27 * slot + d);
  if (v < -1) {
    const int* bi = c.block_index + 3 * slot;
    v = (d == 13) ? slot : hashFind(c.hash, bi[0] + d / 9 - 1, bi[1] + (d / 3) % 3 - 1, bi[2] + d % 3 - 1);
    c.nbr27[27 * slot + d] = v;
  }
  return v;
}
// face neighbour of `slot` (+x,-x,+y,-y,+z,-z), same resolution rule
__device__ __forceinline__ int neighbor6(const XCtx& c, int slot, int dir) {
  int v = __ldcg(c.nbr + 6 * slot + dir);
  if (v < -1) {
    const int* bi = c.block_index + 3 * slot;
    const int d = (dir & 1) ? -1 : 1;
    v = hashFind(c.hash, bi[0] + ((dir >> 1) == 0 ? d : 0), bi[1] + ((dir >> 1) == 1 ? d : 0), bi[2] + ((dir >> 1) == 2 ? d : 0));
    c.nbr[6 * slot + dir] = v;
  }
  return v;
}

// Per-launch tables (the same for every candidate).
__device__ __forceinline__ void initTables(XTables& tab, int tid) {
  // ---- halo copies. Batches 0..5: the six faces (+x,-x,+y,-y,+z,-z), one voxel per lane, so a batch is live or dead for the
  // whole group; lane l of batch k reads cell l of the opposite face (k ^ 1) of its block's slot, so a batch is 1 KiB of
  // contiguous cells and 256 bytes of contiguous flags. Batches 6, 7: edges and corners, each read from one face of its block
  // that holds it (an edge voxel from the face across the first other axis, a corner from the x face).
  for (int i = tid; i < 512; i += kXT) {
    const int k = i >> 6, lane = i & 63;
    unsigned int e = 0;
    int ra = 1, r1 = 1, r2 = 1, axis = 0;  // region coordinates: along `axis`, and the two others in axis order
    int fa = 0;                            // axis of the face the voxel is read from
    bool valid = true;
    if (k < 6) {
      axis = k >> 1, fa = axis;
      ra = (k & 1) ? 0 : 9, r1 = (lane >> 3) + 1, r2 = (lane & 7) + 1;
    } else {
      const int n = i - 384;
      if (n < 96) {  // 12 edges x 8 voxels
        const int edge = n >> 3, cn = edge & 3;
        axis = edge >> 2, fa = axis == 0 ? 1 : 0;
        ra = (n & 7) + 1, r1 = (cn & 1) ? 9 : 0, r2 = (cn & 2) ? 9 : 0;
      } else if (n < 104) {
        const int cn = n - 96;
        ra = (cn & 1) ? 9 : 0, r1 = (cn & 2) ? 9 : 0, r2 = (cn & 4) ? 9 : 0;
      } else {
        valid = false;
      }
    }
    if (valid) {
      const int rx = axis == 0 ? ra : r1, ry = axis == 0 ? r1 : (axis == 1 ? ra : r2), rz = axis == 2 ? ra : r2;
      const int d = (boundaryOff(rx) + 1) * 9 + (boundaryOff(ry) + 1) * 3 + (boundaryOff(rz) + 1);
      const int lx = boundaryLoc(rx), ly = boundaryLoc(ry), lz = boundaryLoc(rz);  // voxel coordinates in block d
      const int lf = fa == 0 ? lx : (fa == 1 ? ly : lz), l1 = fa == 0 ? ly : lx, l2 = fa == 2 ? ly : lz;  // on / across the face
      const int cell = (2 * fa + (lf == 0 ? 1 : 0)) * 64 + l1 * 8 + l2;
      e = (unsigned)rvox(rx, ry, rz) | ((unsigned)cell << 11) | ((unsigned)d << 20) | (1u << 25);
    }
    tab.halo[k][lane] = e;
  }
  // ---- boundary pairs. Slot 0 / 1: the 8x8 interior of the two boundary planes of the pass (one source block each, so the
  // slot is live or dead for the whole group); slots 2, 3: the 2 x 36 border pairs (sources in edge / corner blocks).
  for (int i = tid; i < 6 * 4 * 64; i += kXT) {
    const int pass = i >> 8, j = (i >> 6) & 3, lane = i & 63;
    const int axis = pass >> 1, dir = (pass & 1) ? -1 : 1;
    int plane, u, w;
    bool valid = true;
    if (j < 2) {
      plane = j, u = (lane >> 3) + 1, w = (lane & 7) + 1;
    } else {
      const int n = (j - 2) * 64 + lane;
      plane = n / 36;
      const int q = n % 36;
      if (q < 10) u = 0, w = q;
      else if (q < 20) u = 9, w = q - 10;
      else if (q < 28) u = q - 20 + 1, w = 0;
      else u = q - 28 + 1, w = 9;
      if (n >= 72) valid = false, plane = 0, u = 1, w = 1;
    }
    unsigned int e = 0;
    if (valid) {
      const int sa = dir > 0 ? (plane ? 8 : 0) : (plane ? 9 : 1);  // source coordinate along the axis
      const int so = dir > 0 ? (plane ? 0 : -1) : (plane ? 1 : 0);  // block offset of the source along the axis
      const int da = sa + dir;
      const int A = axis == 0 ? 9 : (axis == 1 ? 3 : 1), U = axis == 0 ? 3 : 9, W = axis == 2 ? 3 : 1;
      const int d = 13 + so * A + boundaryOff(u) * U + boundaryOff(w) * W;
      const int inner = da >= 1 && da <= 8 && u >= 1 && u <= 8 && w >= 1 && w <= 8;
      const int sv = axis == 0 ? rvox(sa, u, w) : (axis == 1 ? rvox(u, sa, w) : rvox(u, w, sa));
      const int dv = axis == 0 ? rvox(da, u, w) : (axis == 1 ? rvox(u, da, w) : rvox(u, w, da));
      e = (unsigned)sv | ((unsigned)dv << 11) | ((unsigned)d << 22) | ((unsigned)inner << 27) | (1u << 28);
    }
    tab.pair[pass][j][lane] = e;
  }
}

// Which source blocks are live in each pass, and which neighbours have to be fetched at all (see the header): bit d of
// live[p] <=> the pairs of pass p whose source block is d are replayed.
struct LiveMasks {
  unsigned int* live;   // [6], in shared memory (indexed by a run-time pass number)
  unsigned int needed;  // members (without B) that take part in a live pair
  unsigned int axes;    // bit a: a pass along axis a is live (liveAxes)
};
__device__ __forceinline__ LiveMasks liveMasks(unsigned int mask, unsigned int* live_smem, bool writer) {
  LiveMasks L;
  L.live = live_smem;
  const unsigned int ok = mask | (1u << 13);  // destinations that matter at all: B or a member
  // D(p+1): blocks whose state after pass p can still reach B; bit d = (dx+1)*9 + (dy+1)*3 + (dz+1)
  const unsigned int D[6] = {0x7FFFE00u, 0x3FE00u, 0x3F000u, 0x7000u, 0x6000u, 0x2000u};
  unsigned int acc = 0;
  L.axes = 0;
#pragma unroll
  for (int p = 0; p < 6; p++) {
    const int axis = p >> 1;
    const int A = axis == 0 ? 9 : (axis == 1 ? 3 : 1);
    const unsigned int lo = axis == 0 ? 0x000001ffu : (axis == 1 ? 0x001c0e07u : 0x01249249u);  // blocks at offset -1 along the axis
    const unsigned int dst_ok = ok & D[p];
    unsigned int lv, dst;
    if ((p & 1) == 0) {  // +dir: sources at offset -1, 0; destination = source + A
      lv = mask & (lo | (lo << A)) & (dst_ok >> A);
      dst = lv << A;
    } else {  // -dir: sources at offset 0, +1; destination = source - A
      lv = mask & ((lo << A) | (lo << (2 * A))) & (dst_ok << A);
      dst = lv >> A;
    }
    if (writer) live_smem[p] = lv;
    if (lv) L.axes |= 1u << axis;
    acc |= lv | dst;
  }
  L.needed = acc & mask & ~(1u << 13);
  return L;
}

// ---- the candidate's own block: one z-row per lane (its 8 cells and its 8 flag words as two 16-byte vectors), through
// registers into the two planes
struct OwnRegs {
  uint4 cell[8];
  uint4 flag[2];
};
__device__ __forceinline__ OwnRegs ownLoad(const unsigned char* blk, int lane64) {
  OwnRegs o;
  const unsigned int* b = reinterpret_cast<const unsigned int*>(blk);
#pragma unroll
  for (int z = 0; z < 8; z++) o.cell[z] = __ldcg(reinterpret_cast<const uint4*>(esdfCell(b, lane64 * 8 + z)));
#pragma unroll
  for (int h = 0; h < 2; h++) o.flag[h] = __ldcg(reinterpret_cast<const uint4*>(esdfFlag(b, lane64 * 8 + 4 * h)));
  return o;
}
__device__ __forceinline__ unsigned int liveAxes(const unsigned int* live) {  // bit a: a pass along axis a is live
  return ((live[0] | live[1]) ? 1u : 0u) | ((live[2] | live[3]) ? 2u : 0u) | ((live[4] | live[5]) ? 4u : 0u);
}
__device__ __forceinline__ void ownToShared(unsigned int* R, const OwnRegs& o, int lane64) {
  uint4* A = reinterpret_cast<uint4*>(R);
  const int v0 = rvox((lane64 >> 3) + 1, (lane64 & 7) + 1, 1);
#pragma unroll
  for (int z = 0; z < 8; z++) A[v0 + z] = o.cell[z];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    R[kFlagBase + v0 + 4 * h] = o.flag[h].x, R[kFlagBase + v0 + 4 * h + 1] = o.flag[h].y;
    R[kFlagBase + v0 + 4 * h + 2] = o.flag[h].z, R[kFlagBase + v0 + 4 * h + 3] = o.flag[h].w;
  }
}
// inner 8x8x8 of the region -> the block in the layer (if `to_layer`), and its six faces -> its slot in an exchange slab, one
// cell and one flag word per lane and face. The block goes in eight steps of one cell and one flag word per lane, warp w of
// the group taking voxels 256 w + 32 k + lane (x = 4 w + k / 2): each warp store is 512 contiguous bytes of cells and 128 of
// flags. On the way the box of the BLOCK OFFSETS the voxels' parents point into is collected and published in c.psum
// (EsdfCtx::psum; one word per warp of the group, so no barrier is needed): the clear pass of later updates reads a
// candidate block only if that box contains a to-clear block.
__device__ __forceinline__ void ownStore(unsigned char* layer_blk, bool to_layer, unsigned char* x_slot, const unsigned int* R,
                                         unsigned int* psum_slot, int lane64) {
  const uint4* A = reinterpret_cast<const uint4*>(R);
  const int x = lane64 >> 3, y = lane64 & 7;
  unsigned int* dl = reinterpret_cast<unsigned int*>(layer_blk);
  uint4* xc = reinterpret_cast<uint4*>(x_slot) + lane64;
  unsigned int* xf = reinterpret_cast<unsigned int*>(x_slot + kXFlagOff) + lane64;
#pragma unroll
  for (int f = 0; f < 6; f++) {  // face f: region coordinate 8 (+) or 1 (-) along f's axis, lane = c1 * 8 + c2 (halo batch order)
    const int fa = f >> 1, p = (f & 1) ? 1 : 8;
    const int v = fa == 0 ? rvox(p, x + 1, y + 1) : (fa == 1 ? rvox(x + 1, p, y + 1) : rvox(x + 1, y + 1, p));
    __stcg(xc + f * 64, A[v]);
    __stcg(xf + f * 64, R[kFlagBase + v]);
  }
  int lo0 = 99, lo1 = 99, lo2 = 99, hi0 = -99, hi1 = -99, hi2 = -99;
  const int w = lane64 >> 5, l = lane64 & 31;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int vx = 4 * w + (k >> 1), vy = ((k & 1) << 2) + (l >> 3), vz = l & 7;
    const int v = (vx * kVps + vy) * kVps + vz, rv = rvox(vx + 1, vy + 1, vz + 1);
    const uint4 a = A[rv];
    if (to_layer) {
      __stcg(reinterpret_cast<uint4*>(esdfCell(dl, v)), a);
      __stcg(esdfFlag(dl, v), R[kFlagBase + rv]);
    }
    if ((a.y | a.z | a.w) != 0u) {
      const int b0 = (vx + (int)a.y) >> 3, b1 = (vy + (int)a.z) >> 3, b2 = (vz + (int)a.w) >> 3;  // floor: arithmetic shift
      lo0 = min(lo0, b0), hi0 = max(hi0, b0), lo1 = min(lo1, b1), hi1 = max(hi1, b1), lo2 = min(lo2, b2), hi2 = max(hi2, b2);
    }
  }
  if (psum_slot) {
    lo0 = __reduce_min_sync(0xffffffffu, lo0), lo1 = __reduce_min_sync(0xffffffffu, lo1), lo2 = __reduce_min_sync(0xffffffffu, lo2);
    hi0 = __reduce_max_sync(0xffffffffu, hi0), hi1 = __reduce_max_sync(0xffffffffu, hi1), hi2 = __reduce_max_sync(0xffffffffu, hi2);
    if ((lane64 & 31) == 0) psum_slot[lane64 >> 5] = parentBoxWord(lo0, hi0, lo1, hi1, lo2, hi2);
  }
}

// ---- halo voxels, as cp.async copies straight into the two region planes -- the 16-byte cell and the flag word of a voxel
// from its block's exchange-slab slot: no registers are held across the wait (the register version held up to 20 words per
// lane and spilled at 96 registers). Only the batches of the members in a live pair are fetched, after the stamps. The cells
// travel .cg, through L2 only. The flag words (here and in ownAsync) are 4-byte copies, which have no .cg form,
// so they go .ca. The L1 lines those leave behind cannot go stale unnoticed: every grid barrier ends with an acquire
// (gridBarrierRA), which invalidates the SM's L1, and within the single-CTA tail the writer is this SM.
__device__ __forceinline__ void cpAsync4(unsigned int* smem_dst, const unsigned int* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned int)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cpAsyncCell(unsigned int* smem_dst, const void* gsrc) {  // 16 bytes, both 16-byte aligned
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned int)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
// ---- the own block split in two (grid rings, processCandidate): first the voxels on the boundary planes of
// the axes `axes` (bit a: the planes 0 and 7 along axis a), which hold every voxel of B the replay reads or writes, then -- only
// if B changed -- the rest. One voxel per lane and x plane (lane = y * 8 + z), as its 16-byte cell (.cg) and its flag word
// (.ca): a warp's copies cover 512 contiguous bytes of cells and 128 of flags. `planes`: copy the voxels on those planes,
// else every other voxel. (.ca: the layer's blocks are written with .cg stores by the owners of earlier rings, and the grid
// barrier between them and this read invalidates the SM's L1; the single-CTA tail does not fetch split.)
__device__ __forceinline__ void ownAsync(unsigned int* R, const unsigned char* blk, int lane64, unsigned int axes, bool planes) {
  const int y = lane64 >> 3, z = lane64 & 7;
  const bool lane_on = ((axes & 2u) && (y == 0 || y == 7)) || ((axes & 4u) && (z == 0 || z == 7));
  const unsigned int* b = reinterpret_cast<const unsigned int*>(blk);
  const int v0 = rvox(1, y + 1, z + 1);
#pragma unroll
  for (int x = 0; x < 8; x++) {
    const bool on = lane_on || ((axes & 1u) && (x == 0 || x == 7));
    if (on == planes) {
      const int v = x * 64 + lane64, rv = v0 + x * kRX;
      cpAsyncCell(R + 4 * rv, esdfCell(b, v));
      cpAsync4(R + kFlagBase + rv, esdfFlag(b, v));
    }
  }
}
// Halo batches `batches` (bit k: batch k of the table), the voxels whose block d has bit d in `blocks` and is allocated.
__device__ __forceinline__ void haloAsync(const XTables& tab, unsigned int* R, const int* row, const unsigned char* X, int lane64,
                                          unsigned int batches, unsigned int blocks) {
#pragma unroll 1
  while (batches) {  // group-uniform
    const int k = __ffs(batches) - 1;
    batches &= batches - 1;
    const unsigned int e = tab.halo[k][lane64];
    const int d = (e >> 20) & 31u;
    const int slot = ((e >> 25) & 1u) && ((blocks >> d) & 1u) ? row[d] : -1;
    if (slot >= 0) {
      const unsigned char* xslot = X + (size_t)slot * kXSlotBytes;
      const int cell = (e >> 11) & 511u, v = e & 2047u;
      cpAsyncCell(R + 4 * v, xslot + 16 * cell);
      cpAsync4(R + kFlagBase + v, reinterpret_cast<const unsigned int*>(xslot + kXFlagOff) + cell);
    }
  }
}
// faces in batch order: +x,-x,+y,-y,+z,-z = blocks 22, 4, 16, 10, 14, 12; everything else is an edge or corner block (batches 6, 7)
constexpr unsigned int kFaceBlocks = (1u << 22) | (1u << 4) | (1u << 16) | (1u << 10) | (1u << 14) | (1u << 12);
__device__ __forceinline__ unsigned int haloBatches(unsigned int needed) {
  unsigned int bl = ((needed >> 22) & 1u) | (((needed >> 4) & 1u) << 1) | (((needed >> 16) & 1u) << 2) | (((needed >> 10) & 1u) << 3) |
                    (((needed >> 14) & 1u) << 4) | (((needed >> 12) & 1u) << 5);
  if (needed & ~kFaceBlocks) bl |= 0xC0u;
  return bl;
}

// ---- the six passes of updateLocalNeighborBands (:1323-1386) restricted to the pairs that matter, updateSingleNeighbor
// (:602-633) per pair. Inside one pass sources and destinations are disjoint planes, so its pairs are independent.
// The loops are NOT unrolled and the pass is a run-time value: a candidate executes this code once, and straight-line code
// that is executed once is fetched from L2 (the first version, six unrolled passes, spent a quarter of its samples waiting for
// instructions).
__device__ __forceinline__ bool replayX(const XTables& tab, unsigned int* R, const LiveMasks& L, int lane64, int group,
                                        float max_sq) {
  uint4* A = reinterpret_cast<uint4*>(R);
  const unsigned int* live_p = L.live;
  bool changed = false;
#pragma unroll 1
  for (int pass = 0; pass < 6; pass++) {
    const unsigned int live = live_p[pass];
    if (!live) continue;  // group-uniform
    const int axis = pass >> 1, dir = (pass & 1) ? -1 : 1;
    const int s0 = axis == 0 ? dir : 0, s1 = axis == 1 ? dir : 0, s2 = axis == 2 ? dir : 0;
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
      unsigned int e = tab.pair[pass][j][lane64];
      if (!((e >> 28) & 1u) || !((live >> ((e >> 22) & 31u)) & 1u)) e = 0;
      if (__any_sync(0xffffffffu, e != 0u)) {  // slots 0 and 1 are live or dead for the whole group
        const int sv = e & 2047u, dv = (e >> 11) & 2047u;  // (voxel 0 for a dead lane: any valid address)
        const uint4 es = A[sv], ns = A[dv];
        const unsigned int ef = R[kFlagBase + sv], nf = R[kFlagBase + dv];
        const bool ok = e != 0u && flagObserved(ef) && flagObserved(nf) && !flagSite(nf) && !(__uint_as_float(es.x) >= max_sq);
        const int d0 = (int)es.y - s0, d1 = (int)es.z - s1, d2 = (int)es.w - s2;
        const float pdist = (float)(d0 * d0 + (d1 * d1 + d2 * d2));
        if (ok && __uint_as_float(ns.x) > pdist) {
          A[dv] = make_uint4(__float_as_uint(pdist), (unsigned)d0, (unsigned)d1, (unsigned)d2);
          changed = changed || ((e >> 27) & 1u);
        }
      }
    }
    groupSync(group);
  }
  return changed;
}

// ---- sweepSingleBand (:542-600) for one line of the block, on registers. AXIS is the line's direction; (a, b) are the two
// other voxel coordinates in axis order. Written for few instructions on a short loop-carried chain (a block's sweep is
// 3 axes x 16 sequential steps on two warps: what it costs is instructions x issue latency):
//   * the running site of the scan is kept RELATIVE TO THE LINE: la = its offset along the line, (lo1, lo2) = its two
//     perpendicular components (constant along the line), lp2 = lo1^2 + lo2^2; its squared distance to the voxel at `pos`
//     is (la - pos)^2 + lp2 and that voxel's new parent (la - pos, lo1, lo2);
//   * squared distances are exact integers (or max_sq), so "sq > n" is the integer test ceil(sq) > n;
//   * "no site seen yet" is lp2 = 2^28 (never closer than anything), "voxel cannot be improved" (unobserved or a site) is
//     ceil(sq) := INT_MIN, so the reference's test `found && observed && !site && sq > d` is ONE compare;
//   * a voxel that offers a site to the scan -- a site itself (offer = its own position: its parent registers are zeroed) or an
//     observed voxel with a valid distance (offer = its parent) -- has its bit in `tk`; the reference's four cases become
//     `improve` and `take = tk && !improve`.
// Chain per voxel: subtract, multiply-add, compare, predicate, select. Forward pass, then backward over the updated registers.
// One copy per axis (compile-time AXIS, unrolled passes) instead of a run-time axis with rolled passes keeps that chain short.
template <int AXIS>
__device__ __forceinline__ bool sweepLineX(unsigned int* R, int a, int b, float max_sq) {
  uint4* A = reinterpret_cast<uint4*>(R);
  const int v0 = AXIS == 0 ? rvox(1, a + 1, b + 1) : (AXIS == 1 ? rvox(a + 1, 1, b + 1) : rvox(a + 1, b + 1, 1));
  constexpr int stride = AXIS == 0 ? kRX : (AXIS == 1 ? kRY : 1);
  constexpr int kNone = 1 << 28, kCap = 1 << 27;
  int T[kVps], pa[kVps], po1[kVps], po2[kVps], pp2[kVps];
  unsigned int tk = 0, dirty = 0;
#pragma unroll
  for (int i = 0; i < kVps; i++) {
    const uint4 q = A[v0 + i * stride];
    const unsigned int fl = R[kFlagBase + v0 + i * stride];
    const float sq = __uint_as_float(q.x);
    const bool o = flagObserved(fl), st = flagSite(fl);
    const int t = min(__float2int_ru(sq), kCap);
    T[i] = (o && !st) ? t : INT_MIN;
    const int qa = (int)(AXIS == 0 ? q.y : (AXIS == 1 ? q.z : q.w));
    const int q1 = (int)(AXIS == 0 ? q.z : q.y);
    const int q2 = (int)(AXIS == 2 ? q.z : q.w);
    pa[i] = st ? 0 : qa, po1[i] = st ? 0 : q1, po2[i] = st ? 0 : q2;
    pp2[i] = po1[i] * po1[i] + po2[i] * po2[i];
    if (o && (st || sq < max_sq)) tk |= 1u << i;
  }
#pragma unroll
  for (int pass = 0; pass < 2; pass++) {
    int la = 0, lo1 = 0, lo2 = 0, lp2 = kNone;
#pragma unroll
    for (int kk = 0; kk < kVps; kk++) {
      const int k = pass ? (kVps - 1 - kk) : kk;  // line position
      const int t = la - k;
      const int pd = t * t + lp2;
      const bool improve = T[k] > pd;  // the running site is closer than the voxel's value
      const bool take = ((tk >> k) & 1u) && !improve;
      const int offer_a = pa[k] + k;
      if (improve) {
        T[k] = pd, pa[k] = t, po1[k] = lo1, po2[k] = lo2, pp2[k] = lp2;
        dirty |= 1u << k;  // (pd < old sq <= max_sq: the voxel now has a valid distance ...
      }
      la = take ? offer_a : la;
      lo1 = take ? po1[k] : lo1;
      lo2 = take ? po2[k] : lo2;
      lp2 = take ? pp2[k] : lp2;
    }
    tk |= dirty;  // ... and offers its parent to the backward scan)
  }
#pragma unroll
  for (int i = 0; i < kVps; i++) {
    if ((dirty >> i) & 1u) {
      const unsigned int x = (unsigned)(AXIS == 0 ? pa[i] : po1[i]);
      const unsigned int y = (unsigned)(AXIS == 0 ? po1[i] : (AXIS == 1 ? pa[i] : po2[i]));
      const unsigned int z = (unsigned)(AXIS == 2 ? pa[i] : po2[i]);
      A[v0 + i * stride] = make_uint4(__float_as_uint((float)T[i]), x, y, z);
    }
  }
  return dirty != 0;
}
// sweepBlockBandKernel (:1390-1431) for the block in the region: x lines, y lines, z lines.
__device__ __forceinline__ bool sweepBlockX(unsigned int* R, int group, int lane64, float max_sq) {
  const int a = lane64 >> 3, b = lane64 & 7;
  bool ch = sweepLineX<0>(R, a, b, max_sq);
  groupSync(group);
  ch |= sweepLineX<1>(R, a, b, max_sq);
  groupSync(group);
  ch |= sweepLineX<2>(R, a, b, max_sq);
  return ch;
}

// Registration of the face neighbours of a block that is a member of ring `target` as candidates of that ring, in three
// steps so that the atomic and the neighbours' rows travel while the block is swept (nothing consumes their results before
// registerFinish):
//   begin : atomicExch on the candidates' stamps (unique registration) + prefetch of their 3x3x3 rows,
//   claim : positions in this CTA's segment for the registrations this group won (shared-memory counter),
//   finish: write the records {slot, row}.
// xs.nb[group][0..5] holds the six face neighbours (slot or < 0).
struct RegState {
  int old;    // lanes 0..5: previous stamp of the neighbour
  int pos;    // lanes 0..5: position won in the CTA's segment, -1: somebody else registered it
  int v[3];   // row entries (w, d) = ((lane + 64 k) / 27, (lane + 64 k) % 27) of the six neighbours
};
__device__ __forceinline__ RegState registerBegin(const XCtx& c, XShared& xs, int group, int lane64, int target) {
  RegState s;
  s.old = target, s.pos = -1;
  if (lane64 < 6) {
    const int nb = xs.nb[group][lane64];
    if (nb >= 0) s.old = atomicExch(c.cand_stamp + nb, target);
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int idx = lane64 + 64 * k;
    s.v[k] = -1;
    if (idx < 162) {
      const int nb = xs.nb[group][idx / 27];
      if (nb >= 0) s.v[k] = __ldcg(c.nbr27 + 27 * nb + idx % 27);  // consumed in registerFinish: stays in flight
    }
  }
  return s;
}
__device__ __forceinline__ void registerClaim(const XCtx& c, XShared& xs, RegState& s, int group, int lane64, int target) {
  if (lane64 < 32) {  // the group's first warp
    const bool win = lane64 < 6 && xs.nb[group][lane64] >= 0 && s.old != target;
    const unsigned int ballot = __ballot_sync(0xffffffffu, win);
    if (ballot) {
      int base = 0;
      if (lane64 == 0) base = atomicAdd(&xs.ncand, __popc(ballot));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (win) s.pos = base + __popc(ballot & ((1u << lane64) - 1u));
      // Never write past the segment (the next CTA's records follow it): the registration is dropped and reported.
      if (s.pos >= c.seg) {
        s.pos = -1;
        atomicOr(c.error, 8);
      }
    }
  }
}
__device__ __forceinline__ void registerFinish(const XCtx& c, XShared& xs, const RegState& s, int group, int lane64,
                                               int* segment) {
  if (lane64 < 6) xs.pos[group][lane64] = s.pos;
  groupSync(group);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int idx = lane64 + 64 * k;
    if (idx < 162) {
      const int w = idx / 27, pos = xs.pos[group][w];
      if (pos >= 0) {
        int v = s.v[k];
        if (v < -1) v = neighbor27(c, xs.nb[group][w], idx % 27);  // never linked: resolve through the hash once
        __stcg(segment + (size_t)pos * kRecInts + 1 + idx % 27, v);
      }
    }
  }
  if (lane64 < 6 && s.pos >= 0) __stcg(segment + (size_t)s.pos * kRecInts, xs.nb[group][lane64]);
}

// One candidate of ring `ring`: gather, replay, and if it changed: sweep, publish, register its neighbours for ring+1.
// The entry is xs.seg[group] (registering CTA, index in its segment); the group is the caller's (threadIdx.x / 64).
// K: the ring's candidate count, -1 in the single-CTA tail. A grid ring with K >= c.split_min_k fetches the own block SPLIT:
// right after a grid barrier every group of every CTA asks for a 10 KiB block at once, and most candidates do not change
// (they outnumber the members 2.5-3.5x), so the candidate first fetches only the boundary planes of B along the live passes'
// axes, with the halo, after the stamps; the rest of B follows only if B changed, with registerBegin's atomics and row loads.
__device__ __noinline__ void processCandidate(int ring, int K) {
  const XCtx& c = x_ctx;
  const XTables& tab = x_tab;
  XShared& xs = x_xs;
  const int cta = blockIdx.x, group = threadIdx.x >> 6, lane64 = threadIdx.x & 63;
  unsigned int* R = x_smem + group * kXRegionWords;
  const int ci = ring & 1, ni = ci ^ 1;
  const bool split = K >= c.split_min_k;
  X_PROF_BEGIN()
  if (lane64 < 28) xs.rec[group][lane64] = __ldcg(c.segment(ci, xs.seg[group][0]) + (size_t)xs.seg[group][1] * kRecInts + lane64);
  groupSync(group);
  X_PROF(0)
  const int slot = xs.rec[group][0];
  const int* row = &xs.rec[group][1];
  const unsigned char* blk = c.blocks + (size_t)slot * kEsdfBlockBytes;
  // membership of the 27 blocks in this ring (sources of the passes); the loads travel with the loads of the own block (when
  // not split)
  int sv = ring - 1;
  if (lane64 < 27 && row[lane64] >= 0) sv = __ldcg(c.stamp[ci] + row[lane64]);
  if (split) {
    const unsigned int m = __ballot_sync(0xffffffffu, lane64 < 27 && sv == ring);
    if (lane64 == 0) xs.mask[group] = m, xs.changed[group] = 0;
  } else {
    OwnRegs own = ownLoad(blk, lane64);
    const unsigned int m = __ballot_sync(0xffffffffu, lane64 < 27 && sv == ring);
    if (lane64 == 0) xs.mask[group] = m, xs.changed[group] = 0;
    ownToShared(R, own, lane64);
  }
  groupSync(group);
  const LiveMasks L = liveMasks(xs.mask[group], xs.live[group], lane64 == 0);
  X_PROF_BIN(1, 9, K)
  // the halo of the members that take part in a live pair, and when split, B's boundary planes along the live passes' axes
  if (split) {
    ownAsync(R, blk, lane64, L.axes, true);
    if (lane64 == 0) atomicAdd(&xs.n_split, 1);
  }
  if (L.needed) haloAsync(tab, R, row, c.X[ci], lane64, haloBatches(L.needed), L.needed);  // group-uniform
  if (L.needed || split) cpAsyncWaitAll();
  groupSync(group);  // (also publishes xs.live[group], written by lane 0 in liveMasks and read by every lane in replayX)
  X_PROF_KBIN(2, 15, K)
  const bool ch = replayX(tab, R, L, lane64, group, c.max_sq);
  if (ch) xs.changed[group] = 1;
  groupSync(group);
  X_PROF(3)
  X_PROF_COUNT(6)
  if (xs.changed[group]) {
    // B is a member of ring+1
    if (lane64 < 6) xs.nb[group][lane64] = row[faceEntry(lane64)];
    if (lane64 == 0) {
      __stcg(c.stamp[ni] + slot, ring + 1);
      atomicAdd(&xs.nchanged, 1);
    }
    groupSync(group);
    if (split) ownAsync(R, blk, lane64, liveAxes(xs.live[group]), false);  // the rest of B (the replay wrote only the planes)
    RegState rs = registerBegin(c, xs, group, lane64, ring + 1);
    if (split) {
      if (lane64 == 0) atomicAdd(&xs.n_rest, 1);
      cpAsyncWaitAll();
      groupSync(group);
    }
    X_PROF(8)
    sweepBlockX(R, group, lane64, c.max_sq);
    registerClaim(c, xs, rs, group, lane64, ring + 1);
    groupSync(group);
    X_PROF(4)
    ownStore(c.blocks + (size_t)slot * kEsdfBlockBytes, true, c.X[ni] + (size_t)slot * kXSlotBytes, R, c.psum + 2 * (size_t)slot, lane64);
    registerFinish(c, xs, rs, group, lane64, c.segment(ni, cta));
    X_PROF_COUNT(7)
  }
  groupSync(group);
  X_PROF_KBIN(5, 18, K)
}

// A member of the initial list of a computeEsdf call (ring `ring`): sweep in place, publish, register its neighbours as
// the candidates of this ring.
__device__ __noinline__ void processSeed(int ring, int slot) {
  const XCtx& c = x_ctx;
  XShared& xs = x_xs;
  const int cta = blockIdx.x, group = threadIdx.x >> 6, lane64 = threadIdx.x & 63;
  unsigned int* R = x_smem + group * kXRegionWords;
  const int ci = ring & 1;
  unsigned char* blk = c.blocks + (size_t)slot * kEsdfBlockBytes;
  OwnRegs own = ownLoad(blk, lane64);
  if (lane64 < 6) xs.nb[group][lane64] = neighbor6(c, slot, lane64);
  if (lane64 == 0) {
    __stcg(c.stamp[ci] + slot, ring);
    xs.changed[group] = 0;
  }
  groupSync(group);
  RegState rs = registerBegin(c, xs, group, lane64, ring);
  ownToShared(R, own, lane64);
  groupSync(group);
  const bool ch = sweepBlockX(R, group, lane64, c.max_sq);
  registerClaim(c, xs, rs, group, lane64, ring);
  if (ch) xs.changed[group] = 1;
  groupSync(group);
  // (an unchanged block keeps its parent box)
  ownStore(blk, xs.changed[group] != 0, c.X[ci] + (size_t)slot * kXSlotBytes, R, xs.changed[group] ? c.psum + 2 * (size_t)slot : nullptr, lane64);
  registerFinish(c, xs, rs, group, lane64, c.segment(ci, cta));
  groupSync(group);
}

// Grid barrier with a release arrival and acquire polling: the same ordering as gridBarrier's two __threadfences (the CTA's
// writes, gathered by the __syncthreads, are released by thread 0's arrival; its acquire load of the final count makes every
// CTA's writes visible, and invalidates the SM's L1), without the heavier sequentially-consistent fences.
__device__ __forceinline__ void gridBarrierRA(unsigned int* bar, unsigned int& generation, unsigned int nctas) {
  __syncthreads();
  if (threadIdx.x == 0) {
    generation++;
    const unsigned int target = generation * nctas;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
    } while (v < target);
  }
  __syncthreads();
}

// Grid barrier + all-gather of the per-CTA counts {registrations, changed blocks}; leaves the exclusive scan of the
// registrations in xs.pre and returns the totals: counts stored to per-CTA slots (two arrays by barrier parity), fence, atomic
// arrival counter polled by thread 0, fence, then one read of the per-CTA slots. (The alternative -- one flag per CTA, every
// CTA polling every other CTA's flag -- needs no read-modify-write on a shared word but grows with the square of the grid.)
__device__ __forceinline__ void counterBarrierScan(XShared& xs, unsigned int* bar, unsigned int& generation, int2* counts, int nctas,
                                                   int cta, int tid, int seg, int ring_inc, int* K, int* M) {
  // Barrier number xs.n_bar selects the parity of the count slots. Every thread reads it here, before the CTA barrier below;
  // thread 0 advances it (and the ring) just before the last CTA barrier of this function, when nobody reads it any more.
  counts += (xs.n_bar & 1) * kMaxCtas;
  __syncthreads();
  if (tid == 0) {
    __stcg(counts + cta, make_int2(min(xs.ncand, seg), xs.nchanged));  // (registrations past the segment were dropped)
    xs.ncand = 0, xs.nchanged = 0;
  }
  gridBarrierRA(bar, generation, nctas);
  int2 v = make_int2(0, 0);
  if (tid < nctas) v = __ldcg(counts + tid);
  const int lane = tid & 31, warp = tid >> 5;
  int inc = v.x, chg = v.y;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) chg += __shfl_xor_sync(0xffffffffu, chg, o);
  if (warp < 8 && lane == 31) xs.warp_tot[0][warp] = inc;
  if (warp < 8 && lane == 0) xs.warp_tot[1][warp] = chg;
  __syncthreads();
  int base = 0, mtot = 0;
#pragma unroll
  for (int w = 0; w < 8; w++) {
    if (w < warp) base += xs.warp_tot[0][w];
    if (w * 32 < nctas) mtot += xs.warp_tot[1][w];
  }
  if (tid < nctas) xs.pre[tid + 1] = base + inc;
  if (tid == 0) xs.pre[0] = 0, xs.next = 0, xs.ring += ring_inc, xs.n_bar++;
  __syncthreads();
  *K = xs.pre[nctas];
  *M = mtot;
}

__global__ void __maxnreg__(NVB_WAVEX_MAXREG) esdfWaveXKernel(EsdfCtx c) {
  XShared& xs = x_xs;
  const int cta = blockIdx.x, nctas = gridDim.x;
  const int tid = threadIdx.x, group = tid >> 6, lane64 = tid & 63;
  // Empty block list: integrateBlocksTemplate returns before touching anything (:226-228).
  if (*(volatile int*)c.work_count == 0) return;
  initTables(x_tab, tid);
  if (tid == 0) {
    xs.ncand = 0, xs.nchanged = 0, xs.next = 0;
    xs.ring = *(volatile int*)c.ring_id;
    xs.generation = 0, xs.n_bar = 0, xs.swept = 0, xs.faces = 0, xs.rings = 0, xs.n_tail = 0, xs.n_split = 0, xs.n_rest = 0;
    XCtx& xc = x_ctx;
    xc.blocks = c.esdf.blocks, xc.block_index = c.esdf.block_index, xc.hash = c.esdf.hash;
    xc.nbr = c.nbr, xc.nbr27 = c.nbr27, xc.cand_stamp = c.cand_stamp, xc.psum = c.psum;
    xc.stamp[0] = c.stamp_a, xc.stamp[1] = c.stamp_b;
    xc.X[0] = c.xslab, xc.X[1] = c.xslab + (size_t)c.esdf.capacity * kXSlotBytes;
    xc.recs[0] = c.xrec, xc.recs[1] = c.xrec + (size_t)nctas * c.xseg * kRecInts;
    xc.seg = c.xseg, xc.split_min_k = c.xsplit_min_k, xc.error = c.error, xc.max_sq = c.max_sq;
  }
#if NVB_WAVEX_PROF
  if (lane64 < kXProfWords) xs.prof[group][lane64] = 0;
#endif
  __syncthreads();
#if NVB_WAVEX_PROF
  long long t_bar = 0, t_work = 0, t0 = globalTimerNs(), t1;
  int dbgK = 0, dbgM = 0;
#define X_DBG(k, m) dbgK = (k), dbgM = (m);
#define X_TIME_WORK()                                                                                                      \
  t1 = globalTimerNs(), t_work += t1 - t0;                                                                                 \
  if (tid == 0 && xs.n_bar < 1000) atomicMax((unsigned long long*)c.phase_max + xs.n_bar, (unsigned long long)(t1 - t0)); \
  if (cta == 0 && tid == 0 && xs.n_bar < 1000)                                                                             \
    c.phase_max[1000 + xs.n_bar] = dbgK, c.phase_max[2000 + xs.n_bar] = dbgM, c.phase_max[3000 + xs.n_bar] = t1 - t0;      \
  t0 = t1;
#define X_TIME_BARRIER() t1 = globalTimerNs(), t_bar += t1 - t0, t0 = t1;
#else
#define X_DBG(k, m)
#define X_TIME_WORK()
#define X_TIME_BARRIER()
#endif
  // Barrier number xs.n_bar of this launch: publishes what this CTA registered / changed in the phase, returns the totals and
  // leaves the exclusive scan of the registrations in xs.pre.
// `inc`: the ring advances by that much with the barrier.
#define X_BARRIER(inc, Kout, Mout)                                                                                        \
  X_TIME_WORK()                                                                                                           \
  counterBarrierScan(xs, c.barrier, xs.generation, reinterpret_cast<int2*>(c.xcounts), nctas, cta, tid, c.xseg, inc,        \
                     &(Kout), &(Mout));                                                                                   \
  X_TIME_BARRIER()
  for (int pass = 0; pass < 2; pass++) {
    // pass 0: blocks with sites; pass 1: the persistent cleared list (:254-257)
    const int* src = pass ? c.cleared_list : c.upd_list;
    const int n0 = pass ? *(volatile int*)c.cleared_count : *(volatile int*)c.upd_count;
    if (n0 == 0) continue;
    // ---- seeds: the call's block list is ring xs.ring
    X_DBG(-1, n0)
    if (lane64 == 0) xs.seeds[group] = n0;  // (n0 itself would be saved to the stack around every processSeed call)
    for (;;) {
      if (lane64 == 0) xs.cur[group] = atomicAdd(&xs.next, 1);
      groupSync(group);
      const long long e = (long long)cta + (long long)xs.cur[group] * nctas;
      if (e >= xs.seeds[group]) break;
      processSeed(xs.ring, __ldcg(src + e));
    }
    int M = xs.seeds[group], K, unused;
    X_BARRIER(0, K, unused)  // K: candidates of ring xs.ring
    if (tid == 0) xs.swept += M;
    while (true) {
      X_DBG(K, M)
      if (NVB_WAVEX_TAIL && K <= kXG) {
        // ---- tail: the ring fits one CTA. CTA 0 runs whole rings with block-level barriers until the wavefront dies out
        // or outgrows it (its registrations all land in its own segment); everybody else waits at ONE grid barrier.
        if (cta == 0) {
          int t = 0;
          if (group < K) {  // where the (at most 8) entries of the current ring live
            for (int s = lane64; s < nctas; s += 64)
              if (xs.pre[s] <= group && group < xs.pre[s + 1]) xs.seg[group][0] = s, xs.seg[group][1] = group - xs.pre[s];
          }
          __syncthreads();
          while (true) {
            if (group < K) processCandidate(xs.ring, -1);
            __syncthreads();
            const int K2 = min(xs.ncand, c.xseg), M2 = xs.nchanged;
            __syncthreads();
            if (tid == 0) xs.ncand = 0, xs.nchanged = 0, xs.faces += 6 * M, xs.rings++, xs.swept += M2, xs.ring++;
            if (tid < kXG) xs.seg[tid][0] = 0, xs.seg[tid][1] = tid;  // the next ring's entries: segment 0, in order
            t++;
            M = M2, K = K2;
            __syncthreads();
            if (M == 0 || K > kXG) break;
          }
          if (tid == 0) xs.n_tail += t, c.xtail[0] = t, c.xtail[1] = K, c.xtail[2] = M;
        }
        {
          int k_unused, m_unused;  // (the tail's counts travel through xtail: CTA 0 alone registered)
          X_BARRIER(0, k_unused, m_unused)
        }
        if (cta != 0) {
          if (tid == 0) xs.bcast[0] = __ldcg(c.xtail + 0), xs.bcast[1] = __ldcg(c.xtail + 1), xs.bcast[2] = __ldcg(c.xtail + 2);
          __syncthreads();
          K = xs.bcast[1], M = xs.bcast[2];
          if (tid == 0) xs.ring += xs.bcast[0];
          __syncthreads();
        }
        if (M == 0) break;
        // the K candidates of the current ring were all registered by CTA 0
        for (int s = tid; s <= nctas; s += kXT) xs.pre[s] = s == 0 ? 0 : K;
        __syncthreads();
        continue;
      }
      // ---- grid ring: candidates dealt round-robin over CTAs, then over the CTA's groups. The loop reads K from xs.pre[nctas]
      // (= K) rather than a register: whatever it keeps live across processCandidate is saved to the stack at every call.
      for (;;) {
        if (lane64 == 0) xs.cur[group] = atomicAdd(&xs.next, 1);
        groupSync(group);
        const long long e = (long long)cta + (long long)xs.cur[group] * nctas;
        if (e >= xs.pre[nctas]) break;
        for (int s = lane64; s < nctas; s += 64)
          if (xs.pre[s] <= e && e < xs.pre[s + 1]) xs.seg[group][0] = s, xs.seg[group][1] = (int)e - xs.pre[s];
        groupSync(group);
        processCandidate(xs.ring, xs.pre[nctas]);
      }
      int K2, M2;
      X_BARRIER(1, K2, M2)
      if (tid == 0) xs.faces += 6 * M, xs.rings++, xs.swept += M2;
      M = M2, K = K2;
      if (M == 0) break;
    }
    if (tid == 0) xs.ring++;  // the next computeEsdf call's stamps must not alias this one's
    __syncthreads();
  }
#undef X_BARRIER
#undef X_TIME_WORK
#undef X_TIME_BARRIER
#undef X_DBG
  if (tid == 0 && xs.n_split) {  // (the counts are final: the last ring ended with a CTA barrier)
    atomicAdd((unsigned long long*)&c.stats[kStatSplitCandidates], (unsigned long long)xs.n_split);
    atomicAdd((unsigned long long*)&c.stats[kStatRestFetches], (unsigned long long)xs.n_rest);
  }
  if (cta == 0 && tid == 0) {
    *c.ring_id = xs.ring + 1;
    c.stats[kStatCleared] = *(volatile int*)c.cleared_count;
    c.stats[kStatSwept] = xs.swept, c.stats[kStatFaces] = xs.faces, c.stats[kStatRings] = xs.rings;
    c.stats[kStatTailRings] = xs.n_tail, c.stats[kStatBarriers] = xs.n_bar;
#if NVB_WAVEX_PROF
    c.stats[kStatBarrierNs] = t_bar, c.stats[kStatWorkNs] = t_work;
    long long sum_max = 0;
    for (int q = 0; q < xs.n_bar && q < 1000; q++) sum_max += (long long)c.phase_max[q];
    c.stats[kStatSlowestCtaWorkNs] = sum_max;
    for (int q = 0; q < kXProfWords; q++) c.phase_max[kXProfBase + q] = xs.prof[0][q];
#endif
  }
}

}  // namespace

int esdfWaveXGrid(int num_sms, int reserved_sms) {
  int grid = num_sms < kMaxCtas ? num_sms : kMaxCtas;
  if (reserved_sms > 0 && grid - reserved_sms >= 8) grid -= reserved_sms;
  return grid;
}
size_t esdfWaveXFlagBytes() { return 2 * (size_t)kMaxCtas * sizeof(int2); }
size_t esdfWaveXSlabBytes(int capacity) { return 2 * (size_t)capacity * kXSlotBytes; }

// Grid rings with at least this many candidates fetch their candidates' own blocks split (processCandidate). 0: every grid
// ring (K > 8; the single-CTA tail and the seeds fetch whole blocks). 80-frame c2 bench on one H100 SXM at a 700 W power
// limit, two runs each: threshold 0 / 256 / 1 040 / never -> 2 835, 2 833 / 2 811, 2 814 / 2 732, 2 723 / 2 651, 2 582 frames/s.
constexpr int kSplitMinK = 0;
int esdfWaveXSplitMinK() {
  // Test hook: NVB_WAVEX_SPLIT_MIN_K=<n> replaces kSplitMinK (0: every grid ring fetches split, 1000000000: none does).
  const char* e = getenv("NVB_WAVEX_SPLIT_MIN_K");
  const int v = e ? atoi(e) : kSplitMinK;
  return v < 0 ? 0 : v;
}

cudaError_t launchEsdfComputeX(const EsdfCtx& c, int num_sms, int reserved_sms, cudaStream_t stream, int* launches) {
  static int per_sm = -1;
  if (per_sm < 0) {
    cudaFuncSetAttribute(esdfWaveXKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kXSmemBytes);
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, esdfWaveXKernel, kXT, kXSmemBytes) != cudaSuccess) v = 0;
    per_sm = v;
  }
  if (per_sm <= 0) return cudaErrorLaunchOutOfResources;
  EsdfCtx cc = c;
  void* args[] = {&cc};
  (*launches)++;
  // `reserved_sms` SMs are left to the other resident kernels: the raycast / compaction / TSDF kernels of the next frame then
  // run there instead of stealing issue slots from ring-critical CTAs (80-frame C2 bench on one H100 SXM at a 400 W power
  // limit, nvb_mapper_set_esdf_reserved_sms = 0 / 2 / 4 / 8, two runs each: 2367, 2339 / 2404, 2407 / 2399, 2378 / 2379, 2336 frames/s),
  // and a multi-GPU rank's NCCL all-gather can start -- and wait for its peers -- while a wavefront is in flight (a
  // cooperative grid that fills every SM serialises the two).
  const int grid = esdfWaveXGrid(num_sms, reserved_sms);
  return cudaLaunchCooperativeKernel((const void*)esdfWaveXKernel, dim3(grid), dim3(kXT), args, kXSmemBytes, stream);
}

}  // namespace nvb
