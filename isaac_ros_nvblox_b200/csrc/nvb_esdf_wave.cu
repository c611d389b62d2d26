// nvb_esdf_wave.cu -- the ESDF wavefront (computeEsdf, nvblox/src/integrators/esdf_integrator.cu:1465-1496)
// as ONE cooperative persistent launch.
//
// computeEsdf(list): sweep(list); while (list not empty) { list = updateNeighborBands(list); sweep(list); }
// runs twice per update: for the blocks with sites and for the persistent "cleared" list (:254-257).
// The result depends on the order of the passes (x,y,z in-block sweeps; +x,-x,+y,-y,+z,-z face propagation,
// each seeing the previous ones), so that order is kept: per ring three axis phases and one sweep phase,
// separated by grid barriers.
//
// What a phase costs is the SLOWEST CTA's dependent chain plus a grid barrier, ~18 rings x 4 phases per
// frame. The design therefore minimises round trips and
// imbalance per phase, not bytes:
//   * Ring membership is a per-slot stamp (stamp[r & 1][slot] == r): the face operations test "is my
//     neighbour a member of this ring" with one load that travels with the voxel loads.
//   * Ring r+1's member list is built unique with atomicExch on that stamp. Updated blocks are first recorded
//     in shared memory during the three axis phases and appended once per ring (two dependent L2 atomics per
//     ring instead of per phase); a warp reserves its list range with one atomicAdd. No sort/unique launch.
//   * Members are dealt round-robin from the list (CTA c takes entries c, c+G, ...): every CTA gets
//     ceil(n/G) blocks. (Static slot ownership was tried first: it was far from balanced, and the slowest CTA sets the pace.)
//     A CTA keeps its members and their six neighbour slots (nbr table, built at allocation) in shared
//     memory for the three axis phases: an axis phase is ONE L2 round trip (face voxels + neighbour stamp).
//   * The +dir/-dir passes of an axis are fused per block interface (exact, see axisMembers): 3 phases, not 6;
//     one warp per interface, two face voxels per lane, no block-level synchronisation inside the phase.
//   * A block's three-axis sweep is a ~2 000-instruction dependent chain on two warps; it runs on registers
//     with an integer, branch-free formulation (sweepLineRegs).
//   * 256-thread CTAs with up to 128 registers (half an SM's register file) so that the next frame's
//     raycast / compaction / TSDF kernels co-reside while the wavefront runs on its side stream.
#include "nvb_esdf_wave_common.cuh"

namespace nvb {

namespace {

#ifndef NVB_WAVE_THREADS
#define NVB_WAVE_THREADS 256
#endif
constexpr int kWT = NVB_WAVE_THREADS;   // threads per CTA. Design reasoning, not measured on the H100: the phase time is one block's
                                        // dependent chain rather than the thread count, and 1024 threads would cap registers at 64
                                        // (spills). 256 x 128 registers = half of an SM's register file, so the next frame's kernels
                                        // co-reside.
constexpr int kWG = kWT / 64;           // groups of 64 threads
constexpr size_t kWaveSmemBytes = waveSmemBytes<kWT>();
constexpr size_t kGesSmemBytes = gesSmemBytes<kWT>();
using WaveSharedT = WaveShared<kWT>;
using GesSharedT = GesShared<kWT>;


__global__ void __maxnreg__(NVB_WAVE_MAXREG) esdfWaveKernel(EsdfCtx c) {
  extern __shared__ __align__(16) unsigned int smem[];
  __shared__ WaveSharedT sh;
  const int cta = blockIdx.x, nctas = gridDim.x;
  // Empty block list: integrateBlocksTemplate returns before touching anything (:226-228).
  if (*(volatile int*)c.work_count == 0) return;
  if (threadIdx.x == 0) sh.npend = 0;
  __syncthreads();
  unsigned int generation = 0;
  int ring = *(volatile int*)c.ring_id;
  int* stamp[2] = {c.stamp_a, c.stamp_b};
  int* list[2] = {c.ring_a, c.ring_b};
  long long swept = 0, faces = 0, rings = 0;
  // CTA 0 keeps a coarse time split (ns): barriers (incl. waiting for the slowest CTA), axis phases,
  // sweep phases
  long long t_bar = 0, t_axis = 0, t_sweep = 0, n_bar = 0, t0 = globalTimerNs(), t1;
#define NVB_TICK(acc)   \
  t1 = globalTimerNs(); \
  acc += t1 - t0;       \
  t0 = t1;
  // every CTA: duration of its own work in the phase that ends at barrier #n_bar -> max over CTAs
  long long tw0 = globalTimerNs();
#define NVB_PHASE_MAX()                                                                                   \
  if (threadIdx.x == 0 && n_bar < 1000) {                                                                 \
    atomicMax((unsigned long long*)c.phase_max + n_bar, (unsigned long long)(globalTimerNs() - tw0));     \
  }
#define NVB_PHASE_BEGIN() tw0 = globalTimerNs();
#define NVB_BARRIER(acc)                      \
  NVB_TICK(acc)                               \
  NVB_PHASE_MAX()                             \
  gridBarrier(c.barrier, generation, nctas);  \
  NVB_TICK(t_bar)                             \
  n_bar++;                                    \
  NVB_PHASE_BEGIN()
  auto share = [&](int count) { return (count > cta) ? (count - cta + nctas - 1) / nctas : 0; };
  auto roundsOf = [&](int count) { return ((count + nctas - 1) / nctas + kWaveMaxMembers - 1) / kWaveMaxMembers; };
  for (int pass = 0; pass < 2; pass++) {
    // pass 0: blocks with sites; pass 1: the persistent cleared list (:254-257)
    int n = pass ? *(volatile int*)c.cleared_count : *(volatile int*)c.upd_count;
    if (n == 0) continue;
    int ci = ring & 1;
    const int* cur = pass ? c.cleared_list : c.upd_list;  // the first ring's members are read straight from the source list
    bool initial = true;  // members of `cur` still have to be stamped as ring `ring`
    int spec = 0;         // leading entries of this CTA's share already in sh.members (speculative fetch)
    // Loop invariant: the n members of `cur` (ring `ring`) have received their face updates and wait for their sweep.
    while (n > 0) {
      const int ni = ci ^ 1;
      if (kTail > 0 && n <= kTail) {
        // ---- tail mode: the ring fits one CTA. CTA 0 runs whole rings (sweep, three axis phases, hand-over) with
        // block-level synchronisation only, until the wavefront dies out or outgrows the tail; everybody else
        // waits at ONE grid barrier. A ring costs its dependent chain instead of chain + 4 barriers + the
        // list hand-over through L2.
        if (cta == 0) {
          int t = 0, tn = n, tci = ci, tring = ring;
          int k = loadMembers(sh, cur, tn, 0, 1, 0, initial ? stamp[tci] : nullptr, tring);
          while (true) {
            const int tni = tci ^ 1;
            sweepMembers(c, sh, k, smem, true);
            swept += k;
#pragma unroll 1
            for (int axis = 0; axis < 3; axis++) {
              axisMembers(c, sh, axis, k, stamp[tci], tring, stamp[tni], list[tni], c.ring_count + tni);
              __syncthreads();
            }
            faces += 6ll * k;
            rings++, t++;
            k = flushLocal(sh, stamp[tni], tring, list[tni]);
            tring++, tci = tni, tn = k;
            if (tn == 0 || tn > kTail) break;
          }
          if (threadIdx.x == 0) c.tail_state[0] = t, c.tail_state[1] = tn;
        }
        NVB_BARRIER(t_sweep)
        if (threadIdx.x == 0) sh.scan[0] = __ldcg(c.tail_state + 0), sh.scan[1] = __ldcg(c.tail_state + 1);
        __syncthreads();
        const int t = sh.scan[0];
        n = sh.scan[1];
        __syncthreads();
        ring += t;
        ci ^= (t & 1);
        cur = list[ci];
        initial = false, spec = 0;
        continue;
      }
      // ---- grid mode
      const int rounds = roundsOf(n);
      // sweep phase
      for (int r = 0; r < rounds; r++) {
        const int k = loadMembers(sh, cur, n, cta, nctas, r * kWaveMaxMembers, initial ? stamp[ci] : nullptr, ring,
                                  r == 0 ? spec : 0);
        sweepMembers(c, sh, k, smem, rounds == 1);
      }
      if (cta == 0 && threadIdx.x == 0) c.ring_count[ni] = 0;  // append counter of ring+1
      NVB_BARRIER(t_sweep)
      swept += n;
      // axis phases
#pragma unroll 1
      for (int axis = 0; axis < 3; axis++) {
        for (int r = 0; r < rounds; r++) {
          int k = share(n);
          if (rounds > 1) {
            k = loadMembers(sh, cur, n, cta, nctas, r * kWaveMaxMembers, nullptr, 0, 0);
            prefetchNeighbors(c, sh, k);
            __syncthreads();
          }
          axisMembers(c, sh, axis, k, stamp[ci], ring, stamp[ni], list[ni], c.ring_count + ni);
          if (rounds > 1) flushPending(sh, stamp[ni], ring, list[ni], c.ring_count + ni);
        }
        if (axis == 2 && rounds == 1) flushPending(sh, stamp[ni], ring, list[ni], c.ring_count + ni);
        NVB_BARRIER(t_axis)
      }
      faces += 6ll * n;
      rings++;
      // ring+1 = the blocks appended during the three axis phases. Its member count and the first entries of this
      // CTA's share are fetched in the same round trip (entries past the count are ignored).
      {
        const int j = threadIdx.x;
        const long long idx = (long long)cta + (long long)j * nctas;
        int e = 0;
        if (j < kSpec && idx < c.esdf.capacity) e = __ldcg(list[ni] + idx);
        const int n_next = *(volatile int*)(c.ring_count + ni);
        if (j < kSpec) sh.members[j] = e;
        spec = kSpec;
        __syncthreads();
        n = n_next;
      }
      ring++;
      ci = ni;
      cur = list[ni];
      initial = false;
    }
    ring++;
    if (cta == 0 && threadIdx.x == 0) c.ring_count[0] = c.ring_count[1] = 0;
    NVB_BARRIER(t_sweep)
  }
#undef NVB_TICK
  if (cta == 0 && threadIdx.x == 0) {
    *c.ring_id = ring + 1;
    c.stats[kStatCleared] = *(volatile int*)c.cleared_count;
    c.stats[kStatSwept] = swept, c.stats[kStatFaces] = faces, c.stats[kStatRings] = rings;
    c.stats[kStatBarrierNs] = t_bar, c.stats[kStatAxisNs] = t_axis, c.stats[kStatSweepNs] = t_sweep, c.stats[kStatBarriers] = n_bar;
    long long sum_max = 0;
    for (int q = 0; q < n_bar && q < 1000; q++) sum_max += (long long)c.phase_max[q];
    c.stats[kStatSlowestCtaWorkNs] = sum_max;
  }
}



__global__ void __maxnreg__(NVB_WAVE_MAXREG) esdfWaveGesKernel(EsdfCtx c) {
  extern __shared__ __align__(16) unsigned int smem[];
  __shared__ WaveSharedT sh;
  __shared__ GesSharedT gs;
  const int cta = blockIdx.x, nctas = gridDim.x;
  const int tid = threadIdx.x, group = tid >> 6, lane64 = tid & 63;
  if (*(volatile int*)c.work_count == 0) return;
  if (tid == 0) sh.npend = 0;
  if (tid < kWG) gs.done_n[tid] = 0;
  if (tid == 0) gs.overflow = 0;
  gesInitTables(gs, tid);
  __syncthreads();
  unsigned int generation = 0;
  int ring = *(volatile int*)c.ring_id;
  int* stamp[2] = {c.stamp_a, c.stamp_b};
  int* list[2] = {c.ring_a, c.ring_b};
  int* clist[2] = {c.cand_a, c.cand_b};
  int* ccount = c.ges_counts;      // [parity] candidates of the ring with that parity
  int* mcount = c.ges_counts + 2;  // [parity] members of the ring with that parity
  long long swept = 0, faces = 0, rings = 0, n_bar = 0, t_bar = 0, t_work = 0, t0 = globalTimerNs(), t1;
  unsigned int* R = smem + group * kRegionWords;
  long long tg = 0, te = 0, ts = 0, ncand = 0, nchg = 0, tq;  // CTA 0 / group 0: gather, emulate, sweep+store time (SM clock cycles: %globaltimer costs ~a round trip per read)
#define GES_BARRIER()                                                                                           \
  t1 = globalTimerNs(), t_work += t1 - t0;                                                                      \
  if (tid == 0 && n_bar < 1000) atomicMax((unsigned long long*)c.phase_max + n_bar, (unsigned long long)(t1 - t0)); \
  t0 = t1;                                                                                                      \
  gridBarrier(c.barrier, generation, nctas);                                                                    \
  t1 = globalTimerNs(), t_bar += t1 - t0, t0 = t1;                                                              \
  n_bar++;
  auto roundsOf = [&](int count) { return ((count + nctas - 1) / nctas + kWaveMaxMembers - 1) / kWaveMaxMembers; };
  for (int pass = 0; pass < 2; pass++) {
    const int* src = pass ? c.cleared_list : c.upd_list;
    int n0 = pass ? *(volatile int*)c.cleared_count : *(volatile int*)c.upd_count;
    if (n0 == 0) continue;
    int ci = ring & 1;
    bool initial = true;
    // ---- large rings: four-phase rings (sweep | x | y | z, member lists with unique append), exactly as in
    // esdfWaveKernel. A large ring has several candidates per 64-thread group, which the gather-replay below would
    // process one after the other; here the per-member work is smaller and the four barriers amortise.
    {
      auto share = [&](int count) { return (count > cta) ? (count - cta + nctas - 1) / nctas : 0; };
      int spec = 0;
      while (n0 > c.ges_switch) {
        const int ni = ci ^ 1;
        const int rounds = roundsOf(n0);
        for (int r = 0; r < rounds; r++) {
          const int k = loadMembers(sh, src, n0, cta, nctas, r * kWaveMaxMembers, initial ? stamp[ci] : nullptr, ring,
                                    r == 0 ? spec : 0);
          sweepMembers(c, sh, k, smem, rounds == 1);
        }
        if (cta == 0 && tid == 0) c.ring_count[ni] = 0;  // append counter of ring+1
        GES_BARRIER()
        swept += n0;
#pragma unroll 1
        for (int axis = 0; axis < 3; axis++) {
          for (int r = 0; r < rounds; r++) {
            int k = share(n0);
            if (rounds > 1) {
              k = loadMembers(sh, src, n0, cta, nctas, r * kWaveMaxMembers, nullptr, 0, 0);
              prefetchNeighbors(c, sh, k);
              __syncthreads();
            }
            axisMembers(c, sh, axis, k, stamp[ci], ring, stamp[ni], list[ni], c.ring_count + ni);
            if (rounds > 1) flushPending(sh, stamp[ni], ring, list[ni], c.ring_count + ni);
          }
          if (axis == 2 && rounds == 1) flushPending(sh, stamp[ni], ring, list[ni], c.ring_count + ni);
          GES_BARRIER()
        }
        faces += 6ll * n0;
        rings++;
        {
          const long long idx = (long long)cta + (long long)tid * nctas;
          int e = 0;
          if (tid < kSpec && idx < c.esdf.capacity) e = __ldcg(list[ni] + idx);
          const int n_next = *(volatile int*)(c.ring_count + ni);
          if (tid < kSpec) sh.members[tid] = e;
          spec = kSpec;
          __syncthreads();
          n0 = n_next;
        }
        ring++;
        ci = ni;
        src = list[ni];
        initial = false;
      }
      if (n0 == 0) {  // the wavefront died out in the large-ring regime
        ring++;
        if (cta == 0 && tid == 0) c.ring_count[0] = c.ring_count[1] = 0;
        GES_BARRIER()
        continue;
      }
    }
    // ---- hand-over / initial phase: sweep the current member list in place, stamp it as ring `ring`, register its
    // neighbours as the candidates of that ring
    {
      const int rounds = roundsOf(n0);
      for (int r = 0; r < rounds; r++) {
        const int k = loadMembers(sh, src, n0, cta, nctas, r * kWaveMaxMembers, stamp[ci], ring);
        sweepMembers(c, sh, k, smem, true);
        for (int q = tid; q < k * 6; q += kWT) {
          const int item = q / 6;
          const int nb = item < kNbrCache ? sh.nbr[q] : resolveNeighbor(c, sh.members[item], q % 6);
          if (nb >= 0 && atomicExch(c.cand_stamp + nb, ring) != ring) clist[ci][atomicAdd(ccount + ci, 1)] = nb;
        }
        __syncthreads();
      }
    }
    GES_BARRIER()
    swept += n0;
    int M = n0;
    int K_prev = 0;  // candidates of the previous ring (clist[ni])
    while (true) {
      const int ni = ci ^ 1;
      // ---- phase P: results of the previous ring go from the shadow slab into the layer (nobody reads the layer
      // now); this ring's candidates and their 27-neighbourhood rows come into shared memory
      const int K = *(volatile int*)(ccount + ci);
      const int share = (K > cta) ? (K - cta + nctas - 1) / nctas : 0;
      {
        const int kc = share < kGesMaxCand ? share : kGesMaxCand;
        int myslot = -1;
        if (tid < kc) myslot = __ldcg(clist[ci] + cta + tid * nctas);  // issued before the copies
        if (gs.overflow) {
          // more changed blocks than a group remembers: find them again through the previous ring's candidate
          // list (a candidate that became a member of ring `ring` is a changed block)
          for (int j = group; cta + (long long)j * nctas < K_prev; j += kWG) {
            const int s = __ldcg(clist[ni] + cta + j * nctas);
            if (__ldcg(stamp[ci] + s) == ring) copyShadowToLayer(c, s, lane64);
          }
        } else {
          for (int j = 0; j < gs.done_n[group]; j++) copyShadowToLayer(c, gs.done_slots[group][j], lane64);
        }
        __syncthreads();
        if (tid < kWG) gs.done_n[tid] = 0;
        if (tid == 0) gs.overflow = 0;
        if (tid < kc) gs.cand[tid] = myslot;
        __syncthreads();
        for (int q = tid; q < kc * 27; q += kWT) {
          const int s = gs.cand[q / 27], d = q % 27;
          int v = __ldcg(c.nbr27 + 27 * s + d);
          if (v < -1) {  // never linked (block created outside the ESDF update path): resolve through the hash once
            const int* bi = c.esdf.block_index + 3 * s;
            v = hashFind(c.esdf.hash, bi[0] + d / 9 - 1, bi[1] + (d / 3) % 3 - 1, bi[2] + d % 3 - 1);
            c.nbr27[27 * s + d] = v;
          }
          gs.rows[q] = v;
        }
        if (cta == 0 && tid == 0) ccount[ni] = 0, mcount[ni] = 0;  // filled during the coming phase A
      }
      GES_BARRIER()
      // ---- phase A: every candidate of the ring: gather, replay the six passes, sweep if it changed
      for (int base = 0; base < share; base += kGesMaxCand) {
        const int kc = (share - base) < kGesMaxCand ? (share - base) : kGesMaxCand;
        if (base > 0) {  // further chunks (very large rings only): fetch in place
          __syncthreads();
          if (tid < kc) gs.cand[tid] = __ldcg(clist[ci] + cta + (base + tid) * nctas);
          __syncthreads();
          for (int q = tid; q < kc * 27; q += kWT) {
            const int s = gs.cand[q / 27], d = q % 27;
            int v = __ldcg(c.nbr27 + 27 * s + d);
            if (v < -1) {
              const int* bi = c.esdf.block_index + 3 * s;
              v = hashFind(c.esdf.hash, bi[0] + d / 9 - 1, bi[1] + (d / 3) % 3 - 1, bi[2] + d % 3 - 1);
              c.nbr27[27 * s + d] = v;
            }
            gs.rows[q] = v;
          }
          __syncthreads();
        }
        for (int i = group; i < kc; i += kWG) {
          const int slot = gs.cand[i];
          const int* row = gs.rows + i * 27;
          // membership of the 27 blocks in this ring (sources of the passes); the loads travel with the gather
          int st = ring - 1;
          tq = clock64();
          if (lane64 < 27 && row[lane64] >= 0) st = __ldcg(stamp[ci] + row[lane64]);
          gesGather(c, gs, R, row, lane64);
          const unsigned int m = __ballot_sync(0xffffffffu, lane64 < 27 && st == ring);
          if (lane64 == 0) gs.mask[group] = m, gs.changed[group] = 0;
          groupSync(group);
          tg += clock64() - tq, tq = clock64(), ncand++;
          const bool ch = gesEmulate(gs, R, gs.mask[group], lane64, group, c.max_sq);
          if (ch) gs.changed[group] = 1;
          groupSync(group);
          te += clock64() - tq, tq = clock64();
          if (gs.changed[group]) {
            nchg++;
            // B is a member of ring+1: tell its face neighbours (candidates of ring+1). The exchange is issued
            // now and consumed after the sweep.
            int nb = -1, old = ring + 1;
            if (lane64 < 6) {
              const int face = lane64 == 0 ? 22 : (lane64 == 1 ? 4 : (lane64 == 2 ? 16 : (lane64 == 3 ? 10 : (lane64 == 4 ? 14 : 12))));
              nb = row[face];
              if (nb >= 0) old = atomicExch(c.cand_stamp + nb, ring + 1);
            }
            if (lane64 == 0) {
              stamp[ni][slot] = ring + 1;
              atomicAdd(mcount + ni, 1);
              const int dn = gs.done_n[group];
              if (dn < kGesDoneMax) gs.done_slots[group][dn] = slot, gs.done_n[group] = dn + 1;
              else gs.overflow = 1;
            }
            int pos = -1;
            {
              const int a = lane64 >> 3, b = lane64 & 7;
              sweepLineRegs(R, kRegionFlagWord0, regionVox(1, a + 1, b + 1), 80, 0, a, b, 0, c.max_sq);
              groupSync(group);
              // the exchange is back by now; the position fetch overlaps the other two axes
              if (nb >= 0 && old != ring + 1) pos = atomicAdd(ccount + ni, 1);
              sweepLineRegs(R, kRegionFlagWord0, regionVox(a + 1, 1, b + 1), 8, a, 0, b, 1, c.max_sq);
              groupSync(group);
              sweepLineRegs(R, kRegionFlagWord0, regionVox(a + 1, b + 1, 1), 1, a, b, 0, 2, c.max_sq);
              groupSync(group);
            }
            if (pos >= 0) clist[ni][pos] = nb;
            // inner 8x8x8 -> shadow slab
            unsigned int* dst = reinterpret_cast<unsigned int*>(c.shadow + (size_t)slot * kEsdfBlockBytes);
#pragma unroll
            for (int it = 0; it < 2; it++) {
              const int r = it * 32 + (lane64 >> 1), half = lane64 & 1;  // block z-row (lx, ly); two lanes share a row
              const int zr = ((r >> 3) + 1) * 10 + (r & 7) + 1;
#pragma unroll
              for (int j = 0; j < 4; j++)
                __stcg(reinterpret_cast<uint4*>(esdfCell(dst, r * 8 + 2 * j + half)),
                       *reinterpret_cast<const uint4*>(esdfCell(R, zr * 8 + 2 * j + half)));
              __stcg(reinterpret_cast<uint4*>(esdfFlag(dst, r * 8 + 4 * half)),
                     *reinterpret_cast<const uint4*>(R + kRegionFlagWord0 + zr * 8 + 4 * half));
            }
          }
          groupSync(group);
          ts += clock64() - tq;
        }
      }
      GES_BARRIER()
      const int M_next = *(volatile int*)(mcount + ni);
      faces += 6ll * M;
      rings++;
      swept += M_next;
      ring++;
      ci = ni;
      M = M_next;
      K_prev = K;
      if (M == 0) break;
    }
    ring++;
    if (cta == 0 && tid == 0) ccount[0] = ccount[1] = mcount[0] = mcount[1] = 0;
    GES_BARRIER()
  }
#undef GES_BARRIER
  if (cta == 0 && tid == 0) {
    *c.ring_id = ring + 1;
    c.stats[kStatCleared] = *(volatile int*)c.cleared_count;
    c.stats[kStatSwept] = swept, c.stats[kStatFaces] = faces, c.stats[kStatRings] = rings;
    c.stats[kStatBarrierNs] = t_bar, c.stats[kStatWorkNs] = t_work, c.stats[kStatSweepNs] = 0, c.stats[kStatBarriers] = n_bar;
    long long sum_max = 0;
    for (int q = 0; q < n_bar && q < 1000; q++) sum_max += (long long)c.phase_max[q];
    c.stats[kStatSlowestCtaWorkNs] = sum_max;
    c.phase_max[3990] = tg, c.phase_max[3991] = te, c.phase_max[3992] = ts, c.phase_max[3993] = ncand, c.phase_max[3994] = nchg;
  }
}

}  // namespace

int esdfPersistentMaxCtas(int num_sms) {
  static int per_sm = -1;
  if (per_sm < 0) {
    cudaFuncSetAttribute(esdfWaveKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWaveSmemBytes);
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, esdfWaveKernel, kWT, kWaveSmemBytes) != cudaSuccess) v = 0;
    per_sm = v;
  }
  return per_sm * num_sms;
}

cudaError_t launchEsdfComputeGes(const EsdfCtx& c, int num_sms, cudaStream_t stream, int* launches) {
  static int per_sm = -1;
  if (per_sm < 0) {
    cudaFuncSetAttribute(esdfWaveGesKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGesSmemBytes);
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, esdfWaveGesKernel, kWT, kGesSmemBytes) != cudaSuccess) v = 0;
    per_sm = v;
  }
  if (per_sm <= 0) return cudaErrorLaunchOutOfResources;
  EsdfCtx cc = c;
  void* args[] = {&cc};
  (*launches)++;
  return cudaLaunchCooperativeKernel((const void*)esdfWaveGesKernel, dim3(num_sms), dim3(kWT), args, kGesSmemBytes, stream);
}

cudaError_t launchEsdfComputePersistent(const EsdfCtx& c, int num_sms, cudaStream_t stream, int* launches) {
  const int max_ctas = esdfPersistentMaxCtas(num_sms);
  if (max_ctas <= 0) return cudaErrorLaunchOutOfResources;
  // One CTA per SM: the wavefront is latency-bound, more CTAs only make the barrier slower.
  int grid = num_sms < max_ctas ? num_sms : max_ctas;
  EsdfCtx cc = c;
  void* args[] = {&cc};
  (*launches)++;
  return cudaLaunchCooperativeKernel((const void*)esdfWaveKernel, dim3(grid), dim3(kWT), args, kWaveSmemBytes, stream);
}

}  // namespace nvb
