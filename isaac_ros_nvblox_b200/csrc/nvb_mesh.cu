// nvb_mesh.cu -- marching-cubes mesh of the TSDF layer (MeshIntegrator, mesh/mesh_integrator.h:39-162).
//
// Replaces MeshIntegrator::integrateBlocksGPU (nvblox/src/mesh/mesh_integrator.cu:66-108): isBlockMeshableKernel
// (:313-328), meshBlocksCalculateTableIndicesKernel (:335-452), meshBlocksCalculateVerticesKernel (:454-487),
// weldVerticesCubKernel (:691-803), and updateAppearanceBlockByClosestVoxel for the colour layer
// (mesh_integrator_appearance.cu:98-147).
//
// Kernel shape. The reference keeps one MeshBlock of four growable host-managed vectors per VoxelBlock, builds pointer
// tables on the host, parks a 140-byte PerVoxelMarchingCubesResults per voxel in global memory between its two kernels
// (72 KB per block) and synchronises the stream five times per call. Here the mesh lives in ONE device arena (vertices,
// normals, triangle indices, colours at the same offsets) with a 32-byte header per block in a slab + hash like every
// other layer; a call is
//   count  : one CTA per listed block stages the block and the faces of its 7 upper neighbours as a 9x9x9 (distance,
//            weight) grid in shared memory (5.8 KB, read once), classifies the 512 cubes and reduces their vertex counts;
//   scan   : one CTA turns the counts into arena offsets (the only number the host reads back: the total, to grow the
//            arena when it would overflow);
//   emit   : the same staging again (the TSDF is L2-resident; recomputing the cube is cheaper than the 72 KB round trip),
//            an in-block exclusive scan fixes every cube's output range, vertices + flat normals go straight to the arena;
//   weld   : per block, a bitonic sort of (quantised-position hash, index) pairs in shared memory, head flags, ranks.
// The reference hands out a cube's output range with an atomicAdd (marching_cubes_impl.cuh:11-29), so the order of a block's
// triangles is a race there; here cubes emit in x-major voxel order, which makes the whole mesh -- welded or not --
// bit-reproducible and lets the parity tests compare arrays instead of multisets.
#include "nvb_internal.cuh"
#include "nvb_mc_table.h"

#include <cfloat>

namespace nvb {

namespace {

struct McTables {
  signed char tri[256][16];  // edge numbers, -1 terminated
  unsigned char nverts[256];
};
constexpr int mcHex(char c) { return c <= '9' ? c - '0' : c - 'a' + 10; }
constexpr McTables makeMcTables() {
  McTables t{};
  for (int i = 0; i < 256; i++) {
    int c = 0;
    for (; kMcTriangles[i][c] != 0; c++) t.tri[i][c] = (signed char)mcHex(kMcTriangles[i][c]);
    t.nverts[i] = (unsigned char)c;
    for (; c < 16; c++) t.tri[i][c] = -1;
  }
  return t;
}
__constant__ McTables c_mc = makeMcTables();
__constant__ unsigned char c_edge_corners[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6},
                                                    {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};

constexpr int kMeshThreads = 256;
constexpr int kGrid = 9;  // voxels per side + the upper neighbours' first layer
constexpr int kGridCells = kGrid * kGrid * kGrid;

struct CubeShared {
  float2 g[kGridCells];  // (distance, weight); a missing neighbour block reads as weight = -inf
  int nb[8];             // TSDF slots of the block and its 7 upper neighbours (neighborIndexFromDirection order)
  int warp_sum[kMeshThreads / 32];
  int flag;
};

__device__ __forceinline__ int gridCell(int x, int y, int z) { return (x * kGrid + y) * kGrid + z; }

// Stage block `tslot` (index bx, by, bz) and its upper neighbours' faces.
__device__ __forceinline__ void stageCubeGrid(const MeshCtx& c, CubeShared& s, int tslot, int bx, int by, int bz, int tid) {
  if (tid < 8) {
    s.nb[tid] = tid == 0 ? tslot : hashFind(c.tsdf.hash, bx + ((tid >> 2) & 1), by + ((tid >> 1) & 1), bz + (tid & 1));
  }
  if (tid == 0) s.flag = 0;
  __syncthreads();
  for (int e = tid; e < kGridCells; e += kMeshThreads) {
    const int x = e / (kGrid * kGrid), y = (e / kGrid) % kGrid, z = e % kGrid;
    const int slot = s.nb[((x >> 3) << 2) | ((y >> 3) << 1) | (z >> 3)];
    float2 v = make_float2(0.0f, -INFINITY);
    if (slot >= 0)
      v = *reinterpret_cast<const float2*>(c.tsdf.blocks + (size_t)slot * kTsdfBlockBytes +
                                           (size_t)((((x & 7) << 3) | (y & 7)) << 3 | (z & 7)) * sizeof(float2));
    s.g[e] = v;
  }
  __syncthreads();
}

// calculateVertexConfiguration (marching_cubes_impl.h:6-15) of the cube at voxel (vx, vy, vz); -1 if a corner is missing or
// unobserved (mesh_integrator.cu:383-417).
__device__ __forceinline__ int cubeIndex(const MeshCtx& c, const CubeShared& s, int vx, int vy, int vz, float sdf[8]) {
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int ox = (i == 1 || i == 2 || i == 5 || i == 6), oy = (i == 2 || i == 3 || i == 6 || i == 7), oz = i >> 2;
    const float2 v = s.g[gridCell(vx + ox, vy + oy, vz + oz)];
    if (v.y < c.min_weight) return -1;
    sdf[i] = v.x;
    if (v.x < 0.0f) idx |= 1 << i;
  }
  return idx;
}

// Position of corner i of the cube (mesh_integrator.cu:423-426): block_position + voxel_size * (corner + 0.5 + 8 * block_offset)
__device__ __forceinline__ float cornerCoord(const MeshCtx& c, float block_pos, int v) {
  const int in = v & 7, off = v >> 3;
  return block_pos + c.voxel_size * (((float)in + 0.5f) + (float)(kVps * off));
}

// Exclusive scan of one value per thread over the CTA (256 threads); returns the exclusive prefix, *total = CTA sum.
__device__ __forceinline__ int blockExclusiveScan(CubeShared& s, int v, int tid, int* total) {
  const int lane = tid & 31, warp = tid >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s.warp_sum[warp] = inc;
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kMeshThreads / 32; w++) {
    const int ws = s.warp_sum[w];
    if (w < warp) base += ws;
    tot += ws;
  }
  __syncthreads();
  *total = tot;
  return base + inc - v;
}

__device__ __forceinline__ MeshHeader* meshHeader(const MeshCtx& c, int slot) {
  return reinterpret_cast<MeshHeader*>(c.mesh.blocks + (size_t)slot * kMeshHeaderBytes);
}

// Entry i of the call's list -> (index, TSDF slot). Lists are unique (a set in every caller).
__device__ __forceinline__ bool listEntry(const MeshCtx& c, int i, int* bx, int* by, int* bz, int* tslot) {
  if (c.todo.slots) {
    const int t = c.todo.slots[i];
    c.todo.dirty[t] = 0;  // this block's pending update is being consumed
    *bx = c.tsdf.block_index[3 * t], *by = c.tsdf.block_index[3 * t + 1], *bz = c.tsdf.block_index[3 * t + 2];
    *tslot = *bx == kDeadSlotX ? -1 : t;
  } else {
    *bx = c.in_xyz[3 * i], *by = c.in_xyz[3 * i + 1], *bz = c.in_xyz[3 * i + 2];
    *tslot = hashFind(c.tsdf.hash, *bx, *by, *bz);  // getIndicesInLayer (:53-64)
  }
  return *tslot >= 0;
}

// ---- count: clear the existing mesh block, meshability test, vertex count of the block.
__global__ void __launch_bounds__(kMeshThreads) meshCountKernel(MeshCtx c) {
  __shared__ CubeShared s;
  __shared__ int s_entry[4];
  const int n = c.todo.count ? *c.todo.count : c.in_count_host;
  const int tid = threadIdx.x;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    __syncthreads();
    if (tid == 0) {
      int bx, by, bz, tslot;
      listEntry(c, i, &bx, &by, &bz, &tslot);
      s_entry[0] = bx, s_entry[1] = by, s_entry[2] = bz, s_entry[3] = tslot;
      if (tslot >= 0) {
        // "Clear all blocks if they exist" (:80-87): the block stays allocated with empty vectors
        const int ms = hashFind(c.mesh.hash, bx, by, bz);
        if (ms >= 0) {
          MeshHeader* h = meshHeader(c, ms);
          if (h->cap) atomicAdd(c.arena_state + kArenaGarbage, h->cap);
          h->offset = 0, h->nv = 0, h->nt = 0, h->cap = 0, h->nc = 0;
        }
      }
    }
    __syncthreads();
    const int tslot = s_entry[3];
    if (tslot < 0) {
      if (tid == 0) c.counts[i] = 0;
      continue;
    }
    stageCubeGrid(c, s, tslot, s_entry[0], s_entry[1], s_entry[2], tid);
    // voxel pair of this thread: linear offsets 2 tid, 2 tid + 1 (x-major)
    const int vx = tid >> 5, vy = (tid >> 2) & 7, vz = (tid & 3) * 2;
    bool meshable = false;
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const float2 v = s.g[gridCell(vx, vy, vz + k)];
      meshable = meshable || (fabsf(v.x) <= c.cutoff_distance_m && v.y >= c.min_weight);  // isBlockMeshableKernel
      float sdf[8];
      const int idx = cubeIndex(c, s, vx, vy, vz + k, sdf);
      if (idx >= 0) cnt += c_mc.nverts[idx];
    }
    if (meshable) s.flag = 1;
    int total;
    blockExclusiveScan(s, cnt, tid, &total);
    if (tid == 0) c.counts[i] = s.flag ? total : 0;
  }
}

// ---- scan: counts -> arena offsets; reserves the range in the arena. One CTA.
__global__ void __launch_bounds__(1024) meshScanKernel(MeshCtx c) {
  __shared__ int warp_sum[32];
  __shared__ int carry;
  __shared__ long long base;
  const int n = c.todo.count ? *c.todo.count : c.in_count_host;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int first = 0; first < n; first += 1024) {
    const int i = first + tid;
    const int v = i < n ? c.counts[i] : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    int b = carry;
    for (int w = 0; w < warp; w++) b += warp_sum[w];
    if (i < n) c.offsets[i] = b + inc - v;
    __syncthreads();
    if (tid == 1023) carry = b + inc;
    __syncthreads();
  }
  if (tid == 0) {
    const int total = carry;
    const int used = c.arena_state[kArenaUsed];
    c.arena_state[kArenaLastTotal] = total;
    c.arena_state[kArenaLastBase] = used;
    // the host reads (base, total) before the emit kernel and grows / compacts the arena if base + total does not fit
    base = used;
  }
  __syncthreads();
  const int b = (int)base;
  for (int i = tid; i < n; i += 1024) c.offsets[i] += b;
}

// interpolateVertex (marching_cubes_impl.h:28-43) along cube edge e
__device__ __forceinline__ void edgeVertex(const float pos[8][3], const float sdf[8], int e, float out[3]) {
  const int c0 = c_edge_corners[e][0], c1 = c_edge_corners[e][1];
  const float sa = sdf[c0], sb = sdf[c1];
  const float diff = sa - sb;
  if (fabsf(diff) >= 1e-4f) {
    const float t = sa / diff;
#pragma unroll
    for (int j = 0; j < 3; j++) out[j] = pos[c0][j] + t * (pos[c1][j] - pos[c0][j]);
  } else {
#pragma unroll
    for (int j = 0; j < 3; j++) out[j] = 0.5f * (pos[c0][j] + pos[c1][j]);
  }
}

// ---- emit: vertices, flat normals and identity triangle indices of every listed block with a non-zero count.
__global__ void __launch_bounds__(kMeshThreads) meshEmitKernel(MeshCtx c) {
  __shared__ CubeShared s;
  __shared__ int s_entry[4];
  const int n = c.todo.count ? *c.todo.count : c.in_count_host;
  const int tid = threadIdx.x;
  if (blockIdx.x == 0 && tid == 0) c.arena_state[kArenaUsed] = c.arena_state[kArenaLastBase] + c.arena_state[kArenaLastTotal];
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int count = c.counts[i];
    if (count <= 0) continue;
    __syncthreads();
    if (tid == 0) {
      int bx, by, bz, tslot;
      if (c.todo.slots) {
        const int t = c.todo.slots[i];
        bx = c.tsdf.block_index[3 * t], by = c.tsdf.block_index[3 * t + 1], bz = c.tsdf.block_index[3 * t + 2], tslot = t;
      } else {
        bx = c.in_xyz[3 * i], by = c.in_xyz[3 * i + 1], bz = c.in_xyz[3 * i + 2];
        tslot = hashFind(c.tsdf.hash, bx, by, bz);
      }
      s_entry[0] = bx, s_entry[1] = by, s_entry[2] = bz, s_entry[3] = tslot;
      // allocateBlockAtIndexAsync (:603-611) + the vectors' resize
      bool was_new;
      const int ms = hashFindOrInsert(c.mesh, bx, by, bz, c.error, &was_new);
      if (ms >= 0) {
        MeshHeader* h = meshHeader(c, ms);
        h->offset = c.offsets[i], h->nv = count, h->nt = count, h->cap = count, h->nc = 0;
      }
    }
    __syncthreads();
    const int bx = s_entry[0], by = s_entry[1], bz = s_entry[2];
    stageCubeGrid(c, s, s_entry[3], bx, by, bz, tid);
    const int vx = tid >> 5, vy = (tid >> 2) & 7, vz = (tid & 3) * 2;
    int idx[2], cnt = 0;
    float sdf[2][8];
#pragma unroll
    for (int k = 0; k < 2; k++) {
      idx[k] = cubeIndex(c, s, vx, vy, vz + k, sdf[k]);
      if (idx[k] >= 0) cnt += c_mc.nverts[idx[k]];
    }
    int total;
    int next = c.offsets[i] + blockExclusiveScan(s, cnt, tid, &total);
    // getPositionFromBlockIndex: block_size * index
    const float bp[3] = {c.block_size * (float)bx, c.block_size * (float)by, c.block_size * (float)bz};
#pragma unroll 1
    for (int k = 0; k < 2; k++) {
      if (idx[k] <= 0 || idx[k] == 255) continue;
      float pos[8][3];
#pragma unroll
      for (int q = 0; q < 8; q++) {
        const int ox = (q == 1 || q == 2 || q == 5 || q == 6), oy = (q == 2 || q == 3 || q == 6 || q == 7), oz = q >> 2;
        pos[q][0] = cornerCoord(c, bp[0], vx + ox), pos[q][1] = cornerCoord(c, bp[1], vy + oy);
        pos[q][2] = cornerCoord(c, bp[2], vz + k + oz);
      }
      const signed char* row = c_mc.tri[idx[k]];
      // calculateVertices (marching_cubes_impl.cuh:31-70): the table's triangle (a, b, c) is stored as (c, b, a)
      for (int t = 0; t < 15 && row[t] >= 0; t += 3) {
        float p0[3], p1[3], p2[3];
        edgeVertex(pos, sdf[k], row[t + 2], p0), edgeVertex(pos, sdf[k], row[t + 1], p1), edgeVertex(pos, sdf[k], row[t], p2);
        const float px[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
        const float py[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
        float nx = px[1] * py[2] - px[2] * py[1], ny = px[2] * py[0] - px[0] * py[2], nz = px[0] * py[1] - px[1] * py[0];
        const float sq = (nx * nx + ny * ny) + nz * nz;
        if (sq > 0.0f) {
          const float len = sqrtf(sq);
          nx /= len, ny /= len, nz /= len;
        }
        float* V = c.vertices + 3 * (size_t)next;
        float* N = c.normals + 3 * (size_t)next;
        V[0] = p0[0], V[1] = p0[1], V[2] = p0[2], V[3] = p1[0], V[4] = p1[1], V[5] = p1[2], V[6] = p2[0], V[7] = p2[1], V[8] = p2[2];
#pragma unroll
        for (int q = 0; q < 3; q++) N[3 * q] = nx, N[3 * q + 1] = ny, N[3 * q + 2] = nz;
        const int local = next - c.offsets[i];
        c.triangles[next] = local, c.triangles[next + 1] = local + 1, c.triangles[next + 2] = local + 2;
        next += 3;
      }
    }
  }
}

// ---- weld (weldVerticesCubKernel<128, 20>, :691-803). One CTA per listed block.
constexpr int kWeldMax = 128 * 20;  // blocks with this many vertices or more keep them all
constexpr int kWeldPad = 4096;
constexpr size_t kWeldSmemBytes = (size_t)kWeldPad * 8 + (size_t)kWeldPad * 4 * 2 + (size_t)kWeldMax * 12;

__global__ void __launch_bounds__(kMeshThreads) meshWeldKernel(MeshCtx c) {
  extern __shared__ __align__(16) unsigned char weld_smem[];
  unsigned long long* key = reinterpret_cast<unsigned long long*>(weld_smem);  // later: staged vertices of the heads
  int* idx = reinterpret_cast<int*>(weld_smem + (size_t)kWeldPad * 8);
  int* rank = idx + kWeldPad;
  float* stage_n = reinterpret_cast<float*>(rank + kWeldPad);
  float* stage_v = reinterpret_cast<float*>(key);
  __shared__ int warp_sum[kMeshThreads / 32];
  __shared__ int s_ms;
  const int n = c.todo.count ? *c.todo.count : c.in_count_host;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int nv = c.counts[i];
    if (nv <= 0 || nv >= kWeldMax) continue;
    const int off = c.offsets[i];
    int P = 32;
    while (P < nv) P <<= 1;
    __syncthreads();
    for (int q = tid; q < P; q += kMeshThreads) {
      unsigned long long k = ~0ull;
      int id = 0x7fffffff;
      if (q < nv) {
        // Index3DHash(Index3D(x * 1000, y * 1000, z * 1000)) (core/hash.h:32-40)
        const float* v = c.vertices + 3 * (size_t)(off + q);
        const int x = (int)(v[0] * 1000.0f), y = (int)(v[1] * 1000.0f), z = (int)(v[2] * 1000.0f);
        const unsigned long long sl = 17191ull;
        k = (unsigned long long)(long long)x + (unsigned long long)(long long)y * sl + (unsigned long long)(long long)z * (sl * sl);
        id = q;
      }
      key[q] = k, idx[q] = id;
    }
    __syncthreads();
    // bitonic sort by (key, index): the index tie-break reproduces the stable radix sort
    for (int k2 = 2; k2 <= P; k2 <<= 1) {
      for (int j = k2 >> 1; j > 0; j >>= 1) {
        for (int q = tid; q < P; q += kMeshThreads) {
          const int p = q ^ j;
          if (p > q) {
            const unsigned long long ka = key[q], kb = key[p];
            const int ia = idx[q], ib = idx[p];
            const bool a_gt_b = ka > kb || (ka == kb && ia > ib);
            const bool up = (q & k2) == 0;
            if (a_gt_b == up) key[q] = kb, key[p] = ka, idx[q] = ib, idx[p] = ia;
          }
        }
        __syncthreads();
      }
    }
    // head flags + inclusive scan (FlagHeads + InclusiveSum), blocked: thread t owns sorted positions [t * per, (t+1) * per)
    const int per = P / kMeshThreads > 0 ? P / kMeshThreads : 1;
    const int lo = tid * per;
    int local = 0;
    for (int q = lo; q < lo + per && q < nv; q++) local += (q == 0 || key[q] != key[q - 1]) ? 1 : 0;
    int inc = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    int run = inc - local, heads = 0;
    for (int w = 0; w < kMeshThreads / 32; w++) {
      if (w < warp) run += warp_sum[w];
      heads += warp_sum[w];
    }
    for (int q = lo; q < lo + per && q < nv; q++) {
      const bool head = q == 0 || key[q] != key[q - 1];
      run += head ? 1 : 0;
      rank[q] = head ? run : -run;  // negative: not a head
    }
    __syncthreads();
    // the keys are dead: their storage now stages the heads' vertices
    for (int q = tid; q < nv; q += kMeshThreads) {
      const int r = rank[q], id = idx[q];
      const int pos = (r > 0 ? r : -r) - 1;
      c.triangles[off + id] = pos;  // block->triangles[thread_inds[i]] = head_indices[i] - 1
      if (r > 0) {
        const float* v = c.vertices + 3 * (size_t)(off + id);
        const float* nn = c.normals + 3 * (size_t)(off + id);
        stage_v[3 * pos] = v[0], stage_v[3 * pos + 1] = v[1], stage_v[3 * pos + 2] = v[2];
        stage_n[3 * pos] = nn[0], stage_n[3 * pos + 1] = nn[1], stage_n[3 * pos + 2] = nn[2];
      }
    }
    if (tid == 0) {
      int bx, by, bz;
      if (c.todo.slots) {
        const int t = c.todo.slots[i];
        bx = c.tsdf.block_index[3 * t], by = c.tsdf.block_index[3 * t + 1], bz = c.tsdf.block_index[3 * t + 2];
      } else {
        bx = c.in_xyz[3 * i], by = c.in_xyz[3 * i + 1], bz = c.in_xyz[3 * i + 2];
      }
      s_ms = hashFind(c.mesh.hash, bx, by, bz);
    }
    __syncthreads();
    for (int q = tid; q < 3 * heads; q += kMeshThreads) {
      c.vertices[3 * (size_t)off + q] = stage_v[q];
      c.normals[3 * (size_t)off + q] = stage_n[q];
    }
    if (tid == 0 && s_ms >= 0) meshHeader(c, s_ms)->nv = heads;  // vertices / normals shrink, `triangles` keeps its length
  }
}

// ---- colour (updateAppearanceGPU, mesh_integrator_appearance.cu:281-380)
__global__ void __launch_bounds__(kMeshThreads) meshColorKernel(MeshCtx c) {
  __shared__ int s_ms, s_cs;
  const int n = c.todo.count ? *c.todo.count : c.in_count_host;
  const int tid = threadIdx.x;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    __syncthreads();
    int bx, by, bz;
    if (c.todo.slots) {
      const int t = c.todo.slots[i];
      bx = c.tsdf.block_index[3 * t], by = c.tsdf.block_index[3 * t + 1], bz = c.tsdf.block_index[3 * t + 2];
    } else {
      bx = c.in_xyz[3 * i], by = c.in_xyz[3 * i + 1], bz = c.in_xyz[3 * i + 2];
    }
    if (tid == 0) {
      s_ms = bx == kDeadSlotX ? -1 : hashFind(c.mesh.hash, bx, by, bz);
      s_cs = (c.color.blocks && s_ms >= 0) ? hashFind(c.color.hash, bx, by, bz) : -1;
    }
    __syncthreads();
    if (s_ms < 0) continue;
    MeshHeader* h = meshHeader(c, s_ms);
    const int nv = h->nv, off = h->offset;
    if (tid == 0) h->nc = nv;  // expandAppearanceToMatchVertices
    const float bp[3] = {c.block_size * (float)bx, c.block_size * (float)by, c.block_size * (float)bz};
    for (int q = tid; q < nv; q += kMeshThreads) {
      uchar4 out = make_uchar4(127, 127, 127, 255);  // Color::Gray() (core/color.h:59)
      if (s_cs >= 0) {
        const float* v = c.vertices + 3 * (size_t)(off + q);
        int vi[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
          vi[j] = (int)((v[j] - bp[j]) / c.voxel_size);
          vi[j] = vi[j] > kVps - 1 ? kVps - 1 : vi[j];
          vi[j] = vi[j] < 0 ? 0 : vi[j];
        }
        const unsigned char* cv = c.color.blocks + (size_t)s_cs * kColorBlockBytes + (size_t)((vi[0] * kVps + vi[1]) * kVps + vi[2]) * 8;
        out = make_uchar4(cv[0], cv[1], cv[2], 255);
      }
      c.colors[off + q] = out;
    }
  }
}

// ---- read-back helpers
__global__ void meshHeadersKernel(MeshCtx c, const int* xyz, int n, int* out4) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ms = hashFind(c.mesh.hash, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
  int4 o = make_int4(-1, -1, -1, -1);
  if (ms >= 0) {
    const MeshHeader* h = meshHeader(c, ms);
    o = make_int4(h->offset, h->nv, h->nt, h->nc);
  }
  reinterpret_cast<int4*>(out4)[i] = o;
}

// Packs the listed blocks' segments back to back: src4 = (offset, nv, nt, nc) per block, dst3 = exclusive sums of
// (nv, nt, nc) per block.
__global__ void meshPackKernel(MeshCtx c, const int* src4, const int* dst3, int n, float* v_out, float* n_out, int* t_out,
                               uchar4* c_out) {
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int4 h = reinterpret_cast<const int4*>(src4)[i];
    if (h.x < 0) continue;
    const int dv = dst3[3 * i], dt = dst3[3 * i + 1], dc = dst3[3 * i + 2];
    for (int q = threadIdx.x; q < 3 * h.y; q += blockDim.x) {
      v_out[3 * (size_t)dv + q] = c.vertices[3 * (size_t)h.x + q];
      n_out[3 * (size_t)dv + q] = c.normals[3 * (size_t)h.x + q];
    }
    for (int q = threadIdx.x; q < h.z; q += blockDim.x) t_out[dt + q] = c.triangles[h.x + q];
    for (int q = threadIdx.x; q < h.w; q += blockDim.x) c_out[dc + q] = c.colors[h.x + q];
  }
}

// Arena compaction: live segments (by header slot) move to a fresh arena in slot order.
__global__ void meshCompactSizesKernel(MeshCtx c, int nslots, int* sizes) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nslots) return;
  sizes[s] = c.mesh.block_index[3 * s] == kDeadSlotX ? 0 : meshHeader(c, s)->cap;
}
__global__ void meshCompactMoveKernel(MeshCtx c, int nslots, const int* new_offsets, float* v2, float* n2, int* t2, uchar4* c2) {
  for (int s = blockIdx.x; s < nslots; s += gridDim.x) {
    if (c.mesh.block_index[3 * s] == kDeadSlotX) continue;
    MeshHeader* h = meshHeader(c, s);
    const int cap = h->cap, src = h->offset, dst = new_offsets[s];
    if (cap == 0) continue;
    for (int q = threadIdx.x; q < 3 * h->nv; q += blockDim.x) {
      v2[3 * (size_t)dst + q] = c.vertices[3 * (size_t)src + q];
      n2[3 * (size_t)dst + q] = c.normals[3 * (size_t)src + q];
    }
    for (int q = threadIdx.x; q < h->nt; q += blockDim.x) t2[dst + q] = c.triangles[src + q];
    for (int q = threadIdx.x; q < h->nc; q += blockDim.x) c2[dst + q] = c.colors[src + q];
    __syncthreads();
    if (threadIdx.x == 0) h->offset = dst;
    __syncthreads();
  }
}

}  // namespace

size_t meshWeldSmemBytes() { return kWeldSmemBytes; }

void launchMeshCount(const MeshCtx& c, int upper, int num_sms, cudaStream_t stream) {
  int grid = upper < num_sms * 8 ? upper : num_sms * 8;
  if (grid < 1) grid = 1;
  meshCountKernel<<<grid, kMeshThreads, 0, stream>>>(c);
  meshScanKernel<<<1, 1024, 0, stream>>>(c);
}
void launchMeshScan(const MeshCtx& c, cudaStream_t stream) { meshScanKernel<<<1, 1024, 0, stream>>>(c); }
void launchMeshEmit(const MeshCtx& c, int upper, int num_sms, cudaStream_t stream) {
  int grid = upper < num_sms * 8 ? upper : num_sms * 8;
  if (grid < 1) grid = 1;
  meshEmitKernel<<<grid, kMeshThreads, 0, stream>>>(c);
  if (c.weld) {
    static bool attr = false;
    if (!attr) {
      cudaFuncSetAttribute(meshWeldKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWeldSmemBytes);
      attr = true;
    }
    int wgrid = upper < num_sms * 2 ? upper : num_sms * 2;
    if (wgrid < 1) wgrid = 1;
    meshWeldKernel<<<wgrid, kMeshThreads, kWeldSmemBytes, stream>>>(c);
  }
}
void launchMeshColor(const MeshCtx& c, int upper, int num_sms, cudaStream_t stream) {
  int grid = upper < num_sms * 8 ? upper : num_sms * 8;
  if (grid < 1) grid = 1;
  meshColorKernel<<<grid, kMeshThreads, 0, stream>>>(c);
}
void launchMeshHeaders(const MeshCtx& c, const int* xyz_dev, int n, int* out4, cudaStream_t stream) {
  if (n > 0) meshHeadersKernel<<<(n + 255) / 256, 256, 0, stream>>>(c, xyz_dev, n, out4);
}
void launchMeshPack(const MeshCtx& c, const int* src4, const int* dst3, int n, float* v_out, float* n_out, int* t_out,
                    unsigned char* c_out, int num_sms, cudaStream_t stream) {
  if (n <= 0) return;
  int grid = n < num_sms * 8 ? n : num_sms * 8;
  meshPackKernel<<<grid, 256, 0, stream>>>(c, src4, dst3, n, v_out, n_out, t_out, reinterpret_cast<uchar4*>(c_out));
}
void launchMeshCompactSizes(const MeshCtx& c, int nslots, int* sizes, cudaStream_t stream) {
  if (nslots > 0) meshCompactSizesKernel<<<(nslots + 255) / 256, 256, 0, stream>>>(c, nslots, sizes);
}
void launchMeshCompactMove(const MeshCtx& c, int nslots, const int* new_offsets, float* v2, float* n2, int* t2,
                           unsigned char* c2, int num_sms, cudaStream_t stream) {
  if (nslots <= 0) return;
  int grid = nslots < num_sms * 8 ? nslots : num_sms * 8;
  meshCompactMoveKernel<<<grid, 256, 0, stream>>>(c, nslots, new_offsets, v2, n2, t2, reinterpret_cast<uchar4*>(c2));
}

}  // namespace nvb
