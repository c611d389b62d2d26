// nvb_merge.cu -- device-resident merge of the ranks' updated-block index lists (the one exchange step of the multi-GPU
// path, SURVEY.md section 8(e): every rank integrates its own camera's frames into its own map replica and the ranks only tell
// each other WHICH blocks they touched).
//
// Protocol (isaac_ros_nvblox_b200/multi_gpu.py BatchMerger): every rank appends the block lists of the frames of a batch to a
// SEGMENT in its own HBM -- int32 [count, x0, y0, z0, x1, ...] with a fixed capacity, written by appendFrameKernel on the
// mapper's stream straight from the frame list the view calculator left on the device -- one fixed-size ncclAllGather moves the
// segments (no count exchange, no host round trip), and unionSegments* below turn the gathered segments into the sorted unique
// union, identical on every rank: AABB reduction, marking into a bitset over the AABB, ordered ballot/popc compaction (x fastest,
// then y, then z: the view calculator's order), all sized from device memory. Nothing here synchronises with the host.
#include "nvb_internal.cuh"

namespace nvb {

namespace {

constexpr int kMergeThreads = 256;
constexpr int kMergeTileWords = 64;

__global__ void unionInitKernel(UnionState* state) {
  if (threadIdx.x < 3) state->aabb_min[threadIdx.x] = INT32_MAX;
  else if (threadIdx.x < 6) state->aabb_max[threadIdx.x - 3] = INT32_MIN;
  else if (threadIdx.x == 6) state->error = 0;
  else if (threadIdx.x == 7) state->words = 0;
}

__device__ __forceinline__ bool segmentEntry(const int* segs, int num_segments, int stride, int cap, long long i, int* x, int* y, int* z) {
  const int s = (int)(i / cap), e = (int)(i % cap);
  if (s >= num_segments) return false;
  const int* seg = segs + (size_t)s * stride;
  int n = seg[0];
  n = n < 0 ? 0 : (n > cap ? cap : n);
  if (e >= n) return false;
  *x = seg[1 + 3 * e], *y = seg[2 + 3 * e], *z = seg[3 + 3 * e];
  return true;
}

__global__ void unionAabbKernel(const int* __restrict__ segs, int num_segments, int stride, int cap, UnionState* state) {
  int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  const long long total = (long long)num_segments * cap;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int x, y, z;
    if (segmentEntry(segs, num_segments, stride, cap, i, &x, &y, &z)) {
      lo[0] = min(lo[0], x), lo[1] = min(lo[1], y), lo[2] = min(lo[2], z);
      hi[0] = max(hi[0], x), hi[1] = max(hi[1], y), hi[2] = max(hi[2], z);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
    hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
  }
  if ((threadIdx.x & 31) == 0 && lo[0] <= hi[0]) {
#pragma unroll
    for (int a = 0; a < 3; a++) atomicMin(&state->aabb_min[a], lo[a]), atomicMax(&state->aabb_max[a], hi[a]);
  }
}

__device__ __forceinline__ bool unionGrid(const UnionState* state, long long cap_bits, int* sx, int* sxy, long long* cells) {
  const int* lo = state->aabb_min;
  const int* hi = state->aabb_max;
  if (lo[0] > hi[0]) return false;  // no entries
  const long long dx = (long long)hi[0] - lo[0] + 1, dy = (long long)hi[1] - lo[1] + 1, dz = (long long)hi[2] - lo[2] + 1;
  *cells = dx * dy * dz;
  if (*cells > cap_bits) return false;
  *sx = (int)dx, *sxy = (int)(dx * dy);
  return true;
}

__global__ void unionMarkKernel(const int* __restrict__ segs, int num_segments, int stride, int cap, UnionState* state,
                                unsigned int* bits, long long cap_bits) {
  int sx, sxy;
  long long cells;
  if (!unionGrid(state, cap_bits, &sx, &sxy, &cells)) {
    // entries, but the AABB does not fit
    if (blockIdx.x == 0 && threadIdx.x == 0 && state->aabb_min[0] <= state->aabb_max[0]) state->error = 1;
    return;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) state->words = (int)((cells + 31) / 32);
  const long long total = (long long)num_segments * cap;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int x, y, z;
    if (segmentEntry(segs, num_segments, stride, cap, i, &x, &y, &z)) {
      const int* lo = state->aabb_min;
      const long long lin = (long long)(x - lo[0]) + (long long)(y - lo[1]) * sx + (long long)(z - lo[2]) * sxy;
      atomicOr(bits + (lin >> 5), 1u << (lin & 31));
    }
  }
}

// Ordered compaction: tile t owns 64 bitset words; its output offset is the popcount of all preceding words, which every tile
// recomputes for itself (the bitset is a few KB in L2), so tiles are independent (the scheme of compactAllocateKernel).
__global__ void __launch_bounds__(kMergeThreads) unionCompactKernel(const UnionState* state, const unsigned int* bits, long long cap_bits,
                                                                    int* out_xyz, int out_cap, int* out_count) {
  __shared__ int s_incl[kMergeTileWords];
  __shared__ unsigned int s_word[kMergeTileWords];
  __shared__ int s_red[kMergeThreads / 32];
  int sx, sxy;
  long long cells;
  if (!unionGrid(state, cap_bits, &sx, &sxy, &cells)) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *out_count = 0;
    return;
  }
  const int num_words = (int)((cells + 31) / 32);
  const int num_tiles = (num_words + kMergeTileWords - 1) / kMergeTileWords;
  const int tid = threadIdx.x;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int w0 = tile * kMergeTileWords;
    unsigned int word = 0;
    if (tid < kMergeTileWords && w0 + tid < num_words) word = bits[w0 + tid];
    if (tid < kMergeTileWords) {
      s_word[tid] = word;
      int incl = __popc(word);
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, incl, off);
        if ((tid & 31) >= off) incl += n;
      }
      s_incl[tid] = incl;
    }
    int part = 0;
    for (int w = tid; w < w0; w += kMergeThreads) part += __popc(bits[w]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) part += __shfl_down_sync(0xffffffffu, part, off);
    if ((tid & 31) == 0) s_red[tid >> 5] = part;
    __syncthreads();
    if (tid >= 32 && tid < kMergeTileWords) s_incl[tid] += s_incl[31];
    __syncthreads();
    const int total = s_incl[kMergeTileWords - 1];
    int prefix = 0;
    for (int q = 0; q < kMergeThreads / 32; q++) prefix += s_red[q];
    if (tile == num_tiles - 1 && tid == 0) *out_count = prefix + total;
    for (int j = tid; j < total; j += kMergeThreads) {
      int lo = 0, hi = kMergeTileWords - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_incl[mid] > j) hi = mid;
        else lo = mid + 1;
      }
      const unsigned int wv = s_word[lo];
      const int rank = j - (s_incl[lo] - __popc(wv));
      const int bit = (int)__fns(wv, 0, rank + 1);
      const long long lin = (long long)(w0 + lo) * 32 + bit;
      const int o = prefix + j;
      if (o < out_cap) {
        out_xyz[3 * o] = (int)(lin % sx) + state->aabb_min[0];
        out_xyz[3 * o + 1] = (int)((lin / sx) % (sxy / sx)) + state->aabb_min[1];
        out_xyz[3 * o + 2] = (int)(lin / sxy) + state->aabb_min[2];
      }
    }
    __syncthreads();
  }
}

__global__ void unionClearKernel(const UnionState* state, unsigned int* bits) {
  const int n = state->words;
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n; w += gridDim.x * blockDim.x) bits[w] = 0u;
}

// The frame list the view calculator left on the device ({x, y, z, slot} + count) -> appended to a segment.
__global__ void appendFrameKernel(const int4* __restrict__ frame, const int* __restrict__ frame_count, int* seg, int cap, int* error) {
  __shared__ int s_base, s_n;
  if (threadIdx.x == 0) {
    const int have = seg[0];
    int n = *frame_count;
    if (have + n > cap) {  // a full segment drops the rest and raises the mapper's device error flag (-> NVB_ERR_CAPACITY)
      n = cap - have > 0 ? cap - have : 0;
      atomicOr(error, 4);
    }
    s_base = have, s_n = n;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < s_n; i += blockDim.x) {
    const int4 v = frame[i];
    const int o = s_base + i;
    seg[1 + 3 * o] = v.x, seg[2 + 3 * o] = v.y, seg[3 + 3 * o] = v.z;
  }
  __syncthreads();
  if (threadIdx.x == 0) seg[0] = s_base + s_n;
}

}  // namespace

void launchAppendFrame(const int4* frame, const int* frame_count, int* seg, int cap, int* error, cudaStream_t stream) {
  appendFrameKernel<<<1, 1024, 0, stream>>>(frame, frame_count, seg, cap, error);
}

void launchUnionSegments(const int* segs, int num_segments, int stride, int cap, int* state_words, unsigned int* bits,
                         long long cap_bits, int* out_xyz, int out_cap, int* out_count, cudaStream_t stream) {
  UnionState* state = reinterpret_cast<UnionState*>(state_words);
  const long long total = (long long)num_segments * cap;
  int grid = (int)((total + kMergeThreads - 1) / kMergeThreads);
  grid = grid < 1 ? 1 : (grid > 592 ? 592 : grid);
  unionInitKernel<<<1, 32, 0, stream>>>(state);
  unionAabbKernel<<<grid, kMergeThreads, 0, stream>>>(segs, num_segments, stride, cap, state);
  unionMarkKernel<<<grid, kMergeThreads, 0, stream>>>(segs, num_segments, stride, cap, state, bits, cap_bits);
  unionCompactKernel<<<kHelperCtas, kMergeThreads, 0, stream>>>(state, bits, cap_bits, out_xyz, out_cap, out_count);
  unionClearKernel<<<kHelperCtas, 256, 0, stream>>>(state, bits);
}

}  // namespace nvb
