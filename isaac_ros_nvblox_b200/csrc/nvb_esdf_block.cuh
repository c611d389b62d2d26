// nvb_esdf_block.cuh -- the ESDF layer's block format: the one place that knows where a voxel's words live.
//
// A block of the ESDF layer holds its 512 voxels (v = (x * 8 + y) * 8 + z) as two planes:
//   bytes [0, 8192)     512 cells of 16 bytes {squared_distance_vox f32, parent_direction x, y, z i32},
//   bytes [8192, 10240) 512 flag words (byte 0 is_inside, 1 observed, 2 is_site, 3 padding, kept as stored).
// The reference's EsdfVoxel (map/voxels.h:55-74) is the same five words as one 20-byte record. A 16-byte cell is one aligned
// vector access and the flags of 32 consecutive voxels are one 128-byte line, where a 20-byte record is 16-byte aligned one
// time in four; the shared-memory regions and the exchange slab of the wavefront use the same split. Everything the library
// hands to or takes from its callers (nvb_layer_get_blocks / set_blocks, map files, voxel queries) is in the record form:
// the block copies convert with esdfVoxelToRecord / esdfVoxelFromRecord. A new block is all zero bytes in both forms.
#pragma once
#include <algorithm>

#include "nvb_internal.cuh"

namespace nvb {

constexpr int kEsdfCellWords = 4;
constexpr int kEsdfFlagWord0 = kVpb * kEsdfCellWords;  // word offset of the flag plane (2048)
constexpr int kEsdfRecordWords = 5;                    // the reference's EsdfVoxel
static_assert((kEsdfFlagWord0 + kVpb) * 4 == kEsdfBlockBytes, "ESDF block = cell plane + flag plane");
static_assert(kEsdfRecordWords * 4 * kVpb == kEsdfBlockBytes, "ESDF block = 512 EsdfVoxel records");

// Voxel v's cell (4 words) and flag word in a block, or in a block image staged in shared memory. W: (const) unsigned int.
template <class W>
__host__ __device__ __forceinline__ W* esdfCell(W* blk, int v) {
  return blk + kEsdfCellWords * v;
}
template <class W>
__host__ __device__ __forceinline__ W* esdfFlag(W* blk, int v) {
  return blk + kEsdfFlagWord0 + v;
}

// Voxel v of a block <-> its 20-byte record `rec` (five words).
__host__ __device__ __forceinline__ void esdfVoxelToRecord(const unsigned int* blk, int v, unsigned int* rec) {
  const unsigned int* c = esdfCell(blk, v);
  rec[0] = c[0], rec[1] = c[1], rec[2] = c[2], rec[3] = c[3], rec[4] = *esdfFlag(blk, v);
}
__host__ __device__ __forceinline__ void esdfVoxelFromRecord(const unsigned int* rec, unsigned int* blk, int v) {
  unsigned int* c = esdfCell(blk, v);
  c[0] = rec[0], c[1] = rec[1], c[2] = rec[2], c[3] = rec[3], *esdfFlag(blk, v) = rec[4];
}

// n whole blocks in place, on the host (map files).
inline void esdfBlocksToRecords(unsigned char* data, size_t n) {
  std::vector<unsigned int> blk(kEsdfBlockBytes / 4);
  for (size_t b = 0; b < n; b++) {
    unsigned int* words = reinterpret_cast<unsigned int*>(data + b * kEsdfBlockBytes);
    std::copy(words, words + blk.size(), blk.begin());
    for (int v = 0; v < kVpb; v++) esdfVoxelToRecord(blk.data(), v, words + kEsdfRecordWords * v);
  }
}
inline void esdfBlocksFromRecords(unsigned char* data, size_t n) {
  std::vector<unsigned int> rec(kEsdfBlockBytes / 4);
  for (size_t b = 0; b < n; b++) {
    unsigned int* words = reinterpret_cast<unsigned int*>(data + b * kEsdfBlockBytes);
    std::copy(words, words + rec.size(), rec.begin());
    for (int v = 0; v < kVpb; v++) esdfVoxelFromRecord(rec.data() + kEsdfRecordWords * v, words, v);
  }
}

}  // namespace nvb
