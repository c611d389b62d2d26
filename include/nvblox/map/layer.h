// nvblox/map/layer.h -- VoxelBlockLayer<V> queries (reference: nvblox/include/nvblox/map/layer.h:76-311)
// answered from the device-resident slab + hash of libnvblox_b200.so.
#pragma once
#include <memory>
#include <vector>
#include "nvblox/map/blox.h"
#include "nvblox_b200.h"
namespace nvblox {
template <typename VoxelType>
class VoxelBlockLayer {
 public:
  using BlockType = VoxelBlock<VoxelType>;
  VoxelBlockLayer(NvbMapper* m, int layer_id) : m_(m), id_(layer_id) {}
  NvbMapper* mapper_handle() const { return m_; }  // (not in the reference: the layers here are views of a mapper's device map)
  int layer_id() const { return id_; }
  float voxel_size() const { return nvb_mapper_voxel_size(m_); }
  float block_size() const { return nvb_mapper_block_size(m_); }
  MemoryType memory_type() const { return MemoryType::kDevice; }
  int numBlocks() const {
    int32_t n = 0;
    b200_detail::check(nvb_layer_num_blocks(m_, id_, &n), "numBlocks", nvb_last_error());
    return n;
  }
  size_t size() const { return (size_t)numBlocks(); }
  std::vector<Index3D> getAllBlockIndices() const {
    const int n = numBlocks();
    std::vector<Index3D> out((size_t)n);
    std::vector<int32_t> raw((size_t)n * 3 + 3);
    int32_t cnt = 0;
    b200_detail::check(nvb_layer_block_indices(m_, id_, raw.data(), n, &cnt), "getAllBlockIndices", nvb_last_error());
    for (int i = 0; i < n; i++) out[i] = Index3D(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
    return out;
  }
  // BlockLayer::getBlockAtIndex (map/layer.h:103-104): a handle whose get() is the block's device address, null if the block
  // is not allocated.
  typename BlockType::ConstPtr getBlockAtIndex(const Index3D& idx) const {
    const int32_t k[3] = {idx[0], idx[1], idx[2]};
    void* p = nullptr;
    b200_detail::check(nvb_layer_block_device_ptr(m_, id_, k, &p), "getBlockAtIndex", nvb_last_error());
    return typename BlockType::ConstPtr(static_cast<const BlockType*>(p));
  }
  typename BlockType::Ptr getBlockAtIndex(const Index3D& idx) {
    const int32_t k[3] = {idx[0], idx[1], idx[2]};
    void* p = nullptr;
    b200_detail::check(nvb_layer_block_device_ptr(m_, id_, k, &p), "getBlockAtIndex", nvb_last_error());
    return typename BlockType::Ptr(static_cast<BlockType*>(p));
  }
  bool isBlockAllocated(const Index3D& idx) const { return getBlockAtIndex(idx) != nullptr; }
  // Host copy of one block (the reference's tests read kUnified layers directly).
  std::shared_ptr<BlockType> getBlockAtIndexHost(const Index3D& idx) const {
    auto blk = std::make_shared<BlockType>();
    const int32_t k[3] = {idx[0], idx[1], idx[2]};
    uint8_t found = 0;
    b200_detail::check(nvb_layer_get_blocks(m_, id_, k, 1, blk.get(), &found), "getBlockAtIndexHost", nvb_last_error());
    return found ? blk : nullptr;
  }
  bool getVoxel(const Index3D& block_idx, const Index3D& voxel_idx, VoxelType* out) const {
    auto b = getBlockAtIndexHost(block_idx);
    if (!b) return false;
    *out = b->voxels[voxel_idx[0]][voxel_idx[1]][voxel_idx[2]];
    return true;
  }
  // VoxelBlockLayer::getVoxels (map/layer.h:265-276): the voxel holding each position and whether its block exists. Runs on
  // the GPU (nvb_layer_query_voxels); a missing voxel is VoxelType{}.
  void getVoxels(const std::vector<Vector3f>& positions_L, std::vector<VoxelType>* voxels_ptr,
                 std::vector<bool>* success_flags_ptr) const {
    const size_t n = positions_L.size();
    std::vector<float> xyz(n * 3);
    for (size_t i = 0; i < n; i++) xyz[3 * i] = positions_L[i][0], xyz[3 * i + 1] = positions_L[i][1], xyz[3 * i + 2] = positions_L[i][2];
    voxels_ptr->assign(n, VoxelType{});
    std::vector<uint8_t> ok(n, 0);
    b200_detail::check(nvb_layer_query_voxels(m_, id_, xyz.data(), NVB_MEM_HOST, (int64_t)n, voxels_ptr->data(), ok.data()),
                       "getVoxels", nvb_last_error());
    success_flags_ptr->assign(ok.begin(), ok.end());
  }
 // The mapper this layer belongs to (DynamicsDetection::computeDynamics runs on the owner of its FreespaceLayer).
  NvbMapper* c_abi() const { return m_; }
 private:
  NvbMapper* m_;
  int id_;
};
using TsdfLayer = VoxelBlockLayer<TsdfVoxel>;
using OccupancyLayer = VoxelBlockLayer<OccupancyVoxel>;
using FreespaceLayer = VoxelBlockLayer<FreespaceVoxel>;
using ColorLayer = VoxelBlockLayer<ColorVoxel>;
using EsdfLayer = VoxelBlockLayer<EsdfVoxel>;
}  // namespace nvblox
