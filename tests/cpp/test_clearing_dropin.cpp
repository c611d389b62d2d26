// Replays nvblox_ros' map-clearing calls through nvblox/nvblox.h only: the node's timer calls
// Mapper::clearOutsideRadius(T_L_C.translation(), map_clearing_radius_m) (nvblox_node.cpp:1567-1583), the ESDF service builds
// its shapes like getShapesToClear (conversions/esdf_and_gradients_conversions.cu:127-172) and calls clearTsdfInsideShapes,
// then updateEsdf; the layer publisher asks getClearedBlocks({}) which blocks to delete (layer_publishing.cpp:716,804).
// The results are checked against the reference's definitions and the validateEsdf invariants
// (tests/test_esdf_integrator.cpp:339-460). Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <set>
#include <tuple>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

static Vector3f voxelCentre(float block_size, const Index3D& b, int x, int y, int z) {
  // getCenterPositionFromBlockIndexAndVoxelIndex (core/internal/impl/indexing_impl.h:51-81)
  const float vs = block_size * (1.0f / 8), hv = block_size * (0.5f / 8);
  const int v[3] = {x, y, z};
  Vector3f p;
  for (int k = 0; k < 3; k++) p[k] = (block_size * (float)b[k] + vs * (float)v[k]) + hv;
  return p;
}

int main() {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  constexpr float kVoxel = 0.05f;
  Camera camera(300.f, 300.f, 320.f, 240.f, 640, 480);
  DepthImage depth(480, 640, MemoryType::kUnified);
  for (int r = 0; r < 480; r++) for (int c = 0; c < 640; c++) depth(r, c) = 5.0f;  // a wall 5 m ahead
  ColorImage red(480, 640, MemoryType::kUnified);
  for (int r = 0; r < 480; r++) for (int c = 0; c < 640; c++) red(r, c) = Color::Red();
  Mapper mapper(kVoxel);
  Transform T_L_C = Transform::Identity();
  mapper.integrateDepth(depth, T_L_C, camera);
  mapper.integrateColor(red, T_L_C, camera);
  mapper.updateEsdf();
  TsdfLayer tsdf = mapper.tsdf_layer();
  EsdfLayer esdf = mapper.esdf_layer();
  ColorLayer color = mapper.color_layer();
  const float bs = tsdf.block_size();
  const int n0 = tsdf.numBlocks();
  EXPECT(n0 > 1000 && esdf.numBlocks() == n0);

  // --- clear_map_outside_radius timer
  const float radius = 5.5f;
  const std::vector<Index3D> all = tsdf.getAllBlockIndices();
  std::set<std::tuple<int, int, int>> expect_removed;
  for (const Index3D& b : all)
    if (isBlockOutsideRadius(b, bs, T_L_C.translation(), radius)) expect_removed.insert(std::make_tuple(b[0], b[1], b[2]));
  EXPECT(!expect_removed.empty() && (int)expect_removed.size() < n0);
  mapper.clearOutsideRadius(T_L_C.translation(), radius);
  const int n1 = tsdf.numBlocks();
  EXPECT(n1 == n0 - (int)expect_removed.size());
  EXPECT(esdf.numBlocks() == n1);
  EXPECT(color.numBlocks() <= n1);
  for (const Index3D& b : tsdf.getAllBlockIndices()) EXPECT(!isBlockOutsideRadius(b, bs, T_L_C.translation(), radius));
  const std::vector<Index3D> cleared = mapper.getClearedBlocks({});
  EXPECT(cleared.size() == expect_removed.size());
  for (size_t i = 0; i < cleared.size(); i++) {
    EXPECT(expect_removed.count(std::make_tuple(cleared[i][0], cleared[i][1], cleared[i][2])) == 1);
    EXPECT(tsdf.getBlockAtIndex(cleared[i]) == nullptr && esdf.getBlockAtIndex(cleared[i]) == nullptr);
  }
  EXPECT(mapper.getClearedBlocks({}).empty());

  // --- EsdfAndGradients service: shapes as getShapesToClear builds them (AABB = min + size, empty ones and
  // non-positive radii dropped), then clearTsdfInsideShapes and updateEsdf
  std::vector<BoundingShape> shapes;
  const Vector3f aabb_min(-1.0f, -1.0f, 4.6f), aabb_size(2.0f, 1.5f, 0.8f);
  AxisAlignedBoundingBox aabb(aabb_min, Vector3f(aabb_min[0] + aabb_size[0], aabb_min[1] + aabb_size[1], aabb_min[2] + aabb_size[2]));
  if (!aabb.isEmpty()) shapes.push_back(BoundingShape(aabb));
  AxisAlignedBoundingBox empty_box(Vector3f(1.0f, 1.0f, 1.0f), Vector3f(0.0f, 0.0f, 0.0f));
  if (!empty_box.isEmpty()) shapes.push_back(BoundingShape(empty_box));
  BoundingSphere sphere(Vector3f(2.0f, 0.5f, 5.0f), 0.7f), no_sphere(Vector3f(0.0f, 0.0f, 5.0f), 0.0f);
  if (sphere.radius() > 0.f) shapes.push_back(BoundingShape(sphere));
  if (no_sphere.radius() > 0.f) shapes.push_back(BoundingShape(no_sphere));
  EXPECT(shapes.size() == 2 && shapes[0].type() == ShapeType::kAABB && shapes[1].type() == ShapeType::kSphere);
  mapper.clearTsdfInsideShapes(shapes);
  EXPECT(tsdf.numBlocks() == n1);  // nothing is deallocated
  long cleared_voxels = 0, touched_blocks = 0;
  for (const Index3D& b : tsdf.getAllBlockIndices()) {
    bool touched = false;
    for (const BoundingShape& s : shapes) touched = touched || s.touchesBlock(b, bs);
    if (!touched) continue;
    touched_blocks++;
    auto blk = tsdf.getBlockAtIndexHost(b);
    for (int x = 0; x < 8; x++) for (int y = 0; y < 8; y++) for (int z = 0; z < 8; z++) {
      bool inside = false;
      for (const BoundingShape& s : shapes) inside = inside || s.contains(voxelCentre(bs, b, x, y, z));
      if (!inside) continue;
      const TsdfVoxel& v = blk->voxels[x][y][z];
      EXPECT(v.weight == 0.0f && v.distance == 0.0f);
      cleared_voxels++;
    }
  }
  EXPECT(touched_blocks > 0 && cleared_voxels > 1000);
  mapper.updateEsdf();
  EXPECT(esdf.numBlocks() == n1);
  long sites = 0;
  for (const Index3D& b : esdf.getAllBlockIndices()) {
    auto blk = esdf.getBlockAtIndexHost(b);
    for (int x = 0; x < 8; x++) for (int y = 0; y < 8; y++) for (int z = 0; z < 8; z++) {
      const EsdfVoxel& v = blk->voxels[x][y][z];
      if (!v.observed) continue;
      if (v.is_site) { sites++; EXPECT(v.squared_distance_vox == 0.0f); }
      else if (v.parent_direction != Index3D::Zero()) {
        const Index3D& p = v.parent_direction;
        EXPECT(v.squared_distance_vox == (float)(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
      }
      bool inside = false;  // a cleared voxel is unobserved in the TSDF, so it is no site
      for (const BoundingShape& s : shapes) inside = inside || s.contains(voxelCentre(bs, b, x, y, z));
      EXPECT(!(inside && v.is_site));
    }
  }
  EXPECT(sites > 1000);
  EXPECT(mapper.getClearedBlocks({}).empty());  // shape clearing deallocates nothing

  // --- ShapeClearer on the colour layer: Color::Gray(), weight 0
  ShapeClearer<ColorLayer> color_clearer;
  const std::vector<Index3D> color_touched = color_clearer.clear(shapes, &color);
  EXPECT(!color_touched.empty());
  long grey = 0;
  for (const Index3D& b : color_touched) {
    auto blk = color.getBlockAtIndexHost(b);
    for (int x = 0; x < 8; x++) for (int y = 0; y < 8; y++) for (int z = 0; z < 8; z++) {
      bool inside = false;
      for (const BoundingShape& s : shapes) inside = inside || s.contains(voxelCentre(bs, b, x, y, z));
      if (inside) { EXPECT(blk->voxels[x][y][z].color == Color::Gray() && blk->voxels[x][y][z].weight == 0.0f); grey++; }
    }
  }
  EXPECT(grey > 0);
  std::printf("clearing drop-in ok: %d of %d blocks cleared, %ld voxels inside shapes, %ld sites\n", n0 - n1, n0, cleared_voxels, sites);
  return 0;
}
