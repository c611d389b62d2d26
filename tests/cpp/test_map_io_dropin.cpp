// Replays nvblox_ros' map file services through nvblox/nvblox.h only (nvblox_node.cpp, the save_map, load_map and save_ply
// handlers): Mapper::saveLayerCake(filename), Mapper::loadMap(filename) on a second mapper, the Mapper(map_filepath)
// constructor, io::outputVoxelLayerToPly on the TSDF, ESDF and freespace layers and io::outputColorMeshLayerToPly.
// argv[1]: a directory to write into. Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <fstream>
#include <string>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

static bool sameBlocks(const TsdfLayer& a, const TsdfLayer& b) {
  const auto ia = a.getAllBlockIndices();
  if (ia.size() != b.getAllBlockIndices().size()) return false;
  for (const Index3D& k : ia) {
    auto x = a.getBlockAtIndexHost(k), y = b.getBlockAtIndexHost(k);
    if (!x || !y) return false;
    for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) for (int l = 0; l < 8; l++)
      if (x->voxels[i][j][l].distance != y->voxels[i][j][l].distance || x->voxels[i][j][l].weight != y->voxels[i][j][l].weight)
        return false;
  }
  return true;
}

static long plyVertices(const std::string& path) {
  std::ifstream f(path);
  std::string line;
  std::getline(f, line);
  if (line != "ply") return -1;
  while (std::getline(f, line))
    if (line.rfind("element vertex ", 0) == 0) return std::stol(line.substr(15));
  return -1;
}

int main(int argc, char** argv) {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  const std::string dir = argc > 1 ? argv[1] : ".";
  // a plane at 1.5 m in front of a 160 x 120 camera
  Camera cam(100.0f, 100.0f, 80.0f, 60.0f, 160, 120);
  DepthImage depth(120, 160, MemoryType::kHost);
  for (int r = 0; r < 120; r++) for (int c = 0; c < 160; c++) depth(r, c) = 1.5f;
  Transform T = Transform::Identity();
  Mapper mapper(0.05f, MemoryType::kDevice, ProjectiveLayerType::kTsdfWithFreespace);
  mapper.integrateDepth(depth, T, cam);
  mapper.updateEsdf(UpdateFullLayer::kYes);
  mapper.updateFreespace(1000, T, cam, depth, UpdateFullLayer::kYes);
  mapper.updateColorMesh(UpdateFullLayer::kYes);
  EXPECT(mapper.tsdf_layer().numBlocks() > 0);

  const std::string map_path = dir + "/dropin.nvblx";
  EXPECT(mapper.saveLayerCake(map_path));                   // ~/save_map
  Mapper loaded(0.1f);
  EXPECT(loaded.loadMap(map_path));                         // ~/load_map
  EXPECT(loaded.voxel_size_m() == 0.05f);
  EXPECT(sameBlocks(mapper.tsdf_layer(), loaded.tsdf_layer()));
  EXPECT(loaded.esdf_layer().numBlocks() == mapper.esdf_layer().numBlocks());
  EXPECT(loaded.color_mesh_layer().numBlocks() > 0);
  Mapper from_file(map_path);                               // Mapper(map_filepath)
  EXPECT(sameBlocks(mapper.tsdf_layer(), from_file.tsdf_layer()));
  EXPECT(!loaded.loadMap(dir + "/missing.nvblx"));
  EXPECT(sameBlocks(mapper.tsdf_layer(), loaded.tsdf_layer()));

  // ~/save_ply
  EXPECT(io::outputVoxelLayerToPly(mapper.tsdf_layer(), dir + "/tsdf.ply"));
  EXPECT(io::outputVoxelLayerToPly(mapper.esdf_layer(), dir + "/esdf.ply"));
  EXPECT(io::outputVoxelLayerToPly(mapper.freespace_layer(), dir + "/freespace.ply"));
  EXPECT(io::outputColorMeshLayerToPly(mapper.color_mesh_layer(), dir + "/mesh.ply"));
  EXPECT(plyVertices(dir + "/tsdf.ply") > 0 && plyVertices(dir + "/esdf.ply") > 0 && plyVertices(dir + "/mesh.ply") > 0);
  EXPECT(plyVertices(dir + "/freespace.ply") == 512L * mapper.freespace_layer().numBlocks());
  EXPECT(mapper.saveTsdfAsPly(dir + "/tsdf2.ply") && mapper.saveColorMeshAsPly(dir + "/mesh2.ply"));
  std::printf("map io drop-in ok: %d TSDF blocks, %ld TSDF points\n", mapper.tsdf_layer().numBlocks(),
              plyVertices(dir + "/tsdf.ply"));
  return 0;
}
