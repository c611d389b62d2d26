// nvblox/io/mesh_io.h -- io::outputColorMeshLayerToPly (reference: nvblox/include/nvblox/io/mesh_io.h, src/io/mesh_io.cpp):
// the mesh blocks appended in the layer's block order (MeshBlockLayer::getMesh), triangle indices offset by the vertices
// before their block, written through PlyWriter.
#pragma once
#include <string>
#include <vector>
#include "nvblox/io/ply_writer.h"
#include "nvblox/mesh/mesh_block.h"
namespace nvblox {
namespace io {
inline bool outputColorMeshLayerToPly(const ColorMeshLayer& layer, const std::string& filename) {
  std::vector<Vector3f> vertices, normals;
  std::vector<Color> colors;
  std::vector<int> triangles;
  for (const Index3D& idx : layer.getAllBlockIndices()) {
    auto b = layer.getBlockAtIndex(idx);
    if (!b) continue;
    const int base = (int)vertices.size();
    vertices.insert(vertices.end(), b->vertices.begin(), b->vertices.end());
    normals.insert(normals.end(), b->vertex_normals.begin(), b->vertex_normals.end());
    colors.insert(colors.end(), b->vertex_appearances.begin(), b->vertex_appearances.end());
    for (int t : b->triangles) triangles.push_back(t + base);
  }
  PlyWriter writer(filename);
  writer.setPoints(&vertices);
  writer.setTriangles(&triangles);
  if (!normals.empty()) writer.setNormals(&normals);
  if (!colors.empty()) writer.setColors(&colors);
  return writer.write();
}
inline bool outputColorMeshLayerToPly(const ColorMeshLayer& layer, const char* filename) {
  return outputColorMeshLayerToPly(layer, std::string(filename));
}
}  // namespace io
}  // namespace nvblox
