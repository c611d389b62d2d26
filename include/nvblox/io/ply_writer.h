// nvblox/io/ply_writer.h -- io::PlyWriter (reference: nvblox/include/nvblox/io/ply_writer.h, src/io/ply_writer.cpp): an
// ASCII PLY of points with optional normals, intensities, colours and triangles, numbers in the default ostream format.
// Header-only here, shared by pointcloud_io.h and mesh_io.h.
#pragma once
#include <fstream>
#include <string>
#include <vector>
#include "nvblox/core/types.h"
#include "nvblox/map/voxels.h"
namespace nvblox {
namespace io {
class PlyWriter {
 public:
  explicit PlyWriter(const std::string& filename) : filename_(filename) {}
  void setPoints(const std::vector<Vector3f>* points) { points_ = points; }
  void setNormals(const std::vector<Vector3f>* normals) { normals_ = normals; }
  void setIntensities(const std::vector<float>* intensities) { intensities_ = intensities; }
  void setColors(const std::vector<Color>* colors) { colors_ = colors; }
  void setTriangles(const std::vector<int>* triangles) { triangles_ = triangles; }
  // false, and no file, without points or with a per-point array of another size
  bool write() {
    if (!points_ || points_->empty()) return false;
    const size_t n = points_->size();
    if ((normals_ && normals_->size() != n) || (intensities_ && intensities_->size() != n) || (colors_ && colors_->size() != n))
      return false;
    std::ofstream f(filename_);
    if (!f) return false;
    f << "ply" << std::endl << "format ascii 1.0" << std::endl << "element vertex " << n << std::endl;
    f << "property float x" << std::endl << "property float y" << std::endl << "property float z" << std::endl;
    if (normals_) f << "property float nx" << std::endl << "property float ny" << std::endl << "property float nz" << std::endl;
    if (intensities_) f << "property float intensity" << std::endl;
    if (colors_) f << "property uchar red" << std::endl << "property uchar green" << std::endl << "property uchar blue" << std::endl;
    if (triangles_) {
      f << "element face " << triangles_->size() / 3 << std::endl;
      f << "property list uchar int vertex_indices" << std::endl;
    }
    f << "end_header" << std::endl;
    for (size_t i = 0; i < n; i++) {
      const Vector3f& p = (*points_)[i];
      f << p[0] << " " << p[1] << " " << p[2];
      if (normals_) f << " " << (*normals_)[i][0] << " " << (*normals_)[i][1] << " " << (*normals_)[i][2];
      if (intensities_) f << " " << (*intensities_)[i];
      if (colors_)
        f << " " << std::to_string((*colors_)[i].r) << " " << std::to_string((*colors_)[i].g) << " " << std::to_string((*colors_)[i].b);
      f << std::endl;
    }
    if (triangles_)
      for (size_t i = 0; i + 2 < triangles_->size(); i += 3)
        f << 3 << " " << (*triangles_)[i] << " " << (*triangles_)[i + 1] << " " << (*triangles_)[i + 2] << " " << std::endl;
    return true;
  }

 private:
  std::string filename_;
  const std::vector<Vector3f>* points_ = nullptr;
  const std::vector<Vector3f>* normals_ = nullptr;
  const std::vector<float>* intensities_ = nullptr;
  const std::vector<Color>* colors_ = nullptr;
  const std::vector<int>* triangles_ = nullptr;
};
}  // namespace io
}  // namespace nvblox
