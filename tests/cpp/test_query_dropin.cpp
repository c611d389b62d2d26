// Point queries through nvblox/nvblox.h only: VoxelBlockLayer::getVoxels on the TSDF and ESDF layers of a mapped wall,
// checked voxel for voxel against the host copies of their blocks, and interpolation::interpolateOnCPU (single point and
// vector) of the TSDF, whose distance across the wall is linear in the point's depth (test_3d_interpolation.cpp's
// linear-field idea). Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <vector>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  constexpr float kVoxel = 0.05f;
  Camera camera(300.f, 300.f, 320.f, 240.f, 640, 480);
  DepthImage depth(480, 640, MemoryType::kUnified);
  for (int r = 0; r < 480; r++) for (int c = 0; c < 640; c++) depth(r, c) = 3.0f;  // a wall 3 m ahead
  Mapper mapper(kVoxel);
  mapper.integrateDepth(depth, Transform::Identity(), camera);
  mapper.updateEsdf();
  TsdfLayer tsdf = mapper.tsdf_layer();
  EsdfLayer esdf = mapper.esdf_layer();
  const float bs = tsdf.block_size();

  // getVoxels: points on a grid across the wall, some in unallocated blocks
  std::vector<Vector3f> pts;
  for (int i = -6; i <= 6; i++) for (int k = 0; k < 40; k++) pts.push_back(Vector3f(0.137f * i, -0.071f * i, 2.0f + 0.05f * k));
  pts.push_back(Vector3f(0.0f, 0.0f, -50.0f));  // no block there
  std::vector<TsdfVoxel> tv;
  std::vector<EsdfVoxel> ev;
  std::vector<bool> tok, eok;
  tsdf.getVoxels(pts, &tv, &tok);
  esdf.getVoxels(pts, &ev, &eok);
  EXPECT(tv.size() == pts.size() && eok.size() == pts.size());
  int found = 0;
  for (size_t i = 0; i < pts.size(); i++) {
    Index3D b, v;
    for (int a = 0; a < 3; a++) {  // getBlockAndVoxelIndexFromPositionInLayer
      b[a] = (int)std::floor(pts[i][a] / bs);
      v[a] = std::min((int)((pts[i][a] - bs * (float)b[a]) * (float)(1.0 / (double)(bs / 8))), 7);
    }
    auto tb = tsdf.getBlockAtIndexHost(b);
    EXPECT(tok[i] == (tb != nullptr));
    if (!tb) continue;
    found++;
    const TsdfVoxel& t = tb->voxels[v[0]][v[1]][v[2]];
    EXPECT(tv[i].distance == t.distance && tv[i].weight == t.weight);
    auto eb = esdf.getBlockAtIndexHost(b);
    EXPECT(eok[i] == (eb != nullptr));
    if (eb) {
      const EsdfVoxel& e = eb->voxels[v[0]][v[1]][v[2]];
      EXPECT(ev[i].squared_distance_vox == e.squared_distance_vox && ev[i].observed == e.observed && ev[i].is_inside == e.is_inside);
    }
  }
  EXPECT(!tok.back() && found > 100);

  // interpolateOnCPU on the TSDF near the wall: distance ~ 3 - z (linear along the optical axis, within a voxel's error)
  std::vector<Vector3f> near;
  for (int k = 0; k < 20; k++) near.push_back(Vector3f(0.01f, 0.02f, 2.92f + 0.008f * k));
  std::vector<float> d;
  std::vector<bool> ok;
  interpolation::interpolateOnCPU(near, tsdf, &d, &ok);
  int good = 0;
  for (size_t i = 0; i < near.size(); i++) {
    if (!ok[i]) continue;
    good++;
    EXPECT(std::fabs(d[i] - (3.0f - near[i][2])) < 2.0f * kVoxel);
    float one = -1.0f;
    EXPECT(interpolation::interpolateOnCPU(near[i], tsdf, &one) && one == d[i]);
  }
  EXPECT(good >= 10);
  float untouched = 42.0f;
  EXPECT(!interpolation::interpolateOnCPU(Vector3f(0.0f, 0.0f, -50.0f), tsdf, &untouched) && untouched == 42.0f);
  float e = 0.0f;
  EXPECT(interpolation::interpolateOnCPU(Vector3f(0.0f, 0.0f, 2.6f), esdf, &e) && e > 0.0f);
  std::printf("query drop-in ok: %d voxels found, %d interpolated points\n", found, good);
  return 0;
}
