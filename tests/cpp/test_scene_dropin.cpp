// primitives::Scene through nvblox/nvblox.h only, with the reference test's calls (tests/test_scene.cpp: BlankMap, PlaneScene,
// a camera offset from the plane, TypesList) and nvblox_torch's py_scene.cu calls (createDummyMap's primitives, the AABB,
// getPrimitiveTypeList with Primitive::toString, generateLayerFromScene<TsdfVoxel> with 4-voxel truncation, updateEsdf).
// The GPU-generated TSDF voxels equal max(getSignedDistanceToPoint, -max_dist) of the host mirror bit for bit, with weight 1.
// Exit code 0 = pass, 77 = no GPU.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include "nvblox/nvblox.h"
using namespace nvblox;
#define EXPECT(c) do { if (!(c)) { std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
  // TypesList (host only)
  {
    primitives::Scene scene;
    scene.addPrimitive(std::make_unique<primitives::Plane>(Vector3f(1.0f, 0.0, 0.0), Vector3f(-1, 0, 0)));
    scene.addPrimitive(std::make_unique<primitives::Sphere>(Vector3f(0.0f, 0.0, 0.0), 1.0));
    scene.addPrimitive(std::make_unique<primitives::Cube>(Vector3f(0.0f, 0.0, 0.0), Vector3f(1.0, 1.0, 1.0)));
    scene.addPrimitive(std::make_unique<primitives::Cylinder>(Vector3f(0.0f, 0.0, 0.0), 1.0, 1.0));
    const std::vector<primitives::Primitive::Type> type_list = scene.getPrimitiveTypeList();
    EXPECT(type_list.size() == 4);
    EXPECT(type_list[0] == primitives::Primitive::Type::kPlane && type_list[1] == primitives::Primitive::Type::kSphere);
    EXPECT(type_list[2] == primitives::Primitive::Type::kCube && type_list[3] == primitives::Primitive::Type::kCylinder);
    EXPECT(primitives::Primitive::toString(type_list[3]) == "kCylinder");
    Vector3f p;
    float d = 0.0f;
    EXPECT(scene.getRayIntersection(Vector3f(-3.0f, 0.0f, 0.0f), Vector3f(1.0f, 0.0f, 0.0f), 10.0f, &p, &d) && d == 2.0f);
    EXPECT(scene.aabb().min()[0] == -5.0f && scene.aabb().max()[2] == 9.0f);
  }
  if (nvb_device_count() == 0) { std::fprintf(stderr, "no CUDA device\n"); return 77; }
  Camera camera(300.f, 300.f, 320.f, 240.f, 640, 480);
  // BlankMap
  {
    primitives::Scene scene;
    scene.aabb() = AxisAlignedBoundingBox(Vector3f(-3.0f, -3.0f, 0.0f), Vector3f(3.0f, 3.0f, 3.0f));
    constexpr float max_dist = 1.0;
    EXPECT(scene.getSignedDistanceToPoint(Vector3f::Zero(), max_dist) == max_dist);
    DepthImage depth_frame(camera.height(), camera.width(), MemoryType::kUnified);
    scene.generateDepthImageFromScene(camera, Transform::Identity(), max_dist, &depth_frame);
    for (int i = 0; i < depth_frame.numel(); i++) EXPECT(depth_frame(i) == 0.0f);
  }
  // PlaneScene, and the same plane seen from 1 m further back
  for (int offset = 0; offset < 2; offset++) {
    primitives::Scene scene;
    scene.addPrimitive(std::make_unique<primitives::Plane>(primitives::Plane(Vector3f(0.0f, 0.0, 1.0f), Vector3f(0, 0, -1))));
    Transform T_S_C = Transform::Identity();
    T_S_C(2, 3) = -1.0f * (float)offset;
    DepthImage depth_frame(camera.height(), camera.width(), MemoryType::kUnified);
    scene.generateDepthImageFromScene(camera, T_S_C, 4.0f, &depth_frame, -1.0f);
    for (int i = 0; i < depth_frame.numel(); i++) EXPECT(std::fabs(depth_frame(i) - (1.0f + offset)) < 1e-6f);
  }
  // py_scene.cu: createDummyMap, then the TSDF layer of a mapper and its ESDF
  {
    primitives::Scene scene;
    scene.aabb() = AxisAlignedBoundingBox(Vector3f(-5.5f, -5.5f, -0.5f), Vector3f(5.5f, 5.5f, 5.5f));
    scene.addPlaneBoundaries(-5.0f, 5.0f, -5.0f, 5.0f);
    scene.addGroundLevel(0.0f);
    scene.addCeiling(5.0f);
    scene.addPrimitive(std::make_unique<primitives::Cube>(Vector3f(0.0f, 0.0f, 2.0f), Vector3f(2.0f, 2.0f, 2.0f)));
    scene.addPrimitive(std::make_unique<primitives::Sphere>(Vector3f(0.0f, 0.0f, 2.0f), 2.0f));
    EXPECT(scene.getPrimitiveTypeList().size() == 8);
    const float voxel_size = 0.2f;
    Mapper mapper(voxel_size);
    TsdfLayer tsdf_layer = mapper.tsdf_layer();
    const float max_distance = 4.F * voxel_size;
    scene.generateLayerFromScene<TsdfVoxel>(max_distance, &tsdf_layer);
    const std::vector<Index3D> blocks = tsdf_layer.getAllBlockIndices();
    EXPECT(blocks.size() == 8 * 8 * 5);  // floor(+-5.5 / 1.6) = -4..3, floor(-0.5 / 1.6) .. floor(5.5 / 1.6) = -1..3
    const float bs = tsdf_layer.block_size();
    for (size_t i = 0; i < blocks.size(); i += 17) {
      auto blk = tsdf_layer.getBlockAtIndexHost(blocks[i]);
      EXPECT(blk != nullptr);
      for (int x = 0; x < 8; x++)
        for (int y = 0; y < 8; y++)
          for (int z = 0; z < 8; z++) {
            const Vector3f c((bs * (float)blocks[i][0] + voxel_size * (float)x) + bs * (0.5f / 8),
                             (bs * (float)blocks[i][1] + voxel_size * (float)y) + bs * (0.5f / 8),
                             (bs * (float)blocks[i][2] + voxel_size * (float)z) + bs * (0.5f / 8));
            const TsdfVoxel& v = blk->voxels[x][y][z];
            if (!scene.aabb().contains(c)) continue;
            const float d = scene.getSignedDistanceToPoint(c, max_distance);
            const float want = d < -max_distance ? -max_distance : d;
            EXPECT(std::memcmp(&v.distance, &want, sizeof(float)) == 0 && v.weight == 1.0f);
          }
    }
    mapper.updateEsdf();
    EXPECT(mapper.esdf_layer().numBlocks() == (int)blocks.size());
  }
  std::printf("scene drop-in: ok\n");
  return 0;
}
