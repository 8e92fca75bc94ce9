// C++ test of the mesh methods of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp, stand-alone mode): six submaps of
// a sensor moving 1 m per submap along a corridor (floor, side walls and end walls). The mesh must have vertices on the
// walls and floor within a few centimetres, faces whose ids are below the vertex count, band voxels whose weights add up to
// the walked voxels, and a PLY file of the stated size. Built on a CPU-only machine (where it must fail loudly for lack of
// a GPU, exit code 3) and run on the H100 by tests/test_mesh_adapter.py with an output directory as argv[1].
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg_pcl.hpp"

int main(int argc, char** argv) {
  try {
    b200reg::ScanMatcherSession session;
    for (int k = 0; k < 6; k++) {
      std::vector<float> pts;  // x y z intensity, sensor frame: the sensor is at (k, 0, 1.5)
      const float sx = (float)k;
      for (int az = 0; az < 720; az++)
        for (int el = 0; el < 16; el++) {
          const float a = az * 0.00872665f, e = -0.35f + 0.04f * el;
          const float dx = std::cos(e) * std::cos(a), dy = std::cos(e) * std::sin(a), dz = std::sin(e);
          float t = 1e9f;
          if (dz < 0) t = std::fmin(t, -1.5f / dz);  // floor z = 0
          if (dy > 0) t = std::fmin(t, 4.1f / dy);   // walls y = +-4.1
          if (dy < 0) t = std::fmin(t, -4.1f / dy);
          if (dx > 0) t = std::fmin(t, (30.f - sx) / dx);
          if (dx < 0) t = std::fmin(t, (-20.f - sx) / dx);
          if (t > 40.f) continue;
          pts.insert(pts.end(), {t * dx, t * dy, t * dz, 0.f});
        }
      const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, (double)sx, 0, 1.5, 1};
      if (b200sm_import_submap(session.handle(), pts.data(), pts.size() / 4, 16, 12, pose, (double)k) != B200REG_OK)
        throw std::runtime_error(std::string("import: ") + b200sm_last_error(session.handle()));
    }
    const b200sm_mesh_info info = session.buildMesh();
    std::vector<float> xyz;
    std::vector<unsigned> faces;
    session.mesh(xyz, faces);
    std::vector<int> ijk;
    std::vector<long long> sum;
    std::vector<unsigned> weight;
    session.meshVoxels(ijk, sum, weight);
    size_t near = 0, bad_face = 0;
    unsigned long long walked = 0;
    for (size_t v = 0; v < xyz.size(); v += 3) {
      const float x = xyz[v], y = xyz[v + 1], z = xyz[v + 2];
      const float d = std::fmin(std::fmin(std::fabs(z), std::fabs(std::fabs(y) - 4.1f)), std::fmin(std::fabs(x - 30.f), std::fabs(x + 20.f)));
      near += d < 0.05f;
    }
    for (unsigned f : faces) bad_face += f >= info.n_vertices;
    for (unsigned w : weight) walked += w;
    const std::string path = std::string(argc > 1 ? argv[1] : ".") + "/mesh.ply";
    const size_t bytes = session.saveMeshPly(path);
    FILE* f = std::fopen(path.c_str(), "rb");
    long size = -1;
    if (f) {
      std::fseek(f, 0, SEEK_END);
      size = std::ftell(f);
      std::fclose(f);
    }
    std::printf("rays %llu band %llu vertices %llu faces %llu near %zu file %ld\n", info.n_rays, info.n_band_voxels, info.n_vertices,
                info.n_faces, near, size);
    const bool ok = info.n_faces > 1000 && xyz.size() == 3 * info.n_vertices && faces.size() == 3 * info.n_faces && bad_face == 0 &&
                    near * 10 >= info.n_vertices * 9 && weight.size() == info.n_band_voxels && walked == info.n_walked &&
                    size == (long)bytes && bytes > 13 * info.n_faces + 12 * info.n_vertices;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
