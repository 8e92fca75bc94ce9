// C++ test of the OctoMap methods of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp, stand-alone mode): six submaps
// of a sensor moving 1 m per submap along a corridor (floor, side walls and end walls). The OctoMap must have occupied and
// free voxels and leaves, a tree whose size adds up, and a .bt file of the stated size that starts with OctoMap's first
// header line and states that size. Built on a CPU-only machine (where it must fail loudly for lack of a GPU, exit code 3)
// and run on the H100 by tests/test_octomap_adapter.py with an output directory as argv[1].
#include <cmath>
#include <cstdio>
#include <cstring>
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
    const b200sm_octomap_info info = session.buildOctoMap();
    const std::string path = std::string(argc > 1 ? argv[1] : ".") + "/map.bt";
    const size_t bytes = session.saveOctoMapBt(path);
    std::vector<char> file(bytes + 1, 0);
    FILE* f = std::fopen(path.c_str(), "rb");
    size_t got = 0;
    if (f) {
      got = std::fread(file.data(), 1, file.size(), f);
      std::fclose(f);
    }
    const std::string size_line = "\nsize " + std::to_string(info.tree_size) + "\nres 0.2\ndata\n";
    std::printf("rays %llu occupied %llu free %llu inner %llu size %llu file %zu\n", info.n_rays, info.n_occupied_voxels,
                info.n_free_voxels, info.n_inner_nodes, info.tree_size, got);
    const bool ok = info.n_occupied_voxels > 1000 && info.n_free_voxels > info.n_occupied_voxels && info.n_occupied_leaves > 0 &&
                    info.n_free_leaves > 0 && info.tree_size == info.n_inner_nodes + info.n_occupied_leaves + info.n_free_leaves &&
                    got == bytes && bytes == info.n_bytes && std::strncmp(file.data(), "# Octomap OcTree binary file\n", 29) == 0 &&
                    std::string(file.data(), got).find(size_line) != std::string::npos;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
