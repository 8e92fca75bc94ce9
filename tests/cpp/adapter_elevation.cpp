// C++ test of the elevation-map methods of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp, stand-alone mode): four
// submaps of a grid of points over a 5 degree ramp beside a 1 m wall, 0.1 m apart. The ramp must read 5 degrees and be
// traversable, the wall lethal, and the traversability pair must be saved. Built on a CPU-only machine (where it must fail
// loudly for lack of a GPU, exit code 3) and run on the H100 by tests/test_elevation_adapter.py with an output directory as
// argv[1].
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg_pcl.hpp"

int main(int argc, char** argv) {
  try {
    b200reg::ScanMatcherSession session;
    const float slope = std::tan(5.0f * 3.14159265f / 180.0f);
    for (int k = 0; k < 4; k++) {
      std::vector<float> pts;  // x y z intensity, robot frame of a robot at (k, 0, 0)
      for (int i = 0; i < 100; i++)
        for (int j = 0; j < 60; j++) {
          const float x = 0.05f + 0.1f * i, y = 0.05f + 0.1f * j;  // map frame
          const float z = y < 5.0f ? slope * x : 1.0f;              // the wall: y in [5, 6)
          pts.insert(pts.end(), {x - (float)k, y, z, 0.f});
        }
      const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, (double)k, 0, 0, 1};
      if (b200sm_import_submap(session.handle(), pts.data(), pts.size() / 4, 16, 12, pose, (double)k) != B200REG_OK)
        throw std::runtime_error(std::string("import: ") + b200sm_last_error(session.handle()));
    }
    const b200sm_elevation_info info = session.buildElevationMap();
    std::vector<signed char> value;
    std::vector<float> tan_slope;
    session.elevationMap(value, nullptr, &tan_slope);
    size_t ramp = 0, ramp_ok = 0, wall = 0, wall_ok = 0;
    for (unsigned y = 0; y < info.height; y++)
      for (unsigned x = 0; x < info.width; x++) {
        const size_t q = (size_t)y * info.width + x;
        if (x >= 3 && x + 3 < info.width && y >= 3 && y < 45) {
          ramp++;
          ramp_ok += value[q] >= 0 && value[q] < 100 && std::fabs(std::atan(tan_slope[q]) * 180.0f / 3.14159265f - 5.0f) < 0.2f;
        }
        if (y >= 50) {
          wall++;
          wall_ok += value[q] == 100 || (y >= 53 && value[q] >= 0);  // the wall's top away from its edge is flat
        }
      }
    const std::string dir = std::string(argc > 1 ? argv[1] : ".");
    session.saveTraversabilityMap(dir + "/traversability.pgm", dir + "/traversability.yaml");
    FILE* f = std::fopen((dir + "/traversability.pgm").c_str(), "rb");
    long size = -1;
    if (f) {
      std::fseek(f, 0, SEEK_END);
      size = std::ftell(f);
      std::fclose(f);
    }
    std::printf("cells %u x %u observed %llu lethal %llu ramp %zu/%zu wall %zu/%zu file %ld\n", info.width, info.height, info.n_observed,
                info.n_lethal, ramp_ok, ramp, wall_ok, wall, size);
    const bool ok = info.width == 100 && info.height == 60 && ramp > 1000 && ramp_ok == ramp && wall_ok == wall &&
                    size > (long)(info.width * info.height) && info.n_lethal > 0;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
