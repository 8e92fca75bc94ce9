// C++ test of the map-consistency method of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp, stand-alone mode): two
// submaps of a floor and a wall, the second 2 cm off. The adapter's buildMapConsistency must return exactly the info the
// C-ABI's b200sm_build_map_consistency returns for the same session and parameters, with valid queries and a finite MME.
// Built on a CPU-only machine (where it must fail loudly for lack of a GPU, exit code 3) and run on the H100 by
// tests/test_map_consistency_adapter.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg_pcl.hpp"

int main() {
  try {
    b200reg::ScanMatcherSession session;
    for (int k = 0; k < 2; k++) {
      std::vector<float> pts;  // x y z intensity: a floor and a wall at x = 3
      for (int i = 0; i < 60; i++)
        for (int j = 0; j < 60; j++) {
          pts.insert(pts.end(), {0.05f * i, 0.05f * j, 0.003f * (float)((i * 7 + j * 3) % 5), 0.f});
          pts.insert(pts.end(), {3.0f + 0.003f * (float)((i + j) % 4), 0.05f * j, 0.05f * i, 0.f});
        }
      const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0.02 * k, 0, 0, 1};
      if (b200sm_import_submap(session.handle(), pts.data(), pts.size() / 4, 16, 12, pose, (double)k) != B200REG_OK)
        throw std::runtime_error(std::string("import: ") + b200sm_last_error(session.handle()));
    }
    const b200sm_map_consistency_params p{0.3, 10, 2};
    const b200sm_map_consistency_info a = session.buildMapConsistency({}, &p);
    b200sm_map_consistency_info b{};
    if (b200sm_build_map_consistency(session.handle(), nullptr, &p, &b) != B200REG_OK)
      throw std::runtime_error(std::string("build: ") + b200sm_last_error(session.handle()));
    const b200sm_map_consistency_info d = session.buildMapConsistency();
    std::printf("points %llu queries %llu valid %llu mme %.6f mpv %.3g defaults: queries %llu\n", a.n_points, a.n_queries, a.n_valid,
                a.mme, a.mpv, d.n_queries);
    const bool ok = std::memcmp(&a, &b, sizeof(a)) == 0 && a.n_points == 14400 && a.n_queries == 7200 && a.n_valid > 0 &&
                    std::isfinite(a.mme) && d.n_queries == 14400;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
