// C++ test of ScanMatcherSession::saveSession / loadSession (include/b200reg_pcl.hpp, stand-alone mode): a session of nine
// ray-cast corridor submaps (intensity = ring, one submap empty) is saved with two loop edges and adjusted poses into the
// directory given as argv[1], then loaded into a fresh session. Every submap's rows, pose and distance must come back
// bitwise, with the segments and the graph. Built on a CPU-only machine (where it must fail loudly for lack of a GPU,
// exit code 3) and run on the H100 by tests/test_session_io_adapter.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg_pcl.hpp"

namespace {
std::vector<float> corridor_scan(float sx) {
  std::vector<float> pts;  // x y z intensity, sensor frame: the sensor is at (sx, 0, 1.5)
  for (int az = 0; az < 360; az++)
    for (int el = 0; el < 16; el++) {
      const float a = az * 0.0174533f, e = -0.35f + 0.04f * el;
      const float dx = std::cos(e) * std::cos(a), dy = std::cos(e) * std::sin(a), dz = std::sin(e);
      float t = 1e9f;
      if (dz < 0) t = std::fmin(t, -1.5f / dz);
      if (dy > 0) t = std::fmin(t, 3.f / dy);
      if (dy < 0) t = std::fmin(t, -4.f / dy);
      if (dx > 0) t = std::fmin(t, (30.f - sx) / dx);
      if (dx < 0) t = std::fmin(t, (-20.f - sx) / dx);
      if (t > 40.f) continue;
      pts.insert(pts.end(), {t * dx, t * dy, t * dz, (float)el + 0.25f * sx});
    }
  return pts;
}
}  // namespace

int main(int argc, char** argv) {
  try {
    if (argc < 2) throw std::invalid_argument("usage: adapter_session_io <dir>");
    b200reg::ScanMatcherSession a;
    std::vector<std::vector<float>> clouds;
    for (int k = 0; k < 9; k++) {
      clouds.push_back(k == 4 ? std::vector<float>() : corridor_scan((float)k));
      const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, (double)k, 0.01 * k, 1.5, 1};
      if (b200sm_import_submap(a.handle(), clouds[k].data(), clouds[k].size() / 4, 16, 12, pose, 1.0 * k) != B200REG_OK)
        throw std::runtime_error(std::string("import: ") + b200sm_last_error(a.handle()));
    }
    std::vector<b200sm_loop_edge> edges(2);
    for (int l = 0; l < 2; l++) {
      edges[l].from = l;
      edges[l].to = 8 - l;
      const double Z[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 8.0 - 2 * l, 0.08 - 0.02 * l, 0, 1};
      std::memcpy(edges[l].relative_pose, Z, sizeof(Z));
    }
    std::vector<double> poses;
    a.poseAdjust(edges, poses, 3);
    const b200sm_session_io_info saved = a.saveSession(argv[1], edges, 3, poses);
    b200reg::ScanMatcherSession b;
    std::vector<b200sm_loop_edge> edges_back;
    std::vector<double> poses_back;
    int k = 0;
    const b200sm_session_io_info loaded = b.loadSession(argv[1], edges_back, poses_back, k);
    bool same = b.numSubmaps() == 9 && k == 3 && edges_back.size() == 2 && poses_back == poses &&
                loaded.n_points == saved.n_points && loaded.n_submaps == 9 && loaded.adjusted == 1;
    for (size_t l = 0; same && l < edges_back.size(); l++)
      same = edges_back[l].from == edges[l].from && edges_back[l].to == edges[l].to &&
             std::memcmp(edges_back[l].relative_pose, edges[l].relative_pose, sizeof(edges[l].relative_pose)) == 0;
    for (size_t i = 0; same && i < 9; i++) {
      std::vector<float> p(clouds[i].size() + 4), q(clouds[i].size() + 4);
      double pa[16], pb[16], da = 0, db = 0;
      size_t na = 0, nb = 0;
      b200sm_get_submap(a.handle(), i, p.data(), p.size() / 4, &na, pa, &da);
      b200sm_get_submap(b.handle(), i, q.data(), q.size() / 4, &nb, pb, &db);
      same = na == nb && na == clouds[i].size() / 4 && std::memcmp(p.data(), q.data(), 16 * na) == 0 &&
             std::memcmp(pa, pb, sizeof(pa)) == 0 && da == db;
    }
    std::vector<double> poses_b;
    b.poseAdjust(edges_back, poses_b, k);
    same = same && poses_b == poses;
    std::printf("saved %zu submaps %zu points %llu bytes; loaded %zu submaps, k %d, %zu edges: %s\n", saved.n_submaps, saved.n_points,
                saved.n_bytes, loaded.n_submaps, k, edges_back.size(), same ? "identical" : "DIFFERENT");
    return same ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
