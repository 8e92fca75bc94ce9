// C++ test of relocalisation through the adapter (include/b200reg_pcl.hpp, stand-alone mode): a prior map set from host
// memory, a session started far from the sensor with the heading wrong, ScanMatcherSession::relocalize with the default
// parameters but fewer headings, then a frame of localizeCloud from the adopted pose. Built on a CPU-only machine (where it
// must fail loudly for lack of a GPU, exit code 3) and run on the H100 by tests/test_relocalize_adapter.py.
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "b200reg_pcl.hpp"

static float frand(unsigned& s) {
  s = s * 1664525u + 1013904223u;
  return (float)((s >> 8) & 0xffffff) / 16777216.0f;
}

int main() {
  try {
    b200reg::PointCloud map;
    unsigned seed = 17;
    for (int i = 0; i < 120000; i++) {  // a floor, a wall along x with pilasters every 5 m, and cross walls at irregular x
      b200reg::PointXYZI p;
      float u = 120.f * frand(seed) - 60.f, v = 40.f * frand(seed) - 20.f;
      int kind = i % 3;
      static const float walls[6] = {-47.f, -31.f, -8.f, 13.f, 22.f, 51.f};
      if (kind == 0) { p.x = u; p.y = v; p.z = 0.02f * frand(seed); }
      else if (kind == 1) { p.x = u; p.y = 10.f - (std::fmod(u + 60.f, 5.f) < 1.f ? 1.f : 0.f); p.z = 4.f * frand(seed); }
      else { p.x = walls[i % 6] + 0.02f * frand(seed); p.y = v; p.z = 4.f * frand(seed); }
      p.intensity = (float)i;
      map.points.push_back(p);
    }
    b200reg::NormalDistributionsTransform reg;
    reg.setResolution(2.0f);
    reg.setTransformationEpsilon(0.01);
    reg.setNeighborhoodSearchMethod(b200reg::DIRECT7);
    b200reg::ScanMatcherSession session;
    session.setParams(0.5f, 0.4f, 10, 1.5, true, 0.5, 25.0);
    session.setPriorMap(&map.points[0].x, map.size(), sizeof(b200reg::PointXYZI), offsetof(b200reg::PointXYZI, intensity));
    session.setLocalizationParams(30.0, 1.0);
    auto scan_at = [&](float sx) {  // the map's points within 25 m of (sx, 0, 0), in the sensor frame
      b200reg::PointCloud s;
      for (size_t i = 0; i < map.size(); i += 3) {
        b200reg::PointXYZI q = map.points[i + (i / 3) % 3];
        q.x -= sx;
        if (q.x * q.x + q.y * q.y < 25.f * 25.f) s.points.push_back(q);
      }
      return s;
    };
    const double start[3] = {-40.0, 6.0, 0.0}, quat[4] = {0.0, 0.0, std::sin(1.0), std::cos(1.0)};  // 2 rad off
    session.setInitialPose(start, quat);
    b200reg::PointCloud scan = scan_at(0.3f);
    b200sm_relocalize_params p{0.25, 0.3, 3.0, 72, 6, 0.3, 4, 1.0};
    std::vector<b200sm_relocalize_row> rows;
    b200sm_relocalize_result info{};
    const int best = session.relocalize(reg.handle(), &scan.points[0].x, scan.size(), sizeof(b200reg::PointXYZI),
                                        offsetof(b200reg::PointXYZI, intensity), &p, rows, &info);
    bool ok = best >= 0 && !rows.empty() && info.n_rows == (int)rows.size() && info.m > 0 && info.width > 0;
    for (size_t r = 1; r < rows.size(); r++) ok = ok && rows[r - 1].score >= rows[r].score;
    for (size_t r = 0; r < rows.size(); r++)
      if (ok && rows[r].status == B200REG_OK && rows[r].converged && rows[r].fitness < p.accept_fitness)
        ok = rows[(size_t)best].fitness <= rows[r].fitness;
    ok = ok && std::fabs(rows[(size_t)best].final_T[12] - 0.3f) < 0.1f && std::fabs(rows[(size_t)best].final_T[13]) < 0.1f;
    double pose[7];
    float fin[16];
    scan = scan_at(0.7f);
    session.localizeCloud(reg.handle(), &scan.points[0].x, scan.size(), sizeof(b200reg::PointXYZI), offsetof(b200reg::PointXYZI, intensity),
                          pose, fin);
    ok = ok && std::fabs(pose[0] - 0.7) < 0.1 && std::fabs(pose[1]) < 0.1;
    std::printf("relocalize: grid %lld x %lld, m %lld, best row %d x=%.3f y=%.3f (search %.3f ms), next frame x=%.3f y=%.3f\n",
                info.width, info.height, info.m, best, best >= 0 ? rows[(size_t)best].final_T[12] : 0.f,
                best >= 0 ? rows[(size_t)best].final_T[13] : 0.f, info.search_ms, pose[0], pose[1]);
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
