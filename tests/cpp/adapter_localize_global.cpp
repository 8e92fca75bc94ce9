// C++ test of global localisation through the adapter (include/b200reg_pcl.hpp, stand-alone mode): a prior map set from host
// memory, a session started 1.7 m / 1.2 m off the sensor with no guess list, ScanMatcherSession::localizeGlobal over an
// (x, y, yaw) grid, the grid read back with globalSearch and scored again with NormalDistributionsTransform::scorePoses on the
// same target and source (bitwise the session's scores), then a frame of localizeCloud from the adopted pose. Built on a
// CPU-only machine (where it must fail loudly for lack of a GPU, exit code 3) and run on the H100 by
// tests/test_localize_global_adapter.py.
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
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
    unsigned seed = 11;
    for (int i = 0; i < 120000; i++) {  // a floor, a wall along x with pilasters every 5 m, and cross walls every 20 m
      b200reg::PointXYZI p;
      float u = 120.f * frand(seed) - 60.f, v = 40.f * frand(seed) - 20.f;
      int kind = i % 3;
      if (kind == 0) { p.x = u; p.y = v; p.z = 0.02f * frand(seed); }
      else if (kind == 1) { p.x = u; p.y = 10.f - (std::fmod(u + 60.f, 5.f) < 1.f ? 1.f : 0.f); p.z = 4.f * frand(seed); }
      else { p.x = 20.f * std::floor(u / 20.f) + 0.02f * frand(seed); p.y = v; p.z = 4.f * frand(seed); }
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
    session.setLocalizationParams(30.0, 1.0);  // >= radius + scan_max_range
    auto scan_at = [&](float sx) {  // the map's points within 25 m of (sx, 0, 0), in the sensor frame
      b200reg::PointCloud s;
      for (size_t i = 0; i < map.size(); i += 3) {
        b200reg::PointXYZI q = map.points[i + (i / 3) % 3];
        q.x -= sx;
        if (q.x * q.x + q.y * q.y < 25.f * 25.f) s.points.push_back(q);
      }
      return s;
    };
    const double start[3] = {2.0, 1.2, 0.0}, quat[4] = {0.0, 0.0, 0.0, 1.0};
    session.setInitialPose(start, quat);
    b200reg::PointCloud scan = scan_at(0.3f);
    const b200sm_global_search spec{3.0, 0.5, 8, 4};  // radius, step, yaw_steps, top_k
    std::vector<int> cand;
    std::vector<b200reg_batch_result> rows;
    b200sm_global_result info{};
    const int best = session.localizeGlobal(reg.handle(), &scan.points[0].x, scan.size(), sizeof(b200reg::PointXYZI),
                                            offsetof(b200reg::PointXYZI, intensity), spec, cand, rows, &info);
    std::vector<float> poses;
    std::vector<double> scores, again;
    std::vector<long long> hits, hits_again;
    session.globalSearch(poses, scores, hits);
    reg.scorePoses(poses, again, hits_again);  // the engine's target and source are the session's cut and filtered scan
    bool ok = best >= 0 && rows.size() == 4 && cand.size() == 4 && info.n_refined == 4 && info.n_hypotheses == (long long)scores.size() &&
              poses.size() == 16 * scores.size() && std::fabs(rows[best].final_T[12] - 0.3f) < 0.1f &&
              std::fabs(rows[best].final_T[13]) < 0.1f;
    ok = ok && again.size() == scores.size() && std::memcmp(again.data(), scores.data(), scores.size() * sizeof(double)) == 0 &&
         hits_again == hits;
    for (size_t r = 1; r < cand.size(); r++) ok = ok && scores[cand[r - 1]] >= scores[cand[r]];
    double pose[7];
    float fin[16];
    scan = scan_at(0.7f);
    session.localizeCloud(reg.handle(), &scan.points[0].x, scan.size(), sizeof(b200reg::PointXYZI), offsetof(b200reg::PointXYZI, intensity),
                          pose, fin);
    ok = ok && std::fabs(pose[0] - 0.7) < 0.1 && std::fabs(pose[1]) < 0.1;
    std::printf("localize_global: %lld hypotheses, best row %d (hypothesis %d) x=%.3f y=%.3f, next frame x=%.3f y=%.3f\n",
                info.n_hypotheses, best, best >= 0 ? cand[best] : -1, best >= 0 ? rows[best].final_T[12] : 0.f,
                best >= 0 ? rows[best].final_T[13] : 0.f, pose[0], pose[1]);
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
