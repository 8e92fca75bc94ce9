// C++ test of the localisation methods of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp, stand-alone mode): a prior
// map set from host memory, the initial pose from three hypotheses, then frames of a sensor moving 0.4 m per frame in x,
// each registered against the cut of the map around the pose. Built on a CPU-only machine (where it must fail loudly for
// lack of a GPU, exit code 3) and run on the H100 by tests/test_localize_adapter.py.
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
    session.setLocalizationParams(30.0, 1.0);
    // the scan at sensor position (sx, 0, 0): the map's points within 25 m, in the sensor frame
    auto scan_at = [&](float sx) {
      b200reg::PointCloud s;
      for (size_t i = 0; i < map.size(); i += 3) {
        b200reg::PointXYZI q = map.points[i + (i / 3) % 3];
        q.x -= sx;
        if (q.x * q.x + q.y * q.y < 25.f * 25.f) s.points.push_back(q);
      }
      return s;
    };
    double pose[7];
    float fin[16];
    b200reg::PointCloud scan = scan_at(0.3f);
    std::vector<float> guesses;
    for (float gx : {-0.5f, 0.2f, 1.0f}) {  // column-major 4x4 translations
      float G[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, gx, 0, 0, 1};
      guesses.insert(guesses.end(), G, G + 16);
    }
    std::vector<b200reg_batch_result> rows;
    const int best = session.localizeInit(reg.handle(), &scan.points[0].x, scan.size(), sizeof(b200reg::PointXYZI),
                                          offsetof(b200reg::PointXYZI, intensity), guesses, rows);
    bool ok = rows.size() == 3 && best >= 0 && std::fabs(rows[best].final_T[12] - 0.3f) < 0.1f;
    int recuts = 0;
    for (int k = 1; k <= 6; k++) {
      scan = scan_at(0.3f + 0.4f * k);
      recuts += session.localizeCloud(reg.handle(), &scan.points[0].x, scan.size(), sizeof(b200reg::PointXYZI),
                                      offsetof(b200reg::PointXYZI, intensity), pose, fin)
                    ? 1
                    : 0;
      ok = ok && std::fabs(pose[0] - (0.3 + 0.4 * k)) < 0.1 && std::fabs(pose[1]) < 0.1;
    }
    const b200sm_localize_stats st = session.localizeStats();
    std::vector<float> cut;
    session.cutCloud(cut);
    std::printf("localize: best=%d pose x=%.3f y=%.3f recuts=%d cuts=%d cut=%zu of %zu, submaps=%zu\n", best, pose[0], pose[1], recuts,
                st.n_cuts, cut.size() / 4, st.n_map, session.numSubmaps());
    ok = ok && recuts >= 1 && st.n_cuts == recuts + 1 && st.n_map == map.size() && cut.size() == 4 * st.n_cut && st.n_cut > 0 &&
         st.n_cut < st.n_map && session.numSubmaps() == 0;
    for (size_t i = 4; i < cut.size(); i += 4) ok = ok && cut[i + 3] > cut[i - 1];  // map order: the intensities are row numbers
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
