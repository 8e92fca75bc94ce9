// C++ test of ScanMatcherSession::mergeSession (include/b200reg_pcl.hpp, stand-alone mode): session A holds twelve ray-cast
// submaps of a sensor moving 1 m per submap along a corridor with end walls; session B holds eight of the same scans with
// their poses in a frame turned by 0.5 rad and shifted by (40, -7, 0) m. The merge must succeed, size its rows and the
// adjusted poses, append B as a second segment, and place B's submaps where A's copies of them are. Built on a CPU-only
// machine (where it must fail loudly for lack of a GPU, exit code 3) and run on the H100 by tests/test_merge_adapter.py.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg_pcl.hpp"

namespace {
std::vector<float> corridor_scan(float sx) {
  std::vector<float> pts;  // x y z intensity, sensor frame: the sensor is at (sx, 0, 1.5)
  for (int az = 0; az < 720; az++)
    for (int el = 0; el < 16; el++) {
      const float a = az * 0.00872665f, e = -0.35f + 0.04f * el;
      const float dx = std::cos(e) * std::cos(a), dy = std::cos(e) * std::sin(a), dz = std::sin(e);
      float t = 1e9f;
      if (dz < 0) t = std::fmin(t, -1.5f / dz);
      if (dy > 0) t = std::fmin(t, (az % 90 < 10 ? 3.f : 4.f) / dy);  // walls with recesses
      if (dy < 0) t = std::fmin(t, -4.f / dy);
      if (dx > 0) t = std::fmin(t, (30.f - sx) / dx);
      if (dx < 0) t = std::fmin(t, (-20.f - sx) / dx);
      if (t > 40.f) continue;
      pts.insert(pts.end(), {t * dx, t * dy, t * dz, (float)el});
    }
  return pts;
}
void import(b200reg::ScanMatcherSession& s, const std::vector<float>& pts, const double* pose, double d) {
  if (b200sm_import_submap(s.handle(), pts.data(), pts.size() / 4, 16, 12, pose, d) != B200REG_OK)
    throw std::runtime_error(std::string("import: ") + b200sm_last_error(s.handle()));
}
}  // namespace

int main() {
  try {
    b200reg::ScanMatcherSession a, b;
    b200reg::NormalDistributionsTransform ndt;
    ndt.setResolution(1.0f);
    const double c = std::cos(0.5), s = std::sin(0.5), W[3] = {40.0, -7.0, 0.0};
    for (int k = 0; k < 12; k++) {
      const std::vector<float> pts = corridor_scan((float)k);
      const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, (double)k, 0, 1.5, 1};
      import(a, pts, pose, (double)k);
      if (k >= 2 && k < 10) {  // W^-1 * pose, W = Rz(0.5) + W: rotation R^T, translation R^T (p - W)
        const double px = k - W[0], py = -W[1];
        const double pb[16] = {c, -s, 0, 0, s, c, 0, 0, 0, 0, 1, 0, c * px + s * py, -s * px + c * py, 1.5, 1};
        import(b, pts, pb, (double)(k - 2));
      }
    }
    std::vector<b200sm_merge_row> rows;
    std::vector<double> poses;
    const b200sm_merge_result r = a.mergeSession(b, ndt.handle(), rows, poses);
    size_t n = 0, segs = 0, first[4] = {0, 0, 0, 0};
    b200sm_num_submaps(a.handle(), &n);
    b200sm_get_segments(a.handle(), first, 4, &segs);
    double worst = 0;  // B's submap j at its placement against A's copy of it (submap j + 2)
    for (int j = 0; j < 8; j++) {
      double pa[16], pm[16];
      b200sm_get_submap(a.handle(), j + 2, nullptr, 0, &n, pa, nullptr);
      b200sm_get_submap(a.handle(), 12 + j, nullptr, 0, &n, pm, nullptr);
      worst = std::fmax(worst, std::hypot(pa[12] - pm[12], pa[13] - pm[13]));
    }
    b200sm_num_submaps(a.handle(), &n);
    std::printf("merged %d verified %d accepted %d inliers %d rows %zu poses %zu submaps %zu segments %zu [%zu %zu] worst %.4f\n",
                r.merged, r.verified, r.accepted, r.inliers, rows.size(), poses.size(), n, segs, first[0], first[1], worst);
    const bool ok = r.merged == 1 && r.inliers >= 2 && rows.size() == (size_t)r.verified && poses.size() == 16 * 20 && n == 20 &&
                    segs == 2 && first[1] == 12 && r.first_submap == 12 && worst < 0.1;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
