// C++ test of the map-change methods of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp, stand-alone mode): two
// recordings of six submaps each of a sensor moving 1 m per submap along a corridor (floor, side walls and end walls). A
// post stands in the corridor during the first recording and is gone in the second. More than half of the post's points
// must be VANISHED, no point of the second recording may be dropped, and the updated map must be saved as PCD. Built on a
// CPU-only machine (where it must fail loudly for lack of a GPU, exit code 3) and run on the H100 by
// tests/test_map_changes_adapter.py with an output directory as argv[1].
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg_pcl.hpp"

int main(int argc, char** argv) {
  try {
    b200reg::ScanMatcherSession session;
    const int n_day = 6;
    size_t post_points = 0, day1_points = 0;
    for (int k = 0; k < 2 * n_day; k++) {
      std::vector<float> pts;  // x y z intensity (1 = the post), sensor frame: the sensor is at (x, 0, 1.5)
      const float sx = (float)(k % n_day) + (k >= n_day ? 0.5f : 0.f);
      for (int az = 0; az < 720; az++)
        for (int el = 0; el < 16; el++) {
          const float a = az * 0.00872665f, e = -0.35f + 0.04f * el;
          const float dx = std::cos(e) * std::cos(a), dy = std::cos(e) * std::sin(a), dz = std::sin(e);
          float t = 1e9f, label = 0.f;
          if (dz < 0) t = std::fmin(t, -1.5f / dz);                          // floor z = 0
          if (dy > 0) t = std::fmin(t, 4.f / dy);                            // walls y = +-4
          if (dy < 0) t = std::fmin(t, -4.f / dy);
          if (dx > 0) t = std::fmin(t, (30.f - sx) / dx);                    // end walls x = -20 and x = 30
          if (dx < 0) t = std::fmin(t, (-20.f - sx) / dx);
          if (k < n_day && dx > 0) {                                         // the post: x in [8, 8.4], |y| <= 0.2
            const float tp = (8.f - sx) / dx, yp = tp * dy, zp = 1.5f + tp * dz;
            if (std::fabs(yp) <= 0.2f && zp >= 0.f && zp <= 2.f && tp < t) t = tp, label = 1.f;
          }
          if (t > 40.f) continue;
          pts.insert(pts.end(), {t * dx, t * dy, t * dz, label});
          post_points += label > 0.f;
        }
      if (k < n_day) day1_points += pts.size() / 4;
      const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, (double)sx, 0, 1.5, 1};
      if (b200sm_import_submap(session.handle(), pts.data(), pts.size() / 4, 16, 12, pose, (double)k) != B200REG_OK)
        throw std::runtime_error(std::string("import: ") + b200sm_last_error(session.handle()));
    }
    const b200sm_map_change_info info = session.buildMapChanges({}, n_day);
    std::vector<unsigned char> labels;
    session.mapChanges(labels);
    std::vector<float> xyzi;
    std::vector<size_t> offsets;
    session.updatedMap(xyzi, &offsets);
    size_t post_kept = 0, vanished = 0, day2_dropped = 0;
    for (size_t i = 3; i < xyzi.size(); i += 4) post_kept += xyzi[i] > 0.f;
    for (size_t i = 0; i < labels.size(); i++) {
      vanished += labels[i] == B200SM_CHANGE_VANISHED;
      day2_dropped += i >= day1_points && labels[i] == B200SM_CHANGE_VANISHED;
    }
    std::vector<int> ijk;
    std::vector<unsigned> hb, fb, ha, fa;
    std::vector<unsigned char> vlabel;
    session.changeVoxels(ijk, hb, fb, ha, fa, vlabel);
    const std::string path = std::string(argc > 1 ? argv[1] : ".") + "/updated_map.pcd";
    session.saveUpdatedMapPcd(path);
    FILE* f = std::fopen(path.c_str(), "rb");
    long size = -1;
    if (f) {
      std::fseek(f, 0, SEEK_END);
      size = std::ftell(f);
      std::fclose(f);
    }
    std::printf("points %llu updated %llu voxels %llu vanished voxels %llu post %zu kept %zu file %ld\n", info.n_points,
                info.n_updated_points, info.n_voxels, info.n_vanished_voxels, post_points, post_kept, size);
    const bool ok = info.split_submap == n_day && labels.size() == info.n_points && vanished == info.n_vanished_points &&
                    info.n_updated_points * 4 == xyzi.size() && offsets.size() == (size_t)(2 * n_day) + 1 &&
                    offsets.back() == info.n_updated_points && vlabel.size() == info.n_voxels && post_points > 100 &&
                    post_kept * 2 < post_points && day2_dropped == 0 && info.n_points - info.n_updated_points == vanished && size > 0;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only machine: the engine has no CPU fallback
  }
}
