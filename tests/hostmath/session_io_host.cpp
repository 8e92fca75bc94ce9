// CPU harness of lidarslam_ros2_b200/csrc/session_io.hpp (the on-disk form of b200sm_save_session / b200sm_load_session),
// built by tests/test_session_io_cpu.py with g++ -ffp-contract=off as the library builds it. Poses are column-major 4x4
// doubles, as in the manifest.
#include <cstring>
#include <string>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/session_io.hpp"

using namespace b200;

namespace {
sio::Manifest manifest(const int* sc_rs, const double* sc_rh, int n, int m, const int* seg, const unsigned long long* points,
                       const double* dist, const double* pose, int k, int L, const int* loop_ft, const double* loop_rel,
                       const double* adjusted) {
  sio::Manifest M;
  M.sc.num_rings = sc_rs[0];
  M.sc.num_sectors = sc_rs[1];
  M.sc.max_radius = sc_rh[0];
  M.sc.lidar_height = sc_rh[1];
  M.seg_first.assign(seg, seg + m);
  M.points.assign(points, points + n);
  M.distance.assign(dist, dist + n);
  M.pose.assign(pose, pose + 16 * (size_t)n);
  M.k = k;
  M.loops.resize(L);
  for (int l = 0; l < L; l++) {
    M.loops[l].from = loop_ft[2 * l];
    M.loops[l].to = loop_ft[2 * l + 1];
    std::memcpy(M.loops[l].rel, loop_rel + 16 * l, sizeof(M.loops[l].rel));
  }
  M.adjusted = adjusted != nullptr;
  if (adjusted) M.adjusted_pose.assign(adjusted, adjusted + 16 * (size_t)n);
  return M;
}
size_t copy_out(const std::string& s, char* out, size_t cap) {
  if (out) std::memcpy(out, s.data(), std::min(cap, s.size()));
  return s.size();
}
sio::Manifest parsed;  // the last sioh_parse's result
}  // namespace

extern "C" {

// the manifest (which = 0), the g2o text (1) or the binary PCD header of points[0] (2); returns its size, copies min(cap, size)
size_t sioh_write(int which, const int* sc_rs, const double* sc_rh, int n, int m, const int* seg, const unsigned long long* points,
                  const double* dist, const double* pose, int k, int L, const int* loop_ft, const double* loop_rel,
                  const double* adjusted, char* out, size_t cap) {
  const sio::Manifest M = manifest(sc_rs, sc_rh, n, m, seg, points, dist, pose, k, L, loop_ft, loop_rel, adjusted);
  if (which == 2) return copy_out(sio::pcd_binary_header(points[0]), out, cap);
  return copy_out(which == 0 ? sio::write_manifest(M) : sio::write_g2o(M), out, cap);
}

// 1 and counts6 = (n, segments, k, loops, adjusted, 0) on success; 0 with the message in err otherwise
int sioh_parse(const char* text, size_t len, long long* counts6, char* err, size_t err_cap) {
  std::string why;
  sio::Manifest M;
  if (!sio::parse_manifest(std::string(text, len), M, why)) {
    std::snprintf(err, err_cap, "%s", why.c_str());
    return 0;
  }
  parsed = M;
  counts6[0] = (long long)M.n();
  counts6[1] = (long long)M.seg_first.size();
  counts6[2] = M.k;
  counts6[3] = (long long)M.loops.size();
  counts6[4] = M.adjusted ? 1 : 0;
  counts6[5] = 0;
  return 1;
}

// the last parse's values, into arrays sized from its counts (adjusted may be NULL)
void sioh_parsed(int* sc_rs, double* sc_rh, int* seg, unsigned long long* points, double* dist, double* pose, int* loop_ft,
                 double* loop_rel, double* adjusted) {
  const sio::Manifest& M = parsed;
  sc_rs[0] = M.sc.num_rings;
  sc_rs[1] = M.sc.num_sectors;
  sc_rh[0] = M.sc.max_radius;
  sc_rh[1] = M.sc.lidar_height;
  for (size_t s = 0; s < M.seg_first.size(); s++) seg[s] = M.seg_first[s];
  for (size_t i = 0; i < M.n(); i++) {
    points[i] = M.points[i];
    dist[i] = M.distance[i];
  }
  std::memcpy(pose, M.pose.data(), M.pose.size() * sizeof(double));
  for (size_t l = 0; l < M.loops.size(); l++) {
    loop_ft[2 * l] = M.loops[l].from;
    loop_ft[2 * l + 1] = M.loops[l].to;
    std::memcpy(loop_rel + 16 * l, M.loops[l].rel, sizeof(M.loops[l].rel));
  }
  if (adjusted && M.adjusted) std::memcpy(adjusted, M.adjusted_pose.data(), M.adjusted_pose.size() * sizeof(double));
}

// The g2o writer's edges next to pg::build_edges': from / to of both, the writer's measurement Z and build_edges' Z^-1
// (row-major 12: R then t per row). Returns the count of each (they are compared by the caller).
int sioh_edges(int n, const double* pose, int k, int m, const int* seg, int L, const int* loop_ft, const double* loop_rel,
               int* ft_io, int* ft_pg, double* Z12, double* Zinv12, int* n_pg) {
  std::vector<pg::Iso> X(n);
  for (int i = 0; i < n; i++) X[i] = pg::iso_from_colmajor16(pose + 16 * i);
  std::vector<sio::LoopEdge> loops(L);
  std::vector<pg::Iso> rel(L);
  for (int l = 0; l < L; l++) {
    loops[l].from = loop_ft[2 * l];
    loops[l].to = loop_ft[2 * l + 1];
    std::memcpy(loops[l].rel, loop_rel + 16 * l, sizeof(loops[l].rel));
    rel[l] = pg::iso_from_colmajor16(loop_rel + 16 * l);
  }
  const std::vector<int> segs(seg, seg + m);
  const std::vector<sio::GraphEdge> a = sio::graph_edges(X, k, segs, loops);
  const std::vector<pg::Edge> b = pg::build_edges(X, k, segs, loop_ft, rel.data(), L);
  auto put = [](const pg::Iso& I, double* o) {
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) o[r * 4 + c] = I.R[r * 3 + c];
      o[r * 4 + 3] = I.t[r];
    }
  };
  for (size_t e = 0; e < a.size(); e++) {
    ft_io[2 * e] = a[e].from;
    ft_io[2 * e + 1] = a[e].to;
    put(a[e].Z, Z12 + 12 * e);
  }
  for (size_t e = 0; e < b.size(); e++) {
    ft_pg[2 * e] = b[e].from;
    ft_pg[2 * e + 1] = b[e].to;
    put(b[e].zinv, Zinv12 + 12 * e);
  }
  *n_pg = (int)b.size();
  return (int)a.size();
}
}
