// CPU harness of lidarslam_ros2_b200/csrc/relocalize.hpp (the relocalisation search of b200sm_relocalize, run serially),
// built by tests/test_relocalize_cpu.py with g++ -ffp-contract=off as the library builds its host code. One map and one
// scan at a time: rl_set_map builds the pyramid, rl_set_scan the offsets table, rl_search runs the search.
#include <cstring>

#include "../../lidarslam_ros2_b200/csrc/relocalize.hpp"

namespace {
b200::RlParams g_params;
b200::RlHostPyramid g_pyr;
std::vector<b200::RlOff> g_offs;
long long g_m = 0;
std::string g_err;

void copy_err(char* err, int cap) {
  if (err && cap > 0) {
    std::strncpy(err, g_err.c_str(), (size_t)cap - 1);
    err[cap - 1] = 0;
  }
}
}  // namespace

extern "C" {

// params: the layout of b200sm_relocalize_params. Returns 1 when valid.
int rl_valid(const b200::RlParams* p) { return b200::rl_params_valid(*p) ? 1 : 0; }

// 0, or 1 when a limit is exceeded (err). grid6 = i0, j0, W, H, TW, TH.
int rl_set_map(const float* map4, size_t n, const b200::RlParams* p, long long* grid6, char* err, int err_cap) {
  g_params = *p;
  g_err.clear();
  g_m = 0;
  g_offs.clear();
  if (!b200::rl_build_pyramid_host(map4, n, *p, g_pyr, g_err)) {
    copy_err(err, err_cap);
    return 1;
  }
  const b200::RlGrid& g = g_pyr.g;
  const long long v[6] = {g.i0, g.j0, g.W, g.H, g.TW, g.TH};
  std::memcpy(grid6, v, sizeof(v));
  return 0;
}

// level h: stored width and height; the bytes into out when capacity allows
int rl_level(int h, unsigned char* out, size_t capacity, long long* w, long long* hh) {
  if (g_pyr.g.W == 0) {
    *w = *hh = 0;
    return 0;
  }
  *w = b200::rl_level_w(g_pyr.g, h);
  *hh = b200::rl_level_h(g_pyr.g, h);
  const size_t n = (size_t)(*w * *hh);
  if (out && capacity >= n) std::memcpy(out, g_pyr.level(h), n);
  return 0;
}

// another yaw_steps for the next rl_set_scan / rl_search on the same pyramid (a session's pyramid serves any)
void rl_set_yaw_steps(int yaw_steps) { g_params.yaw_steps = yaw_steps; }

// the offsets of the scan under the pose's rotations at its height: m, or -1 when the points exceed their caps (err)
long long rl_set_scan(const float* scan4, size_t n, const double* position, const double* quat, char* err, int err_cap) {
  std::vector<double> rot_d;
  std::vector<float> rot_f;
  b200::rl_rotations(position, quat, g_params.yaw_steps, rot_d, rot_f);
  b200::rl_offsets_host(scan4, n, rot_f, g_params.yaw_steps, position[2], g_params, g_offs, &g_m);
  g_err = b200::rl_check_points(g_m, g_params.yaw_steps);
  if (!g_err.empty()) {
    copy_err(err, err_cap);
    return -1;
  }
  return g_m;
}

// the offsets table (yaw_steps x m pairs)
void rl_offsets(int* out) {
  if (!g_offs.empty()) std::memcpy(out, g_offs.data(), g_offs.size() * sizeof(b200::RlOff));
}

void rl_scores(int h, long long count, const int* kij, long long* out) {
  for (long long q = 0; q < count; q++)
    out[q] = g_m ? b200::rl_score_host(g_pyr, g_offs, g_m, h, b200::RlNode{kij[3 * q], kij[3 * q + 1], kij[3 * q + 2]}) : 0;
}

// info3 = t0, t, n_rows; nodes16; tiles / keys: top_k each. 0, or 1 at a limit of the headings or the frontier (err).
int rl_search(int exhaustive, long long* info3, long long* nodes16, long long* tiles, unsigned long long* keys, char* err, int err_cap) {
  b200::RlHostResult r;
  b200::rl_search_serial(g_pyr, g_offs, g_m, g_params, exhaustive != 0, r);
  if (!r.error.empty()) {
    g_err = r.error;
    copy_err(err, err_cap);
    return 1;
  }
  info3[0] = r.t0;
  info3[1] = r.t;
  info3[2] = (long long)r.tiles.size();
  std::memcpy(nodes16, r.nodes, sizeof(r.nodes));
  for (size_t q = 0; q < r.tiles.size(); q++) {
    tiles[q] = r.tiles[q];
    keys[q] = r.keys[q];
  }
  return 0;
}

// the guess of leaf (k, i, j) of the current grid for the pose (column-major)
void rl_guess_of(const double* position, const double* quat, int k, long long i, long long j, float* col16) {
  std::vector<double> rot_d;
  std::vector<float> rot_f;
  b200::rl_rotations(position, quat, g_params.yaw_steps, rot_d, rot_f);
  b200::rl_guess(rot_d.data() + 9 * (size_t)k, g_pyr.g, g_params.resolution, position[2], i, j, col16);
}

// the verdict of rl_make_grid and rl_check_headings on a box (1 = refused by the grid, 2 = by the headings)
int rl_grid_limit(long long mni, long long mnj, long long mxi, long long mxj, const b200::RlParams* p) {
  b200::RlGrid g;
  std::vector<unsigned long long> off((size_t)p->num_levels + 1);
  if (!b200::rl_make_grid(mni, mnj, mxi, mxj, *p, &g, off.data()).empty()) return 1;
  return b200::rl_check_headings(g, p->yaw_steps).empty() ? 0 : 2;
}
int rl_points_limit(long long m, int yaw_steps) { return b200::rl_check_points(m, yaw_steps).empty() ? 0 : 1; }
}
