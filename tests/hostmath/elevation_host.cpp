// TEST INFRASTRUCTURE: the elevation map of b200sm_build_elevation_map (csrc/elevation_map.hpp) built serially on the host
// from the same header: origins, extent, cell statistics, the window of every cell, the row-flipped image and both files.
// tests/test_elevation_cpu.py compares it with the Python replay (tests/elevationref.py) and the GPU tests compare the
// session with it bit for bit. Build with -ffp-contract=off and, for the sanitised run (-DEL_HOST_MAIN),
// -fsanitize=address,undefined.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/elevation_map.hpp"

using namespace b200;

namespace {

struct Map {
  bool built = false;
  unsigned width = 0, height = 0;
  double origin[2] = {0, 0};
  ElParams p;
  std::vector<uint32_t> n;
  std::vector<long long> lo, top;
  std::vector<float> step, tan_slope, roughness;
  std::vector<signed char> value;
  std::vector<unsigned char> pgm;
  unsigned long long n_points = 0, n_skipped = 0, n_overhang = 0, n_observed = 0, n_lethal = 0, n_traversable = 0, n_unknown = 0;
};
Map g_map;

}  // namespace

extern "C" {

// params: resolution, max_range, sensor_origin x y z, clearance, min_points, window_cells, min_cells, max_slope, max_step,
// max_roughness, occupied_thresh, free_thresh. points: 4 floats per row, submap k = rows offsets[k] .. offsets[k + 1];
// poses: 16 doubles per submap, column-major. Returns 0, or -1 (parameters), -2 (an origin out of range), -3 (more than
// 2^28 cells), -4 (no submaps), -5 (no point, or every point skipped), -6 (the height extent). A refusal keeps the last map.
int elh_build(const double* params, const float* points, const long long* offsets, const double* poses, int n_sub) {
  ElParams p;
  p.resolution = params[0];
  p.max_range = params[1];
  for (int k = 0; k < 3; k++) p.sensor_origin[k] = params[2 + k];
  p.clearance = params[5];
  p.min_points = (int)params[6];
  p.window_cells = (int)params[7];
  p.min_cells = (int)params[8];
  p.max_slope = params[9];
  p.max_step = params[10];
  p.max_roughness = params[11];
  p.occupied_thresh = params[12];
  p.free_thresh = params[13];
  ElConst c;
  if (el_prepare(p, &c)) return -1;
  if (n_sub <= 0) return -4;
  std::vector<float> T(12 * (size_t)n_sub);
  std::vector<long long> O(2 * (size_t)n_sub);
  bool any = false;
  for (int k = 0; k < n_sub; k++) {
    og_pose_f(poses + 16 * (size_t)k, &T[12 * (size_t)k]);
    if (offsets[k + 1] == offsets[k]) continue;  // an empty submap's origin plays no part
    any = true;
    if (!el_origin(c, p, &T[12 * (size_t)k], &O[2 * (size_t)k], &O[2 * (size_t)k + 1])) return -2;
  }
  if (!any) return -5;
  // the cell and height of every point, -1 cell when skipped
  struct Pt {
    int cx, cy;
    long long Z;
    bool ok;
  };
  std::vector<Pt> pts((size_t)offsets[n_sub]);
  int x0 = INT32_MAX, y0 = INT32_MAX, x1 = INT32_MIN, y1 = INT32_MIN;
  unsigned long long used = 0, skipped = 0;
  long long zmin = EL_LO_EMPTY, zmax = EL_TOP_EMPTY;
  for (int k = 0; k < n_sub; k++)
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(&T[12 * (size_t)k], points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      Pt& q = pts[(size_t)i];
      q.ok = el_point(c, O[2 * (size_t)k], O[2 * (size_t)k + 1], e, &q.cx, &q.cy, &q.Z);
      if (!q.ok) {
        skipped++;
        continue;
      }
      used++;
      x0 = std::min(x0, q.cx);
      x1 = std::max(x1, q.cx);
      y0 = std::min(y0, q.cy);
      y1 = std::max(y1, q.cy);
      zmin = std::min(zmin, q.Z);
      zmax = std::max(zmax, q.Z);
    }
  if (used == 0) return -5;
  const unsigned long long W = (unsigned long long)((long long)x1 - x0 + 1), H = (unsigned long long)((long long)y1 - y0 + 1);
  if (W * H > OG_MAX_CELLS) return -3;
  if (zmax - zmin >= EL_HEIGHT_EXTENT) return -6;
  Map& M = g_map;
  M = Map();
  M.p = p;
  M.width = (unsigned)W;
  M.height = (unsigned)H;
  M.origin[0] = (double)x0 * p.resolution;
  M.origin[1] = (double)y0 * p.resolution;
  M.n_points = used;
  M.n_skipped = skipped;
  const size_t cells = (size_t)(W * H);
  M.n.assign(cells, 0);
  M.lo.assign(cells, EL_LO_EMPTY);
  M.top.assign(cells, EL_TOP_EMPTY);
  auto at = [&](const Pt& q) { return (size_t)(q.cy - y0) * W + (size_t)(q.cx - x0); };
  for (const Pt& q : pts)
    if (q.ok) {
      M.n[at(q)]++;
      M.lo[at(q)] = std::min(M.lo[at(q)], q.Z);
    }
  for (const Pt& q : pts)
    if (q.ok) {
      if (q.Z > M.lo[at(q)] + c.C) M.n_overhang++;
      else M.top[at(q)] = std::max(M.top[at(q)], q.Z);
    }
  M.step.resize(cells);
  M.tan_slope.resize(cells);
  M.roughness.resize(cells);
  M.value.resize(cells);
  M.pgm.resize(cells);
  for (long long y = 0; y < (long long)H; y++)
    for (long long x = 0; x < (long long)W; x++) {
      const size_t q = (size_t)y * W + (size_t)x;
      auto h = [&](int du, int dv) -> long long {
        const long long gx = x + du, gy = y + dv;
        if (gx < 0 || gy < 0 || gx >= (long long)W || gy >= (long long)H) return EL_NONE;
        const size_t g = (size_t)gy * W + (size_t)gx;
        return M.n[g] >= (unsigned)c.min_points ? M.top[g] : EL_NONE;
      };
      const int v = el_window(c, h, &M.step[q], &M.tan_slope[q], &M.roughness[q]);
      M.value[q] = (signed char)v;
      M.pgm[(H - 1 - (size_t)y) * W + (size_t)x] = og_pixel(v, c.og.occ_value, c.og.free_value);
      M.n_observed += h(0, 0) != EL_NONE;
      M.n_lethal += v == 100;
      M.n_traversable += v >= 0 && v < 100;
      M.n_unknown += v < 0;
    }
  M.built = true;
  return 0;
}

// width, height, n_points, n_skipped, n_overhang, n_observed, n_lethal, n_traversable, n_unknown; origin x, y
void elh_info(unsigned long long* info, double* origin) {
  const Map& M = g_map;
  const unsigned long long v[9] = {M.width, M.height, M.n_points, M.n_skipped, M.n_overhang, M.n_observed, M.n_lethal, M.n_traversable,
                                   M.n_unknown};
  std::memcpy(info, v, sizeof(v));
  origin[0] = M.origin[0];
  origin[1] = M.origin[1];
}

// any pointer may be NULL; each holds width * height cells
void elh_get(uint32_t* n, long long* h, long long* lo, float* step, float* tan_slope, float* roughness, signed char* value,
             unsigned char* pgm) {
  const Map& M = g_map;
  const size_t k = M.value.size();
  if (!k) return;
  if (n) std::memcpy(n, M.n.data(), 4 * k);
  if (h) std::memcpy(h, M.top.data(), 8 * k);
  if (lo) std::memcpy(lo, M.lo.data(), 8 * k);
  if (step) std::memcpy(step, M.step.data(), 4 * k);
  if (tan_slope) std::memcpy(tan_slope, M.tan_slope.data(), 4 * k);
  if (roughness) std::memcpy(roughness, M.roughness.data(), 4 * k);
  if (value) std::memcpy(value, M.value.data(), k);
  if (pgm) std::memcpy(pgm, M.pgm.data(), k);
}

// the map_server pair, as b200sm_save_traversability_map writes it; 0 or -1
int elh_save(const char* pgm_path, const char* yaml_path) {
  const Map& M = g_map;
  if (!M.built) return -1;
  const std::string head = og_pgm_header(M.width, M.height, M.p.resolution);
  const std::string yaml = og_yaml(pgm_path, M.p.resolution, M.origin, M.p.occupied_thresh, M.p.free_thresh);
  FILE* f = std::fopen(pgm_path, "wb");
  if (!f) return -1;
  bool ok = std::fwrite(head.data(), 1, head.size(), f) == head.size() && std::fwrite(M.pgm.data(), 1, M.pgm.size(), f) == M.pgm.size();
  ok = (std::fclose(f) == 0) && ok;
  FILE* y = std::fopen(yaml_path, "wb");
  if (!y) return -1;
  ok = std::fwrite(yaml.data(), 1, yaml.size(), y) == yaml.size() && ok;
  ok = (std::fclose(y) == 0) && ok;
  return ok ? 0 : -1;
}

// the constants of a parameter set, for the replay's cross-check: S, R, C, K, G, G2; returns el_prepare's verdict (0 / -1)
int elh_const(const double* params, double* out) {
  ElParams p;
  p.resolution = params[0];
  p.max_range = params[1];
  for (int k = 0; k < 3; k++) p.sensor_origin[k] = params[2 + k];
  p.clearance = params[5];
  p.min_points = (int)params[6];
  p.window_cells = (int)params[7];
  p.min_cells = (int)params[8];
  p.max_slope = params[9];
  p.max_step = params[10];
  p.max_roughness = params[11];
  p.occupied_thresh = params[12];
  p.free_thresh = params[13];
  ElConst c;
  if (el_prepare(p, &c)) return -1;
  const double v[6] = {c.og.S, (double)c.og.R, (double)c.C, (double)c.K, c.G, c.G2};
  std::memcpy(out, v, sizeof(v));
  return 0;
}

}  // extern "C"

#ifdef EL_HOST_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that builds maps
// from generated hilly submaps with non-finite rows, negative coordinates and empty submaps, and checks that the submaps
// in reverse order give the same map and that every value is -1..100.
#include <cmath>
#include <limits>

int main() {
  int failures = 0;
  const double params[14] = {0.25, 20.0, 0.0, 0.0, 0.4, 2.0, 2, 3, 6, 20.0, 0.15, 0.05, 0.65, 0.25};
  for (int trial = 0; trial < 6; trial++) {
    const int n_sub = 1 + trial * 2;
    std::vector<float> pts;
    std::vector<long long> off{0};
    std::vector<double> poses;
    uint64_t st = 0x9E3779B97F4A7C15ull * (uint64_t)(trial + 1);
    auto rnd = [&]() {
      st = st * 6364136223846793005ull + 1442695040888963407ull;
      return (double)(st >> 11) * (1.0 / 9007199254740992.0);
    };
    for (int k = 0; k < n_sub; k++) {
      const int n = (k % 3 == 2) ? 0 : 2000 + 37 * k;
      for (int i = 0; i < n; i++) {
        float x = (float)(rnd() * 30 - 15), y = (float)(rnd() * 30 - 15);
        float z = (float)(0.3 * std::sin(0.4 * x) + 0.1 * y + (i % 17 == 3 ? 3.0 : 0.0) + 0.01 * rnd());
        if (i % 41 == 7) x = std::numeric_limits<float>::quiet_NaN();
        if (i % 43 == 9) z = std::numeric_limits<float>::infinity();
        pts.insert(pts.end(), {x, y, z, 0.0f});
      }
      off.push_back(off.back() + n);
      const double yaw = rnd() * 6.283185307179586, tx = rnd() * 20 - 15, ty = rnd() * 20 - 15;
      const double P[16] = {std::cos(yaw), std::sin(yaw), 0, 0, -std::sin(yaw), std::cos(yaw), 0, 0, 0, 0, 1, 0, tx, ty, 1.2, 1};
      poses.insert(poses.end(), P, P + 16);
    }
    if (elh_build(params, pts.data(), off.data(), poses.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    const Map first = g_map;
    for (signed char v : first.value)
      if (v < -1 || v > 100) failures++;
    std::vector<float> rp;
    std::vector<long long> ro{0};
    std::vector<double> rpo;
    for (int k = n_sub - 1; k >= 0; k--) {
      rp.insert(rp.end(), pts.begin() + 4 * off[k], pts.begin() + 4 * off[k + 1]);
      ro.push_back(ro.back() + (off[k + 1] - off[k]));
      rpo.insert(rpo.end(), poses.begin() + 16 * k, poses.begin() + 16 * (k + 1));
    }
    if (elh_build(params, rp.data(), ro.data(), rpo.data(), n_sub) != 0 || g_map.top != first.top || g_map.n != first.n ||
        g_map.value != first.value || g_map.pgm != first.pgm || g_map.width != first.width || g_map.origin[0] != first.origin[0] ||
        std::memcmp(g_map.roughness.data(), first.roughness.data(), 4 * first.roughness.size()) != 0) {
      std::printf("MISMATCH trial=%d\n", trial);
      failures++;
    }
  }
  std::printf("elevation_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
