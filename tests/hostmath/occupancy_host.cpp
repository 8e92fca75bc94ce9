// TEST INFRASTRUCTURE: the occupancy grid of b200sm_build_occupancy_grid (csrc/occupancy_grid.hpp) built serially on the
// host from the same header: origins, extent, one hit and one free bitmap per submap over the grid, the per-submap fold,
// the values, the row-flipped image and both files. tests/test_occupancy_cpu.py compares it with the Python replay
// (tests/occupancyref.py) and the GPU tests compare the session with it byte for byte. Build with -ffp-contract=off and,
// for the sanitised run (-DOG_HOST_MAIN), -fsanitize=address,undefined.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/occupancy_grid.hpp"

using namespace b200;

namespace {

struct Grid {
  bool built = false;
  unsigned width = 0, height = 0;
  double origin[2] = {0, 0};
  OgParams p;
  std::vector<uint32_t> hits, frees;
  std::vector<signed char> values;
  std::vector<unsigned char> pgm;
  unsigned long long n_rays = 0, n_skipped = 0, n_occupied = 0, n_free = 0, n_unknown = 0;
};
Grid g_grid;

}  // namespace

extern "C" {

// params: resolution, z_min, z_max, max_range, sensor_origin x y z, occupied_thresh, free_thresh.
// points: 4 floats per row (x, y, z, unused), submap k = rows offsets[k] .. offsets[k + 1]; poses: 16 doubles per submap,
// column-major. Returns 0, or -1 (parameters), -2 (an origin out of range), -3 (more than 2^28 cells), -4 (no submaps).
int ogh_build(const double* params, const float* points, const long long* offsets, const double* poses, int n_sub) {
  OgParams p;
  p.resolution = params[0];
  p.z_min = params[1];
  p.z_max = params[2];
  p.max_range = params[3];
  for (int k = 0; k < 3; k++) p.sensor_origin[k] = params[4 + k];
  p.occupied_thresh = params[7];
  p.free_thresh = params[8];
  OgConst c;
  if (og_prepare(p, &c)) return -1;
  if (n_sub <= 0) return -4;
  std::vector<float> T(12 * (size_t)n_sub);
  std::vector<long long> O(3 * (size_t)n_sub);
  for (int k = 0; k < n_sub; k++) {
    og_pose_f(poses + 16 * (size_t)k, &T[12 * (size_t)k]);
    if (!og_origin(c, p, &T[12 * (size_t)k], &O[3 * (size_t)k])) return -2;
  }
  // extent: every origin cell and every ray's endpoint cell
  int x0 = og_cell(O[0]), x1 = x0, y0 = og_cell(O[1]), y1 = y0;
  unsigned long long rays = 0, skipped = 0;
  for (int k = 0; k < n_sub; k++) {
    const long long* o = &O[3 * (size_t)k];
    x0 = std::min(x0, og_cell(o[0]));
    x1 = std::max(x1, og_cell(o[0]));
    y0 = std::min(y0, og_cell(o[1]));
    y1 = std::max(y1, og_cell(o[1]));
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(&T[12 * (size_t)k], points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      int hx, hy;
      OgSeg s;
      if (og_ray(c, o[0], o[1], o[2], e[0], e[1], e[2], &hx, &hy, &s) < 0) {
        skipped++;
        continue;
      }
      rays++;
      x0 = std::min(x0, hx);
      x1 = std::max(x1, hx);
      y0 = std::min(y0, hy);
      y1 = std::max(y1, hy);
    }
  }
  const unsigned long long W = (unsigned long long)((long long)x1 - x0 + 1), H = (unsigned long long)((long long)y1 - y0 + 1);
  if (W * H > OG_MAX_CELLS) return -3;
  Grid& G = g_grid;
  G = Grid();
  G.p = p;
  G.width = (unsigned)W;
  G.height = (unsigned)H;
  G.origin[0] = (double)x0 * p.resolution;
  G.origin[1] = (double)y0 * p.resolution;
  G.n_rays = rays;
  G.n_skipped = skipped;
  const size_t cells = (size_t)(W * H);
  G.hits.assign(cells, 0);
  G.frees.assign(cells, 0);
  std::vector<unsigned char> hit(cells), fre(cells);
  for (int k = 0; k < n_sub; k++) {
    std::fill(hit.begin(), hit.end(), 0);
    std::fill(fre.begin(), fre.end(), 0);
    const long long* o = &O[3 * (size_t)k];
    auto at = [&](int cx, int cy) -> size_t {
      if (cx < x0 || cx > x1 || cy < y0 || cy > y1) std::abort();  // a walk never leaves the grid
      return (size_t)(cy - y0) * W + (size_t)(cx - x0);
    };
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(&T[12 * (size_t)k], points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      int hx, hy;
      OgSeg s;
      const int f = og_ray(c, o[0], o[1], o[2], e[0], e[1], e[2], &hx, &hy, &s);
      if (f < 0) continue;
      if (f & 1) hit[at(hx, hy)] = 1;
      if (f & 2) og_walk(s, [&](int cx, int cy) { fre[at(cx, cy)] = 1; });
    }
    for (size_t q = 0; q < cells; q++) {
      if (hit[q]) G.hits[q]++;
      else if (fre[q]) G.frees[q]++;
    }
  }
  G.values.resize(cells);
  G.pgm.resize(cells);
  for (size_t y = 0; y < H; y++)
    for (size_t x = 0; x < W; x++) {
      const size_t q = y * W + x;
      const int v = og_value(G.hits[q], G.frees[q]);
      G.values[q] = (signed char)v;
      const unsigned char px = og_pixel(v, c.occ_value, c.free_value);
      G.pgm[(H - 1 - y) * W + x] = px;
      if (v < 0) G.n_unknown++;
      else if (px == 0) G.n_occupied++;
      else if (px == 254) G.n_free++;
    }
  G.built = true;
  return 0;
}

// width, height, n_rays, n_skipped, n_occupied, n_free, n_unknown; origin x, y
void ogh_info(unsigned long long* info, double* origin) {
  const Grid& G = g_grid;
  const unsigned long long v[7] = {G.width, G.height, G.n_rays, G.n_skipped, G.n_occupied, G.n_free, G.n_unknown};
  std::memcpy(info, v, sizeof(v));
  origin[0] = G.origin[0];
  origin[1] = G.origin[1];
}

// any pointer may be NULL; each holds width * height cells
void ogh_get(signed char* values, uint32_t* hits, uint32_t* frees, unsigned char* pgm) {
  const Grid& G = g_grid;
  const size_t n = G.values.size();
  if (!n) return;
  if (values) std::memcpy(values, G.values.data(), n);
  if (hits) std::memcpy(hits, G.hits.data(), 4 * n);
  if (frees) std::memcpy(frees, G.frees.data(), 4 * n);
  if (pgm) std::memcpy(pgm, G.pgm.data(), n);
}

// the map_server pair, as b200sm_save_occupancy_map writes it; 0 or -1
int ogh_save(const char* pgm_path, const char* yaml_path) {
  const Grid& G = g_grid;
  if (!G.built) return -1;
  const std::string head = og_pgm_header(G.width, G.height, G.p.resolution);
  const std::string yaml = og_yaml(pgm_path, G.p.resolution, G.origin, G.p.occupied_thresh, G.p.free_thresh);
  FILE* f = std::fopen(pgm_path, "wb");
  if (!f) return -1;
  bool ok = std::fwrite(head.data(), 1, head.size(), f) == head.size() && std::fwrite(G.pgm.data(), 1, G.pgm.size(), f) == G.pgm.size();
  ok = (std::fclose(f) == 0) && ok;
  FILE* y = std::fopen(yaml_path, "wb");
  if (!y) return -1;
  ok = std::fwrite(yaml.data(), 1, yaml.size(), y) == yaml.size() && ok;
  ok = (std::fclose(y) == 0) && ok;
  return ok ? 0 : -1;
}

// the walk alone, for the tests: up to cap cells (x, y), returns the walk's length
long long ogh_walk(long long xa, long long ya, long long xb, long long yb, int* cells, long long cap) {
  long long n = 0;
  og_walk(OgSeg{xa, ya, xb, yb}, [&](int cx, int cy) {
    if (n < cap) {
      cells[2 * n] = cx;
      cells[2 * n + 1] = cy;
    }
    n++;
  });
  return n;
}

}  // extern "C"

#ifdef OG_HOST_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that builds
// grids from generated submaps with non-finite rows, negative coordinates, empty submaps and rays across the band, and
// checks that a permutation of the submaps gives the same grid and that hits + frees never exceeds the submap count.
#include <limits>

int main() {
  int failures = 0;
  const double params[9] = {0.25, 0.3, 2.5, 20.0, 0.0, 0.0, 0.4, 0.65, 0.25};
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
      const int n = (k % 3 == 2) ? 0 : 200 + 37 * k;
      for (int i = 0; i < n; i++) {
        float x = (float)(rnd() * 50 - 25), y = (float)(rnd() * 50 - 25), z = (float)(rnd() * 6 - 3);
        if (i % 41 == 7) x = std::numeric_limits<float>::quiet_NaN();
        if (i % 43 == 9) z = std::numeric_limits<float>::infinity();
        pts.insert(pts.end(), {x, y, z, 0.0f});
      }
      off.push_back(off.back() + n);
      const double yaw = rnd() * 6.283185307179586, tx = rnd() * 20 - 15, ty = rnd() * 20 - 15;
      const double P[16] = {std::cos(yaw), std::sin(yaw), 0, 0, -std::sin(yaw), std::cos(yaw), 0, 0, 0, 0, 1, 0, tx, ty, 1.2, 1};
      poses.insert(poses.end(), P, P + 16);
    }
    if (ogh_build(params, pts.data(), off.data(), poses.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    const Grid first = g_grid;
    for (size_t q = 0; q < first.hits.size(); q++)
      if (first.hits[q] + first.frees[q] > (unsigned)n_sub) failures++;
    // the submaps in reverse order
    std::vector<float> rp;
    std::vector<long long> ro{0};
    std::vector<double> rpo;
    for (int k = n_sub - 1; k >= 0; k--) {
      rp.insert(rp.end(), pts.begin() + 4 * off[k], pts.begin() + 4 * off[k + 1]);
      ro.push_back(ro.back() + (off[k + 1] - off[k]));
      rpo.insert(rpo.end(), poses.begin() + 16 * k, poses.begin() + 16 * (k + 1));
    }
    if (ogh_build(params, rp.data(), ro.data(), rpo.data(), n_sub) != 0 || g_grid.hits != first.hits || g_grid.frees != first.frees ||
        g_grid.pgm != first.pgm || g_grid.width != first.width || g_grid.origin[0] != first.origin[0]) {
      std::printf("MISMATCH trial=%d\n", trial);
      failures++;
    }
  }
  std::printf("occupancy_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
