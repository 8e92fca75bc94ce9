// TEST INFRASTRUCTURE: the map consistency of b200sm_build_map_consistency (csrc/map_consistency.hpp) built serially on the
// host from the same header: fixed point, box, the 27 cells around every query, the moments, the per-query values and the
// per-submap rows. tests/test_map_consistency_cpu.py compares it with the Python replay (tests/consistencyref.py) and the
// GPU tests compare the session with it bit for bit. Build with -ffp-contract=off and, for the sanitised run
// (-DMC_HOST_MAIN), -fsanitize=address,undefined.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/map_consistency.hpp"

using namespace b200;

namespace {

struct Build {
  bool built = false;
  McConst c{};
  int box_lo[3] = {0, 0, 0};
  unsigned dims[3] = {0, 0, 0};
  std::vector<uint32_t> n;
  std::vector<double> h, plane;
  // per submap: points, queries, valid, neighbours, sum_h_q, sum_plane_q
  std::vector<unsigned long long> rows;
  unsigned long long n_points = 0, n_skipped = 0, n_cells = 0, n_candidates = 0;
};
Build g_build;

constexpr int ROW = 6;

}  // namespace

extern "C" {

// params: radius, min_neighbors, query_stride. points: 4 floats per row, submap k = rows offsets[k] .. offsets[k + 1];
// poses: 16 doubles per submap, column-major. Returns 0, or -1 (parameters), -2 (no submaps), -3 (a coordinate of 2^46
// or more), -4 (a box of more than 2^31 - 1 cells), -5 (2^31 points or more). A refusal keeps the last build.
int mch_build(const double* params, const float* points, const long long* offsets, const double* poses, int n_sub) {
  McParams p;
  p.radius = params[0];
  p.min_neighbors = (int)params[1];
  p.query_stride = (int)params[2];
  McConst c;
  if (mc_prepare(p, &c)) return -1;
  if (n_sub <= 0) return -2;
  const long long total = offsets[n_sub];
  if ((unsigned long long)total > MC_MAX_POINTS) return -5;
  std::vector<long long> X(3 * (size_t)total);
  std::vector<char> ok((size_t)total, 0);
  std::vector<int> sub_of((size_t)total);
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  unsigned long long skipped = 0, used = 0;
  for (int k = 0; k < n_sub; k++) {
    float T[12];
    og_pose_f(poses + 16 * (size_t)k, T);
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(T, points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      sub_of[(size_t)i] = k;
      const int v = mc_point(c, e, &X[3 * (size_t)i]);
      if (v == MC_POINT_RANGE) return -3;
      if (v == MC_POINT_SKIPPED) {
        skipped++;
        continue;
      }
      ok[(size_t)i] = 1;
      used++;
      for (int a = 0; a < 3; a++) {
        lo[a] = std::min(lo[a], og_cell(X[3 * (size_t)i + a]));
        hi[a] = std::max(hi[a], og_cell(X[3 * (size_t)i + a]));
      }
    }
  }
  unsigned dims[3] = {0, 0, 0};
  unsigned long long cells = 0;
  if (used && !sm_box(lo, hi, dims, &cells)) return -4;
  Build& B = g_build;
  B = Build();
  B.c = c;
  B.n_points = (unsigned long long)total;
  B.n_skipped = skipped;
  B.n.assign((size_t)total, 0);
  double nan;
  const unsigned long long nb = MC_NAN_BITS;
  std::memcpy(&nan, &nb, 8);
  B.h.assign((size_t)total, nan);
  B.plane.assign((size_t)total, nan);
  B.rows.assign(ROW * (size_t)n_sub, 0);
  for (int k = 0; k < n_sub; k++) B.rows[ROW * (size_t)k] = (unsigned long long)(offsets[k + 1] - offsets[k]);
  if (used) {
    for (int a = 0; a < 3; a++) {
      B.box_lo[a] = lo[a];
      B.dims[a] = dims[a];
    }
    auto lin = [&](long long x, long long y, long long z) -> long long {
      const long long wx = x - lo[0], wy = y - lo[1], wz = z - lo[2];
      if (wx < 0 || wy < 0 || wz < 0 || wx >= dims[0] || wy >= dims[1] || wz >= dims[2]) return -1;
      return (wz * dims[1] + wy) * dims[0] + wx;
    };
    // the non-skipped points sorted by cell
    std::vector<std::pair<long long, unsigned>> order;
    order.reserve((size_t)used);
    for (long long i = 0; i < total; i++)
      if (ok[(size_t)i])
        order.push_back({lin(og_cell(X[3 * i]), og_cell(X[3 * i + 1]), og_cell(X[3 * i + 2])), (unsigned)i});
    std::sort(order.begin(), order.end());
    for (size_t r = 0; r < order.size(); r++) B.n_cells += r == 0 || order[r].first != order[r - 1].first;
    for (long long i = 0; i < total; i += c.stride) {
      if (!ok[(size_t)i]) continue;
      const long long* P = &X[3 * (size_t)i];
      const int cx = og_cell(P[0]), cy = og_cell(P[1]), cz = og_cell(P[2]);
      McMoments m;
      for (int dz = -1; dz <= 1; dz++)
        for (int dy = -1; dy <= 1; dy++)
          for (int dx = -1; dx <= 1; dx++) {
            const long long key = lin((long long)cx + dx, (long long)cy + dy, (long long)cz + dz);
            if (key < 0) continue;
            auto it = std::lower_bound(order.begin(), order.end(), std::make_pair(key, 0u));
            for (; it != order.end() && it->first == key; ++it) {
              const long long* Q = &X[3 * (size_t)it->second];
              B.n_candidates++;
              mc_accumulate(m, Q[0] - P[0], Q[1] - P[1], Q[2] - P[2]);
            }
          }
      unsigned long long* row = &B.rows[ROW * (size_t)sub_of[(size_t)i]];
      B.n[(size_t)i] = (uint32_t)m.n;
      row[1] += 1;
      row[3] += (unsigned long long)m.n;
      double h, pv;
      long long qh, ql;
      if (mc_query(c, m, &h, &pv, &qh, &ql)) {
        B.h[(size_t)i] = h;
        B.plane[(size_t)i] = pv;
        row[2] += 1;
        row[4] += (unsigned long long)qh;
        row[5] += (unsigned long long)ql;
      }
    }
  }
  B.built = true;
  return 0;
}

// box_lo[3], dims[3], n_points, n_skipped, n_cells, n_candidates (10 long longs); per submap n_points, n_queries, n_valid,
// n_neighbors, sum_h_q, sum_plane_q (6 long longs each, n_sub rows), and the per-submap mme, mpv and the map's (2 n_sub + 2
// doubles: the map's last)
void mch_info(long long* info, long long* rows, double* means) {
  const Build& B = g_build;
  for (int a = 0; a < 3; a++) {
    info[a] = B.box_lo[a];
    info[3 + a] = B.dims[a];
  }
  info[6] = (long long)B.n_points;
  info[7] = (long long)B.n_skipped;
  info[8] = (long long)B.n_cells;
  info[9] = (long long)B.n_candidates;
  const size_t n_sub = B.rows.size() / ROW;
  std::memcpy(rows, B.rows.data(), B.rows.size() * 8);
  long long sh = 0, sp = 0;
  unsigned long long valid = 0;
  for (size_t k = 0; k < n_sub; k++) {
    const unsigned long long* r = &B.rows[ROW * k];
    means[2 * k] = mc_mme((long long)r[4], r[2]);
    means[2 * k + 1] = mc_mpv(B.c, (long long)r[5], r[2]);
    sh += (long long)r[4];
    sp += (long long)r[5];
    valid += r[2];
  }
  means[2 * n_sub] = mc_mme(sh, valid);
  means[2 * n_sub + 1] = mc_mpv(B.c, sp, valid);
}

void mch_get(uint32_t* n, double* h, double* plane) {
  const Build& B = g_build;
  const size_t k = B.n.size();
  if (!k) return;
  std::memcpy(n, B.n.data(), 4 * k);
  std::memcpy(h, B.h.data(), 8 * k);
  std::memcpy(plane, B.plane.data(), 8 * k);
}

void mch_log(const double* x, double* out, long long n) {
  for (long long i = 0; i < n; i++) out[i] = mc_log(x[i]);
}

// a6: a00 a01 a02 a11 a12 a22 per matrix
void mch_lambda(const double* a6, double* out, long long n) {
  for (long long i = 0; i < n; i++) {
    const double* a = a6 + 6 * i;
    out[i] = mc_lambda_min(a[0], a[1], a[2], a[3], a[4], a[5]);
  }
}

// sm_box's verdict on inclusive cell bounds: 0 with dims, or -4
int mch_box(const int* lo, const int* hi, unsigned* dims) {
  unsigned long long cells;
  return sm_box(lo, hi, dims, &cells) ? 0 : -4;
}

// S, S2, r2, c0 of a parameter set; mc_prepare's verdict (0 / -1)
int mch_const(const double* params, double* out) {
  McParams p;
  p.radius = params[0];
  p.min_neighbors = (int)params[1];
  p.query_stride = (int)params[2];
  McConst c;
  if (mc_prepare(p, &c)) return -1;
  out[0] = c.S;
  out[1] = c.S2;
  out[2] = c.r2;
  out[3] = c.c0;
  return 0;
}

}  // extern "C"

#ifdef MC_HOST_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that builds
// from generated wall-and-floor submaps with non-finite rows, negative coordinates and empty submaps, and checks that the
// submaps in reverse order give the same per-point values (permuted) and the same map totals.
#include <cmath>
#include <limits>

int main() {
  int failures = 0;
  const double params[3] = {0.3, 10, 1};
  for (int trial = 0; trial < 4; trial++) {
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
      const int n = (k % 3 == 2) ? 0 : 1500 + 37 * k;
      for (int i = 0; i < n; i++) {
        float x = (float)(rnd() * 6 - 3), y = (float)(rnd() * 6 - 3), z = (float)(0.02 * rnd());
        if (i % 3 == 0) {  // a wall
          z = (float)(rnd() * 2);
          x = (float)(-1.0 + 0.01 * rnd());
        }
        if (i % 41 == 7) x = std::numeric_limits<float>::quiet_NaN();
        if (i % 43 == 9) z = std::numeric_limits<float>::infinity();
        pts.insert(pts.end(), {x, y, z, 0.0f});
      }
      off.push_back(off.back() + n);
      const double yaw = 0.05 * rnd(), tx = rnd() * 0.2 - 5, ty = rnd() * 0.2 - 5;
      const double P[16] = {std::cos(yaw), std::sin(yaw), 0, 0, -std::sin(yaw), std::cos(yaw), 0, 0, 0, 0, 1, 0, tx, ty, -0.5, 1};
      poses.insert(poses.end(), P, P + 16);
    }
    if (mch_build(params, pts.data(), off.data(), poses.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    const Build first = g_build;
    std::vector<float> rp;
    std::vector<long long> ro{0};
    std::vector<double> rpo;
    for (int k = n_sub - 1; k >= 0; k--) {
      rp.insert(rp.end(), pts.begin() + 4 * off[k], pts.begin() + 4 * off[k + 1]);
      ro.push_back(ro.back() + (off[k + 1] - off[k]));
      rpo.insert(rpo.end(), poses.begin() + 16 * k, poses.begin() + 16 * (k + 1));
    }
    if (mch_build(params, rp.data(), ro.data(), rpo.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    // point i of submap k sits at ro[n_sub - 1 - k] + (i - off[k]) in the reversed map
    for (int k = 0; k < n_sub; k++)
      for (long long i = off[k]; i < off[k + 1]; i++) {
        const size_t j = (size_t)(ro[n_sub - 1 - k] + (i - off[k]));
        if (first.n[(size_t)i] != g_build.n[j] || std::memcmp(&first.h[(size_t)i], &g_build.h[j], 8) != 0 ||
            std::memcmp(&first.plane[(size_t)i], &g_build.plane[j], 8) != 0)
          failures++;
      }
    if (first.n_candidates != g_build.n_candidates || first.n_cells != g_build.n_cells) failures++;
  }
  std::printf("consistency_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
