// TEST INFRASTRUCTURE: the map changes of b200sm_build_map_changes (csrc/map_changes.hpp) built serially on the host from
// the same header: the split, origins, rays, the box of both epochs' endpoint voxels, the rank index over it, one hit and
// one free bitmap per submap, folded into the counts of the submap's epoch, the voxel labels, the point labels and the
// updated map. tests/test_map_changes_cpu.py compares it with the Python replay (tests/changeref.py) and the GPU tests
// compare the session with it bit for bit. Build with -ffp-contract=off and, for the sanitised run (-DCH_HOST_MAIN),
// -fsanitize=address,undefined.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/map_changes.hpp"

using namespace b200;

namespace {

struct Build {
  int lo[3] = {0, 0, 0};
  unsigned dims[3] = {0, 0, 0};
  long long split = 0;
  unsigned long long n_rays = 0, n_skipped = 0, n_app_vox = 0, n_van_vox = 0, n_app_pts = 0, n_van_pts = 0;
  std::vector<int> ijk;  // 3 per voxel, rank order
  std::vector<uint32_t> hits[2], frees[2];
  std::vector<unsigned char> label;        // per voxel
  std::vector<unsigned char> point_label;  // per point, assembly order
  std::vector<float> points;               // the assembled map, 4 floats per point
  std::vector<long long> offsets;          // updated map offsets per submap, n_sub + 1
};
Build g_build;

}  // namespace

extern "C" {

// params: resolution, max_range, sensor_origin x y z, ray_fraction, min_frees, dynamic_thresh. split_submap as the C-ABI
// takes it; last_segment_first: the session's last segment's first submap (0: one segment). points: 4 floats per row,
// submap k = rows offsets[k] .. offsets[k + 1]; poses: 16 doubles per submap, column-major. Returns 0, or -1
// (parameters), -2 (an origin out of range), -3 (a box of more than 2^31 - 1 cells), -4 (no submaps), -5 (the split).
int chh_build(const double* params, long long split_submap, long long last_segment_first, const float* points, const long long* offsets,
              const double* poses, int n_sub) {
  SmParams p;
  p.resolution = params[0];
  p.max_range = params[1];
  for (int k = 0; k < 3; k++) p.sensor_origin[k] = params[2 + k];
  p.ray_fraction = params[5];
  p.min_frees = params[6] >= 0 && params[6] <= 4294967295.0 ? (unsigned)params[6] : 0u;
  p.dynamic_thresh = params[7];
  SmConst c;
  if (sm_prepare(p, &c)) return -1;
  if (n_sub <= 0) return -4;
  unsigned long long split = 0;
  if (ch_split(split_submap, (unsigned long long)n_sub, (unsigned long long)last_segment_first, &split)) return -5;
  std::vector<float> T(12 * (size_t)n_sub);
  std::vector<long long> O(3 * (size_t)n_sub);
  for (int k = 0; k < n_sub; k++) {
    og_pose_f(poses + 16 * (size_t)k, &T[12 * (size_t)k]);
    if (!sm_origin(c, p, &T[12 * (size_t)k], &O[3 * (size_t)k])) return -2;
  }
  const size_t n = (size_t)offsets[n_sub];
  std::vector<unsigned char> is_ray(n);
  std::vector<int> vox(3 * n);
  std::vector<long long> end(3 * n);
  std::vector<float> moved(4 * n);
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  unsigned long long rays = 0, skipped = 0;
  for (int k = 0; k < n_sub; k++)
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(&T[12 * (size_t)k], points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      moved[4 * i] = e[0];
      moved[4 * i + 1] = e[1];
      moved[4 * i + 2] = e[2];
      moved[4 * i + 3] = points[4 * i + 3];
      int* v = &vox[3 * i];
      long long* f = &end[3 * i];
      if (!sm_ray(c, &O[3 * (size_t)k], e[0], e[1], e[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) {
        skipped++;
        continue;
      }
      is_ray[i] = 1;
      rays++;
      for (int a = 0; a < 3; a++) {
        lo[a] = std::min(lo[a], v[a]);
        hi[a] = std::max(hi[a], v[a]);
      }
    }
  unsigned dims[3] = {0, 0, 0};
  unsigned long long cells = 0;
  if (rays && !sm_box(lo, hi, dims, &cells)) return -3;
  Build& B = g_build;
  B = Build();
  B.split = (long long)split;
  B.n_rays = rays;
  B.n_skipped = skipped;
  B.points = moved;
  if (rays)
    for (int a = 0; a < 3; a++) {
      B.lo[a] = lo[a];
      B.dims[a] = dims[a];
    }
  const size_t n_words = (size_t)((cells + 31) / 32);
  std::vector<uint32_t> bits(n_words), prefix(n_words);
  auto lin_of = [&](int x, int y, int z, unsigned* lin) {
    const long long wx = (long long)x - B.lo[0], wy = (long long)y - B.lo[1], wz = (long long)z - B.lo[2];
    if (wx < 0 || wy < 0 || wz < 0 || wx >= B.dims[0] || wy >= B.dims[1] || wz >= B.dims[2]) return false;
    *lin = (unsigned)((wz * (long long)B.dims[1] + wy) * (long long)B.dims[0] + wx);
    return true;
  };
  auto rank_of = [&](int x, int y, int z, unsigned* r) {
    unsigned lin;
    if (!lin_of(x, y, z, &lin)) return false;
    const uint32_t w = bits[lin >> 5], bit = lin & 31u;
    if (!((w >> bit) & 1u)) return false;
    *r = prefix[lin >> 5] + (unsigned)__builtin_popcount(w & ((1u << bit) - 1u));
    return true;
  };
  for (size_t i = 0; i < n; i++) {
    if (!is_ray[i]) continue;
    unsigned lin;
    if (!lin_of(vox[3 * i], vox[3 * i + 1], vox[3 * i + 2], &lin)) std::abort();  // an endpoint is always in the box
    bits[lin >> 5] |= 1u << (lin & 31u);
  }
  unsigned n_vox = 0;
  for (size_t w = 0; w < n_words; w++) {
    prefix[w] = n_vox;
    n_vox += (unsigned)__builtin_popcount(bits[w]);
  }
  B.ijk.resize(3 * (size_t)n_vox);
  for (size_t w = 0; w < n_words; w++)
    for (unsigned b = 0; b < 32; b++)
      if ((bits[w] >> b) & 1u) {
        const unsigned long long lin = w * 32ull + b, plane = (unsigned long long)B.dims[0] * B.dims[1];
        const unsigned r = prefix[w] + (unsigned)__builtin_popcount(bits[w] & ((1u << b) - 1u));
        B.ijk[3 * (size_t)r] = B.lo[0] + (int)(lin % plane % B.dims[0]);
        B.ijk[3 * (size_t)r + 1] = B.lo[1] + (int)(lin % plane / B.dims[0]);
        B.ijk[3 * (size_t)r + 2] = B.lo[2] + (int)(lin / plane);
      }
  // per submap: hit and free booleans over the occupied voxels, folded into the counts of the submap's epoch
  for (int e = 0; e < 2; e++) {
    B.hits[e].assign(n_vox, 0);
    B.frees[e].assign(n_vox, 0);
  }
  std::vector<unsigned char> hit(n_vox), fre(n_vox);
  for (int k = 0; k < n_sub; k++) {
    const int e = (unsigned long long)k < split ? CH_BEFORE : CH_AFTER;
    std::fill(hit.begin(), hit.end(), 0);
    std::fill(fre.begin(), fre.end(), 0);
    const long long* o = &O[3 * (size_t)k];
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      if (!is_ray[i]) continue;
      unsigned r;
      if (!rank_of(vox[3 * i], vox[3 * i + 1], vox[3 * i + 2], &r)) std::abort();
      hit[r] = 1;
      const long long* f = &end[3 * i];
      sm_walk(o[0], o[1], o[2], f[0], f[1], f[2], [&](int x, int y, int z) {
        unsigned rw;
        if (rank_of(x, y, z, &rw)) fre[rw] = 1;
      });
    }
    for (unsigned v = 0; v < n_vox; v++) {
      if (hit[v]) B.hits[e][v]++;
      else if (fre[v]) B.frees[e][v]++;
    }
  }
  B.label.resize(n_vox);
  for (unsigned v = 0; v < n_vox; v++) {
    B.label[v] = ch_voxel_label(B.hits[CH_BEFORE][v], B.frees[CH_BEFORE][v], B.hits[CH_AFTER][v], B.frees[CH_AFTER][v], c.min_frees,
                                c.dyn_value);
    B.n_app_vox += B.label[v] == CH_APPEARED;
    B.n_van_vox += B.label[v] == CH_VANISHED;
  }
  B.point_label.assign(n, CH_UNCHANGED);
  B.offsets.assign((size_t)n_sub + 1, 0);
  long long kept = 0;
  for (int k = 0; k < n_sub; k++) {
    const int e = (unsigned long long)k < split ? CH_BEFORE : CH_AFTER;
    B.offsets[k] = kept;
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      unsigned r;
      if (is_ray[i] && rank_of(vox[3 * i], vox[3 * i + 1], vox[3 * i + 2], &r)) B.point_label[i] = ch_point_label(B.label[r], e);
      B.n_app_pts += B.point_label[i] == CH_APPEARED;
      B.n_van_pts += B.point_label[i] == CH_VANISHED;
      kept += B.point_label[i] != CH_VANISHED;
    }
  }
  B.offsets[n_sub] = kept;
  return 0;
}

// lo x y z, W, H, D, split, n_rays, n_skipped, n_voxels, n_appeared_voxels, n_vanished_voxels, n_points, n_appeared_points,
// n_vanished_points, n_updated_points
void chh_info(long long* info) {
  const Build& B = g_build;
  const long long v[16] = {B.lo[0], B.lo[1], B.lo[2], B.dims[0], B.dims[1], B.dims[2], B.split, (long long)B.n_rays,
                           (long long)B.n_skipped, (long long)B.label.size(), (long long)B.n_app_vox, (long long)B.n_van_vox,
                           (long long)B.point_label.size(), (long long)B.n_app_pts, (long long)B.n_van_pts,
                           B.offsets.empty() ? 0 : B.offsets.back()};
  std::memcpy(info, v, sizeof(v));
}

// any pointer may be NULL: ijk (3 ints per voxel), the four counts and the label per voxel in rank order; the label per point
void chh_voxels(int* ijk, uint32_t* hits_b, uint32_t* frees_b, uint32_t* hits_a, uint32_t* frees_a, unsigned char* label,
                unsigned char* point_label) {
  const Build& B = g_build;
  const size_t n = B.label.size();
  if (n) {
    if (ijk) std::memcpy(ijk, B.ijk.data(), 3 * n * sizeof(int));
    if (hits_b) std::memcpy(hits_b, B.hits[CH_BEFORE].data(), n * 4);
    if (frees_b) std::memcpy(frees_b, B.frees[CH_BEFORE].data(), n * 4);
    if (hits_a) std::memcpy(hits_a, B.hits[CH_AFTER].data(), n * 4);
    if (frees_a) std::memcpy(frees_a, B.frees[CH_AFTER].data(), n * 4);
    if (label) std::memcpy(label, B.label.data(), n);
  }
  if (point_label && !B.point_label.empty()) std::memcpy(point_label, B.point_label.data(), B.point_label.size());
}

// the updated map (4 floats per kept point, assembly order) and its per-submap offsets (n_sub + 1)
void chh_updated(float* out, long long* offsets) {
  const Build& B = g_build;
  size_t m = 0;
  for (size_t i = 0; i < B.point_label.size(); i++)
    if (B.point_label[i] != CH_VANISHED) {
      if (out) std::memcpy(out + 4 * m, &B.points[4 * i], 4 * sizeof(float));
      m++;
    }
  if (offsets) std::memcpy(offsets, B.offsets.data(), B.offsets.size() * sizeof(long long));
}

}  // extern "C"

#ifdef CH_HOST_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that builds the
// changes of generated submaps with non-finite rows, negative coordinates and empty submaps at several splits, and checks
// that the submaps of each epoch in reverse order give the same voxels, counts and labels, that each epoch's counts never
// exceed its submaps, that an AFTER point is never dropped, and that the offsets add up.
#include <cmath>
#include <limits>

int main() {
  int failures = 0;
  const double params[8] = {0.25, 20.0, 0.0, 0.0, 0.3, 0.85, 2, 0.4};
  for (int trial = 0; trial < 6; trial++) {
    const int n_sub = 2 + trial * 2;
    std::vector<float> pts;
    std::vector<long long> off{0};
    std::vector<double> poses;
    uint64_t st = 0x9E3779B97F4A7C15ull * (uint64_t)(trial + 7);
    auto rnd = [&]() {
      st = st * 6364136223846793005ull + 1442695040888963407ull;
      return (double)(st >> 11) * (1.0 / 9007199254740992.0);
    };
    const int split = 1 + trial % (n_sub - 1);
    for (int k = 0; k < n_sub; k++) {
      const int n = (k % 3 == 2) ? 0 : 200 + 37 * k;
      for (int i = 0; i < n; i++) {
        float x = (float)(rnd() * 30 - 15), y = (float)(rnd() * 30 - 15), z = (float)(rnd() * 6 - 3);
        if (i % 41 == 7) x = std::numeric_limits<float>::quiet_NaN();
        if (i % 43 == 9) z = std::numeric_limits<float>::infinity();
        pts.insert(pts.end(), {x, y, z, (float)i});
      }
      off.push_back(off.back() + n);
      const double yaw = rnd() * 6.283185307179586, tx = rnd() * 10 - 7, ty = rnd() * 10 - 7;
      const double P[16] = {std::cos(yaw), std::sin(yaw), 0, 0, -std::sin(yaw), std::cos(yaw), 0, 0, 0, 0, 1, 0, tx, ty, 1.2, 1};
      poses.insert(poses.end(), P, P + 16);
    }
    if (chh_build(params, split, 0, pts.data(), off.data(), poses.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    const Build first = g_build;
    for (size_t q = 0; q < first.label.size(); q++)
      if (first.hits[0][q] + first.frees[0][q] > (unsigned)split || first.hits[1][q] + first.frees[1][q] > (unsigned)(n_sub - split) ||
          first.hits[0][q] + first.hits[1][q] == 0)
        failures++;
    long long kept = 0;
    for (size_t i = 0; i < first.point_label.size(); i++) {
      kept += first.point_label[i] != CH_VANISHED;
      if (i >= (size_t)off[split] && first.point_label[i] == CH_VANISHED) failures++;
    }
    if (kept != first.offsets.back()) failures++;
    // each epoch's submaps in reverse order, the split where it was
    std::vector<float> rp;
    std::vector<long long> ro{0};
    std::vector<double> rpo;
    auto take = [&](int k) {
      rp.insert(rp.end(), pts.begin() + 4 * off[k], pts.begin() + 4 * off[k + 1]);
      ro.push_back(ro.back() + (off[k + 1] - off[k]));
      rpo.insert(rpo.end(), poses.begin() + 16 * k, poses.begin() + 16 * (k + 1));
    };
    for (int k = split - 1; k >= 0; k--) take(k);
    for (int k = n_sub - 1; k >= split; k--) take(k);
    if (chh_build(params, split, 0, rp.data(), ro.data(), rpo.data(), n_sub) != 0 || g_build.hits[0] != first.hits[0] ||
        g_build.frees[0] != first.frees[0] || g_build.hits[1] != first.hits[1] || g_build.frees[1] != first.frees[1] ||
        g_build.ijk != first.ijk || g_build.label != first.label || g_build.offsets.back() != first.offsets.back() ||
        g_build.n_app_pts != first.n_app_pts || g_build.n_van_pts != first.n_van_pts) {
      std::printf("MISMATCH trial=%d\n", trial);
      failures++;
    }
  }
  std::printf("map_changes_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
