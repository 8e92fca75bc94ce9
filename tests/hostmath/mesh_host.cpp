// TEST INFRASTRUCTURE: the surface mesh of b200sm_build_mesh (csrc/mesh.hpp) built serially on the host from the same
// header: origins, rays, the widened box of the endpoint voxels, the band walks into a rank index over it, the fused sums
// and weights, the ACTIVE cells, their vertices and the faces. tests/test_mesh_cpu.py compares it with the Python replay
// (tests/meshref.py) and the GPU tests compare the session with it bit for bit. Build with -ffp-contract=off and, for the
// sanitised run (-DMS_HOST_MAIN), -fsanitize=address,undefined.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/mesh.hpp"

using namespace b200;

namespace {

struct Build {
  int lo[3] = {0, 0, 0};
  unsigned dims[3] = {0, 0, 0};
  unsigned long long n_points = 0, n_rays = 0, n_skipped = 0, n_walked = 0, n_observed = 0;
  std::vector<int> ijk;  // 3 per band voxel, rank order
  std::vector<long long> sum;
  std::vector<uint32_t> weight;
  std::vector<float> vertices;    // 3 per vertex
  std::vector<uint32_t> faces;    // 3 per face
};
Build g_build;

// The ACTIVE cells, vertices and faces of B's band voxels (lo, dims, ijk in rank order, sum, weight). 0, or -6 for 2^32
// faces or more.
int extract_mesh(Build& B, unsigned min_weight, double resolution) {
  const unsigned long long cells = (unsigned long long)B.dims[0] * B.dims[1] * B.dims[2];
  const size_t n_words = (size_t)((cells + 31) / 32);
  const unsigned n_vox = (unsigned)B.sum.size();
  std::vector<uint32_t> bits(n_words), prefix(n_words);
  auto lin_of = [&](int x, int y, int z, unsigned* lin) {
    const long long wx = (long long)x - B.lo[0], wy = (long long)y - B.lo[1], wz = (long long)z - B.lo[2];
    if (wx < 0 || wy < 0 || wz < 0 || wx >= B.dims[0] || wy >= B.dims[1] || wz >= B.dims[2]) return false;
    *lin = (unsigned)((wz * (long long)B.dims[1] + wy) * (long long)B.dims[0] + wx);
    return true;
  };
  for (unsigned v = 0; v < n_vox; v++) {
    unsigned lin;
    if (!lin_of(B.ijk[3 * (size_t)v], B.ijk[3 * (size_t)v + 1], B.ijk[3 * (size_t)v + 2], &lin)) std::abort();
    bits[lin >> 5] |= 1u << (lin & 31u);
  }
  unsigned acc = 0;
  for (size_t w = 0; w < n_words; w++) {
    prefix[w] = acc;
    acc += (unsigned)__builtin_popcount(bits[w]);
  }
  auto rank_of = [&](int x, int y, int z, unsigned* r) {
    unsigned lin;
    if (!lin_of(x, y, z, &lin)) return false;
    const uint32_t w = bits[lin >> 5], bit = lin & 31u;
    if (!((w >> bit) & 1u)) return false;
    *r = prefix[lin >> 5] + (unsigned)__builtin_popcount(w & ((1u << bit) - 1u));
    return true;
  };
  struct { unsigned min_weight; double resolution; } c{min_weight, resolution};
  B.vertices.clear();
  B.faces.clear();
  B.n_observed = 0;
  auto observed = [&](int x, int y, int z, unsigned* r) { return rank_of(x, y, z, r) && B.weight[*r] >= c.min_weight; };
  for (unsigned v = 0; v < n_vox; v++) B.n_observed += B.weight[v] >= c.min_weight;
  // ACTIVE cells by their lowest corner's rank, and their vertex ids
  std::vector<uint32_t> vid(n_vox, 0xffffffffu);
  unsigned n_vert = 0;
  for (unsigned v = 0; v < n_vox; v++) {
    const int* q = &B.ijk[3 * (size_t)v];
    double D[8];
    bool neg[8];
    bool all = true;
    int n_neg = 0;
    for (int m = 0; m < 8 && all; m++) {
      unsigned r;
      if (!observed(q[0] + (m & 1), q[1] + ((m >> 1) & 1), q[2] + ((m >> 2) & 1), &r)) all = false;
      else {
        D[m] = ms_dist(B.sum[r], B.weight[r]);
        neg[m] = ms_neg(B.sum[r]);
        n_neg += neg[m];
      }
    }
    if (!all || n_neg == 0 || n_neg == 8) continue;
    vid[v] = n_vert++;
    float xyz[3];
    ms_vertex(D, neg, q[0], q[1], q[2], c.resolution, xyz);
    B.vertices.insert(B.vertices.end(), xyz, xyz + 3);
  }
  unsigned long long n_faces = 0;
  for (unsigned v = 0; v < n_vox; v++) {
    if (B.weight[v] < c.min_weight) continue;
    const int* q = &B.ijk[3 * (size_t)v];
    const bool vn = ms_neg(B.sum[v]);
    for (int a = 0; a < 3; a++) {
      unsigned w;
      if (!observed(q[0] + (a == 0), q[1] + (a == 1), q[2] + (a == 2), &w) || ms_neg(B.sum[w]) == vn) continue;
      unsigned ids[4];
      bool all = true;
      for (int m = 0; m < 4 && all; m++) {
        int cc[3];
        ms_edge_cell(a, m & 1, m >> 1, q[0], q[1], q[2], cc);
        unsigned r;
        if (!rank_of(cc[0], cc[1], cc[2], &r) || vid[r] == 0xffffffffu) all = false;
        else ids[m] = vid[r];
      }
      if (!all) continue;
      unsigned tri[6];
      ms_quad(ids, vn, tri);
      B.faces.insert(B.faces.end(), tri, tri + 6);
      n_faces += 2;
    }
  }
  if (n_faces > 0xffffffffull) return -6;
  return 0;
}

}  // namespace

extern "C" {

// params: resolution, truncation, max_range, sensor_origin x y z, min_weight. points: 4 floats per row, submap k = rows
// offsets[k] .. offsets[k + 1]; poses: 16 doubles per submap, column-major. Returns 0, or -1 (parameters), -2 (an origin
// out of range), -3 (a box of more than 2^31 - 1 voxels), -4 (no submaps), -6 (2^32 faces or more).
int msh_build(const double* params, const float* points, const long long* offsets, const double* poses, int n_sub) {
  MsParams p;
  p.resolution = params[0];
  p.truncation = params[1];
  p.max_range = params[2];
  for (int k = 0; k < 3; k++) p.sensor_origin[k] = params[3 + k];
  p.min_weight = params[6] >= 0 && params[6] <= 4294967295.0 ? (unsigned)params[6] : 0u;
  MsConst c;
  if (ms_prepare(p, &c)) return -1;
  if (n_sub <= 0) return -4;
  std::vector<float> T(12 * (size_t)n_sub);
  std::vector<long long> O(3 * (size_t)n_sub);
  for (int k = 0; k < n_sub; k++) {
    og_pose_f(poses + 16 * (size_t)k, &T[12 * (size_t)k]);
    if (!ms_origin(c, p, &T[12 * (size_t)k], &O[3 * (size_t)k])) return -2;
  }
  const size_t n = (size_t)offsets[n_sub];
  std::vector<unsigned char> is_ray(n);
  std::vector<long long> end(3 * n);
  std::vector<int> sub_of(n);
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  unsigned long long rays = 0, skipped = 0;
  for (int k = 0; k < n_sub; k++)
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(&T[12 * (size_t)k], points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      int v[3];
      long long* f = &end[3 * i];
      sub_of[i] = k;
      if (!sm_ray(c.sm, &O[3 * (size_t)k], e[0], e[1], e[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) {
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
  int blo[3] = {0, 0, 0};
  unsigned long long cells = 0;
  if (rays && !ms_box(lo, hi, c.r, blo, dims, &cells)) return -3;
  Build& B = g_build;
  B = Build();
  B.n_points = n;
  B.n_rays = rays;
  B.n_skipped = skipped;
  if (rays)
    for (int a = 0; a < 3; a++) {
      B.lo[a] = blo[a];
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
  // the band walk of ray i: visit(x, y, z, s)
  auto band = [&](size_t i, auto&& visit) {
    const long long* o = &O[3 * (size_t)sub_of[i]];
    const long long* E = &end[3 * i];
    long long A[3], Bp[3];
    double L;
    if (!ms_band(c.T, o, E[0], E[1], E[2], A, Bp, &L)) return;
    sm_walk(A[0], A[1], A[2], Bp[0], Bp[1], Bp[2], [&](int x, int y, int z) {
      visit(x, y, z, ms_sdf(c.T, E[0], E[1], E[2], E[0] - o[0], E[1] - o[1], E[2] - o[2], L, x, y, z));
    });
  };
  for (size_t i = 0; i < n; i++) {
    if (!is_ray[i]) continue;
    band(i, [&](int x, int y, int z, long long) {
      unsigned lin;
      if (!lin_of(x, y, z, &lin)) std::abort();  // the header's bound: every walk stays in the widened box
      bits[lin >> 5] |= 1u << (lin & 31u);
    });
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
  B.sum.assign(n_vox, 0);
  B.weight.assign(n_vox, 0);
  for (size_t i = 0; i < n; i++) {
    if (!is_ray[i]) continue;
    band(i, [&](int x, int y, int z, long long s) {
      unsigned r;
      if (!rank_of(x, y, z, &r)) std::abort();
      B.sum[r] += s;
      B.weight[r] += 1;
      B.n_walked++;
    });
  }
  return extract_mesh(B, c.min_weight, c.resolution);
}

// The extraction alone on a given field: box lo[3], dims[3], n band voxels ijk (3 ints each, ascending linear index in the
// box), sum, weight. Returns 0 or -6; msh_info / msh_arrays read the result.
int msh_extract(const int* lo, const unsigned* dims, const int* ijk, const long long* sum, const uint32_t* weight, long long n,
                double resolution, unsigned min_weight) {
  Build& B = g_build;
  B = Build();
  for (int a = 0; a < 3; a++) {
    B.lo[a] = lo[a];
    B.dims[a] = dims[a];
  }
  B.ijk.assign(ijk, ijk + 3 * n);
  B.sum.assign(sum, sum + n);
  B.weight.assign(weight, weight + n);
  return extract_mesh(B, min_weight, resolution);
}

// ms_box: 1 and the box (blo[3], dims[3]) when the bounds lo[3], hi[3] widened by r make at most 2^31 - 1 voxels, else 0
int msh_box(const int* lo, const int* hi, int r, int* blo, unsigned* dims) {
  unsigned long long cells = 0;
  return ms_box(lo, hi, r, blo, dims, &cells) ? 1 : 0;
}

// lo x y z, W, H, D, n_points, n_rays, n_skipped, n_walked, n_band_voxels, n_observed_voxels, n_vertices, n_faces
void msh_info(long long* info) {
  const Build& B = g_build;
  const long long v[14] = {B.lo[0], B.lo[1], B.lo[2], B.dims[0], B.dims[1], B.dims[2], (long long)B.n_points, (long long)B.n_rays,
                           (long long)B.n_skipped, (long long)B.n_walked, (long long)B.sum.size(), (long long)B.n_observed,
                           (long long)(B.vertices.size() / 3), (long long)(B.faces.size() / 3)};
  std::memcpy(info, v, sizeof(v));
}

// any pointer may be NULL: ijk (3 ints per band voxel), sum, weight in rank order; vertices (3 floats), faces (3 uint32)
void msh_arrays(int* ijk, long long* sum, uint32_t* weight, float* vertices, uint32_t* faces) {
  const Build& B = g_build;
  const size_t n = B.sum.size();
  if (n) {
    if (ijk) std::memcpy(ijk, B.ijk.data(), 3 * n * sizeof(int));
    if (sum) std::memcpy(sum, B.sum.data(), n * sizeof(long long));
    if (weight) std::memcpy(weight, B.weight.data(), n * sizeof(uint32_t));
  }
  if (vertices && !B.vertices.empty()) std::memcpy(vertices, B.vertices.data(), B.vertices.size() * sizeof(float));
  if (faces && !B.faces.empty()) std::memcpy(faces, B.faces.data(), B.faces.size() * sizeof(uint32_t));
}

}  // extern "C"

#ifdef MS_HOST_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that builds the
// mesh of generated submaps with non-finite rows, negative coordinates, zero-length rays and empty submaps, and checks that
// the submaps and points in reverse order give the same field, vertices and faces, that every face's vertices are distinct
// ids below the vertex count, and that the weights add up to the walked voxels.
#include <cmath>
#include <limits>

int main() {
  int failures = 0;
  const double params[7] = {0.25, 0.75, 20.0, 0.0, 0.0, 0.3, 2};
  for (int trial = 0; trial < 6; trial++) {
    const int n_sub = 2 + trial * 2;
    std::vector<float> pts;
    std::vector<long long> off{0};
    std::vector<double> poses;
    uint64_t st = 0x9E3779B97F4A7C15ull * (uint64_t)(trial + 11);
    auto rnd = [&]() {
      st = st * 6364136223846793005ull + 1442695040888963407ull;
      return (double)(st >> 11) * (1.0 / 9007199254740992.0);
    };
    for (int k = 0; k < n_sub; k++) {
      const int n = (k % 3 == 2) ? 0 : 6000 + 41 * k;
      for (int i = 0; i < n; i++) {
        // points on a sphere of radius 4 around the submap's sensor (the sensors within 0.3 m of each other), and some
        // scattered ones
        const double th = rnd() * 6.283185307179586, u = rnd() * 2 - 1, rad = (i % 5 == 0) ? 1 + rnd() * 10 : 4.0;
        float x = (float)(rad * std::sqrt(1 - u * u) * std::cos(th)), y = (float)(rad * std::sqrt(1 - u * u) * std::sin(th)),
              z = (float)(rad * u - 0.3);
        if (i % 41 == 7) x = std::numeric_limits<float>::quiet_NaN();
        if (i % 43 == 9) z = std::numeric_limits<float>::infinity();
        if (i % 47 == 3) x = 0.f, y = 0.f, z = 0.3f;  // at the sensor origin (0, 0, 0.3): a zero-length ray
        pts.insert(pts.end(), {x, y, z, (float)i});
      }
      off.push_back(off.back() + n);
      const double yaw = rnd() * 6.283185307179586, tx = rnd() * 0.3 - 7, ty = rnd() * 0.3 - 7;
      const double P[16] = {std::cos(yaw), std::sin(yaw), 0, 0, -std::sin(yaw), std::cos(yaw), 0, 0, 0, 0, 1, 0, tx, ty, 1.2, 1};
      poses.insert(poses.end(), P, P + 16);
    }
    if (msh_build(params, pts.data(), off.data(), poses.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    const Build first = g_build;
    unsigned long long w = 0;
    for (uint32_t x : first.weight) w += x;
    if (w != first.n_walked) failures++;
    const uint32_t nv = (uint32_t)(first.vertices.size() / 3);
    for (size_t f = 0; f < first.faces.size(); f += 3) {
      const uint32_t a = first.faces[f], b = first.faces[f + 1], c = first.faces[f + 2];
      if (a >= nv || b >= nv || c >= nv || a == b || b == c || a == c) failures++;
    }
    // submaps and the points of each in reverse order
    std::vector<float> rp;
    std::vector<long long> ro{0};
    std::vector<double> rpo;
    for (int k = n_sub - 1; k >= 0; k--) {
      for (long long i = off[k + 1] - 1; i >= off[k]; i--) rp.insert(rp.end(), pts.begin() + 4 * i, pts.begin() + 4 * i + 4);
      ro.push_back(ro.back() + (off[k + 1] - off[k]));
      rpo.insert(rpo.end(), poses.begin() + 16 * k, poses.begin() + 16 * (k + 1));
    }
    if (msh_build(params, rp.data(), ro.data(), rpo.data(), n_sub) != 0 || g_build.ijk != first.ijk || g_build.sum != first.sum ||
        g_build.weight != first.weight || g_build.faces != first.faces || g_build.vertices.size() != first.vertices.size() ||
        (!first.vertices.empty() &&
         std::memcmp(g_build.vertices.data(), first.vertices.data(), first.vertices.size() * sizeof(float)) != 0)) {
      std::printf("MISMATCH trial=%d\n", trial);
      failures++;
    }
    if (first.faces.empty()) failures++;
  }
  std::printf("mesh_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
