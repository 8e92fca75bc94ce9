// Scan Context (G. Kim and A. Kim, IROS 2018) of a submap and the distance between two of them, as the place search of the
// scan-matcher session (b200sm_search_loop_place) defines them. The kernels (place_recognition.cu) and a host compile
// (tests/hostmath/scan_context_host.cpp, g++ -ffp-contract=off) both use the functions below, so a descriptor, a column norm
// and a distance are the same bits on either side: every double product, sum, quotient and square root is rounded on its
// own (__dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn on the device). There is no atan2: libm and CUDA differ in its last
// ulp, which would move points across sector edges. The angle is instead compared against a table of sector directions
// made once on the host, and both sides read the table's bits.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#ifdef __CUDACC__
#define SC_HD __host__ __device__ __forceinline__
#else
#define SC_HD inline
#endif
#ifdef __CUDA_ARCH__
#define SC_NO_UNROLL _Pragma("unroll 1")  // K13b: no double-division call unrolled into a copy that spills around it
#else
#define SC_NO_UNROLL
#endif

namespace b200 {

constexpr int SC_MAX_RINGS = 128, SC_MAX_SECTORS = 720, SC_MAX_BINS = 8192, SC_MAX_TOP_K = 1024;

struct ScParams {
  int num_rings = 20, num_sectors = 60;
  double max_radius = 80.0, lidar_height = 2.0;
};

inline bool sc_params_valid(const ScParams& p) {
  return p.num_rings >= 1 && p.num_rings <= SC_MAX_RINGS && p.num_sectors >= 1 && p.num_sectors <= SC_MAX_SECTORS &&
         p.num_rings * p.num_sectors <= SC_MAX_BINS && std::isfinite(p.max_radius) && p.max_radius > 0 &&
         std::isfinite(p.lidar_height);
}

SC_HD double sc_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
SC_HD double sc_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
SC_HD double sc_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
SC_HD double sc_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
SC_HD double sc_sqrt(double a) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
SC_HD bool sc_finite(float v) {
#ifdef __CUDA_ARCH__
  return isfinite(v);
#else
  return std::isfinite(v);
#endif
}

// The tables the binning reads. ring_b[k - 1] = B_k = t_k * t_k with t_k = (k * max_radius) / num_rings, k = 1..num_rings
// (ring_b[num_rings - 1] is the outer bound); sector_u[2 k], sector_u[2 k + 1] = cos, sin of a_k = (2 pi k) / num_sectors,
// k = 0..num_sectors-1.
inline void sc_tables(const ScParams& p, std::vector<double>& ring_b, std::vector<double>& sector_u) {
  ring_b.resize(p.num_rings);
  for (int k = 1; k <= p.num_rings; k++) {
    const double t = ((double)k * p.max_radius) / p.num_rings;
    ring_b[k - 1] = t * t;
  }
  sector_u.resize(2 * (size_t)p.num_sectors);
  for (int k = 0; k < p.num_sectors; k++) {
    const double a = (2.0 * 3.141592653589793 * (double)k) / p.num_sectors;  // math.pi
    sector_u[2 * k] = std::cos(a);
    sector_u[2 * k + 1] = std::sin(a);
  }
}

SC_HD int sc_half(double x, double y) { return (y < 0 || (y == 0 && x < 0)) ? 1 : 0; }

// angle(a) <= angle(b) on [0, 2 pi): the lower half-plane first, then the sign of the cross product a x b
SC_HD bool sc_angle_le(double ax, double ay, double bx, double by) {
  const int ha = sc_half(ax, ay), hb = sc_half(bx, by);
  if (ha != hb) return ha < hb;
  return sc_sub(sc_mul(ax, by), sc_mul(ay, bx)) >= 0;
}

// The bin of point (x, y, z), ring * num_sectors + sector, or -1 when the point is skipped (a non-finite coordinate, or
// q = x^2 + y^2 beyond the outer bound). ring = #{k in 1..R-1 : B_k <= q}; sector = #{k in 1..S-1 : angle(u_k) <=
// angle(p)}; the origin is bin 0. Both counts are binary searches: B_k is non-decreasing in k, and the sector directions
// are at least 2 pi / 720 apart, so the rounded comparison against u_k is monotone in k as well.
SC_HD int sc_bin(float x, float y, float z, const double* ring_b, int num_rings, const double* sector_u, int num_sectors) {
  if (!sc_finite(x) || !sc_finite(y) || !sc_finite(z)) return -1;
  const double dx = x, dy = y;
  const double q = sc_add(sc_mul(dx, dx), sc_mul(dy, dy));
  if (q > ring_b[num_rings - 1]) return -1;
  int lo = 0, hi = num_rings - 1;  // ring in [lo, hi]: the count of B_1..B_{R-1} that are <= q
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ring_b[mid - 1] <= q) lo = mid;
    else hi = mid - 1;
  }
  const int ring = lo;
  if (dx == 0 && dy == 0) return ring * num_sectors;
  lo = 0;
  hi = num_sectors - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sc_angle_le(sector_u[2 * mid], sector_u[2 * mid + 1], dx, dy)) lo = mid;
    else hi = mid - 1;
  }
  return ring * num_sectors + lo;
}

// The value a point puts in its bin: z + (float)lidar_height, in float.
SC_HD float sc_value(float z, float height) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(z, height);
#else
  return z + height;
#endif
}

// Float <-> an unsigned of the same order (+0 above -0), so that a bin's maximum is an integer atomicMax. 0 is the key of
// no float that sc_value can give (it would be a NaN with every bit set): it marks an empty bin.
SC_HD uint32_t sc_order_key(float v) {
  uint32_t u;
  std::memcpy(&u, &v, 4);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
SC_HD float sc_from_key(uint32_t k) {
  if (k == 0) return 0.0f;
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float v;
  std::memcpy(&v, &u, 4);
  return v;
}

// n_j = sqrt(sum_i (double)D[i][j]^2), ascending i; D is ring-major with num_sectors columns
SC_HD double sc_column_norm(const float* D, int num_rings, int num_sectors, int j) {
  double a = 0;
  for (int i = 0; i < num_rings; i++) {
    const double v = D[i * num_sectors + j];
    a = sc_add(a, sc_mul(v, v));
  }
  return sc_sqrt(a);
}

// d_s: the mean cosine over the column pairs (j, (j + s) mod S) whose norms are both non-zero, subtracted from 1; 1.0 when
// there is no such pair
SC_HD double sc_distance_at(const float* Q, const double* nQ, const float* C, const double* nC, int num_rings, int num_sectors, int s) {
  double sum = 0;
  int m = 0;
  SC_NO_UNROLL
  for (int j = 0; j < num_sectors; j++) {
    int c = j + s;
    if (c >= num_sectors) c -= num_sectors;
    if (nQ[j] > 0 && nC[c] > 0) {
      double dot = 0;
      for (int i = 0; i < num_rings; i++) dot = sc_add(dot, sc_mul((double)Q[i * num_sectors + j], (double)C[i * num_sectors + c]));
      sum = sc_add(sum, sc_div(dot, sc_mul(nQ[j], nC[c])));
      m++;
    }
  }
  return m ? sc_sub(1.0, sc_div(sum, (double)m)) : 1.0;
}

// D = min_s d_s and the lowest s that attains it
inline double sc_distance(const float* Q, const double* nQ, const float* C, const double* nC, int num_rings, int num_sectors, int* shift) {
  double best = sc_distance_at(Q, nQ, C, nC, num_rings, num_sectors, 0);
  int bs = 0;
  for (int s = 1; s < num_sectors; s++) {
    const double d = sc_distance_at(Q, nQ, C, nC, num_rings, num_sectors, s);
    if (d < best) {
      best = d;
      bs = s;
    }
  }
  *shift = bs;
  return best;
}

// The candidates of a place search: the rows r < n with D[r] < threshold, ordered by (D[r], ids[r]) ascending
inline std::vector<int> sc_rank(const double* D, const int* ids, size_t n, double threshold) {
  std::vector<int> rows;
  for (size_t r = 0; r < n; r++)
    if (D[r] < threshold) rows.push_back((int)r);
  std::sort(rows.begin(), rows.end(), [&](int a, int b) { return D[a] < D[b] || (D[a] == D[b] && ids[a] < ids[b]); });
  return rows;
}

// The initial guess of the verification: G = P_cand * Rz(2 pi s / num_sectors) * P_new^-1, row-major doubles (the
// products summed in ascending k from 0, the inverse an Isometry's: R^T, -R^T t), then cast to float column-major.
inline void sc_guess(const double* P_cand, const double* P_new, int shift, int num_sectors, float* G_colmajor16) {
  const double th = 2.0 * 3.141592653589793 * (double)shift / (double)num_sectors;
  const double c = std::cos(th), sn = std::sin(th);
  const double Rz[16] = {c, -sn, 0, 0, sn, c, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  double A[16], inv[16] = {P_new[0], P_new[4], P_new[8], 0, P_new[1], P_new[5], P_new[9], 0, P_new[2], P_new[6], P_new[10], 0,
                           0, 0, 0, 1};
  for (int r = 0; r < 3; r++) inv[r * 4 + 3] = -(inv[r * 4 + 0] * P_new[3] + inv[r * 4 + 1] * P_new[7] + inv[r * 4 + 2] * P_new[11]);
  for (int r = 0; r < 4; r++)
    for (int col = 0; col < 4; col++) {
      double a = 0;
      for (int k = 0; k < 4; k++) a += P_cand[r * 4 + k] * Rz[k * 4 + col];
      A[r * 4 + col] = a;
    }
  for (int r = 0; r < 4; r++)
    for (int col = 0; col < 4; col++) {
      double a = 0;
      for (int k = 0; k < 4; k++) a += A[r * 4 + k] * inv[k * 4 + col];
      G_colmajor16[col * 4 + r] = (float)a;
    }
}

}  // namespace b200
