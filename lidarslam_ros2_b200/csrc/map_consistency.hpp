// The map consistency of the session (b200sm_build_map_consistency): a ground-truth-free measure of how crisp the assembled
// map is. Every query point gets the covariance of its neighbours within `radius`; from it come the differential entropy
// h = 1/2 ln det(2 pi e Sigma), whose mean is the Mean Map Entropy (MME, Razlaw et al., 2015), and the smallest eigenvalue
// of Sigma, whose mean is the Mean Plane Variance (MPV). Double walls and blur from a bad pose or a wrong loop edge raise
// both. The kernels (consistency.cu) and a host compile (tests/hostmath/consistency_host.cpp, g++ -ffp-contract=off) both
// use the functions below, so every value is the same on either side, bit for bit.
//
// Definitions (this text is the contract; tests/consistencyref.py replays it in Python integers and doubles):
//  * Points: those b200sm_assemble_map(s, poses, ...) returns, in map order (submap by submap), each moved by its submap's
//    float pose (og_transform). A point with a non-finite coordinate is SKIPPED: counted, neither a query nor a neighbour.
//  * Fixed point, as the occupancy grid's: S = 2^16 / radius, X = floor((double)x * S), one rounded multiply (og_fixed).
//    Every non-skipped coordinate must satisfy |X| < 2^46, else the build is refused. The point's CELL is (X >> 16,
//    Y >> 16, Z >> 16): cells are `radius` on a side.
//  * Neighbourhood. The QUERIES are the non-skipped points whose map index is a multiple of query_stride. Neighbour j of
//    query i is a non-skipped point (i itself included) with D = P_j - P_i (int64) and Dx^2 + Dy^2 + Dz^2 <= 2^32, the
//    radius squared, exact. Only the 27 cells around the query's cell can hold one. The query keeps n and the nine int64
//    moments sum D_a, sum D_a D_b. |D_a| <= 2^16 for a neighbour, so every term is below 2^33 in magnitude and every sum
//    is exact for maps below 2^31 points (refused otherwise): the sums do not depend on the order of the work.
//  * Per query, in double, one rounding per operation in the order written below (mc_add etc.: __dadd_rn ... on the
//    device, -ffp-contract=off on the host): C_ab = (S_ab - S_a S_b / n) / n, the int64 sums converted first (units^2);
//    det C by mc_det's cofactor expansion. The query is VALID iff n >= min_neighbors and det C >= 1 (unit^6; about
//    (radius / 2^16)^2 per eigenvalue, which bounds h from below). h = 1/2 (c0 + mc_log(det C)) with c0 = 3 mc_log(2 pi e)
//    - 6 mc_log(S) (one value per build). plane_var = lambda_min(C) / S^2 (m^2), lambda_min from mc_lambda_min's fixed
//    cyclic Jacobi sweeps. An invalid query reads MC_NAN in both; a point that is not a query reads MC_NAN and n = 0.
//  * Aggregates, per submap and for the whole map: queries, valid queries, neighbours summed over all queries, and over the
//    valid queries sum rint(h * 2^24) and sum rint(plane_var / radius^2 * 2^30) in int64 (|h| < 64 for radius in
//    [0.01, 100], and plane_var <= radius^2, so both sums stay below 2^61 for maps below 2^31 points). MME = sum_h 2^-24 /
//    valid, MPV = sum_plane 2^-30 radius^2 / valid (NaN without a valid query). Integer sums: the device's atomics give
//    the host's bits.
//  * Box. The cells of the non-skipped points span a box [x0, x1] x [y0, y1] x [z0, z1] with the static map's linear index
//    and limit (sm_box): more than 2^31 - 1 cells is refused before anything is sized from it. A box that large is a real
//    limit for a kilometre-scale map at a small radius (2 km x 2 km x 50 m at 0.3 m is 2.2e9 cells); a second indexing
//    scheme over sorted cell keys would lift it.
#pragma once
#include <cstring>

#include "static_map.hpp"

namespace b200 {

constexpr double MC_COORD_LIMIT = OG_ORIGIN_LIMIT;               // 2^46: |X| of a non-skipped coordinate
constexpr long long MC_RADIUS2 = 1LL << 32;                     // the radius squared in fixed point
constexpr unsigned long long MC_MAX_POINTS = 0x7fffffffull;     // 2^31 - 1: the map's points
constexpr double MC_H_SCALE = 16777216.0;                       // 2^24
constexpr double MC_PLANE_SCALE = 1073741824.0;                 // 2^30
constexpr unsigned long long MC_NAN_BITS = 0x7ff8000000000000ull;  // the NaN of an invalid query or a non-query point
constexpr int MC_JACOBI_SWEEPS = 6;

struct McParams {
  double radius = 0.5;
  int min_neighbors = 10;
  int query_stride = 1;
};

// What a build computes from the parameters once, on the host.
struct McConst {
  double S;      // 2^16 / radius
  double S2;     // S * S
  double r2;     // radius * radius
  double c0;     // 3 mc_log(2 pi e) - 6 mc_log(S)
  long long min_neighbors;
  long long stride;
};

// The nine moments and the count of one query's neighbourhood.
struct McMoments {
  long long n = 0, sx = 0, sy = 0, sz = 0, sxx = 0, sxy = 0, sxz = 0, syy = 0, syz = 0, szz = 0;
};

OG_HD double mc_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
OG_HD double mc_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
OG_HD double mc_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
OG_HD double mc_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
OG_HD double mc_sqrt(double a) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
OG_HD double mc_i2d(long long v) {  // round to nearest, ties to even
#ifdef __CUDA_ARCH__
  return __ll2double_rn(v);
#else
  return (double)v;
#endif
}
OG_HD long long mc_rint(double v) {  // round to nearest, ties to even
#ifdef __CUDA_ARCH__
  return __double2ll_rn(v);
#else
  return std::llrint(v);
#endif
}
OG_HD unsigned long long mc_bits(double v) {
#ifdef __CUDA_ARCH__
  return (unsigned long long)__double_as_longlong(v);
#else
  unsigned long long b;
  std::memcpy(&b, &v, 8);
  return b;
#endif
}
OG_HD double mc_from_bits(unsigned long long b) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)b);
#else
  double v;
  std::memcpy(&v, &b, 8);
  return v;
#endif
}

// The natural logarithm of a positive normal x with + - * / only: x = m 2^e with m in [sqrt(2)/2, sqrt(2)), f = m - 1
// (exact), s = f / (2 + f), z = s^2, R = sum_{k=1..11} 2 z^k / (2k + 1) by Horner, ln m = f - s (f - R) (the odd series
// 2 atanh(s) = 2s + s R with 2s = f - s f), and ln x = e ln2_hi + (ln m + e ln2_lo), ln2_hi with 21 trailing zero bits so
// that e ln2_hi is exact. Within 2 ulp of the correctly rounded logarithm on [1, 2^100] (a test).
OG_HD double mc_log(double x) {
  const unsigned long long b = mc_bits(x);
  int e = (int)((b >> 52) & 0x7ffull) - 1023;
  double m = mc_from_bits((b & 0xfffffffffffffull) | 0x3ff0000000000000ull);  // [1, 2)
  if (m > 0x1.6a09e667f3bcdp+0) {                                              // sqrt(2)
    m = mc_mul(m, 0.5);
    e += 1;
  }
  const double f = mc_sub(m, 1.0);
  const double s = mc_div(f, mc_add(2.0, f));
  const double z = mc_mul(s, s);
  double R = 0x1.642c8590b2164p-4;  // 2/23, then 2/21 ... 2/3
  R = mc_add(0x1.8618618618618p-4, mc_mul(z, R));
  R = mc_add(0x1.af286bca1af28p-4, mc_mul(z, R));
  R = mc_add(0x1.e1e1e1e1e1e1ep-4, mc_mul(z, R));
  R = mc_add(0x1.1111111111111p-3, mc_mul(z, R));
  R = mc_add(0x1.3b13b13b13b14p-3, mc_mul(z, R));
  R = mc_add(0x1.745d1745d1746p-3, mc_mul(z, R));
  R = mc_add(0x1.c71c71c71c71cp-3, mc_mul(z, R));
  R = mc_add(0x1.2492492492492p-2, mc_mul(z, R));
  R = mc_add(0x1.999999999999ap-2, mc_mul(z, R));
  R = mc_add(0x1.5555555555555p-1, mc_mul(z, R));
  R = mc_mul(z, R);
  const double lnm = mc_sub(f, mc_mul(s, mc_sub(f, R)));
  const double de = (double)e;
  return mc_add(mc_mul(de, 0x1.62e42fee00000p-1), mc_add(lnm, mc_mul(de, 0x1.a39ef35793c76p-33)));
}

// One Jacobi rotation of a symmetric 3x3 in the plane (p, q), r the third index: zeroes a_pq (Numerical Recipes' form,
// theta = (a_qq - a_pp) / (2 a_pq), t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)), c = 1 / sqrt(t^2 + 1), s = t c).
// Skipped when a_pq is already 0.
OG_HD void mc_rotate(double& app, double& aqq, double& apq, double& arp, double& arq) {
  if (apq == 0.0) return;
  const double theta = mc_div(mc_sub(aqq, app), mc_mul(2.0, apq));
  const double at = theta < 0.0 ? -theta : theta;
  double t = mc_div(1.0, mc_add(at, mc_sqrt(mc_add(mc_mul(theta, theta), 1.0))));
  if (theta < 0.0) t = -t;
  const double c = mc_div(1.0, mc_sqrt(mc_add(mc_mul(t, t), 1.0)));
  const double s = mc_mul(t, c);
  const double tp = mc_mul(t, apq);
  app = mc_sub(app, tp);
  aqq = mc_add(aqq, tp);
  apq = 0.0;
  const double rp = arp, rq = arq;
  arp = mc_sub(mc_mul(c, rp), mc_mul(s, rq));
  arq = mc_add(mc_mul(s, rp), mc_mul(c, rq));
}

// The smallest eigenvalue of the symmetric matrix (a00 a01 a02; a11 a12; a22): MC_JACOBI_SWEEPS cyclic sweeps over
// (0, 1), (0, 2), (1, 2), then the least diagonal entry. Within 1e-12 of the largest eigenvalue of numpy's eigvalsh (a test).
OG_HD double mc_lambda_min(double a00, double a01, double a02, double a11, double a12, double a22) {
  for (int sweep = 0; sweep < MC_JACOBI_SWEEPS; sweep++) {
    mc_rotate(a00, a11, a01, a02, a12);
    mc_rotate(a00, a22, a02, a01, a12);
    mc_rotate(a11, a22, a12, a01, a02);
  }
  const double m = a00 < a11 ? a00 : a11;
  return m < a22 ? m : a22;
}

// det of the symmetric matrix by the cofactor expansion along its first row
OG_HD double mc_det(double c00, double c01, double c02, double c11, double c12, double c22) {
  const double m0 = mc_sub(mc_mul(c11, c22), mc_mul(c12, c12));
  const double m1 = mc_sub(mc_mul(c01, c22), mc_mul(c12, c02));
  const double m2 = mc_sub(mc_mul(c01, c12), mc_mul(c11, c02));
  return mc_add(mc_sub(mc_mul(c00, m0), mc_mul(c01, m1)), mc_mul(c02, m2));
}

enum : int { MC_POINT_OK = 0, MC_POINT_SKIPPED, MC_POINT_RANGE };

// A moved point e into fixed point X[3]: MC_POINT_SKIPPED when a coordinate is not finite, MC_POINT_RANGE when a product
// is not inside (-2^46, 2^46) (the build is refused), else MC_POINT_OK.
OG_HD int mc_point(const McConst& c, const float* e, long long* X) {
  for (int a = 0; a < 3; a++)
    if (e[a] - e[a] != 0.0f) return MC_POINT_SKIPPED;  // NaN or an infinity
  for (int a = 0; a < 3; a++)
    if (!og_fixed(e[a], c.S, MC_COORD_LIMIT, &X[a])) return MC_POINT_RANGE;
  return MC_POINT_OK;
}

// A candidate at offset D from the query: accumulated when it is a neighbour
OG_HD void mc_accumulate(McMoments& m, long long dx, long long dy, long long dz) {
  const long long xx = dx * dx, yy = dy * dy, zz = dz * dz;
  if (xx + yy + zz > MC_RADIUS2) return;
  m.n += 1;
  m.sx += dx;
  m.sy += dy;
  m.sz += dz;
  m.sxx += xx;
  m.sxy += dx * dy;
  m.sxz += dx * dz;
  m.syy += yy;
  m.syz += dy * dz;
  m.szz += zz;
}

// covariance entry (S_ab - S_a S_b / n) / n
OG_HD double mc_cov(double sab, double sa, double sb, double n) { return mc_div(mc_sub(sab, mc_div(mc_mul(sa, sb), n)), n); }

// One query's values: true when valid, with *h, *plane_var and the quantised *qh, *ql; false leaves them alone.
OG_HD bool mc_query(const McConst& c, const McMoments& m, double* h, double* plane_var, long long* qh, long long* ql) {
  if (m.n < c.min_neighbors) return false;
  const double n = mc_i2d(m.n), sx = mc_i2d(m.sx), sy = mc_i2d(m.sy), sz = mc_i2d(m.sz);
  const double c00 = mc_cov(mc_i2d(m.sxx), sx, sx, n), c01 = mc_cov(mc_i2d(m.sxy), sx, sy, n), c02 = mc_cov(mc_i2d(m.sxz), sx, sz, n);
  const double c11 = mc_cov(mc_i2d(m.syy), sy, sy, n), c12 = mc_cov(mc_i2d(m.syz), sy, sz, n), c22 = mc_cov(mc_i2d(m.szz), sz, sz, n);
  const double det = mc_det(c00, c01, c02, c11, c12, c22);
  if (!(det >= 1.0)) return false;
  *h = mc_mul(0.5, mc_add(c.c0, mc_log(det)));
  *plane_var = mc_div(mc_lambda_min(c00, c01, c02, c11, c12, c22), c.S2);
  *qh = mc_rint(mc_mul(*h, MC_H_SCALE));
  *ql = mc_rint(mc_mul(mc_div(*plane_var, c.r2), MC_PLANE_SCALE));
  return true;
}

// ---- host side: parameters, aggregates ----

// nullptr when p is valid (and *c filled), else the reason
inline const char* mc_prepare(const McParams& p, McConst* c) {
  if (!(p.radius >= 0.01 && p.radius <= 100.0)) return "radius must be in [0.01, 100] m";
  if (p.min_neighbors < 4) return "min_neighbors must be >= 4";
  if (p.query_stride < 1) return "query_stride must be >= 1";
  c->S = 65536.0 / p.radius;
  c->S2 = c->S * c->S;
  c->r2 = p.radius * p.radius;
  c->c0 = mc_sub(mc_mul(3.0, mc_log(0x1.114580b45d475p+4)), mc_mul(6.0, mc_log(c->S)));  // 2 pi e
  c->min_neighbors = p.min_neighbors;
  c->stride = p.query_stride;
  return nullptr;
}

// MME from the quantised sum of h over `valid` queries (NaN when there is none)
inline double mc_mme(long long sum_h, unsigned long long valid) {
  return valid ? mc_div(mc_mul(mc_i2d(sum_h), 1.0 / MC_H_SCALE), mc_i2d((long long)valid)) : mc_from_bits(MC_NAN_BITS);
}
// MPV (m^2) from the quantised sum of plane_var / radius^2
inline double mc_mpv(const McConst& c, long long sum_plane, unsigned long long valid) {
  return valid ? mc_div(mc_mul(mc_mul(mc_i2d(sum_plane), 1.0 / MC_PLANE_SCALE), c.r2), mc_i2d((long long)valid))
               : mc_from_bits(MC_NAN_BITS);
}

}  // namespace b200
