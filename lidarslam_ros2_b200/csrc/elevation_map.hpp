// The 2.5D elevation and traversability map of the session's map (b200sm_build_elevation_map): a surface height per 2D
// cell under the robot's clearance, and the slope, step and roughness of a window of cells around it, classified as nav2's
// map_server reads a trinary map. The kernels (elevation.cu) and a host compile (tests/hostmath/elevation_host.cpp, g++
// -ffp-contract=off) both use the functions below, with occupancy_grid.hpp's fixed point, transform, skip rule, image rule
// and files, so every layer is bitwise the same on either side. Every double step is written out with one rounding per
// operation in a fixed order (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn on the device); the one
// transcendental, tan(max_slope), is evaluated once on the host.
//
// Definitions (this text is the contract; tests/elevationref.py replays it in Python integers and doubles):
//  * Points. S = 2^16 / resolution. Submap k's float pose T moves every point p of its cloud to e = transform_point(T, p),
//    bitwise the point b200sm_assemble_map returns, and its origin is o = transform_point(T, (float)sensor_origin), whose X
//    and Y must lie inside (-2^46, 2^46) in fixed point (else the build is refused). A point is skipped exactly as
//    occupancy_grid.hpp skips a ray (og_ray): a coordinate of e out of range (non-finite included), or a horizontal offset
//    from o beyond R = floor(max_range * S). og_ray is called with the height band set to the whole line, so it never clips
//    and decides nothing but the skip. Skipped points are counted (n_skipped), the others are n_points.
//  * Cell statistics. Point (X, Y, Z) lies in cell (X >> 16, Y >> 16), the occupancy grid's lattice. Each cell keeps n, the
//    number of its points (uint32), lo, their minimum Z, and top, the maximum Z among its points with Z <= lo + C, where
//    C = floor(clearance * S). Points with Z > lo + C are overhangs (canopy, a bridge deck, a ceiling): they count in
//    n_overhang and in n, and change nothing else. A cell is OBSERVED when n >= min_points; its surface height is h = top.
//    Every statistic is an integer min, max or count, so the grid does not depend on the order of points, submaps or
//    blocks. An empty cell reads lo = EL_LO_EMPTY and top = EL_TOP_EMPTY (byte-filled 0x7f.. and 0x80..).
//  * Bounds. The extent of heights, max Z - min Z over every non-skipped point, must be below 2^40 (checked once after the
//    statistics pass; 2^24 cells of height). With window_cells r <= 8 a window has m <= 289 cells, |u|, |v| <= 8 and
//    heights relative to the centre |z| < 2^40, so every moment sum is an exact int64 below 2^53 (|Σ u z| < 289 * 8 * 2^40
//    < 2^52), the centred products P, Q below 2^61 and D below 2^42.
//  * Window. For an observed cell c, the window is the observed cells (i, j) with |i - ic| <= r, |j - jc| <= r (c included;
//    cells beyond the grid are not observed); m is their number. u = i - ic, v = j - jc, z = h - h_c. Over the window:
//      step = max h - min h (exact);
//      sums Su, Sv, Suu, Suv, Svv, Sz, Suz, Svz (int64);
//      A = m Suu - Su^2, B = m Suv - Su Sv, Cc = m Svv - Sv^2, D = A Cc - B^2 (= m * det of the normal equations), and
//      P = m Suz - Su Sz, Q = m Svz - Sv Sz (int64, exact);
//      the least-squares plane z ~ a u + b v + d in double, each operation rounded once, in this order:
//      a = (P*Cc - Q*B) / D, b = (Q*A - P*B) / D, d = ((Sz - a*Su) - b*Sv) / m (integers converted to double first);
//      s2 = a*a + b*b; tan_slope = sqrt(s2) / 2^16 (height units per cell over 2^16 units per cell);
//      residuals in row-major window order (v, then u, ascending): e = z - ((a*u + b*v) + d), sum = sum + e*e from 0;
//      roughness = sqrt(sum / m) / S (metres).
//  * Unknown. Value -1 when c is not observed, m < min_cells, or D == 0 (a degenerate plane: the observed cells are
//    collinear; exact, since D is an integer). The float layers of an unknown cell are NaN (0x7fc00000).
//  * Value. 100 (lethal) when step > K = floor(max_step * S), s2 > G2 = G*G with G = tan(max_slope) * 2^16 (host double), or
//    roughness > max_roughness. Otherwise floor(99 x + 0.5), at most 99, where x is the largest of step / K,
//    sqrt(s2) / G and roughness / max_roughness (each a double division). The float layers are step / S, tan_slope and roughness, each rounded once to float from those doubles.
//  * Extent. The grid is axis-aligned in the map frame: the bounding box of the cells of every non-skipped point; a build
//    with none is refused. origin = ((double)i0 * resolution, (double)j0 * resolution). More than 2^28 cells is refused
//    before the grid is allocated (the extent is measured on the device first, by occupancy's K14a). The session keeps
//    EL_BYTES_PER_CELL = 34 bytes per cell: n (4), lo and top (8 + 8), step, tan_slope, roughness (4 each), value and image
//    byte (1 + 1).
//  * Image and files: og_pixel with rint(occupied_thresh * 100) and rint(free_thresh * 100), rows from the top, and
//    occupancy's PGM and YAML text, so nav2 reads the pair as a trinary map of where the robot may drive.
#pragma once
#include "occupancy_grid.hpp"

namespace b200 {

constexpr long long EL_HEIGHT_EXTENT = 1LL << 40;
constexpr int EL_MAX_WINDOW = 8;
constexpr long long EL_LO_EMPTY = 0x7f7f7f7f7f7f7f7fLL;                  // above every Z (|Z| < 2^52)
constexpr long long EL_TOP_EMPTY = (long long)0x8080808080808080ULL;     // below every Z
constexpr long long EL_NONE = EL_TOP_EMPTY;                             // a window cell that is not observed
constexpr unsigned EL_NAN_BITS = 0x7fc00000u;
constexpr int EL_BYTES_PER_CELL = 34;

struct ElParams {
  double resolution = 0.1;
  double max_range = 100.0;
  double sensor_origin[3] = {0.0, 0.0, 0.0};
  double clearance = 2.0;
  int min_points = 2;
  int window_cells = 3;
  int min_cells = 6;
  double max_slope = 20.0;  // degrees
  double max_step = 0.15;
  double max_roughness = 0.05;
  double occupied_thresh = 0.65, free_thresh = 0.25;
};

// What a build computes from the parameters once, on the host.
struct ElConst {
  OgConst og;             // S, R; the band the whole line
  long long C;            // floor(clearance * S)
  long long K;            // floor(max_step * S)
  double G, G2;           // tan(max_slope) * 2^16, G * G
  double max_roughness;
  int r, min_points, min_cells;
};

OG_HD double el_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
OG_HD double el_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
OG_HD double el_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
OG_HD double el_sqrt(double a) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}
OG_HD float el_nan() {
#ifdef __CUDA_ARCH__
  return __int_as_float((int)EL_NAN_BITS);
#else
  float f;
  const unsigned b = EL_NAN_BITS;
  std::memcpy(&f, &b, sizeof(f));
  return f;
#endif
}

// One point of a submap whose origin is (xo, yo): false when it is skipped, else its cell and fixed-point height.
OG_HD bool el_point(const ElConst& c, long long xo, long long yo, const float* e, int* cx, int* cy, long long* Z) {
  OgSeg s;
  if (og_ray(c.og, xo, yo, 0, e[0], e[1], e[2], cx, cy, &s) < 0) return false;
  og_fixed(e[2], c.og.S, OG_COORD_LIMIT, Z);  // in range: og_ray checked it
  return true;
}

// The layers of one cell. h(u, v) is the surface height of the cell at offset (u, v), EL_NONE when that cell is not
// observed or lies beyond the grid. Returns the value (-1, 0..99 or 100).
template <class Height>
OG_HD int el_window(const ElConst& c, Height&& h, float* step_m, float* tan_slope, float* roughness) {
  *step_m = *tan_slope = *roughness = el_nan();
  const long long hc = h(0, 0);
  if (hc == EL_NONE) return -1;
  const int r = c.r;
  long long m = 0, su = 0, sv = 0, suu = 0, suv = 0, svv = 0, sz = 0, suz = 0, svz = 0, zmin = hc, zmax = hc;
  for (int v = -r; v <= r; v++)
    for (int u = -r; u <= r; u++) {
      const long long hz = h(u, v);
      if (hz == EL_NONE) continue;
      const long long z = hz - hc;
      m++;
      su += u;
      sv += v;
      suu += u * u;
      suv += u * v;
      svv += v * v;
      sz += z;
      suz += u * z;
      svz += v * z;
      zmin = hz < zmin ? hz : zmin;
      zmax = hz > zmax ? hz : zmax;
    }
  if (m < c.min_cells) return -1;
  const long long A = m * suu - su * su, B = m * suv - su * sv, Cc = m * svv - sv * sv;
  const long long D = A * Cc - B * B;
  if (D == 0) return -1;
  const long long P = m * suz - su * sz, Q = m * svz - sv * sz;
  const double dP = (double)P, dQ = (double)Q, dA = (double)A, dB = (double)B, dC = (double)Cc, dD = (double)D;
  const double a = el_div(el_sub(og_mul(dP, dC), og_mul(dQ, dB)), dD);
  const double b = el_div(el_sub(og_mul(dQ, dA), og_mul(dP, dB)), dD);
  const double d = el_div(el_sub(el_sub((double)sz, og_mul(a, (double)su)), og_mul(b, (double)sv)), (double)m);
  const double s2 = el_add(og_mul(a, a), og_mul(b, b));
  double sum = 0.0;
  for (int v = -r; v <= r; v++)
    for (int u = -r; u <= r; u++) {
      const long long hz = h(u, v);
      if (hz == EL_NONE) continue;
      const double e = el_sub((double)(hz - hc), el_add(el_add(og_mul(a, (double)u), og_mul(b, (double)v)), d));
      sum = el_add(sum, og_mul(e, e));
    }
  const double rough = el_div(el_sqrt(el_div(sum, (double)m)), c.og.S);
  const long long step = zmax - zmin;
  const double root = el_sqrt(s2);
  *step_m = (float)el_div((double)step, c.og.S);
  *tan_slope = (float)el_div(root, 65536.0);
  *roughness = (float)rough;
  if (step > c.K || s2 > c.G2 || rough > c.max_roughness) return 100;
  double x = el_div((double)step, (double)c.K);
  const double xs = el_div(root, c.G), xr = el_div(rough, c.max_roughness);
  if (xs > x) x = xs;
  if (xr > x) x = xr;
  const int value = (int)floor(el_add(og_mul(99.0, x), 0.5));
  return value < 99 ? value : 99;
}

// ---- host side: parameters and origins ----

// nullptr when p is valid (and *c filled), else the reason
inline const char* el_prepare(const ElParams& p, ElConst* c) {
  if (!std::isfinite(p.resolution) || !(p.resolution > 0)) return "resolution must be finite and > 0";
  const double S = 65536.0 / p.resolution;
  if (!std::isfinite(S)) return "resolution too small";
  if (!std::isfinite(p.max_range) || !(p.max_range > 0)) return "max_range must be finite and > 0";
  const double Rd = p.max_range * S;
  if (!(Rd <= (double)OG_RANGE_LIMIT)) return "max_range / resolution must be <= 2^14";
  for (int k = 0; k < 3; k++)
    if (!std::isfinite(p.sensor_origin[k])) return "sensor_origin must be finite";
  long long C, K;
  if (!(p.clearance >= 0) || !og_fixed(p.clearance, S, OG_COORD_LIMIT, &C)) return "clearance must be >= 0 and below 2^36 cells";
  if (p.min_points < 1) return "min_points must be >= 1";
  if (p.window_cells < 1 || p.window_cells > EL_MAX_WINDOW) return "window_cells must be in 1..8";
  const int side = 2 * p.window_cells + 1;
  if (p.min_cells < 3 || p.min_cells > side * side) return "min_cells must be in 3..(2 window_cells + 1)^2";
  if (!(p.max_slope > 0 && p.max_slope < 90)) return "max_slope must be in (0, 90) degrees";
  if (!(p.max_step > 0) || !og_fixed(p.max_step, S, OG_COORD_LIMIT, &K) || K < 1)
    return "max_step must be finite, at least one fixed-point unit and below 2^36 cells";
  if (!std::isfinite(p.max_roughness) || !(p.max_roughness > 0)) return "max_roughness must be finite and > 0";
  if (!(p.free_thresh >= 0 && p.free_thresh < p.occupied_thresh && p.occupied_thresh <= 1))
    return "thresholds must satisfy 0 <= free_thresh < occupied_thresh <= 1";
  c->og.S = S;
  c->og.R = (long long)std::floor(Rd);
  c->og.zlo = -(1LL << 62);
  c->og.zhi = 1LL << 62;
  c->og.occ_value = (int)std::rint(p.occupied_thresh * 100.0);
  c->og.free_value = (int)std::rint(p.free_thresh * 100.0);
  c->C = C;
  c->K = K;
  c->G = std::tan(p.max_slope * (3.14159265358979323846 / 180.0)) * 65536.0;
  c->G2 = c->G * c->G;
  if (!(c->G > 0)) return "max_slope must be in (0, 90) degrees";
  c->max_roughness = p.max_roughness;
  c->r = p.window_cells;
  c->min_points = p.min_points;
  c->min_cells = p.min_cells;
  return nullptr;
}

// The horizontal origin of a submap's points in fixed point; false when it is out of range
inline bool el_origin(const ElConst& c, const ElParams& p, const float* T, long long* xo, long long* yo) {
  float of[3];
  og_transform(T, (float)p.sensor_origin[0], (float)p.sensor_origin[1], (float)p.sensor_origin[2], of);
  return og_fixed(of[0], c.og.S, OG_ORIGIN_LIMIT, xo) && og_fixed(of[1], c.og.S, OG_ORIGIN_LIMIT, yo);
}

}  // namespace b200
