// The 2D occupancy grid of the session's map (b200sm_build_occupancy_grid): free space ray-cast from each submap's sensor
// origin to its points, hits and frees counted per submap, classified as nav2's map_server reads a trinary map. The kernels
// (occupancy.cu) and a host compile (tests/hostmath/occupancy_host.cpp, g++ -ffp-contract=off) both use the functions below,
// so every decision — which point is skipped, which cells a ray frees, which cell it hits — is the same on either side. The
// only floating-point steps are the float transform of a point (transform_point's order, one rounding per operation) and one
// rounded double multiply per coordinate into fixed point; everything after that is integer arithmetic.
//
// Definitions (this text is the contract; tests/occupancyref.py replays it in Python integers):
//  * Fixed point. S = 2^16 / resolution (one double division on the host). A map-frame coordinate v becomes
//    V = floor((double)v * S), the product rounded once. A coordinate whose product is not inside (-2^52, 2^52) — a
//    non-finite one included — is out of range. The cell of V is V >> 16 (an arithmetic shift: floor, not truncation, for
//    negative V). Cell (i, j) covers map x in [i, i + 1) * resolution as far as the rounded S allows.
//  * Rays. Submap k's float pose T (the double pose cast entry by entry) moves every point p of its cloud to
//    e = transform_point(T, p), bitwise the point b200sm_assemble_map returns. The ray's origin is o = transform_point(T,
//    (float)sensor_origin). A point is skipped (neither hit nor free) when a coordinate of e is out of range or when its
//    horizontal offset dx = Xe - Xo, dy = Ye - Yo exceeds R = floor(max_range * S): |dx| > R, |dy| > R or
//    dx^2 + dy^2 > R^2. Every other point is a ray (counted in n_rays; the skipped ones in n_skipped).
//  * Bounds that keep every product inside int64: R <= 2^30 (max_range / resolution <= 2^14, checked with the parameters);
//    every origin's X, Y, Z inside (-2^46, 2^46), and |Zlo - Zo|, |Zhi - Zo| <= 2^32 (checked per call, before anything
//    runs: a sensor origin farther than 2^16 cells from the band is refused). Then |dx|, |dy| <= 2^30, the clip's products
//    dx * (Zb - Zo) are below 2^62 in magnitude, the walk's cross products below 2^60, and every cell index fits an int32.
//  * Height band. Zlo = floor(z_min * S), Zhi = floor(z_max * S). An endpoint is in the band when Zlo <= Ze <= Zhi. The 3D
//    segment o -> e is clipped to the band: with dz = Ze - Zo, the part with Zlo <= Zo + t dz <= Zhi, t in [0, 1]. A
//    boundary crossed at t = n / dz (n = Zb - Zo) moves the segment's end there, at X = Xo + floor(dx * n / dz) (exact
//    floor division of the integer product), Y likewise; an end inside the band stays where it is. A segment that never
//    enters the band (dz == 0 with Zo outside it, or both ends beyond the same side) frees nothing. The origin may be above
//    or below the band.
//  * Traversal. The free cells of a ray are the cells of a 4-connected walk of the clipped 2D segment A -> B, both end
//    cells included: from cell(A), nx = |cell(Bx) - cell(Ax)| steps in x and ny in y. While both remain, the next step is
//    the axis whose next cell boundary the segment reaches first (Amanatides & Woo), compared as Dx * |uy| against
//    Dy * |ux| in int64, where u = B - A and Dx is the distance from A to that boundary ((i + 1) * 2^16 - Xa moving up,
//    Xa - i * 2^16 moving down, i the current cell). TIE RULE: at an exact corner (equal products) the walk steps in x
//    first, then y. When one axis has no step left, the other takes the rest. No walk leaves the box of its two end cells.
//  * Per-submap update (OctoMap's computeUpdate): within one submap, a cell is HIT when at least one in-band endpoint lies
//    in it, and FREE when at least one clipped segment's walk crosses it and it is not hit in that submap. A cell's `hits`
//    counts the submaps that hit it and `frees` those that freed it (uint32). Both are counts of per-submap booleans, so
//    the grid does not depend on the order of points, submaps or batches.
//  * Value. -1 when hits + frees == 0, else (200 hits + n) / (2 n) with n = hits + frees in integer division: 100 hits / n
//    rounded half up, 0..100 as in nav_msgs/OccupancyGrid. Counts, not clamped log-odds: a clamped sum depends on the order
//    of its updates.
//  * Extent. The grid is axis-aligned in the map frame: the bounding box of the cells of every origin and every ray's
//    endpoint (in band or not). A walk stays in the box of its end cells, so no walk leaves the grid. origin = ((double)i0 *
//    resolution, (double)j0 * resolution), the lower-left corner of cell (0, 0) as map_server's YAML means it; data are
//    row-major from that corner (OccupancyGrid.data). More than 2^28 cells is refused before the grid is allocated:
//    the extent is measured on the device, so the only allocations before the check are the bounds pass's own
//    per-submap table and bounds (144 bytes per submap) and its counters.
//  * Trinary image, as nav2's map_saver writes one from an OccupancyGrid (restated here from nav2's documented behaviour;
//    this text is the contract): value >= rint(occupied_thresh * 100) -> 0; else value >= 0 and value <=
//    rint(free_thresh * 100) -> 254; otherwise (value -1 included) -> 205. Rows run from the top (largest y) down.
//  * Files. PGM: "P5", one comment line, "width height", "255", each followed by '\n', then the bytes. YAML: image (the
//    PGM's basename as a double-quoted scalar: '\\' and '"' escaped, control bytes as \xHH, so that a name with ": ",
//    '#' or a leading indicator reads back as itself), mode: trinary, resolution, origin: [x, y, 0], negate: 0,
//    occupied_thresh, free_thresh, every number printed with the fewest significant digits (at most 17) that read back to
//    the same double.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#ifdef __CUDACC__
#define OG_HD __host__ __device__ __forceinline__
#else
#define OG_HD inline
#endif

namespace b200 {

constexpr int OG_FRAC_BITS = 16;
constexpr long long OG_ONE = 1LL << OG_FRAC_BITS;
constexpr double OG_COORD_LIMIT = 4503599627370496.0;  // 2^52: |v * S| of an endpoint coordinate
constexpr double OG_ORIGIN_LIMIT = 70368744177664.0;   // 2^46: |v * S| of an origin coordinate and of the band
constexpr long long OG_RANGE_LIMIT = 1LL << 30;        // R
constexpr long long OG_BAND_REACH = 1LL << 32;         // |Zlo - Zo|, |Zhi - Zo|
constexpr unsigned long long OG_MAX_CELLS = 1ull << 28;

struct OgParams {
  double resolution = 0.05;
  double z_min = 0.2, z_max = 2.0;
  double max_range = 100.0;
  double sensor_origin[3] = {0.0, 0.0, 0.0};
  double occupied_thresh = 0.65, free_thresh = 0.25;
};

// What a build computes from the parameters once, on the host.
struct OgConst {
  double S;            // 2^16 / resolution
  long long R;         // floor(max_range * S)
  long long zlo, zhi;  // floor(z_min * S), floor(z_max * S)
  int occ_value, free_value;  // rint(occupied_thresh * 100), rint(free_thresh * 100)
};

// The clipped 2D segment of a ray, fixed point.
struct OgSeg {
  long long xa, ya, xb, yb;
};

OG_HD double og_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
OG_HD float og_fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
OG_HD float og_fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// transform_point of common.cuh: ((T0 x + T1 y) + T2 z) + T3 per row, T 3x4 row-major float
OG_HD void og_transform(const float* T, float x, float y, float z, float* o) {
  o[0] = og_fadd(og_fadd(og_fadd(og_fmul(T[0], x), og_fmul(T[1], y)), og_fmul(T[2], z)), T[3]);
  o[1] = og_fadd(og_fadd(og_fadd(og_fmul(T[4], x), og_fmul(T[5], y)), og_fmul(T[6], z)), T[7]);
  o[2] = og_fadd(og_fadd(og_fadd(og_fmul(T[8], x), og_fmul(T[9], y)), og_fmul(T[10], z)), T[11]);
}

// V = floor(v * S) when |v * S| < limit (false for a product outside it, NaN and infinities included)
OG_HD bool og_fixed(double v, double S, double limit, long long* V) {
  const double p = og_mul(v, S);
  if (!(p > -limit && p < limit)) return false;
  *V = (long long)floor(p);
  return true;
}

OG_HD int og_cell(long long V) { return (int)(V >> OG_FRAC_BITS); }  // arithmetic shift: floor(V / 2^16)

// floor(a / b) for b != 0
OG_HD long long og_floor_div(long long a, long long b) {
  long long q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) q -= 1;
  return q;
}

// One point of a submap whose origin is (xo, yo, zo) (fixed point). Returns -1 when the point is skipped; otherwise a
// bitmask: 1 = the endpoint is in the band (it hits cell (*hx, *hy)), 2 = the segment enters the band (*seg is its clipped
// 2D part). (*hx, *hy) is the endpoint's cell either way: it bounds the grid.
OG_HD int og_ray(const OgConst& c, long long xo, long long yo, long long zo, float ex, float ey, float ez, int* hx, int* hy,
                 OgSeg* seg) {
  long long xe, ye, ze;
  if (!og_fixed(ex, c.S, OG_COORD_LIMIT, &xe) || !og_fixed(ey, c.S, OG_COORD_LIMIT, &ye) || !og_fixed(ez, c.S, OG_COORD_LIMIT, &ze))
    return -1;
  const long long dx = xe - xo, dy = ye - yo;
  if (dx > c.R || dx < -c.R || dy > c.R || dy < -c.R || dx * dx + dy * dy > c.R * c.R) return -1;
  *hx = og_cell(xe);
  *hy = og_cell(ye);
  int flags = (ze >= c.zlo && ze <= c.zhi) ? 1 : 0;
  const long long dz = ze - zo;
  long long na = 0, nb = 0;  // numerators of the clip parameters over dz
  bool clip_a = false, clip_b = false;
  if (dz == 0) {
    if (zo < c.zlo || zo > c.zhi) return flags;
  } else if (dz > 0) {
    if (zo > c.zhi || ze < c.zlo) return flags;
    if (zo < c.zlo) { clip_a = true; na = c.zlo - zo; }
    if (ze > c.zhi) { clip_b = true; nb = c.zhi - zo; }
  } else {
    if (zo < c.zlo || ze > c.zhi) return flags;
    if (zo > c.zhi) { clip_a = true; na = c.zhi - zo; }
    if (ze < c.zlo) { clip_b = true; nb = c.zlo - zo; }
  }
  seg->xa = clip_a ? xo + og_floor_div(dx * na, dz) : xo;
  seg->ya = clip_a ? yo + og_floor_div(dy * na, dz) : yo;
  seg->xb = clip_b ? xo + og_floor_div(dx * nb, dz) : xe;
  seg->yb = clip_b ? yo + og_floor_div(dy * nb, dz) : ye;
  return flags | 2;
}

// The 4-connected walk of a clipped segment: visit(cx, cy) for every cell, cell(A) first and cell(B) last.
template <class Visit>
OG_HD void og_walk(const OgSeg& s, Visit&& visit) {
  int cx = og_cell(s.xa), cy = og_cell(s.ya);
  const int ex = og_cell(s.xb), ey = og_cell(s.yb);
  const long long ux = s.xb - s.xa, uy = s.yb - s.ya;
  const long long ax = ux < 0 ? -ux : ux, ay = uy < 0 ? -uy : uy;
  const int sx = ex > cx ? 1 : -1, sy = ey > cy ? 1 : -1;
  int nx = ex > cx ? ex - cx : cx - ex, ny = ey > cy ? ey - cy : cy - ey;
  visit(cx, cy);
  while (nx + ny > 0) {
    bool step_x;
    if (nx == 0) {
      step_x = false;
    } else if (ny == 0) {
      step_x = true;
    } else {
      const long long bx = sx > 0 ? (long long)(cx + 1) * OG_ONE - s.xa : s.xa - (long long)cx * OG_ONE;
      const long long by = sy > 0 ? (long long)(cy + 1) * OG_ONE - s.ya : s.ya - (long long)cy * OG_ONE;
      step_x = bx * ay <= by * ax;  // the tie (an exact corner) steps x first
    }
    if (step_x) {
      cx += sx;
      nx--;
    } else {
      cy += sy;
      ny--;
    }
    visit(cx, cy);
  }
}

OG_HD int og_value(unsigned hits, unsigned frees) {
  const unsigned long long n = (unsigned long long)hits + frees;
  if (n == 0) return -1;
  return (int)((200ull * hits + n) / (2ull * n));
}

OG_HD unsigned char og_pixel(int value, int occ_value, int free_value) {
  if (value < 0) return 205;
  if (value >= occ_value) return 0;
  if (value <= free_value) return 254;
  return 205;
}

// ---- host side: parameters, origins, text ----

// nullptr when p is valid (and *c filled), else the reason
inline const char* og_prepare(const OgParams& p, OgConst* c) {
  if (!std::isfinite(p.resolution) || !(p.resolution > 0)) return "resolution must be finite and > 0";
  const double S = 65536.0 / p.resolution;
  if (!std::isfinite(S)) return "resolution too small";
  if (!std::isfinite(p.z_min) || !std::isfinite(p.z_max) || !(p.z_min < p.z_max)) return "z_min, z_max must be finite, z_min < z_max";
  if (!std::isfinite(p.max_range) || !(p.max_range > 0)) return "max_range must be finite and > 0";
  const double Rd = p.max_range * S;
  if (!(Rd <= (double)OG_RANGE_LIMIT)) return "max_range / resolution must be <= 2^14";
  for (int k = 0; k < 3; k++)
    if (!std::isfinite(p.sensor_origin[k])) return "sensor_origin must be finite";
  if (!(p.free_thresh >= 0 && p.free_thresh < p.occupied_thresh && p.occupied_thresh <= 1))
    return "thresholds must satisfy 0 <= free_thresh < occupied_thresh <= 1";
  long long zlo, zhi;
  if (!og_fixed(p.z_min, S, OG_ORIGIN_LIMIT, &zlo) || !og_fixed(p.z_max, S, OG_ORIGIN_LIMIT, &zhi))
    return "z_min / z_max beyond 2^30 cells";
  c->S = S;
  c->R = (long long)std::floor(Rd);
  c->zlo = zlo;
  c->zhi = zhi;
  c->occ_value = (int)std::rint(p.occupied_thresh * 100.0);
  c->free_value = (int)std::rint(p.free_thresh * 100.0);
  return nullptr;
}

// The float pose of a submap (3x4 row-major) from its double pose, column-major 4x4
inline void og_pose_f(const double* pose_colmajor16, float* T) {
  for (int r = 0; r < 3; r++)
    for (int col = 0; col < 4; col++) T[r * 4 + col] = (float)pose_colmajor16[col * 4 + r];
}

// The origin of a submap's rays in fixed point; false when it is out of range (see the bounds above)
inline bool og_origin(const OgConst& c, const OgParams& p, const float* T, long long* o) {
  float of[3];
  og_transform(T, (float)p.sensor_origin[0], (float)p.sensor_origin[1], (float)p.sensor_origin[2], of);
  for (int k = 0; k < 3; k++)
    if (!og_fixed(of[k], c.S, OG_ORIGIN_LIMIT, &o[k])) return false;
  return std::llabs(c.zlo - o[2]) <= OG_BAND_REACH && std::llabs(c.zhi - o[2]) <= OG_BAND_REACH;
}

// the fewest significant digits (at most 17) that read back to v; always with a '.' before an exponent, so that YAML 1.1
// readers take it as a float
inline std::string og_number(double v) {
  char buf[40];
  for (int prec = 1; prec <= 17; prec++) {
    std::snprintf(buf, sizeof(buf), "%.*g", prec, v);
    if (std::strtod(buf, nullptr) == v) break;
  }
  std::string s(buf);
  const size_t e = s.find('e');
  if (e != std::string::npos && s.find('.') == std::string::npos) s.insert(e, ".0");
  return s;
}

inline std::string og_pgm_header(unsigned width, unsigned height, double resolution) {
  return "P5\n# CREATOR: lidarslam_ros2_b200 occupancy grid " + og_number(resolution) + " m/pix\n" + std::to_string(width) + " " +
         std::to_string(height) + "\n255\n";
}

// a YAML double-quoted scalar of s: '\\' and '"' escaped, control bytes as \xHH, every other byte as it is — so that a name
// with ": ", '#' or a leading indicator character reads back as itself
inline std::string og_yaml_quote(const std::string& s) {
  std::string q = "\"";
  for (unsigned char ch : s) {
    if (ch == '\\' || ch == '"') {
      q += '\\';
      q += (char)ch;
    } else if (ch < 0x20 || ch == 0x7f) {
      char buf[8];
      std::snprintf(buf, sizeof(buf), "\\x%02X", ch);
      q += buf;
    } else {
      q += (char)ch;
    }
  }
  return q + "\"";
}

inline std::string og_yaml(const char* pgm_path, double resolution, const double* origin, double occupied_thresh, double free_thresh) {
  std::string image(pgm_path);
  const size_t slash = image.find_last_of('/');
  if (slash != std::string::npos) image = image.substr(slash + 1);
  return "image: " + og_yaml_quote(image) + "\nmode: trinary\nresolution: " + og_number(resolution) + "\norigin: [" + og_number(origin[0]) + ", " +
         og_number(origin[1]) + ", 0]\nnegate: 0\noccupied_thresh: " + og_number(occupied_thresh) +
         "\nfree_thresh: " + og_number(free_thresh) + "\n";
}

}  // namespace b200
