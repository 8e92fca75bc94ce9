// Relocalisation anywhere in the prior map (b200sm_relocalize): an exact branch-and-bound search over (x, y, yaw) of the
// frame's scan against a 2D projection of the map. The kernels (relocalize.cu, K17) and a host compile
// (tests/hostmath/relocalize_host.cpp, g++ -ffp-contract=off) both use the functions below, so every decision — which map
// row and which scan point is projected, which cell it lands in, which node survives — is the same on either side. The only
// floating-point steps are the float rotation of a scan point (transform_point's order, one rounding per operation), one
// rounded double add for its height and one rounded double multiply per coordinate into a cell; everything after that is
// integer arithmetic.
//
// Definitions (this text is the contract; tests/relocref.py replays it in Python integers and numpy float32):
//  * Level-0 grid. inv = 1.0 / resolution (one host division). A map row (x, y, z) is projected when it is finite,
//    z_min <= (double)z <= z_max, and floor((double)x * inv), floor((double)y * inv) lie within +-2^30: its cell is those two
//    floors. The grid is the bounding box of the projected cells: origin cell (i0, j0), W x H cells (W * H <= 2^28). A
//    cell's value g_0 is 1 if any projected row falls in it, else 0.
//  * Pyramid. g_h(i, j) = max(g_{h-1}(i, j), g_{h-1}(i + s, j), g_{h-1}(i, j + s), g_{h-1}(i + s, j + s)), s = 2^{h-1}, with
//    g_0 = 0 outside the grid: g_h(i, j) is the max of g_0 over [i, i + 2^h) x [j, j + 2^h). A window that starts left of or
//    below the grid can still reach into it, so level h is stored over i in [1 - 2^h, W), j in [1 - 2^h, H)
//    ((W + 2^h - 1) x (H + 2^h - 1) bytes); a read outside that range is 0 — its window misses the grid. Levels
//    0 .. num_levels - 1 are kept; all of them together at most 2^32 bytes.
//  * Hypotheses. Heading k = 0 .. yaw_steps - 1 rotates by R_k = (float)(Rz(2 pi k / yaw_steps) * R0) (global_yaw_rotations;
//    R0 the current pose's rotation). Leaf (k, i, j), 0 <= i < W, 0 <= j < H, has translation ((double)(i0 + i) * resolution,
//    (double)(j0 + j) * resolution, z0), the lower corner of the cell, z0 the current z. Its index is (k * H + j) * W + i.
//  * Discretised scan. A point p of the filtered scan is projected when z_min <= (double)(R_k p).z + z0 <= z_max (the third
//    row of R_k is R0's for every k, so the set does not depend on k; a non-finite point never is). Its offsets are
//    dx = floor((double)(R_k p).x * inv), dy likewise, clamped to +-2^30 (a clamped offset reads outside every window, as
//    the unclamped one would). m is the number of projected points; m < 2^24 and yaw_steps * m <= 2^26.
//  * Score. score_h(k, i, j) = sum over the projected points of g_h(i + dx, j + dy): each point counts, duplicates
//    included. score_0 is a leaf's score; score_h bounds every leaf of the node's 2^h x 2^h window from above.
//  * Tiles and the answer. L = num_levels, S = 2^{L-1}. Tile (a, b) is the window [a S, (a + 1) S) x [b S, (b + 1) S) over
//    every heading; TW = ceil(W / S), TH = ceil(H / S), tile index b * TW + a. A tile's best leaf has the highest score, the
//    lowest leaf index on a tie: the highest key (score << 40) | (2^40 - 1 - leaf index). The answer is the first top_k
//    tiles ranked by that key among those whose best scores >= T0 = max(1, ceil(min_score * m)).
//  * Pruned search (rl_search_serial; the device runs the same steps). (1) Every root (k, a S, b S), in the order
//    r = (k * TH + b) * TW + a, is scored at level L - 1; each tile keeps its best root key. (2) Dive: the top_k tiles by
//    that key; from each, descend to the child with the highest key at each level. (3) T = max(T0, the top_k-th largest dive
//    leaf score), or T0 with fewer than top_k dives. (4) Level by level, only nodes with score >= T are expanded into their
//    children (child (di, dj), dj outer, di inner, kept when its corner is inside the grid). The children's count is checked
//    against RL_MAX_FRONTIER before they are written. (5) Every leaf with score >= T folds into its tile's key with a max.
//    Every tile ranked within top_k has its best >= T, and all of its leaves >= T are reached, so the answer is exact.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#ifdef __CUDACC__
#define RL_HD __host__ __device__ __forceinline__
#else
#define RL_HD inline
#endif

namespace b200 {

constexpr int RL_MAX_YAW_STEPS = 4096, RL_MAX_LEVELS = 16, RL_MAX_TOP_K = 64;
constexpr long long RL_COORD_LIMIT = 1LL << 30;                  // |cell| of a map row, |offset| of a scan point
constexpr unsigned long long RL_MAX_CELLS = 1ull << 28;          // W * H
constexpr unsigned long long RL_MAX_PYRAMID_BYTES = 1ull << 32;  // every level
constexpr unsigned long long RL_MAX_LEAVES = 1ull << 40;         // yaw_steps * W * H is below it
constexpr unsigned long long RL_MAX_ROOTS = 1ull << 32;
constexpr unsigned long long RL_MAX_OFFSETS = 1ull << 26;        // yaw_steps * m: the offsets table, 8 bytes each
constexpr long long RL_MAX_POINTS = (1LL << 24) - 1;             // m: a score fits the key's 24 upper bits
constexpr unsigned long long RL_MAX_FRONTIER = 1ull << 26;       // stored nodes of one level, 12 bytes each
constexpr unsigned long long RL_INDEX_MASK = (1ull << 40) - 1;

struct RlParams {
  double resolution = 0.25;
  double z_min = 0.3, z_max = 3.0;
  int yaw_steps = 360, num_levels = 6;
  double min_score = 0.3;
  int top_k = 4;
  double accept_fitness = 1.0;
};

inline bool rl_params_valid(const RlParams& p) {
  return std::isfinite(p.resolution) && p.resolution > 0 && std::isfinite(1.0 / p.resolution) && std::isfinite(p.z_min) &&
         std::isfinite(p.z_max) && p.z_min < p.z_max && p.yaw_steps >= 1 && p.yaw_steps <= RL_MAX_YAW_STEPS &&
         p.num_levels >= 1 && p.num_levels <= RL_MAX_LEVELS && p.min_score >= 0 && p.min_score <= 1 && p.top_k >= 1 &&
         p.top_k <= RL_MAX_TOP_K && std::isfinite(p.accept_fitness) && p.accept_fitness > 0;
}

struct RlOff {  // one point's offsets under one heading (the layout of int2)
  int dx, dy;
};
struct RlNode {
  int k, i, j;
};

// The grid and its tiling
struct RlGrid {
  int i0 = 0, j0 = 0;
  long long W = 0, H = 0;
  int levels = 1, yaw_steps = 1;
  long long S = 1, TW = 0, TH = 0;
};

RL_HD double rl_dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
RL_HD double rl_dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
RL_HD float rl_fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
RL_HD float rl_fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
RL_HD bool rl_finite(float v) {
#ifdef __CUDA_ARCH__
  return isfinite(v);
#else
  return std::isfinite(v);
#endif
}

// A map row's cell; false when the row is not projected.
RL_HD bool rl_project_row(float x, float y, float z, double inv, double z_min, double z_max, int* ci, int* cj) {
  if (!rl_finite(x) || !rl_finite(y) || !rl_finite(z)) return false;
  const double zd = (double)z;
  if (!(z_min <= zd && zd <= z_max)) return false;
  const double fx = floor(rl_dmul((double)x, inv)), fy = floor(rl_dmul((double)y, inv));
  const double lim = (double)RL_COORD_LIMIT;
  if (!(fx >= -lim && fx <= lim && fy >= -lim && fy <= lim)) return false;
  *ci = (int)fx;
  *cj = (int)fy;
  return true;
}

// R p (R row-major 3x3 float) in transform_point's order without the translation: one rounding per operation
RL_HD float rl_rot_row(const float* R, int r, float x, float y, float z) {
  return rl_fadd(rl_fadd(rl_fmul(R[3 * r], x), rl_fmul(R[3 * r + 1], y)), rl_fmul(R[3 * r + 2], z));
}
// Is the scan point projected? R is any heading's rotation (the third row is the same for all of them).
RL_HD bool rl_point_in_band(const float* R, float x, float y, float z, double z0, double z_min, double z_max) {
  const double h = rl_dadd((double)rl_rot_row(R, 2, x, y, z), z0);
  return z_min <= h && h <= z_max;
}
RL_HD int rl_offset(float q, double inv) {
  const double f = floor(rl_dmul((double)q, inv));
  const double lim = (double)RL_COORD_LIMIT;
  return !(f >= -lim) ? -(int)RL_COORD_LIMIT : (!(f <= lim) ? (int)RL_COORD_LIMIT : (int)f);
}
RL_HD RlOff rl_offsets(const float* R, float x, float y, float z, double inv) {
  RlOff o;
  o.dx = rl_offset(rl_rot_row(R, 0, x, y, z), inv);
  o.dy = rl_offset(rl_rot_row(R, 1, x, y, z), inv);
  return o;
}

// level h's storage: margin 2^h - 1 on the low sides
RL_HD long long rl_margin(int h) { return (1LL << h) - 1; }
RL_HD long long rl_level_w(const RlGrid& g, int h) { return g.W + rl_margin(h); }
RL_HD long long rl_level_h(const RlGrid& g, int h) { return g.H + rl_margin(h); }
// g_h(i, j) from level h's bytes; 0 outside the stored range
RL_HD int rl_read(const unsigned char* lvl, long long lw, long long lh, long long margin, long long i, long long j) {
  const long long c = i + margin, r = j + margin;
  return (c >= 0 && c < lw && r >= 0 && r < lh) ? (int)lvl[r * lw + c] : 0;
}
// g_h of stored cell (c, r) of level h from level h - 1 (`prev`)
RL_HD unsigned char rl_level_cell(const unsigned char* prev, const RlGrid& g, int h, long long c, long long r) {
  const long long s = 1LL << (h - 1), m = rl_margin(h), pm = rl_margin(h - 1);
  const long long pw = rl_level_w(g, h - 1), ph = rl_level_h(g, h - 1);
  const long long i = c - m, j = r - m;
  const int v = rl_read(prev, pw, ph, pm, i, j) | rl_read(prev, pw, ph, pm, i + s, j) | rl_read(prev, pw, ph, pm, i, j + s) |
                rl_read(prev, pw, ph, pm, i + s, j + s);  // max of 0 / 1 values
  return (unsigned char)v;
}

RL_HD long long rl_leaf_index(const RlGrid& g, int k, long long i, long long j) { return ((long long)k * g.H + j) * g.W + i; }
RL_HD unsigned long long rl_key(long long score, long long leaf_index) {
  return ((unsigned long long)score << 40) | (RL_INDEX_MASK - (unsigned long long)leaf_index);
}
RL_HD long long rl_key_score(unsigned long long key) { return (long long)(key >> 40); }
RL_HD long long rl_key_index(unsigned long long key) { return (long long)(RL_INDEX_MASK - (key & RL_INDEX_MASK)); }
RL_HD long long rl_tile_of(const RlGrid& g, long long i, long long j) { return (j / g.S) * g.TW + i / g.S; }
RL_HD RlNode rl_root(const RlGrid& g, unsigned long long r) {
  const unsigned long long per = (unsigned long long)g.TW * (unsigned long long)g.TH;
  const unsigned long long rem = r % per;
  RlNode n;
  n.k = (int)(r / per);
  n.i = (int)((long long)(rem % (unsigned long long)g.TW) * g.S);
  n.j = (int)((long long)(rem / (unsigned long long)g.TW) * g.S);
  return n;
}
// child c (0..3: di = c & 1, dj = c >> 1) of a level-h node; false when its corner is outside the grid
RL_HD bool rl_child(const RlGrid& g, RlNode n, int h, int c, RlNode* out) {
  const long long s = 1LL << (h - 1);
  const long long i = n.i + (c & 1) * s, j = n.j + (c >> 1) * s;
  if (i >= g.W || j >= g.H) return false;
  out->k = n.k;
  out->i = (int)i;
  out->j = (int)j;
  return true;
}
RL_HD int rl_child_count(const RlGrid& g, RlNode n, int h) {
  const long long s = 1LL << (h - 1);
  return (1 + (n.i + s < g.W)) * (1 + (n.j + s < g.H));
}

// ---- host: sizes, limits, rotations, guesses ---------------------------------------------------------------------------

// The grid of a bounding box of projected cells (min i, min j, max i, max j) and the limits of its pyramid: W * H cells
// and every level's bytes; "" when they fit, else why not. The limits that depend on the headings are rl_check_headings',
// checked by every search (a pyramid serves searches with any yaw_steps).
inline std::string rl_make_grid(long long mni, long long mnj, long long mxi, long long mxj, const RlParams& p, RlGrid* g,
                                unsigned long long* level_offsets /* num_levels + 1 */) {
  g->i0 = (int)mni;
  g->j0 = (int)mnj;
  g->W = mxi - mni + 1;
  g->H = mxj - mnj + 1;
  g->levels = p.num_levels;
  g->yaw_steps = p.yaw_steps;
  g->S = 1LL << (p.num_levels - 1);
  g->TW = (g->W + g->S - 1) / g->S;
  g->TH = (g->H + g->S - 1) / g->S;
  char msg[240];
  const unsigned long long cells = (unsigned long long)g->W * (unsigned long long)g->H;
  if (cells > RL_MAX_CELLS) {
    std::snprintf(msg, sizeof(msg), "the map's grid is %lld x %lld cells, more than 2^28", g->W, g->H);
    return msg;
  }
  unsigned long long off = 0;
  for (int h = 0; h < p.num_levels; h++) {
    level_offsets[h] = off;
    off += (unsigned long long)rl_level_w(*g, h) * (unsigned long long)rl_level_h(*g, h);
  }
  level_offsets[p.num_levels] = off;
  if (off > RL_MAX_PYRAMID_BYTES) {
    std::snprintf(msg, sizeof(msg), "the pyramid of %d levels over %lld x %lld cells is %llu bytes, more than 2^32", p.num_levels,
                  g->W, g->H, off);
    return msg;
  }
  return "";
}

// The limits of a search with yaw_steps headings over grid g: yaw_steps * W * H < 2^40 leaves and yaw_steps * TW * TH <=
// 2^32 roots; "" when they fit, else why not.
inline std::string rl_check_headings(const RlGrid& g, int yaw_steps) {
  char msg[200];
  const unsigned long long leaves = (unsigned long long)yaw_steps * (unsigned long long)g.W * (unsigned long long)g.H;
  if (leaves >= RL_MAX_LEAVES) {
    std::snprintf(msg, sizeof(msg), "yaw_steps * W * H = %llu leaves, 2^40 or more", leaves);
    return msg;
  }
  const unsigned long long roots = (unsigned long long)yaw_steps * (unsigned long long)g.TW * (unsigned long long)g.TH;
  if (roots > RL_MAX_ROOTS) {
    std::snprintf(msg, sizeof(msg), "%llu roots (yaw_steps * tiles), more than 2^32", roots);
    return msg;
  }
  return "";
}

// "" when m projected points fit the offsets table, else why not
inline std::string rl_check_points(long long m, int yaw_steps) {
  char msg[200];
  if (m > RL_MAX_POINTS || (unsigned long long)m * (unsigned long long)yaw_steps > RL_MAX_OFFSETS) {
    std::snprintf(msg, sizeof(msg), "%lld projected scan points x %d headings: more than 2^24 - 1 points or 2^26 offsets", m, yaw_steps);
    return msg;
  }
  return "";
}

inline long long rl_t0(double min_score, long long m) { return std::max(1LL, (long long)std::ceil(min_score * (double)m)); }

// R_k in double (row-major 3x3 each) for the pose (position, quaternion x y z w), and in float
inline void rl_rotations(const double* position, const double* quat, int yaw_steps, std::vector<double>& rot_d,
                         std::vector<float>& rot_f);

// The guess of leaf (k, i, j): R_k and the cell's lower corner at height z0, float, column-major
inline void rl_guess(const double* rot_k, const RlGrid& g, double resolution, double z0, long long i, long long j, float* col16) {
  for (int k = 0; k < 16; k++) col16[k] = 0.0f;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) col16[c * 4 + r] = (float)rot_k[r * 3 + c];
  col16[12] = (float)((double)((long long)g.i0 + i) * resolution);
  col16[13] = (float)((double)((long long)g.j0 + j) * resolution);
  col16[14] = (float)z0;
  col16[15] = 1.0f;
}

// The top_k tiles by key, descending, among those with a key (!= 0) whose score is >= min_score. Keys of distinct tiles
// differ (a key names a leaf, a leaf lies in one tile), so the order is strict. Only top_k indices are held.
inline std::vector<long long> rl_top_tiles(const std::vector<unsigned long long>& keys, long long min_score, int top_k) {
  std::vector<long long> t;
  const auto higher = [&](long long a, long long b) { return keys[(size_t)a] > keys[(size_t)b]; };
  for (size_t q = 0; q < keys.size(); q++) {
    if (keys[q] == 0 || rl_key_score(keys[q]) < min_score) continue;
    if ((int)t.size() == top_k && keys[q] <= keys[(size_t)t.back()]) continue;
    t.insert(std::upper_bound(t.begin(), t.end(), (long long)q, higher), (long long)q);
    if ((int)t.size() > top_k) t.pop_back();
  }
  return t;
}

// T from the dive leaves' scores
inline long long rl_threshold(std::vector<long long> dive_scores, long long t0, int top_k) {
  if ((int)dive_scores.size() < top_k) return t0;
  std::sort(dive_scores.begin(), dive_scores.end(), std::greater<long long>());
  return std::max(t0, dive_scores[(size_t)top_k - 1]);
}

}  // namespace b200

#include "global_grid.hpp"

namespace b200 {

inline void rl_rotations(const double* position, const double* quat, int yaw_steps, std::vector<double>& rot_d,
                         std::vector<float>& rot_f) {
  double M[16];
  pose_to_matrix_d(position, quat, M);
  global_yaw_rotations(M, yaw_steps, rot_d);
  rot_f.resize(rot_d.size());
  for (size_t q = 0; q < rot_d.size(); q++) rot_f[q] = (float)rot_d[q];
}

// ---- the whole search, serially (the host compile of the tests; the device runs the same steps) -------------------------

struct RlHostPyramid {
  RlGrid g;
  std::vector<unsigned long long> off;
  std::vector<unsigned char> bytes;
  const unsigned char* level(int h) const { return bytes.data() + off[(size_t)h]; }
};

struct RlHostResult {
  std::string error;  // a limit: nothing below is valid
  long long m = 0, t0 = 0, t = 0;
  long long nodes[RL_MAX_LEVELS] = {};
  std::vector<long long> tiles;              // the answer, ranked
  std::vector<unsigned long long> keys;      // their best leaf keys
};

// The pyramid of map rows (x, y, z, w); false (and `error`) when a limit is exceeded; an empty grid (W = H = 0) when no
// row is projected.
inline bool rl_build_pyramid_host(const float* map4, size_t n, const RlParams& p, RlHostPyramid& py, std::string& error) {
  const double inv = 1.0 / p.resolution;
  long long mni = 0, mnj = 0, mxi = -1, mxj = -1;
  bool any = false;
  for (size_t q = 0; q < n; q++) {
    int ci, cj;
    if (!rl_project_row(map4[4 * q], map4[4 * q + 1], map4[4 * q + 2], inv, p.z_min, p.z_max, &ci, &cj)) continue;
    if (!any) {
      mni = mxi = ci;
      mnj = mxj = cj;
      any = true;
    }
    mni = std::min<long long>(mni, ci);
    mxi = std::max<long long>(mxi, ci);
    mnj = std::min<long long>(mnj, cj);
    mxj = std::max<long long>(mxj, cj);
  }
  py.off.assign((size_t)p.num_levels + 1, 0);
  py.g = RlGrid();
  if (!any) return true;
  error = rl_make_grid(mni, mnj, mxi, mxj, p, &py.g, py.off.data());
  if (!error.empty()) return false;
  py.bytes.assign((size_t)py.off[(size_t)p.num_levels], 0);
  for (size_t q = 0; q < n; q++) {
    int ci, cj;
    if (!rl_project_row(map4[4 * q], map4[4 * q + 1], map4[4 * q + 2], inv, p.z_min, p.z_max, &ci, &cj)) continue;
    py.bytes[(size_t)((cj - py.g.j0) * py.g.W + (ci - py.g.i0))] = 1;
  }
  for (int h = 1; h < p.num_levels; h++) {
    unsigned char* out = py.bytes.data() + py.off[(size_t)h];
    const long long lw = rl_level_w(py.g, h), lh = rl_level_h(py.g, h);
    for (long long r = 0; r < lh; r++)
      for (long long c = 0; c < lw; c++) out[r * lw + c] = rl_level_cell(py.level(h - 1), py.g, h, c, r);
  }
  return true;
}

// The offsets table (yaw_steps x m, heading-major) of the scan points (x, y, z, w) under R_k (rot_f, 9 floats each)
inline void rl_offsets_host(const float* scan4, size_t n, const std::vector<float>& rot_f, int yaw_steps, double z0,
                            const RlParams& p, std::vector<RlOff>& offs, long long* m) {
  const double inv = 1.0 / p.resolution;
  std::vector<size_t> kept;
  for (size_t q = 0; q < n; q++)
    if (rl_point_in_band(rot_f.data(), scan4[4 * q], scan4[4 * q + 1], scan4[4 * q + 2], z0, p.z_min, p.z_max)) kept.push_back(q);
  *m = (long long)kept.size();
  offs.resize((size_t)yaw_steps * kept.size());
  for (int k = 0; k < yaw_steps; k++)
    for (size_t t = 0; t < kept.size(); t++) {
      const float* s = scan4 + 4 * kept[t];
      offs[(size_t)k * kept.size() + t] = rl_offsets(rot_f.data() + 9 * (size_t)k, s[0], s[1], s[2], inv);
    }
}

inline long long rl_score_host(const RlHostPyramid& py, const std::vector<RlOff>& offs, long long m, int h, RlNode n) {
  const long long lw = rl_level_w(py.g, h), lh = rl_level_h(py.g, h), mg = rl_margin(h);
  const RlOff* o = offs.data() + (size_t)n.k * (size_t)m;
  long long s = 0;
  for (long long t = 0; t < m; t++) s += rl_read(py.level(h), lw, lh, mg, (long long)n.i + o[t].dx, (long long)n.j + o[t].dy);
  return s;
}

// The pruned search (exhaustive = false) or the definition itself (every leaf scored).
inline void rl_search_serial(const RlHostPyramid& py, const std::vector<RlOff>& offs, long long m, const RlParams& p,
                             bool exhaustive, RlHostResult& res) {
  RlGrid g = py.g;
  g.yaw_steps = p.yaw_steps;
  if (g.W) {
    res.error = rl_check_headings(g, p.yaw_steps);
    if (!res.error.empty()) return;
  }
  const int L = g.levels;
  res.m = m;
  res.t0 = rl_t0(p.min_score, m);
  if (m == 0 || g.W == 0) return;
  const size_t n_tiles = (size_t)(g.TW * g.TH);
  std::vector<unsigned long long> leaf_keys(n_tiles, 0);
  if (exhaustive) {
    for (int k = 0; k < g.yaw_steps; k++)
      for (long long j = 0; j < g.H; j++)
        for (long long i = 0; i < g.W; i++) {
          const long long s = rl_score_host(py, offs, m, 0, RlNode{k, (int)i, (int)j});
          unsigned long long& t = leaf_keys[(size_t)rl_tile_of(g, i, j)];
          t = std::max(t, rl_key(s, rl_leaf_index(g, k, i, j)));
        }
    res.t = res.t0;
    res.nodes[0] = (long long)g.yaw_steps * g.W * g.H;
  } else {
    const unsigned long long roots = (unsigned long long)g.yaw_steps * n_tiles;
    res.nodes[L - 1] = (long long)roots;
    std::vector<unsigned long long> root_keys(n_tiles, 0);
    for (unsigned long long r = 0; r < roots; r++) {
      const RlNode n = rl_root(g, r);
      unsigned long long& t = root_keys[(size_t)rl_tile_of(g, n.i, n.j)];
      t = std::max(t, rl_key(rl_score_host(py, offs, m, L - 1, n), rl_leaf_index(g, n.k, n.i, n.j)));
    }
    std::vector<long long> dives;
    for (long long tile : rl_top_tiles(root_keys, 0, p.top_k)) {
      const long long idx = rl_key_index(root_keys[(size_t)tile]);
      RlNode n{(int)(idx / (g.W * g.H)), (int)(idx % g.W), (int)((idx / g.W) % g.H)};
      long long score = rl_key_score(root_keys[(size_t)tile]);
      for (int h = L - 1; h >= 1; h--) {
        unsigned long long best = 0;
        RlNode pick = n;
        for (int c = 0; c < 4; c++) {
          RlNode ch;
          if (!rl_child(g, n, h, c, &ch)) continue;
          const unsigned long long key = rl_key(rl_score_host(py, offs, m, h - 1, ch), rl_leaf_index(g, ch.k, ch.i, ch.j));
          if (key > best) {
            best = key;
            pick = ch;
          }
        }
        n = pick;
        score = rl_key_score(best);
      }
      dives.push_back(score);
    }
    res.t = rl_threshold(dives, res.t0, p.top_k);
    const long long T = res.t;
    if (L == 1) {
      for (size_t q = 0; q < n_tiles; q++)
        if (rl_key_score(root_keys[q]) >= T) leaf_keys[q] = root_keys[q];
    } else {
      std::vector<RlNode> front;
      unsigned long long count = 0;
      for (unsigned long long r = 0; r < roots; r++) {
        const RlNode n = rl_root(g, r);
        if (rl_score_host(py, offs, m, L - 1, n) >= T) count += (unsigned long long)rl_child_count(g, n, L - 1);
      }
      for (int h = L - 2; h >= 0; h--) {
        if (count > RL_MAX_FRONTIER) {
          char msg[160];
          std::snprintf(msg, sizeof(msg), "level %d would store %llu nodes, more than 2^26", h, count);
          res.error = msg;
          return;
        }
        std::vector<RlNode> next;
        if (h == L - 2) {
          for (unsigned long long r = 0; r < roots; r++) {
            const RlNode n = rl_root(g, r);
            if (rl_score_host(py, offs, m, L - 1, n) < T) continue;
            for (int c = 0; c < 4; c++) {
              RlNode ch;
              if (rl_child(g, n, L - 1, c, &ch)) next.push_back(ch);
            }
          }
        } else {
          for (const RlNode& n : front) {
            if (rl_score_host(py, offs, m, h + 1, n) < T) continue;
            for (int c = 0; c < 4; c++) {
              RlNode ch;
              if (rl_child(g, n, h + 1, c, &ch)) next.push_back(ch);
            }
          }
        }
        front.swap(next);
        res.nodes[h] = (long long)front.size();
        count = 0;
        if (h > 0) {
          for (const RlNode& n : front)
            if (rl_score_host(py, offs, m, h, n) >= T) count += (unsigned long long)rl_child_count(g, n, h);
        } else {
          for (const RlNode& n : front) {
            const long long s = rl_score_host(py, offs, m, 0, n);
            if (s < T) continue;
            unsigned long long& t = leaf_keys[(size_t)rl_tile_of(g, n.i, n.j)];
            t = std::max(t, rl_key(s, rl_leaf_index(g, n.k, n.i, n.j)));
          }
        }
      }
    }
  }
  res.tiles = rl_top_tiles(leaf_keys, res.t0, p.top_k);
  for (long long t : res.tiles) res.keys.push_back(leaf_keys[(size_t)t]);
}

}  // namespace b200
