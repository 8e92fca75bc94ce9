// The static map of the session (b200sm_build_static_map): the assembled map without the points of objects that moved
// while it was recorded. Every submap's points are rays from its sensor origin, cast through a 3D voxel grid; a voxel that
// some submaps' rays end in but that more submaps' rays pass through is dynamic, and the points ending in it are dropped.
// The kernels (static_map.cu) and a host compile (tests/hostmath/static_map_host.cpp, g++ -ffp-contract=off) both use
// the functions below and those of occupancy_grid.hpp, so every decision is the same on either side. The only
// floating-point steps are the float transform of a point and one rounded double multiply per coordinate into fixed point.
//
// Definitions (this text is the contract; tests/staticmapref.py replays it in Python integers):
//  * Fixed point, as the occupancy grid's: S = 2^16 / resolution, V = floor((double)v * S) (og_fixed), the voxel of V is
//    V >> 16 (og_cell). Voxel (i, j, k) covers map x in [i, i + 1) * resolution, y, z likewise.
//  * Rays. Submap k's float pose T (the double pose cast entry by entry, og_pose_f) moves each point p to
//    e = og_transform(T, p), bitwise the point b200sm_assemble_map returns. The ray's origin is O = the fixed point of
//    og_transform(T, (float)sensor_origin); an origin coordinate whose product is not inside (-2^46, 2^46) is refused
//    before anything runs. A point is SKIPPED (neither hit nor free, and never removed) when a coordinate of e is out of
//    range (its product not inside (-2^52, 2^52), non-finite included) or when d = E - O has |d_a| > R on some axis or
//    dx^2 + dy^2 + dz^2 > R^2, R = floor(max_range * S). Every other point is a RAY (n_rays; the others n_skipped).
//  * Bounds that keep every product inside int64: R <= 2^30 (max_range / resolution <= 2^14, checked with the parameters)
//    and |O_a| < 2^46. Then |d_a| <= 2^30, |d|^2 <= 3 * 2^60, |d_a * q| <= 2^46 and |u_a| <= |d_a| <= 2^30 (u = E' - O,
//    below). The walk only compares axes with a step left, and on such an axis the next boundary lies between O and E', so
//    0 <= B_a <= |u_a| and every cross product B_a |u_b| is at most 2^60. |E_a| < 2^46 + 2^30, so every voxel index a
//    ray touches (its endpoint's, and its walk's, which lie between voxel(O) and voxel(E')) is at most 2^30 + 2^14 in
//    magnitude: it fits an int32.
//  * Occupied voxels: the voxel of every ray's endpoint E. The BOX is their bounding box [x0, x1] x [y0, y1] x [z0, z1]
//    (no ray: an empty box, nothing is removed). A box of more than 2^31 - 1 cells is refused before anything is sized from
//    it. Cell (x, y, z) of the box has the linear index (z - z0) W H + (y - y0) W + (x - x0) (W, H, D its dimensions), and
//    the occupied voxels are numbered (their RANK) in ascending linear index.
//  * Freed part of a ray. q = rint(ray_fraction * 2^16) (0 < ray_fraction <= 1, q >= 1). The freed segment runs from O to
//    E' = O + ((d * q) >> 16), the shift arithmetic (a floor). Its voxels are a 6-connected 3D Amanatides-Woo walk from
//    voxel(O) to voxel(E'), both included: n_a = |voxel(E'_a) - voxel(O_a)| steps on axis a; while more than one axis has
//    steps left, the next step is the axis whose next voxel boundary the segment reaches first, compared by
//    cross-multiplication in int64 (axis a before b when B_a |u_b| <= B_b |u_a|, u = E' - O, B_a the distance from O to
//    that boundary: (c + 1) 2^16 - O_a moving up, O_a - c 2^16 moving down, c the current voxel). TIE RULE: x first, then
//    y, then z, at exact edges and corners. An axis with no step left takes none. A walk voxel outside the box or not
//    occupied is ignored.
//  * Per-submap update (OctoMap's computeUpdate): a voxel is HIT by submap k when an endpoint of k's rays lies in it, and
//    FREE for k when a walk of k crosses it and k does not hit it. `hits` and `frees` (uint32) count the submaps: counts
//    of per-submap booleans, so nothing depends on the order of points, submaps or batches.
//  * Classification. A voxel is DYNAMIC iff frees >= min_frees and og_value(hits, frees) (100 hits / (hits + frees)
//    rounded half up) <= rint(100 * dynamic_thresh).
//  * Static map: the assembled map in assembly order (submap by submap) minus every ray whose endpoint voxel is dynamic.
//    Skipped points, non-finite ones included, are kept; no other point is dropped.
#pragma once
#include "occupancy_grid.hpp"

namespace b200 {

constexpr unsigned long long SM_MAX_CELLS = 0x7fffffffull;  // 2^31 - 1: the int32 linear index of the box

struct SmParams {
  double resolution = 0.2;
  double max_range = 100.0;
  double sensor_origin[3] = {0.0, 0.0, 0.0};
  double ray_fraction = 0.85;
  unsigned min_frees = 2;
  double dynamic_thresh = 0.4;
};

// What a build computes from the parameters once, on the host.
struct SmConst {
  double S;       // 2^16 / resolution
  long long R;    // floor(max_range * S)
  long long q;    // rint(ray_fraction * 2^16), 1 .. 2^16
  unsigned min_frees;
  int dyn_value;  // rint(100 * dynamic_thresh)
};

// One point of a submap whose origin is o (fixed point). Returns false when the point is skipped; otherwise its endpoint
// voxel (*vx, *vy, *vz) and the end E' of its freed segment (*ex, *ey, *ez, fixed point).
OG_HD bool sm_ray(const SmConst& c, const long long* o, float px, float py, float pz, int* vx, int* vy, int* vz, long long* ex,
                  long long* ey, long long* ez) {
  long long X, Y, Z;
  if (!og_fixed(px, c.S, OG_COORD_LIMIT, &X) || !og_fixed(py, c.S, OG_COORD_LIMIT, &Y) || !og_fixed(pz, c.S, OG_COORD_LIMIT, &Z))
    return false;
  const long long R = c.R, q = c.q;
  const long long dx = X - o[0], dy = Y - o[1], dz = Z - o[2];
  if (dx > R || dx < -R || dy > R || dy < -R || dz > R || dz < -R || dx * dx + dy * dy + dz * dz > R * R) return false;
  *vx = og_cell(X);
  *vy = og_cell(Y);
  *vz = og_cell(Z);
  *ex = o[0] + ((dx * q) >> OG_FRAC_BITS);
  *ey = o[1] + ((dy * q) >> OG_FRAC_BITS);
  *ez = o[2] + ((dz * q) >> OG_FRAC_BITS);
  return true;
}

// The 6-connected walk from fixed point A to B: visit(x, y, z) for every voxel, voxel(A) first and voxel(B) last. (Scalars
// rather than per-axis arrays: an array indexed by the chosen axis would live in local memory on the device.)
template <class Visit>
OG_HD void sm_walk(long long xa, long long ya, long long za, long long xb, long long yb, long long zb, Visit&& visit) {
  int cx = og_cell(xa), cy = og_cell(ya), cz = og_cell(za);
  const int ex = og_cell(xb), ey = og_cell(yb), ez = og_cell(zb);
  const long long ux = xb < xa ? xa - xb : xb - xa, uy = yb < ya ? ya - yb : yb - ya, uz = zb < za ? za - zb : zb - za;
  const int sx = ex > cx ? 1 : -1, sy = ey > cy ? 1 : -1, sz = ez > cz ? 1 : -1;
  int nx = ex > cx ? ex - cx : cx - ex, ny = ey > cy ? ey - cy : cy - ey, nz = ez > cz ? ez - cz : cz - ez;
  visit(cx, cy, cz);
  while (nx + ny + nz > 0) {
    // distance from A to the next boundary on each axis: t_a = b_a / u_a, compared as b_a u_b <= b_b u_a
    const long long bx = sx > 0 ? (long long)(cx + 1) * OG_ONE - xa : xa - (long long)cx * OG_ONE;
    const long long by = sy > 0 ? (long long)(cy + 1) * OG_ONE - ya : ya - (long long)cy * OG_ONE;
    const long long bz = sz > 0 ? (long long)(cz + 1) * OG_ONE - za : za - (long long)cz * OG_ONE;
    if (nx > 0 && (ny == 0 || bx * uy <= by * ux) && (nz == 0 || bx * uz <= bz * ux)) {  // ties step x first
      cx += sx;
      nx--;
    } else if (ny > 0 && (nz == 0 || by * uz <= bz * uy)) {  // then y
      cy += sy;
      ny--;
    } else {
      cz += sz;
      nz--;
    }
    visit(cx, cy, cz);
  }
}

OG_HD bool sm_dynamic(unsigned hits, unsigned frees, unsigned min_frees, int dyn_value) {
  return frees >= min_frees && og_value(hits, frees) <= dyn_value;
}

// ---- host side: parameters, origins, box ----

// nullptr when p is valid (and *c filled), else the reason
inline const char* sm_prepare(const SmParams& p, SmConst* c) {
  if (!std::isfinite(p.resolution) || !(p.resolution > 0)) return "resolution must be finite and > 0";
  const double S = 65536.0 / p.resolution;
  if (!std::isfinite(S)) return "resolution too small";
  if (!std::isfinite(p.max_range) || !(p.max_range > 0)) return "max_range must be finite and > 0";
  const double Rd = p.max_range * S;
  if (!(Rd <= (double)OG_RANGE_LIMIT)) return "max_range / resolution must be <= 2^14";
  for (int k = 0; k < 3; k++)
    if (!std::isfinite(p.sensor_origin[k])) return "sensor_origin must be finite";
  if (!(p.ray_fraction > 0 && p.ray_fraction <= 1)) return "ray_fraction must be in (0, 1]";
  if (p.min_frees < 1) return "min_frees must be >= 1";
  if (!(p.dynamic_thresh >= 0 && p.dynamic_thresh <= 1)) return "dynamic_thresh must be in [0, 1]";
  c->S = S;
  c->R = (long long)std::floor(Rd);
  c->q = (long long)std::rint(p.ray_fraction * (double)OG_ONE);
  if (c->q < 1) return "ray_fraction * 2^16 must round to at least 1";
  c->min_frees = p.min_frees;
  c->dyn_value = (int)std::rint(p.dynamic_thresh * 100.0);
  return nullptr;
}

// The origin of a submap's rays in fixed point; false when a coordinate is beyond 2^30 voxels
inline bool sm_origin(const SmConst& c, const SmParams& p, const float* T, long long* o) {
  float of[3];
  og_transform(T, (float)p.sensor_origin[0], (float)p.sensor_origin[1], (float)p.sensor_origin[2], of);
  for (int k = 0; k < 3; k++)
    if (!og_fixed(of[k], c.S, OG_ORIGIN_LIMIT, &o[k])) return false;
  return true;
}

// The box's dimensions from its inclusive voxel bounds lo[3], hi[3]; false when it has more than 2^31 - 1 cells
inline bool sm_box(const int* lo, const int* hi, unsigned* dims, unsigned long long* cells) {
  unsigned long long n = 1;
  for (int k = 0; k < 3; k++) {
    const long long w = (long long)hi[k] - lo[k] + 1;
    if (w < 1 || w > (long long)SM_MAX_CELLS) return false;
    dims[k] = (unsigned)w;
    n *= (unsigned long long)w;
    if (n > SM_MAX_CELLS) return false;
  }
  *cells = n;
  return true;
}

}  // namespace b200
