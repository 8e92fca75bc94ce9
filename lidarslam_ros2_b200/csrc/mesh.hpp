// The surface mesh of the session's map (b200sm_build_mesh): a truncated signed distance field (TSDF) fused from every
// submap's rays, extracted by naive surface nets and saved as binary PLY. The kernels (mesh.cu), a host compile
// (tests/hostmath/mesh_host.cpp, g++ -ffp-contract=off) and an exact Python replay (tests/meshref.py) all follow the text
// below, so every voxel, vertex and face is the same on each side. The double steps are one rounding each: __dmul_rn,
// __ddiv_rn, __dadd_rn, __dsub_rn and __dsqrt_rn on the device, IEEE double with contraction off on the host.
//
// Definitions (this text is the contract):
//  * Parameters: resolution (metres per voxel, > 0), truncation (metres; 1 <= truncation / resolution <= 16, the ratio one
//    rounded division), max_range (the static map's rule: max_range / resolution <= 2^14), sensor_origin (the LiDAR in the
//    robot frame) and min_weight (>= 1).
//  * Rays: the static map's (static_map.hpp): its S and R (sm_prepare), origins O (sm_origin) and skip rule (sm_ray), so
//    n_rays and n_skipped are the static map's. The endpoint E is sm_ray's with the whole ray kept (q = 2^16: E' = E);
//    ray_fraction plays no part. A ray with E == O (zero length) walks nothing.
//  * Band segment of a ray, d = E - O: T = floor(truncation * S); L = sqrt((double)(d . d)) (d . d an int64, < 3 * 2^60);
//    k = (double)T / L; off_a = floor((double)d_a * k) (one rounded multiply); B = E + off; A = E - off, or A = O when
//    L <= T. The ray's band voxels are sm_walk(A, B), the static map's 6-connected walk with its tie rule.
//  * Signed distance of a walked voxel v: C_a = v_a 2^16 + 2^15 (its centre); dot = sum_a (E_a - C_a) d_a in int64;
//    s = floor((double)dot / L) clamped to [-T, T], positive on the sensor's side of E. Bound: |off_a| <= T + 1, so every
//    walked voxel is within r = (T >> 16) + 1 voxels of voxel(E) on each axis (A = O only when |d_a| <= L <= T); then
//    |E_a - C_a| < (r + 1) 2^16 <= 18 * 2^16 < 2^21 and |d_a| <= 2^30, every term is below 2^51 and the sum below 2^53:
//    (double)dot is exact.
//  * Fusion: every walked voxel gets sum += s (int64) and weight += 1 (uint32), a ray visiting it once. The map has fewer
//    than 2^32 points, so weight < 2^32; |s| <= T <= 2^20, so |sum| < 2^52. Integer atomics: the field does not depend on the
//    order of points, submaps or launches.
//  * Band box: the static map's box of every ray's endpoint voxel (K15a's bounds) widened by r on every side; by the bound
//    above every walk stays inside it. A widened box of more than 2^31 - 1 voxels is refused before anything is sized from
//    it. BAND voxels (those some walk visits) are ranked in ascending linear index, as the static map's occupied voxels.
//  * Observed and sign: a band voxel is OBSERVED when weight >= min_weight. Its sign is NEG when sum < 0, POS otherwise
//    (the tie at 0 is POS). Its distance D = (double)sum / (double)weight, one rounded division.
//  * Cells: cell (i, j, k) has the voxels (i + a, j + b, k + c), a, b, c in {0, 1}, as corners, corner index a + 2b + 4c.
//    It is ACTIVE when all eight corners are observed and their signs are not all equal. Its vertex is the mean of the
//    crossings of its sign-changing edges, taken in this order (ms_vertex): x-edges 0-1, 2-3, 4-5, 6-7, then y-edges 0-2,
//    1-3, 4-6, 5-7, then z-edges 0-4, 1-5, 2-6, 3-7. On edge p -> q the crossing is t = D_p / (D_p - D_q) along the edge's
//    axis, the corner p's offsets (0 or 1) on the other two; the three coordinates are summed over the edges in that order
//    and divided by the edge count (u). Its position in metres is (float)((((double)i + 0.5) + u_x) * resolution), y and z
//    likewise: voxel (i, j, k)'s centre is ((i + 0.5) resolution, ...). Vertex ids are the ACTIVE cells' ranks in ascending
//    linear index of their lowest corner voxel (always a band voxel).
//  * Faces: for every pair of observed voxels v and w = v + e_a of different sign, the four cells that share the edge are
//    c_ST, S, T in {0, 1}: for a = x, cell (i, j - 1 + S, k - 1 + T) in the plane (y, z); for a = y, cell (i - 1 + T, j,
//    k - 1 + S) in (z, x); for a = z, cell (i - 1 + S, j - 1 + T, k) in (x, y) (v = (i, j, k)). If all four are ACTIVE the
//    edge gives the quad c00 c10 c11 c01 split on the c00-c11 diagonal: (c00, c10, c11), (c00, c11, c01) when v is NEG,
//    (c00, c11, c10), (c00, c01, c11) when v is POS, so the right-hand normal points from the NEG voxel to the POS one,
//    towards free space. One inactive cell and the edge gives no face. Order: the rank of v, the axis x, y, z, the two
//    triangles.
//  * Where the mesh is not manifold: a cell face whose four voxels alternate in sign (a checkerboard) has four
//    sign-changing edges around it, and the dual edge between the two cells on either side of it is shared by four quads,
//    not two. Surface nets does not resolve that ambiguity; DESIGN.md section 7b reports how often it happens on the drive.
//  * PLY: "ply\n", "format binary_little_endian 1.0\n", "element vertex V\n", "property float x\n" (y, z), "element face
//    F\n", "property list uchar uint vertex_indices\n", "end_header\n"; then V records of three little-endian floats and F
//    records of a 0x03 byte and three little-endian uint32. F > 2^32 - 1 is refused.
#pragma once
#include "static_map.hpp"

namespace b200 {

struct MsParams {
  double resolution = 0.2;
  double truncation = 0.6;
  double max_range = 100.0;
  double sensor_origin[3] = {0.0, 0.0, 0.0};
  unsigned min_weight = 2;
};

// What a build computes from the parameters once, on the host.
struct MsConst {
  SmConst sm;   // the static map's S and R, q = 2^16
  long long T;  // floor(truncation * S), 2^16 - 1 .. 2^20
  int r;        // (T >> 16) + 1: the box's widening
  unsigned min_weight;
  double resolution;
};

OG_HD double ms_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
OG_HD double ms_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
OG_HD double ms_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
OG_HD double ms_sqrt(double a) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(a);
#else
  return std::sqrt(a);
#endif
}

// The band segment of a ray from O to E. False when the ray has zero length (it walks nothing); else A, B and L.
OG_HD bool ms_band(long long T, const long long* o, long long ex, long long ey, long long ez, long long* a, long long* b, double* L) {
  const long long dx = ex - o[0], dy = ey - o[1], dz = ez - o[2];
  const long long dd = dx * dx + dy * dy + dz * dz;
  if (dd == 0) return false;
  const double l = ms_sqrt((double)dd);
  const double k = ms_div((double)T, l);
  const long long fx = (long long)floor(og_mul((double)dx, k)), fy = (long long)floor(og_mul((double)dy, k)),
                  fz = (long long)floor(og_mul((double)dz, k));
  b[0] = ex + fx;
  b[1] = ey + fy;
  b[2] = ez + fz;
  if (l <= (double)T) {
    a[0] = o[0];
    a[1] = o[1];
    a[2] = o[2];
  } else {
    a[0] = ex - fx;
    a[1] = ey - fy;
    a[2] = ez - fz;
  }
  *L = l;
  return true;
}

// s of voxel (x, y, z) on the ray O -> E of length L (d = E - O)
OG_HD long long ms_sdf(long long T, long long ex, long long ey, long long ez, long long dx, long long dy, long long dz, double L, int x,
                       int y, int z) {
  const long long dot = (ex - ((long long)x * OG_ONE + OG_ONE / 2)) * dx + (ey - ((long long)y * OG_ONE + OG_ONE / 2)) * dy +
                        (ez - ((long long)z * OG_ONE + OG_ONE / 2)) * dz;
  long long s = (long long)floor(ms_div((double)dot, L));
  if (s > T) s = T;
  if (s < -T) s = -T;
  return s;
}

OG_HD bool ms_neg(long long sum) { return sum < 0; }
OG_HD double ms_dist(long long sum, unsigned weight) { return ms_div((double)sum, (double)weight); }

// The vertex of an ACTIVE cell (i, j, k) from its corners' D and signs (corner index a + 2b + 4c): xyz in metres.
OG_HD void ms_vertex(const double* D, const bool* neg, int i, int j, int k, double resolution, float* xyz) {
  // the twelve edges (p, q, axis) in the contract's order
  const int P[12] = {0, 2, 4, 6, 0, 1, 4, 5, 0, 1, 2, 3};
  const int Q[12] = {1, 3, 5, 7, 2, 3, 6, 7, 4, 5, 6, 7};
  double sx = 0.0, sy = 0.0, sz = 0.0;
  int n = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int e = 0; e < 12; e++) {
    const int p = P[e], q = Q[e], axis = e >> 2;
    if (neg[p] == neg[q]) continue;
    const double t = ms_div(D[p], ms_sub(D[p], D[q]));
    sx = ms_add(sx, axis == 0 ? t : (double)(p & 1));
    sy = ms_add(sy, axis == 1 ? t : (double)((p >> 1) & 1));
    sz = ms_add(sz, axis == 2 ? t : (double)((p >> 2) & 1));
    n++;
  }
  const double dn = (double)n;
  xyz[0] = (float)og_mul(ms_add(ms_add((double)i, 0.5), ms_div(sx, dn)), resolution);
  xyz[1] = (float)og_mul(ms_add(ms_add((double)j, 0.5), ms_div(sy, dn)), resolution);
  xyz[2] = (float)og_mul(ms_add(ms_add((double)k, 0.5), ms_div(sz, dn)), resolution);
}

// The cell c_ST of the edge from voxel (i, j, k) along axis a (0 x, 1 y, 2 z): its lowest corner voxel
OG_HD void ms_edge_cell(int a, int S, int T, int i, int j, int k, int* c) {
  if (a == 0) {
    c[0] = i;
    c[1] = j - 1 + S;
    c[2] = k - 1 + T;
  } else if (a == 1) {
    c[0] = i - 1 + T;
    c[1] = j;
    c[2] = k - 1 + S;
  } else {
    c[0] = i - 1 + S;
    c[1] = j - 1 + T;
    c[2] = k;
  }
}

// The two triangles of an edge's quad from its cells' vertex ids v[S + 2T] (c00, c10, c01, c11), v_neg: whether the edge's
// lower voxel is NEG. tri[0..5] = the two triangles in order.
OG_HD void ms_quad(const unsigned* v, bool v_neg, unsigned* tri) {
  const unsigned c00 = v[0], c10 = v[1], c01 = v[2], c11 = v[3];
  tri[0] = c00;
  tri[3] = c00;
  if (v_neg) {
    tri[1] = c10;
    tri[2] = c11;
    tri[4] = c11;
    tri[5] = c01;
  } else {
    tri[1] = c11;
    tri[2] = c10;
    tri[4] = c01;
    tri[5] = c11;
  }
}

// ---- host side: parameters, box ----

// nullptr when p is valid (and *c filled), else the reason
inline const char* ms_prepare(const MsParams& p, MsConst* c) {
  SmParams q;
  q.resolution = p.resolution;
  q.max_range = p.max_range;
  for (int k = 0; k < 3; k++) q.sensor_origin[k] = p.sensor_origin[k];
  q.ray_fraction = 1.0;
  if (const char* why = sm_prepare(q, &c->sm)) return why;
  const double ratio = p.truncation / p.resolution;
  if (!std::isfinite(p.truncation) || !(ratio >= 1.0 && ratio <= 16.0)) return "truncation / resolution must be in [1, 16]";
  if (p.min_weight < 1) return "min_weight must be >= 1";
  c->T = (long long)std::floor(p.truncation * c->sm.S);
  c->r = (int)(c->T >> OG_FRAC_BITS) + 1;
  c->min_weight = p.min_weight;
  c->resolution = p.resolution;
  return nullptr;
}

// The static map's origin rule with the mesh's parameters
inline bool ms_origin(const MsConst& c, const MsParams& p, const float* T, long long* o) {
  SmParams q;
  for (int k = 0; k < 3; k++) q.sensor_origin[k] = p.sensor_origin[k];
  return sm_origin(c.sm, q, T, o);
}

// The band box from the endpoint voxels' inclusive bounds lo[3], hi[3]: widened by r; false when it has more than 2^31 - 1
// voxels. blo[3] = its lower corner.
inline bool ms_box(const int* lo, const int* hi, int r, int* blo, unsigned* dims, unsigned long long* cells) {
  int wlo[3], whi[3];
  for (int k = 0; k < 3; k++) {
    wlo[k] = lo[k] - r;  // voxel indices of rays are within 2^30 + 2^14: no overflow
    whi[k] = hi[k] + r;
    blo[k] = wlo[k];
  }
  return sm_box(wlo, whi, dims, cells);
}

}  // namespace b200
