// Device-side exact nearest-neighbour search over an NnGrid (rank index + per-cell point lists): shared by the fitness
// kernel (nn_grid.cu) and the GICP kernels (gicp.cu). See nn_grid.cu for the exactness argument.
#pragma once
#include <cfloat>

#include "common.cuh"
#include "grid_index.cuh"

namespace b200 {

struct NnGeom {
  float origin[3];
  float h, inv_h;
  int dims[3];
};

constexpr int NN_COARSE_SHIFT = 3;  // a coarse cell = 8 x 8 x 8 grid cells

struct NnView {
  const RankWord* index;
  const unsigned* cell_start;
  const float4* sorted;  // xyz + original index (int bits) in w
  NnGeom g;
  // coarse level: tight bounding box of the points of every 8x8x8 block of cells (6 order-preserving uints: min xyz,
  // max xyz; min > max = empty) — the far-query pass of nn_grid.cu prunes with it
  const unsigned* coarse;
  int cdims[3];
  int n_coarse;
};

struct NnGrid;
NnView nn_view(const NnGrid& grid);  // host: device-side view of a built grid (nn_grid.cu)

__device__ __forceinline__ int nn_cell_coord(float v, float o, float inv_h, int dim) {
  int c = (int)floorf((v - o) * inv_h);
  return max(0, min(dim - 1, c));
}

// The squared radius a ring search may trust after ring r: every point in a cell outside ring r is farther than it, and
// its f32 d2 is larger. Cells come from floor(fl(fl(v - o) * inv_h)), whose cell coordinate s' differs from the exact
// (v - o) / h by at most 3 * 2^-24 * |s| (three roundings). A point two rings out is only r - e_p - e_q cells away,
// with e_p <= 3 * 2^-24 * D for a grid point (s <= D, the largest dimension) and the same for the query: a query
// clamped into the grid is farther than its clamped cell says, and one inside has |s| <= D. So after ring r every
// unvisited point is at least (r - delta) h away with delta = D * 2^-20 (> 6 * 2^-24 D with room for the second-order
// terms). The factor 0.99999 keeps the bound below the f32 d2 of such a point, which rounds at most 5 * 2^-24 low.
// (r h)^2 alone is wrong on long axes: at cell 513 of a 1 130-cell grid a point two cells away can be closer than h.
__device__ __forceinline__ float nn_ring_b2(const NnGeom& g, int r) {
  const float delta = (float)max(g.dims[0], max(g.dims[1], g.dims[2])) * 0x1p-20f;
  const float bound = fmaxf((float)r - delta, 0.f) * g.h;
  return bound * bound * 0.99999f;
}

// FLANN L2_Simple: ((dx*dx + dy*dy) + dz*dz) in f32, un-fused
__device__ __forceinline__ float nn_dist2(float qx, float qy, float qz, float4 t) {
  const float dx = __fsub_rn(qx, t.x), dy = __fsub_rn(qy, t.y), dz = __fsub_rn(qz, t.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// visits every point of the Chebyshev ring r around cell (cx, cy, cz); f(float4 point).
// (sub, nsub): a query may be shared by nsub lanes — lane `sub` then takes every nsub-th cell of the ring.
template <typename F>
__device__ __forceinline__ void nn_visit_ring(const NnView& V, int cx, int cy, int cz, int r, F&& f, int sub = 0, int nsub = 1) {
  const NnGeom& g = V.g;
  int turn = 0;
  const int z0 = max(cz - r, 0), z1 = min(cz + r, g.dims[2] - 1);
  const int y0 = max(cy - r, 0), y1 = min(cy + r, g.dims[1] - 1);
  for (int z = z0; z <= z1; z++) {
    const bool zface = (z == cz - r) || (z == cz + r);
    for (int y = y0; y <= y1; y++) {
      const bool yface = (y == cy - r) || (y == cy + r);
      const int step = (zface || yface || r == 0) ? 1 : 2 * r;  // interior rows: only the two x faces
      for (int x = cx - r; x <= cx + r; x += step) {
        if (x < 0 || x >= g.dims[0]) continue;
        if (nsub > 1) {
          const int mine = turn == sub;
          turn = (turn + 1 == nsub) ? 0 : turn + 1;
          if (!mine) continue;
        }
        const int cell = x + g.dims[0] * (y + g.dims[1] * z);
        unsigned rk;
        if (!rank_probe(__ldg(reinterpret_cast<const uint2*>(V.index + (cell >> 5))), cell & 31, rk)) continue;
        const unsigned s = __ldg(V.cell_start + rk), e = __ldg(V.cell_start + rk + 1);
        for (unsigned k = s; k < e; k++) f(__ldg(V.sorted + k));
      }
    }
  }
}

// exact 1-NN; ties → lower index. If max_d2 < FLT_MAX the search also stops once no closer point than max_d2 can exist
// (the caller then tests best < max_d2 itself). The ring expansion is capped at `max_rings`: a query whose
// neighbourhood is still unresolved then (an outlier far from every target point) returns false and is finished by
// the brute-force pass of nn_grid.cu — ring volumes grow with r^3, a linear scan of the cloud does not.
// GROUP (1, 2 or 4) consecutive lanes share the query: each walks its share of every ring's cells and the lexicographic
// (d2, index) minimum is combined inside the group after each ring (all lanes of the group return the same answer). The
// ring walk is a chain of dependent loads; four lanes per query cut that chain to a quarter.
template <int GROUP = 1>
__device__ __forceinline__ bool nn1_search(const NnView& V, float qx, float qy, float qz, float max_d2, int max_rings,
                                           float& best, int& best_i) {
  const NnGeom& g = V.g;
  const int cx = nn_cell_coord(qx, g.origin[0], g.inv_h, g.dims[0]);
  const int cy = nn_cell_coord(qy, g.origin[1], g.inv_h, g.dims[1]);
  const int cz = nn_cell_coord(qz, g.origin[2], g.inv_h, g.dims[2]);
  best = FLT_MAX;
  best_i = -1;
  const int max_r = min(max_rings, max(g.dims[0], max(g.dims[1], g.dims[2])));
  for (int r = 0; r <= max_r; r++) {
    nn_visit_ring(V, cx, cy, cz, r, [&](float4 t) {
      const float d2 = nn_dist2(qx, qy, qz, t);
      const int ti = __float_as_int(t.w);
      if (d2 < best || (d2 == best && (best_i < 0 || ti < best_i))) {
        best = d2;
        best_i = ti;
      }
    }, (int)(threadIdx.x & (GROUP - 1)), GROUP);
    if (GROUP > 1) {
      // only the lanes of this group take part: other groups of the warp are in other rings, or done
      const unsigned gmask = ((1u << GROUP) - 1u) << ((threadIdx.x & 31) & ~(GROUP - 1));
#pragma unroll
      for (int d = 1; d < GROUP; d <<= 1) {
        const float od = __shfl_xor_sync(gmask, best, d);
        const int oi = __shfl_xor_sync(gmask, best_i, d);
        if (oi >= 0 && (od < best || (od == best && (best_i < 0 || oi < best_i)))) {
          best = od;
          best_i = oi;
        }
      }
    }
    const float b2 = nn_ring_b2(g, r);  // every unvisited point has a larger d2
    if (best_i >= 0 && best <= b2) return true;
    if (b2 > max_d2) return true;  // nothing within the caller's radius remains unvisited
  }
  return max_r >= max(g.dims[0], max(g.dims[1], g.dims[2]));  // whole grid visited → resolved
}

}  // namespace b200
