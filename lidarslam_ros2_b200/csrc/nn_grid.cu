// K8 — exact nearest neighbour over the target cloud on a uniform cell grid (rank index + cell lists), and the
// fitness reduction. Replaces pcl::KdTreeFLANN::nearestKSearch(k=1) as used by
// pcl::Registration::getFitnessScore (called at graph_based_slam_component.cpp:231, scanmatcher_component.cpp:376,
// apps/align.cpp:37) and by GICP's searchForNeighbors (gicp_omp.h:340-347).
//
// Exactness: cells are visited in Chebyshev rings around the query's cell; after ring r every unvisited point is at
// least (r - delta)*h away, delta covering the f32 cell assignment, so the search stops as soon as best_d2 is within that
// radius (nn_ring_b2 in nn_search.cuh, with a conservative float margin). Squared
// distances are accumulated in f32 exactly like FLANN's L2_Simple, ((dx*dx + dy*dy) + dz*dz), un-fused; ties go to
// the lower point index.
#include <cfloat>
#include <cmath>

#include "engine.hpp"
#include "nn_search.cuh"

namespace b200 {

namespace {

__global__ void __launch_bounds__(256) nn_mark_kernel(const float4* __restrict__ pts, size_t n, NnGeom g, RankWord* table,
                                                      int* cell_of_point, unsigned* coarse, int cd0, int cd1) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = pts[i];
  int cell = -1;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    int ix = nn_cell_coord(p.x, g.origin[0], g.inv_h, g.dims[0]);
    int iy = nn_cell_coord(p.y, g.origin[1], g.inv_h, g.dims[1]);
    int iz = nn_cell_coord(p.z, g.origin[2], g.inv_h, g.dims[2]);
    cell = ix + g.dims[0] * (iy + g.dims[1] * iz);
    mark_occupied(table, cell);
    // tight bounding box of the 8x8x8 block of cells this point falls into (far-query pruning). ~10^2 points share a
    // block: look before each atomic — a stale (looser) bound can only cause a redundant atomic, never a missing one
    unsigned* a = coarse + 6 * (size_t)((ix >> NN_COARSE_SHIFT) + cd0 * ((iy >> NN_COARSE_SHIFT) + cd1 * (iz >> NN_COARSE_SHIFT)));
    const unsigned ox = float_to_ordered(p.x), oy = float_to_ordered(p.y), oz = float_to_ordered(p.z);
    if (ox < __ldcg(a + 0)) atomicMin(a + 0, ox);
    if (oy < __ldcg(a + 1)) atomicMin(a + 1, oy);
    if (oz < __ldcg(a + 2)) atomicMin(a + 2, oz);
    if (ox > __ldcg(a + 3)) atomicMax(a + 3, ox);
    if (oy > __ldcg(a + 4)) atomicMax(a + 4, oy);
    if (oz > __ldcg(a + 5)) atomicMax(a + 5, oz);
  }
  cell_of_point[i] = cell;
}

__global__ void nn_coarse_init_kernel(unsigned* coarse, int n_coarse) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_coarse * 6) return;
  coarse[i] = (i % 6 < 3) ? 0xffffffffu : 0u;  // min = +inf, max = -inf in the ordered encoding: empty
}

__global__ void __launch_bounds__(256) nn_count_kernel(size_t n, const int* __restrict__ cell_of_point,
                                                       const RankWord* __restrict__ table, unsigned* counts) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cell = cell_of_point[i];
  if (cell < 0) return;
  atomicAdd(&counts[rank_of(table, cell)], 1u);
}

__global__ void __launch_bounds__(256) nn_scatter_kernel(const float4* __restrict__ pts, size_t n,
                                                         const int* __restrict__ cell_of_point,
                                                         const RankWord* __restrict__ table,
                                                         const unsigned* __restrict__ cell_start, unsigned* cursor,
                                                         float4* sorted) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cell = cell_of_point[i];
  if (cell < 0) return;
  unsigned r = rank_of(table, cell);
  unsigned pos = cell_start[r] + atomicAdd(&cursor[r], 1u);
  float4 p = pts[i];
  sorted[pos] = make_float4(p.x, p.y, p.z, __int_as_float((int)i));
}

constexpr int NN_MAX_RINGS = 3;  // 7^3 cells; beyond that a query is an outlier and goes to the brute-force pass

struct NnQueryParams {
  NnView V;
  float T[12];
  int has_T;
  float max_d2;
  int n_points;
};

__device__ __forceinline__ void nn_query_point(const NnQueryParams& P, float4 q4, float& qx, float& qy, float& qz) {
  qx = q4.x; qy = q4.y; qz = q4.z;
  if (P.has_T) {
    const float3 t = transform_point(P.T, q4);
    qx = t.x; qy = t.y; qz = t.z;
  }
}

constexpr int NN_GROUP = 4;  // lanes per query in the ring phase

__global__ void __launch_bounds__(128) nn1_kernel(NnQueryParams P, const float4* __restrict__ queries, size_t n, int* out_idx,
                                                  float* out_d2, unsigned* unresolved_count, int* unresolved_list) {
  const size_t tid = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const size_t i = tid / NN_GROUP;
  const int sub = (int)(threadIdx.x & (NN_GROUP - 1));
  // (whole groups fall out together: n queries occupy n * NN_GROUP consecutive threads, warps are never split mid-group)
  if (i >= n) return;  // (a whole group: its NN_GROUP lanes share i)
  float qx, qy, qz;
  nn_query_point(P, queries[i], qx, qy, qz);
  float best = FLT_MAX;
  int best_i = -1;
  bool resolved = false;
  {
    // An outlier is recognised before any cell is probed: if the query's 8x8x8 block of cells and its 26 neighbours hold no
    // point at all, nothing lies within NN_MAX_RINGS (< 8) rings — the ring search would probe 7^3 cells for nothing (a scan
    // reaching far beyond a local map made this kernel wait for exactly those threads). Straight to the far-query pass.
    const NnView& V = P.V;
    const int bx = nn_cell_coord(qx, V.g.origin[0], V.g.inv_h, V.g.dims[0]) >> NN_COARSE_SHIFT;
    const int by = nn_cell_coord(qy, V.g.origin[1], V.g.inv_h, V.g.dims[1]) >> NN_COARSE_SHIFT;
    const int bz = nn_cell_coord(qz, V.g.origin[2], V.g.inv_h, V.g.dims[2]) >> NN_COARSE_SHIFT;
    bool any = false;
    for (int dz = -1; dz <= 1 && !any; dz++)
      for (int dy = -1; dy <= 1 && !any; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          const int x = bx + dx, y = by + dy, z = bz + dz;
          if (x < 0 || y < 0 || z < 0 || x >= V.cdims[0] || y >= V.cdims[1] || z >= V.cdims[2]) continue;
          const unsigned* a = V.coarse + 6 * (size_t)(x + V.cdims[0] * (y + V.cdims[1] * z));
          if (__ldg(a) <= __ldg(a + 3)) {
            any = true;
            break;
          }
        }
    // the ring walk, shared by the NN_GROUP lanes of this query (the decision above is the same in all of them)
    if (any) resolved = nn1_search<NN_GROUP>(P.V, qx, qy, qz, P.max_d2, NN_MAX_RINGS, best, best_i);
  }
  if (sub != 0) return;
  out_idx[i] = best_i;
  out_d2[i] = best;
  if (!resolved) unresolved_list[atomicAdd(unresolved_count, 1u)] = (int)i;
}

// Phase 2: one WARP per unresolved query (an outlier: nothing within NN_MAX_RINGS rings of its cell — a scan point beyond the
// end of a local map, a query far outside the target's bounding box). A kd-tree answers those in O(log n); ring volumes grow
// with r^3 and a linear scan of the cloud costs n per query (round 1: 0.5 ms of a 1.4 ms loop-closure pair). Here the
// coarse level prunes: pass A takes the smallest "farthest corner" distance over the occupied 8x8x8 blocks — an upper
// bound on the NN distance, every occupied block holds a point inside its box; pass B visits, warp-cooperatively, only the
// blocks whose box is not farther than the current bound, tightening it as it goes. Lexicographic (d2, index) minimum,
// blocks at EQUAL distance are visited too, so the result is the exact NN with the lower-index tie-break of the ring search.
__global__ void __launch_bounds__(256) nn1_far_kernel(NnQueryParams P, const float4* __restrict__ queries,
                                                      const unsigned* __restrict__ unresolved_count,
                                                      const int* __restrict__ unresolved_list, int* out_idx, float* out_d2) {
  const unsigned total = *unresolved_count;
  const int lane = threadIdx.x & 31;
  const unsigned warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), n_warps = gridDim.x * (blockDim.x >> 5);
  const NnView& V = P.V;
  const NnGeom& g = V.g;
  for (unsigned u = warp_global; u < total; u += n_warps) {
    const int qi = unresolved_list[u];
    float qx, qy, qz;
    nn_query_point(P, queries[qi], qx, qy, qz);
    float best = out_d2[qi];  // what the ring phase found (FLT_MAX / -1 when nothing)
    int best_i = out_idx[qi];
    // ---- pass A: an upper bound on the NN distance ----
    float ub = best_i >= 0 ? best : FLT_MAX;
    for (int c = lane; c < V.n_coarse; c += 32) {
      const unsigned* a = V.coarse + 6 * (size_t)c;
      const unsigned m0 = __ldg(a), M0 = __ldg(a + 3);
      if (m0 > M0) continue;  // empty block
      const float fx = fmaxf(fabsf(qx - ordered_to_float(m0)), fabsf(qx - ordered_to_float(M0)));
      const float fy = fmaxf(fabsf(qy - ordered_to_float(__ldg(a + 1))), fabsf(qy - ordered_to_float(__ldg(a + 4))));
      const float fz = fmaxf(fabsf(qz - ordered_to_float(__ldg(a + 2))), fabsf(qz - ordered_to_float(__ldg(a + 5))));
      ub = fminf(ub, (fx * fx + fy * fy + fz * fz) * 1.0001f);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) ub = fminf(ub, __shfl_xor_sync(0xffffffffu, ub, d));
    float bound = fminf(ub, P.max_d2);  // nothing farther can be the answer (or matter to the caller)
    // ---- pass B: the blocks that can hold it ----
    for (int base = 0; base < V.n_coarse; base += 32) {
      const int c = base + lane;
      float lb = FLT_MAX;
      if (c < V.n_coarse) {
        const unsigned* a = V.coarse + 6 * (size_t)c;
        const unsigned m0 = __ldg(a), M0 = __ldg(a + 3);
        if (m0 <= M0) {
          const float dx = fmaxf(fmaxf(ordered_to_float(m0) - qx, qx - ordered_to_float(M0)), 0.f);
          const float dy = fmaxf(fmaxf(ordered_to_float(__ldg(a + 1)) - qy, qy - ordered_to_float(__ldg(a + 4))), 0.f);
          const float dz = fmaxf(fmaxf(ordered_to_float(__ldg(a + 2)) - qz, qz - ordered_to_float(__ldg(a + 5))), 0.f);
          lb = (dx * dx + dy * dy + dz * dz) * 0.9999f;  // never above the rounded distance of a point inside the box
        }
      }
      unsigned mask = __ballot_sync(0xffffffffu, lb <= bound);
      while (mask) {
        const int src = __ffs(mask) - 1;
        mask &= mask - 1;
        const float lbc = __shfl_sync(0xffffffffu, lb, src);
        if (lbc > bound) continue;  // the bound tightened meanwhile (warp-uniform)
        const int cc = base + src;
        const int bx = (cc % V.cdims[0]) << NN_COARSE_SHIFT, by = ((cc / V.cdims[0]) % V.cdims[1]) << NN_COARSE_SHIFT,
                  bz = (cc / (V.cdims[0] * V.cdims[1])) << NN_COARSE_SHIFT;
        for (int t = lane; t < 512; t += 32) {  // the block's 8x8x8 cells, 16 per lane
          const int x = bx + (t & 7), y = by + ((t >> 3) & 7), z = bz + (t >> 6);
          if (x >= g.dims[0] || y >= g.dims[1] || z >= g.dims[2]) continue;
          const int cell = x + g.dims[0] * (y + g.dims[1] * z);
          unsigned rk;
          if (!rank_probe(__ldg(reinterpret_cast<const uint2*>(V.index + (cell >> 5))), cell & 31, rk)) continue;
          const unsigned st = __ldg(V.cell_start + rk), en = __ldg(V.cell_start + rk + 1);
          for (unsigned k = st; k < en; k++) {
            const float4 tp = __ldg(V.sorted + k);
            const float d2 = nn_dist2(qx, qy, qz, tp);
            const int ti = __float_as_int(tp.w);
            if (d2 < best || (d2 == best && (best_i < 0 || ti < best_i))) {
              best = d2;
              best_i = ti;
            }
          }
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {  // lexicographic (d2, index) minimum over the warp
          const float od = __shfl_xor_sync(0xffffffffu, best, d);
          const int oi = __shfl_xor_sync(0xffffffffu, best_i, d);
          if (oi >= 0 && (od < best || (od == best && (best_i < 0 || oi < best_i)))) {
            best = od;
            best_i = oi;
          }
        }
        if (best_i >= 0) bound = fminf(bound, best);
      }
    }
    if (lane == 0) {
      out_idx[qi] = best_i;
      out_d2[qi] = best;
    }
  }
}

__global__ void __launch_bounds__(256) fitness_kernel(const float* __restrict__ d2, const int* __restrict__ idx, size_t n,
                                                      double max_range, double* out2) {
  double s = 0, c = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (idx[i] < 0) continue;
    double d = (double)d2[i];
    if (d <= max_range) {
      s += d;
      c += 1.0;
    }
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, k);
    c += __shfl_xor_sync(0xffffffffu, c, k);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(out2, s);
    atomicAdd(out2 + 1, c);
  }
}

}  // namespace

NnView nn_view(const NnGrid& grid) {
  NnView V;
  V.index = grid.index.ptr;
  V.cell_start = grid.cell_start.ptr;
  V.sorted = grid.sorted.ptr;
  for (int a = 0; a < 3; a++) {
    V.g.origin[a] = grid.origin[a];
    V.g.dims[a] = grid.dims[a];
  }
  V.g.h = grid.h;
  V.g.inv_h = grid.inv_h;
  V.coarse = grid.coarse.ptr;
  for (int a = 0; a < 3; a++) V.cdims[a] = grid.cdims[a];
  V.n_coarse = grid.n_coarse;
  return V;
}

void NnGrid::build(const float4* pts, size_t n, cudaStream_t s, const Bounds* known_bounds) {
  valid = false;
  n_points = n;
  n_cells_occupied = 0;
  if (n == 0) return;
  const Bounds b = grid_bounds(pts, n, known_bounds, bounds_scratch, launches, s);
  if (!b.any) return;
  double ext[3];
  for (int a = 0; a < 3; a++) {
    origin[a] = b.mn[a];
    ext[a] = std::max(1e-3, (double)b.mx[a] - (double)b.mn[a]);
  }
  double vol = ext[0] * ext[1] * ext[2];
  double hh = std::cbrt(vol / (4.0 * (double)n));
  hh = std::max(hh, 1e-3);
  for (;;) {  // keep the cell count below 2^28
    double cells = 1;
    for (int a = 0; a < 3; a++) cells *= std::floor(ext[a] / hh) + 1;
    if (cells <= 268435456.0) break;
    hh *= 1.26;
  }
  h = (float)hh;
  inv_h = 1.0f / h;
  n_cells = 1;
  for (int a = 0; a < 3; a++) {
    dims[a] = (int)std::floor(ext[a] / hh) + 1;
    n_cells *= dims[a];
  }
  n_words = (int)((n_cells + 31) / 32);
  n_coarse = 1;
  for (int a = 0; a < 3; a++) {
    cdims[a] = (dims[a] + (1 << NN_COARSE_SHIFT) - 1) >> NN_COARSE_SHIFT;
    n_coarse *= cdims[a];
  }
  coarse.ensure((size_t)n_coarse * 6);
  nn_coarse_init_kernel<<<(n_coarse * 6 + 255) / 256, 256, 0, s>>>(coarse.ptr, n_coarse);
  // No host round trip below: the cell lists are sized by the upper bound min(points, cells) on the occupied cells; the
  // exclusive scan runs over that many counters (the tail past the occupied cells is zero, so cell_start[rank + 1] of
  // the last occupied cell is the total, as the queries expect).
  const size_t occ_max = (size_t)std::min<long long>((long long)n, n_cells);
  index.ensure((size_t)n_words);
  cell_of_point.ensure(n);
  cell_start.ensure(occ_max + 1);
  cursor.ensure(occ_max);
  sorted.ensure(n);
  scan_scratch.total.ensure(1);
  rank_index_clear(index.ptr, n_words, s);
  B200_CUDA(cudaMemsetAsync(cell_start.ptr, 0, sizeof(unsigned) * (occ_max + 1), s));
  B200_CUDA(cudaMemsetAsync(cursor.ptr, 0, sizeof(unsigned) * occ_max, s));
  NnGeom g;
  for (int a = 0; a < 3; a++) {
    g.origin[a] = origin[a];
    g.dims[a] = dims[a];
  }
  g.h = h;
  g.inv_h = inv_h;
  const int blocks = (int)((n + 255) / 256);
  nn_mark_kernel<<<blocks, 256, 0, s>>>(pts, n, g, index.ptr, cell_of_point.ptr, coarse.ptr, cdims[0], cdims[1]);
  rank_index_scan_async(index.ptr, n_words, scan_scratch, scan_scratch.total.ptr, s);
  nn_count_kernel<<<blocks, 256, 0, s>>>(n, cell_of_point.ptr, index.ptr, cell_start.ptr);
  counter_scan_async(cell_start.ptr, occ_max, scan_tmp, s);
  nn_scatter_kernel<<<blocks, 256, 0, s>>>(pts, n, cell_of_point.ptr, index.ptr, cell_start.ptr, cursor.ptr, sorted.ptr);
  launches += 10;
  B200_CUDA(cudaGetLastError());
  n_cells_occupied = occ_max;  // upper bound; the exact count stays on the device (scan_scratch.total)
  valid = true;
}

void nn1_query(const NnGrid& grid, const float4* queries, size_t n, const float* T12_host, int* d_idx, float* d_d2,
               cudaStream_t s, float max_d2) {
  if (n == 0) return;
  NnQueryParams P;
  P.V = nn_view(grid);
  P.has_T = T12_host ? 1 : 0;
  for (int k = 0; k < 12; k++) P.T[k] = T12_host ? T12_host[k] : 0.f;
  P.max_d2 = max_d2;
  P.n_points = (int)grid.n_points;
  NnGrid& gm = const_cast<NnGrid&>(grid);  // per-grid query scratch
  gm.unresolved.ensure(n + 1);
  gm.unresolved_count.ensure(1);
  B200_CUDA(cudaMemsetAsync(gm.unresolved_count.ptr, 0, sizeof(unsigned), s));
  const int blocks = (int)((n * NN_GROUP + 127) / 128);
  nn1_kernel<<<blocks, 128, 0, s>>>(P, queries, n, d_idx, d_d2, gm.unresolved_count.ptr, gm.unresolved.ptr);
  nn1_far_kernel<<<H100_SMS * 4, 256, 0, s>>>(P, queries, gm.unresolved_count.ptr, gm.unresolved.ptr, d_idx, d_d2);
  B200_CUDA(cudaGetLastError());
}

void fitness_reduce(const float* d_d2, const int* d_idx, size_t n, double max_range, double* d_scratch2, double* sum,
                    long long* count, cudaStream_t s) {
  B200_CUDA(cudaMemsetAsync(d_scratch2, 0, 2 * sizeof(double), s));
  int blocks = (int)std::min<size_t>((n + 255) / 256, H100_SMS * 4);
  if (blocks < 1) blocks = 1;
  fitness_kernel<<<blocks, 256, 0, s>>>(d_d2, d_idx, n, max_range, d_scratch2);
  double res[2];
  B200_CUDA(cudaMemcpyAsync(res, d_scratch2, sizeof(res), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  *sum = res[0];
  *count = (long long)(res[1] + 0.5);
}

}  // namespace b200
