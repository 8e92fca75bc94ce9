// K12 — NDT score of many rigid poses of one scan in one launch (b200reg_ndt_score_poses): the grid search of global
// localisation (b200sm_localize_global).
//
// scores[k] is the score of computeDerivatives (ndt_omp_impl.hpp:179-284) at poses[k], without the derivatives: the
// per-pair arithmetic is the solver's own (transform_point, lookup_cell_fast, accumulate_pair of ndt_solver.cuh), each
// point's pairs are summed in f32 in probe order and that sum is added to an f64 accumulator, as in process_point.
//
// Layout: one warp per pose. Lane l takes points l, l + 32, ... in increasing order and a fixed xor-shuffle tree sums the
// lanes, so a pose's score and hit count depend only on the pose, the clouds and the NDT parameters — not on the number
// of poses, their order or the grid. The CTA stages the scan in shared memory one tile at a time and all its warps read
// it. The rank index and the voxel records are read through L1 / L2 (the map of a cut is a few MB and stays in L2).
//
// Algorithmic bytes per pose into the SMs (mostly L1 hits): N_src * 16 / SCORE_WARPS + N_src * probes * 8 + N_hit * 48.
#include "ndt_solver.cuh"

namespace b200 {

namespace {

constexpr int SCORE_WARPS = 8;  // poses per CTA
constexpr int SCORE_THREADS = SCORE_WARPS * 32;
constexpr int SCORE_TILE = 1024;  // scan points staged per pass (16 KB); a multiple of 32 keeps lane l on points l + 32 i
// register allocation sized for 5 CTAs (40 warps) per SM, at most 48 registers a thread: without the hint ptxas gives
// DIRECT1 40 registers and spills the values that live across the call of the division slow path in lookup_cell_fast
constexpr int SCORE_MIN_CTAS = 5;

struct ScoreParams {
  const float4* src;
  const RankWord* index;
  const VoxelRecord* records;
  const float4* centroids;
  const float* poses;  // count x 16, column-major
  double* scores;
  long long* hits;
  GridGeom geom;
  int n_src, count;
  float resolution, radius2;  // KDTREE: the FLANN radius and (float)(res * res) in double
  float d1f, gd2;             // (float)d1, (float)d2, as the solver forms them
};

// the pairs of one transformed point for the four pclomp::NeighborSearchMethod values, in process_point's probe order
template <int METHOD>
__device__ __forceinline__ void score_point(const ScoreParams& P, const float* T, const float4 p, double& score, int& hits) {
  const float3 xt = transform_point(T, p);
  const GridGeom& g = P.geom;
  const int ri = lookup_cell_fast(xt.x, g.leaf, g.inv_leaf) - g.min_b[0],
            rj = lookup_cell_fast(xt.y, g.leaf, g.inv_leaf) - g.min_b[1],
            rk = lookup_cell_fast(xt.z, g.leaf, g.inv_leaf) - g.min_b[2];
  PairSums ps = {};
  const RankWord* idx = P.index;
  if (METHOD == 2 || METHOD == 3) {  // DIRECT7 / DIRECT1
    const bool ix = (unsigned)ri < (unsigned)g.div_b[0], iy = (unsigned)rj < (unsigned)g.div_b[1],
               iz = (unsigned)rk < (unsigned)g.div_b[2];
    const int lin = ri + rj * g.mul[1] + rk * g.mul[2];
    const int r0 = (ix && iy && iz) ? probe_lin(idx, lin) : -1;
    if (METHOD == 2) {
      int r[7];
      r[0] = r0;
      const bool yz = iy && iz, xz = ix && iz, xy = ix && iy;
      r[1] = (yz && (unsigned)(ri + 1) < (unsigned)g.div_b[0]) ? probe_lin(idx, lin + 1) : -1;
      r[2] = (yz && (unsigned)(ri - 1) < (unsigned)g.div_b[0]) ? probe_lin(idx, lin - 1) : -1;
      r[3] = (xz && (unsigned)(rj + 1) < (unsigned)g.div_b[1]) ? probe_lin(idx, lin + g.mul[1]) : -1;
      r[4] = (xz && (unsigned)(rj - 1) < (unsigned)g.div_b[1]) ? probe_lin(idx, lin - g.mul[1]) : -1;
      r[5] = (xy && (unsigned)(rk + 1) < (unsigned)g.div_b[2]) ? probe_lin(idx, lin + g.mul[2]) : -1;
      r[6] = (xy && (unsigned)(rk - 1) < (unsigned)g.div_b[2]) ? probe_lin(idx, lin - g.mul[2]) : -1;
      // a probe no lane hit adds exact zeros: skipping it changes no bit (ps.score starts at +0 and is never -0)
#pragma unroll
      for (int k = 0; k < 7; k++)
        if (__any_sync(__activemask(), r[k] >= 0))
          accumulate_pair<false>(load_record(P.records + max(r[k], 0)), r[k] >= 0, xt, P.d1f, P.gd2, ps);
    } else {
      accumulate_pair<false>(load_record(P.records + max(r0, 0)), r0 >= 0, xt, P.d1f, P.gd2, ps);
    }
  } else if (METHOD == 1) {  // DIRECT26 (26 cells, centre excluded)
    for (int dz = -1; dz <= 1; dz++)
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          if (dx == 0 && dy == 0 && dz == 0) continue;
          const int ni = ri + dx, nj = rj + dy, nk = rk + dz;
          if ((unsigned)ni >= (unsigned)g.div_b[0] || (unsigned)nj >= (unsigned)g.div_b[1] || (unsigned)nk >= (unsigned)g.div_b[2])
            continue;
          const int r = probe_lin(idx, ni + nj * g.mul[1] + nk * g.mul[2]);
          if (r < 0) continue;
          accumulate_pair<false>(load_record(P.records + r), true, xt, P.d1f, P.gd2, ps);
        }
  } else {  // KDTREE: radiusSearch over the voxel centroids
    for_radius_voxels<false>(g, idx, P.centroids, P.resolution, P.radius2, xt,
                             [&](int r) { accumulate_pair<false>(load_record(P.records + r), true, xt, P.d1f, P.gd2, ps); });
  }
  if (ps.hits) {
    score += (double)ps.score;
    hits += ps.hits;
  }
}

template <int METHOD>
__global__ void __launch_bounds__(SCORE_THREADS, SCORE_MIN_CTAS) ndt_score_poses_kernel(const __grid_constant__ ScoreParams P) {
  __shared__ __align__(16) float4 pts[SCORE_TILE];
  __shared__ float Ts[SCORE_WARPS][12];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long k = (long long)blockIdx.x * SCORE_WARPS + warp;
  const bool live = k < P.count;
  // 3x4 row-major transform of pose k: T[r][c] = poses[k][c * 4 + r]
  if (live && lane < 12) Ts[warp][lane] = __ldg(P.poses + k * 16 + (lane & 3) * 4 + (lane >> 2));
  double score = 0.0;
  int hits = 0;
  for (int base = 0; base < P.n_src; base += SCORE_TILE) {
    const int m = min(SCORE_TILE, P.n_src - base);
    __syncthreads();  // the previous tile is consumed (and, the first time, Ts is written)
    for (int j = threadIdx.x; j < m; j += SCORE_THREADS) pts[j] = __ldg(P.src + base + j);
    __syncthreads();
    if (live)
      for (int j = lane; j < m; j += 32) score_point<METHOD>(P, Ts[warp], pts[j], score, hits);
  }
  if (!live) return;
  long long h = hits;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    score += __shfl_xor_sync(0xffffffffu, score, d);
    h += __shfl_xor_sync(0xffffffffu, h, d);
  }
  if (lane == 0) {
    P.scores[k] = score;
    if (P.hits) P.hits[k] = h;
  }
}

}  // namespace

void ndt_score_poses(const VoxelMap& map, const float4* src, size_t n_src, const NdtConfig& cfg, const float* d_poses, int count,
                     double* d_scores, long long* d_hits, cudaStream_t s) {
  if (count <= 0) return;
  ScoreParams P{};
  P.src = src;
  P.index = map.index.ptr;
  P.records = map.records.ptr;
  P.centroids = map.centroids.ptr;
  P.poses = d_poses;
  P.scores = d_scores;
  P.hits = d_hits;
  P.geom = map.geom;
  P.n_src = (int)n_src;
  P.count = count;
  P.resolution = cfg.resolution;
  P.radius2 = static_cast<float>((double)cfg.resolution * (double)cfg.resolution);
  const GaussConsts gc = gauss_constants(cfg.outlier_ratio, cfg.resolution);
  P.d1f = (float)gc.d1;
  P.gd2 = (float)gc.d2;
  const unsigned blocks = (unsigned)((count + SCORE_WARPS - 1) / SCORE_WARPS);
  switch (cfg.search_method) {
    case 0: ndt_score_poses_kernel<0><<<blocks, SCORE_THREADS, 0, s>>>(P); break;
    case 1: ndt_score_poses_kernel<1><<<blocks, SCORE_THREADS, 0, s>>>(P); break;
    case 3: ndt_score_poses_kernel<3><<<blocks, SCORE_THREADS, 0, s>>>(P); break;
    default: ndt_score_poses_kernel<2><<<blocks, SCORE_THREADS, 0, s>>>(P); break;
  }
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
