// Device-side structures and per-pair helpers shared by the NDT kernels (ndt_solver.cu, ndt_aux.cu, ndt_score.cu).
#pragma once
#include "../../include/b200reg.h"
#include "common.cuh"
#include "engine.hpp"
#include "grid_index.cuh"

namespace b200 {

constexpr int NDT_MAX_CTAS = 256;  // one CTA per SM
// Registrations in flight inside one batch launch = controller CTAs. Every launch (single or batched) leaves this many
// SMs to controllers, so that the evaluator count — and with it the point partition and the fixed summation order —
// is the same for b200reg_align and for b200reg_ndt_align_batch: a batched result is bitwise the single-align result.
#ifndef B200_NDT_MAX_SLOTS
#define B200_NDT_MAX_SLOTS 3  // developer switch for A/B builds
#endif
constexpr int NDT_MAX_SLOTS = B200_NDT_MAX_SLOTS;

enum EvalMode : int {
  EVAL_DERIV = 0,        // fused derivative pass (K1)
  EVAL_DONE = 1,         // solver finished, result written
  EVAL_NEED_HESSIAN = 2  // leave the persistent kernel: host runs the f64 radius-Hessian pass (K2) and resumes
};

enum SolverPhase : int { PH_INITIAL = 0, PH_LS_FIRST = 1, PH_LS_ITER = 2, PH_LS_HESSIAN = 3 };

// what every CTA needs for one evaluation round; written by the controller (or by the host for round 0)
struct alignas(16) NdtControl {  // size is a multiple of 16 bytes: arrays of it are read with 16-byte shared-memory loads
  float T[12];     // 3x4 row-major transform applied to the source points
  float jang[24];  // 8 x 3 f32 angle-Jacobian table   (ndt_omp_impl.hpp:337-345)
  float hang[45];  // 15 x 3 f32 angle-Hessian table    (ndt_omp_impl.hpp:371-391)
  int mode;        // EvalMode
  int compute_hessian;
  int job;         // batch launches: index of the registration this block belongs to (evaluators restage on a change)
  int pad[4];
};
static_assert(sizeof(NdtControl) % 16 == 0, "NdtControl must keep 16-byte alignment in arrays");
constexpr int NDT_CONTROL_WORDS = sizeof(NdtControl) / 4;

// controller state (lives in global memory: a different CTA may run the controller every round)
struct NdtState {
  double p[6], score, g[6], H[36];
  double dir[6], x_t[6];
  double jd[24], hd[45];  // f64 angle tables at x_t, consumed by the K2 pass
  double phi_0, d_phi_0, a_l, f_l, g_l, a_u, f_u, g_u, a_t;
  float final_T[16];
  long long hits_last, hits_total;
  int interval_converged, open_interval, step_iterations;
  int phase, nr_iterations, evaluations, converged;
};

// Signalling between the evaluator CTAs and the controller CTA carries its own validity ("flag in data", as in NCCL's
// LL protocol), so neither direction needs a counter, a fence or a second dependent round trip:
//  * control block, controller -> evaluators: every 32-bit word travels as one 64-bit store {payload, sequence}; an
//    evaluator thread polls ITS word until the sequence number is the expected one. NDT_CTL_COPIES replicas spread
//    the pollers over L2 lines.
//  * partial sums, evaluators -> controller: rows of 32 doubles, double-buffered by round parity; an unwritten slot
//    holds NDT_PARTIAL_EMPTY (a NaN payload no computation produces). The controller's reduction loads double as the
//    poll; it re-arms each row after consuming it, two rounds before the row is written again.
constexpr int NDT_CTL_COPIES = 4;
constexpr int NDT_CTL_LL_WORDS = 96;  // >= NDT_CONTROL_WORDS, whole 128-byte lines
constexpr unsigned long long NDT_PARTIAL_EMPTY = 0xFFF8DEADFFF8DEADull;
constexpr int NDT_MAX_ROUNDS = 60000;  // sequence numbers are epoch * 65536 + round + 1

// one registration of a batch launch (device array, filled by the host before the launch)
struct NdtJob {
  // source points: records of `stride` bytes with x, y, z floats first — 16 for a float4 cloud resident in HBM, the
  // caller's record size when the raw host records were copied straight in (no unpack pass: the evaluators read them
  // once, when they stage the registration's points into shared memory)
  const unsigned char* src;
  int n_src;
  int stride;
  // ready == nullptr: the points are there when the launch starts. Otherwise the controller waits, before it starts this
  // registration, until *ready == ready_tag: the copy stream writes the tag behind the scan's DMA (cuStreamWriteValue32),
  // so later scans of a batch are still being uploaded while earlier ones are already being registered.
  const unsigned* ready;
  unsigned ready_tag;
  int pad;
  double p0[6];         // initial pose parameters (ndt_omp_impl.hpp:103-111)
  float init_final[16]; // final_transformation_ = guess
  NdtControl init;      // control block of the first evaluation (transform = guess, angle tables at p0)
};

struct NdtSolverWork {
  unsigned error;
  unsigned next_job;     // batch launches: next unassigned registration (atomicAdd by the controllers)
  unsigned trace_count;  // traced align(): rounds recorded so far (counts on past NdtLaunch::trace_cap); host-reset per align
  unsigned pad;
  NdtControl control;    // plain copy of the control block, written only when the kernel leaves for a K2 pass
  NdtState state;
  NdtResult result;
  alignas(128) unsigned long long ctl_ll[NDT_MAX_SLOTS][NDT_CTL_COPIES][NDT_CTL_LL_WORDS];
  alignas(128) double partials[NDT_MAX_SLOTS][2][NDT_MAX_CTAS][SLOT_COUNT];
};

struct NdtLaunch {
  const float4* src;
  const RankWord* index;
  const VoxelRecord* records;
  const double* icov_d;
  const float4* centroids;
  NdtSolverWork* work;
  NdtResult* result_host;  // pinned, device-visible host memory: the controller CTA writes the result there on exit
  // batch launches (n_slots >= 1 and jobs != nullptr): n_jobs registrations against the same map, n_slots in flight;
  // result_host is then an array of n_jobs results. jobs == nullptr: the single registration described inline below.
  const NdtJob* jobs;
  int n_jobs;
  int n_slots;
  PoseBoardView board;  // board.world > 0: finished poses are also stored into every peer's pose board (engine.hpp)
  GridGeom geom;
  int n_src;
  int n_voxels;
  int search_method;
  int mode;    // NdtMode
  unsigned epoch;         // launch counter of this handle (high half of the control block's sequence numbers)
  int acc_offset;         // byte offset of the per-thread accumulators in dynamic shared memory (after the rank index)
  int pts_offset;         // byte offset of the staged source points (n_slots x SMEM_POINTS float4) after the accumulators
  int scalar_controller;  // 1: disable the warp-parallel controller fast path (developer switch)
  int resume;  // 1: state/control already in work (after a K2 pass); first round skips the evaluation
  int index_in_smem;
  int max_iterations;
  float resolution;
  float radius2;  // (float)(resolution * resolution) in double, the FLANN radius of KDTREE mode
  double d1, d2, d3;
  double step_size, trans_eps;
  double p0[6];
  float init_final[16];
  NdtControl init;
  // trace != nullptr (single align() launches only): warp 0 of the controller CTA appends one record per round
  b200reg_ndt_trace_record* trace;
  int trace_cap;
  int trace_launch;  // 0 for the first launch of an align(), +1 for every launch resumed after a K2 pass
};

// ---- rank-index probe ----------------------------------------------------------------------------------
// returns the record index of the voxel at absolute cell coordinates (ci, cj, ck), or -1
// (VoxelGridCovariance::getNeighborhoodAtPoint, voxel_grid_covariance_omp_impl.hpp:382-399)
template <bool STAGED>
__device__ __forceinline__ int probe_cell(const GridGeom& g, const RankWord* __restrict__ gidx,
                                          const RankWord* __restrict__ sidx, int ci, int cj, int ck) {
  if (ci < g.min_b[0] || ci > g.max_b[0] || cj < g.min_b[1] || cj > g.max_b[1] || ck < g.min_b[2] || ck > g.max_b[2])
    return -1;
  const int lin = (ci - g.min_b[0]) + (cj - g.min_b[1]) * g.mul[1] + (ck - g.min_b[2]) * g.mul[2];
  uint2 w;
  if (STAGED) w = *reinterpret_cast<const uint2*>(sidx + (lin >> 5));
  else w = __ldg(reinterpret_cast<const uint2*>(gidx + (lin >> 5)));
  unsigned r;
  if (!rank_probe(w, lin & 31, r)) return -1;
  return (int)r;
}

// rank-index probe of a leaf index known to be inside the grid
// (idx points either at the shared-memory copy staged by TMA or at the global table)
__device__ __forceinline__ int probe_lin(const RankWord* __restrict__ idx, int lin) {
  unsigned r;
  if (!rank_probe(*reinterpret_cast<const uint2*>(idx + (lin >> 5)), lin & 31, r)) return -1;
  return (int)r;
}

struct PairSums {  // sums over the voxels hit by one point
  float S0, S1, S2;                    // sum e * s,           s = C x'
  float M00, M01, M02, M11, M12, M22;  // sum e * C
  float Q00, Q01, Q02, Q11, Q12, Q22;  // sum e * s s^T
  float score;                         // sum of the f32 score increments of this point
  int hits;
};

struct Rec {
  float4 a, b, c;
};
__device__ __forceinline__ Rec load_record(const VoxelRecord* __restrict__ rec) {
  Rec r;
  const float4* p = reinterpret_cast<const float4*>(rec);
  r.a = __ldg(p);
  r.b = __ldg(p + 1);
  r.c = __ldg(p + 2);
  return r;
}

// one (point, voxel) pair — updateDerivatives (ndt_omp_impl.hpp:482-535) reduced to its per-pair core.
// Branch-free: a probe that missed reads record 0 and is masked out, so that the compiler may keep the loads and
// the arithmetic of several pairs in flight. All f32: the reference forms score_inc = float(-d1 * e) and
// e' = float(e * d1) through a double product (:499, :508); multiplying by float(d1) instead differs by at most one
// f32 ulp (6e-8 relative), far below the f32 noise of the per-pair products themselves.
template <bool HESS>
__device__ __forceinline__ void accumulate_pair(const Rec& R, bool valid, float3 xt, float d1f, float gd2, PairSums& ps) {
  const float c00 = R.b.z, c01 = R.b.w, c02 = R.c.x, c11 = R.c.y, c12 = R.c.z, c22 = R.c.w;
  // x' = x_trans - mean (float-float mean: within one ulp of the reference's f64 subtraction + cast, :259-262, :490)
  const float x0 = __fsub_rn(__fsub_rn(xt.x, R.a.x), R.a.w);
  const float x1 = __fsub_rn(__fsub_rn(xt.y, R.a.y), R.b.x);
  const float x2 = __fsub_rn(__fsub_rn(xt.z, R.a.z), R.b.y);
  const float s0 = c00 * x0 + c01 * x1 + c02 * x2;
  const float s1 = c01 * x0 + c11 * x1 + c12 * x2;
  const float s2 = c02 * x0 + c12 * x1 + c22 * x2;
  const float q = x0 * s0 + x1 * s1 + x2 * s2;
  const float ex = expf(-gd2 * q * 0.5f);  // :497
  const float e2 = gd2 * ex;               // :501
  const bool ok = valid && !(e2 > 1.0f || e2 < 0.0f || e2 != e2);  // :504-505 (the score increment is dropped too)
  const float e = ok ? e2 * d1f : 0.0f;    // :508
  ps.score += ok ? -d1f * ex : 0.0f;       // :499
  ps.hits += ok ? 1 : 0;
  ps.S0 += e * s0;
  ps.S1 += e * s1;
  ps.S2 += e * s2;
  if (HESS) {
    ps.M00 += e * c00; ps.M01 += e * c01; ps.M02 += e * c02;
    ps.M11 += e * c11; ps.M12 += e * c12; ps.M22 += e * c22;
    const float es0 = e * s0, es1 = e * s1, es2 = e * s2;
    ps.Q00 += es0 * s0; ps.Q01 += es0 * s1; ps.Q02 += es0 * s2;
    ps.Q11 += es1 * s1; ps.Q12 += es1 * s2; ps.Q22 += es2 * s2;
  }
}

// lookup cell of a transformed point: floor(x / leaf) with an IEEE division (impl.hpp:379-381)
__device__ __forceinline__ int lookup_cell(float x, float leaf) { return (int)floorf(__fdiv_rn(x, leaf)); }
// Same result without the division on the common path: q = x * (1/leaf) is within 2 ulp of the IEEE quotient, so
// floor(q) can only differ from floor(x / leaf) when q lies within a few ulp of an integer — only then is the exact
// division evaluated.
__device__ __forceinline__ int lookup_cell_fast(float x, float leaf, float inv_leaf) {
  const float q = __fmul_rn(x, inv_leaf);
  if (fabsf(q - rintf(q)) <= 1e-6f * fabsf(q) + 1e-30f) return (int)floorf(__fdiv_rn(x, leaf));
  return (int)floorf(q);
}

// Radius neighbourhood (VoxelGridCovariance::radiusSearch, voxel_grid_covariance_omp.h:470-499: every voxel centroid c
// with un-fused f32 |c - x|^2 < f32(res^2)). The cells to probe on one axis are derived from the BUILD rule, not from
// the query's lookup cell: floor(x / leaf) and the builder's floor(x * inv_leaf) disagree near a cell face, so a hit
// can lie two lookup cells away from the query. A centroid that passes the test is within res (1 + 2^-22) of x on each
// axis; the voxel's points (whose build cell names the voxel) are within a few ulp of their f32 centroid, so within
// reach = res (1 + 2^-20) + 2^-21 |x| of x. floor(fl(y * inv_leaf)) is non-decreasing in y, so the voxel's cell on
// this axis lies in [build(x - reach) rounded down, build(x + reach) rounded up]: three cells, four near a face.
// Returns false (no neighbour on any axis) when the range misses the grid or x is not finite; the float clamps
// before the int conversion keep huge coordinates from overflowing it.
__device__ __forceinline__ bool radius_cell_range(float x, float res, float inv_leaf, int min_b, int max_b, int& lo, int& hi) {
  const float reach = __fmaf_ru(fabsf(x), 0x1p-21f, __fmul_ru(res, 1.0f + 0x1p-20f));
  float fl = floorf(__fmul_rn(__fsub_rd(x, reach), inv_leaf));
  float fh = floorf(__fmul_rn(__fadd_ru(x, reach), inv_leaf));
  if (!(fh >= (float)min_b && fl <= (float)max_b)) return false;  // also false for NaN and +-inf
  lo = max((int)fmaxf(fl, (float)min_b), min_b);
  hi = min((int)fminf(fh, (float)max_b), max_b);
  return lo <= hi;
}

// Visits the record index of every voxel whose f32 centroid passes the radius test of xt (f(r)), z-y-x ascending.
template <bool STAGED, typename F>
__device__ __forceinline__ void for_radius_voxels(const GridGeom& g, const RankWord* __restrict__ idx, const float4* centroids,
                                                  float res, float radius2, float3 xt, F&& f) {
  int lo[3], hi[3];
  if (!radius_cell_range(xt.x, res, g.inv_leaf, g.min_b[0], g.max_b[0], lo[0], hi[0]) ||
      !radius_cell_range(xt.y, res, g.inv_leaf, g.min_b[1], g.max_b[1], lo[1], hi[1]) ||
      !radius_cell_range(xt.z, res, g.inv_leaf, g.min_b[2], g.max_b[2], lo[2], hi[2]))
    return;
  for (int k = lo[2]; k <= hi[2]; k++)
    for (int j = lo[1]; j <= hi[1]; j++)
      for (int i = lo[0]; i <= hi[0]; i++) {
        const int lin = (i - g.min_b[0]) + (j - g.min_b[1]) * g.mul[1] + (k - g.min_b[2]) * g.mul[2];
        uint2 w;
        if (STAGED) w = *reinterpret_cast<const uint2*>(idx + (lin >> 5));
        else w = __ldg(reinterpret_cast<const uint2*>(idx + (lin >> 5)));
        unsigned r;
        if (!rank_probe(w, lin & 31, r)) continue;
        const float4 c = __ldg(centroids + r);
        const float ex = __fsub_rn(xt.x, c.x), ey = __fsub_rn(xt.y, c.y), ez = __fsub_rn(xt.z, c.z);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
        if (!(d2 < radius2)) continue;
        f((int)r);
      }
}

}  // namespace b200
