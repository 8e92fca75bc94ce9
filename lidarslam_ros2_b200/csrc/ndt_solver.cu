// K1 — fused NDT derivative kernel inside a persistent, cooperative, device-resident Newton loop.
//
// Replaces (Thirdparty/ndt_omp_ros2/include/pclomp/ndt_omp_impl.hpp):
//   computeTransformation :80-171, computeDerivatives :179-284, computePointDerivatives :396-438,
//   updateDerivatives :482-535, computeStepLengthMT :756-916 (+ :632-753), and the neighbourhood lookups
//   voxel_grid_covariance_omp_impl.hpp:373-442; pcl::transformPointCloud (ndt_omp_impl.hpp:100,817,862) is fused
//   into the evaluation.
//
// H100 design (not a translation of the OpenMP loop):
//   * ONE cooperative kernel launch per align(), one 768-thread CTA per SM. Evaluator CTAs keep their source points in
//     SHARED MEMORY for the whole solve and loop   evaluate -> CTA partial row -> wait for the next pose;   the last
//     CTA is the CONTROLLER: it keeps the Newton / More-Thuente state in shared memory and loops
//     fixed-order f64 reduction of the partial rows (its loads are the arrival poll) -> 6x6 solve -> next pose +
//     angle tables -> publish.  The ~5-40 sequential evaluations of a registration cost no launches, no host round
//     trips and no global-memory state traffic; both signalling directions carry their validity in the data words
//     (ndt_solver.cuh), so a hop is one store plus one polling load — no counter, fence or second round trip.
//   * per (point, voxel) pair only e, s = C x' and the sums S += e s, M += e C, Q += e s s^T are formed; the
//     gradient / Hessian contribution J^T(.)J is applied once per POINT (J, H_E depend on the point only):
//     ~35 FMA per pair + ~140 per point instead of ~600 MAC per pair in the reference.
//   * voxel lookup = occupancy-bitmap rank index (common.cuh) staged into shared memory by TMA bulk copies
//     (cp.async.bulk + mbarrier) once per launch; 48-byte voxel records are fetched with batched 16-byte
//     read-only loads (several records of a point are in flight before the first one is consumed).
//   * reductions: per-thread f32 sums of <= a few points in shared memory -> lane L of each warp sums slot L over the
//     warp's 32 columns in f64 (fixed order) -> per-CTA partial -> fixed-order f64 sum over CTAs: bitwise deterministic.
//
// Algorithmic HBM bytes per evaluation (SURVEY.md §8d): N_src*16 + N_src*probes*8 + N_hit*48 + 28*8.
#include "ndt_solver.cuh"

#ifndef B200_SKIP_EMPTY_PROBES
#define B200_SKIP_EMPTY_PROBES 1  // developer switch for A/B measurements (build with -DB200_SKIP_EMPTY_PROBES=0)
#endif

namespace b200 {

std::mutex& cooperative_launch_mutex(int device) {
  static std::mutex m[64];
  return m[(device >= 0 && device < 64) ? device : 0];
}

namespace {

// ONE 768-thread CTA per SM (80 registers/thread fill the register file, so two can never share an SM): 24 warps keep
// the issue slots of the four schedulers busy, the partial sums of an SM are combined in its own shared memory, and the
// controller CTA has to ingest 129 rows instead of 387 (its L2 -> SM bandwidth bounds the reduction). The controller
// CTA owns an SM by construction.
constexpr int SOLVER_THREADS = 768;
constexpr int SOLVER_WARPS = SOLVER_THREADS / 32;
constexpr int SOLVER_MIN_CTAS = 1;
#ifndef B200_SMEM_POINTS
#define B200_SMEM_POINTS 768  // developer switch for A/B builds (768 measured 5 % faster than 1024: more L1 for the records)
#endif
constexpr int SMEM_POINTS = B200_SMEM_POINTS;  // source points of a CTA's chunk staged in shared memory for the whole solve
constexpr int ACC_SLOTS = 27;      // 6 gradient + 21 upper-triangular Hessian sums per thread (f32, in shared memory)
constexpr int ACC_STRIDE = SOLVER_THREADS + 4;  // rows start 16-byte aligned (the warp reduction reads them with LDS.128) and the
                                                // 772-float pitch spreads the eight lanes of a quarter-warp over all 32 banks
constexpr int ACC_BYTES = ACC_SLOTS * ACC_STRIDE * 4;
constexpr int SOLVER_MAX_INDEX_SMEM = 64 * 1024;  // the rank index is staged in shared memory up to this size
constexpr int PTS_BYTES = SMEM_POINTS * 16;  // per slot
constexpr int ACC_BYTES_PAD = (ACC_BYTES + 127) & ~127;
constexpr int SOLVER_MAX_DYN_SMEM = SOLVER_MAX_INDEX_SMEM + ACC_BYTES_PAD + NDT_MAX_SLOTS * PTS_BYTES;  // the rest of the SM stays L1 for the voxel-record gathers (a 100 KB index in shared memory measured slower)  // padded row: slot-major reads by 32 lanes hit 32 different banks
constexpr long long SPIN_TIMEOUT_CYCLES = 4000000000LL;  // ~2 s device-side watchdog, never reached in normal runs

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- TMA bulk copy helpers (cp.async.bulk → UBLKCP) -----------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned phase) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(phase)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// system scope: pose-board words live in a peer GPU's memory (NVLink) or are read while a peer writes them
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void ld_relaxed_gpu_v2(const double* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_relaxed_gpu_v2(double* p, unsigned long long a, unsigned long long b) {
  asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ unsigned ctl_sequence(unsigned epoch, int round) { return epoch * 65536u + (unsigned)round + 1u; }

// ---- per-thread accumulators of one evaluation --------------------------------------------------------------
// The 27 f32 sums of a thread live in SHARED memory (column tid of acc[slot][tid], conflict-free; the warp-level
// reduction then reads them slot-major, see the kernel) so that the
// registers stay available for the batched voxel-record loads; score (f64) and the hit count stay in registers.
struct Accum {
  float (*s)[ACC_STRIDE];  // [ACC_SLOTS][ACC_STRIDE]
  int tid;
  bool first;  // no point applied yet this evaluation: store instead of read-modify-write
  double score;
  int hits;
  // FIRST: the thread's first point with hits (a plain store, no load); the caller branches on `first` once per point
  template <bool FIRST>
  __device__ __forceinline__ void add(int slot, float v) { s[slot][tid] = FIRST ? v : s[slot][tid] + v; }
};

// per-POINT application of J (point gradient, :396-412) and H_E (:414-436) to the pair sums
template <bool HESS, bool FIRST>
__device__ __forceinline__ void apply_point(const float4 p, const PairSums& ps, const NdtControl& c, float gd2, Accum& a) {
  const float x = p.x, y = p.y, z = p.z;
  // the 24 + 45 table floats are read as 16-byte shared-memory vectors (NdtControl: jang at byte 48, hang at 144)
  const float4* jv = reinterpret_cast<const float4*>(c.jang);
  const float4 ja0 = jv[0], ja1 = jv[1], ja2 = jv[2], ja3 = jv[3], ja4 = jv[4], ja5 = jv[5];
  // J columns 3..5: J3 = (0, j0, j1), J4 = (j2, j3, j4), J5 = (j5, j6, j7)
  const float j0 = ja0.x * x + ja0.y * y + ja0.z * z;
  const float j1 = ja0.w * x + ja1.x * y + ja1.y * z;
  const float j2 = ja1.z * x + ja1.w * y + ja2.x * z;
  const float j3 = ja2.y * x + ja2.z * y + ja2.w * z;
  const float j4 = ja3.x * x + ja3.y * y + ja3.z * z;
  const float j5 = ja3.w * x + ja4.x * y + ja4.y * z;
  const float j6 = ja4.z * x + ja4.w * y + ja5.x * z;
  const float j7 = ja5.y * x + ja5.z * y + ja5.w * z;
  a.score += (double)ps.score;
  a.hits += ps.hits;
  a.add<FIRST>(0, ps.S0);
  a.add<FIRST>(1, ps.S1);
  a.add<FIRST>(2, ps.S2);
  a.add<FIRST>(3, j0 * ps.S1 + j1 * ps.S2);
  a.add<FIRST>(4, j2 * ps.S0 + j3 * ps.S1 + j4 * ps.S2);
  a.add<FIRST>(5, j5 * ps.S0 + j6 * ps.S1 + j7 * ps.S2);
  if (HESS) {
    // W = sum e (C - d2 s s^T)
    const float W00 = ps.M00 - gd2 * ps.Q00, W01 = ps.M01 - gd2 * ps.Q01, W02 = ps.M02 - gd2 * ps.Q02;
    const float W11 = ps.M11 - gd2 * ps.Q11, W12 = ps.M12 - gd2 * ps.Q12, W22 = ps.M22 - gd2 * ps.Q22;
    // W * J3, W * J4, W * J5
    const float a0 = W01 * j0 + W02 * j1, a1 = W11 * j0 + W12 * j1, a2 = W12 * j0 + W22 * j1;
    const float b0 = W00 * j2 + W01 * j3 + W02 * j4, b1 = W01 * j2 + W11 * j3 + W12 * j4, b2 = W02 * j2 + W12 * j3 + W22 * j4;
    const float c0 = W00 * j5 + W01 * j6 + W02 * j7, c1 = W01 * j5 + W11 * j6 + W12 * j7, c2 = W02 * j5 + W12 * j6 + W22 * j7;
    // second-derivative vectors a..f dotted with S (rows of hang: a2 a3 b2 b3 c2 c3 d1 d2 d3 e1 e2 e3 f1 f2 f3)
    const float4* hv = reinterpret_cast<const float4*>(c.hang);
    const float4 h0 = hv[0], h1 = hv[1], h2 = hv[2], h3 = hv[3], h4 = hv[4], h5 = hv[5], h6 = hv[6], h7 = hv[7], h8 = hv[8],
                 h9 = hv[9], h10 = hv[10];
    const float h44 = c.hang[44];
    const float hA2 = h0.x * x + h0.y * y + h0.z * z, hA3 = h0.w * x + h1.x * y + h1.y * z;
    const float hB2 = h1.z * x + h1.w * y + h2.x * z, hB3 = h2.y * x + h2.z * y + h2.w * z;
    const float hC2 = h3.x * x + h3.y * y + h3.z * z, hC3 = h3.w * x + h4.x * y + h4.y * z;
    const float hD1 = h4.z * x + h4.w * y + h5.x * z, hD2 = h5.y * x + h5.z * y + h5.w * z, hD3 = h6.x * x + h6.y * y + h6.z * z;
    const float hE1 = h6.w * x + h7.x * y + h7.y * z, hE2 = h7.z * x + h7.w * y + h8.x * z, hE3 = h8.y * x + h8.z * y + h8.w * z;
    const float hF1 = h9.x * x + h9.y * y + h9.z * z, hF2 = h9.w * x + h10.x * y + h10.y * z,
                hF3 = h10.z * x + h10.w * y + h44 * z;
    // upper triangle, row-major: (0,0..5) (1,1..5) (2,2..5) (3,3..5) (4,4..5) (5,5)
    a.add<FIRST>(6 + 0, W00); a.add<FIRST>(6 + 1, W01); a.add<FIRST>(6 + 2, W02);
    a.add<FIRST>(6 + 3, a0); a.add<FIRST>(6 + 4, b0); a.add<FIRST>(6 + 5, c0);
    a.add<FIRST>(6 + 6, W11); a.add<FIRST>(6 + 7, W12); a.add<FIRST>(6 + 8, a1); a.add<FIRST>(6 + 9, b1);
    a.add<FIRST>(6 + 10, c1);
    a.add<FIRST>(6 + 11, W22); a.add<FIRST>(6 + 12, a2); a.add<FIRST>(6 + 13, b2); a.add<FIRST>(6 + 14, c2);
    a.add<FIRST>(6 + 15, (j0 * a1 + j1 * a2) + (hA2 * ps.S1 + hA3 * ps.S2));
    a.add<FIRST>(6 + 16, (j0 * b1 + j1 * b2) + (hB2 * ps.S1 + hB3 * ps.S2));
    a.add<FIRST>(6 + 17, (j0 * c1 + j1 * c2) + (hC2 * ps.S1 + hC3 * ps.S2));
    a.add<FIRST>(6 + 18, (j2 * b0 + j3 * b1 + j4 * b2) + (hD1 * ps.S0 + hD2 * ps.S1 + hD3 * ps.S2));
    a.add<FIRST>(6 + 19, (j2 * c0 + j3 * c1 + j4 * c2) + (hE1 * ps.S0 + hE2 * ps.S1 + hE3 * ps.S2));
    a.add<FIRST>(6 + 20, (j5 * c0 + j6 * c1 + j7 * c2) + (hF1 * ps.S0 + hF2 * ps.S1 + hF3 * ps.S2));
  }
}

// neighbourhood of one transformed point for the four pclomp::NeighborSearchMethod values
template <int METHOD, bool HESS>
__device__ __forceinline__ void process_point(const NdtLaunch& L, const NdtControl& c, const RankWord* idx, const float4 p,
                                              float gd2, Accum& acc) {
  const float3 xt = transform_point(c.T, p);
  const GridGeom& g = L.geom;
  const int ri = lookup_cell_fast(xt.x, g.leaf, g.inv_leaf) - g.min_b[0],
            rj = lookup_cell_fast(xt.y, g.leaf, g.inv_leaf) - g.min_b[1],
            rk = lookup_cell_fast(xt.z, g.leaf, g.inv_leaf) - g.min_b[2];
  PairSums ps = {};
  const float d1f = (float)L.d1;
  if (METHOD == 2 || METHOD == 3) {  // DIRECT7 (voxel_grid_covariance_omp_impl.hpp:418-433) / DIRECT1
    // in-grid tests per axis (impl.hpp:382-392), shared by the probes
    const bool ix = (unsigned)ri < (unsigned)g.div_b[0], iy = (unsigned)rj < (unsigned)g.div_b[1],
               iz = (unsigned)rk < (unsigned)g.div_b[2];
    const int lin = ri + rj * g.mul[1] + rk * g.mul[2];
    int r[7];
    r[0] = (ix && iy && iz) ? probe_lin(idx, lin) : -1;
    if (METHOD == 2) {
      const bool yz = iy && iz, xz = ix && iz, xy = ix && iy;
      r[1] = (yz && (unsigned)(ri + 1) < (unsigned)g.div_b[0]) ? probe_lin(idx, lin + 1) : -1;
      r[2] = (yz && (unsigned)(ri - 1) < (unsigned)g.div_b[0]) ? probe_lin(idx, lin - 1) : -1;
      r[3] = (xz && (unsigned)(rj + 1) < (unsigned)g.div_b[1]) ? probe_lin(idx, lin + g.mul[1]) : -1;
      r[4] = (xz && (unsigned)(rj - 1) < (unsigned)g.div_b[1]) ? probe_lin(idx, lin - g.mul[1]) : -1;
      r[5] = (xy && (unsigned)(rk + 1) < (unsigned)g.div_b[2]) ? probe_lin(idx, lin + g.mul[2]) : -1;
      r[6] = (xy && (unsigned)(rk - 1) < (unsigned)g.div_b[2]) ? probe_lin(idx, lin - g.mul[2]) : -1;
      // A neighbour that NO lane of the warp has (the +-z cells of ground points, the far side of a facade) is skipped as a
      // whole: a warp holds 32 consecutive points of one LiDAR ring, so its lanes mostly miss the same cells. Masked lanes
      // contribute exact zeros, so skipping a probe nobody hit changes no bit of the sums.
#pragma unroll
      for (int k = 0; k < 7; k++)
        if (!B200_SKIP_EMPTY_PROBES || __any_sync(__activemask(), r[k] >= 0))  // (a lane that hit is in the mask itself)
          accumulate_pair<HESS>(load_record(L.records + max(r[k], 0)), r[k] >= 0, xt, d1f, gd2, ps);
    } else {
      accumulate_pair<HESS>(load_record(L.records + max(r[0], 0)), r[0] >= 0, xt, d1f, gd2, ps);
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
          accumulate_pair<HESS>(load_record(L.records + r), true, xt, d1f, gd2, ps);
        }
  } else {  // KDTREE: radiusSearch over voxel centroids (voxel_grid_covariance_omp.h:470-499), over the build cells
    for_radius_voxels<true>(g, idx, L.centroids, L.resolution, L.radius2, xt,
                            [&](int r) { accumulate_pair<HESS>(load_record(L.records + r), true, xt, d1f, gd2, ps); });
  }
  if (ps.hits) {
    if (acc.first) apply_point<HESS, true>(p, ps, c, gd2, acc);
    else apply_point<HESS, false>(p, ps, c, gd2, acc);
    acc.first = false;
  }
}

// =====================================================================================================
// controller (runs warp-uniformly in warp 0 of the controller CTA; state in shared memory)
// =====================================================================================================
// LU with partial pivoting entirely in registers (all indices static after unrolling). Returns false when a pivot
// collapses (rank deficiency) — the caller then uses the SVD path that reproduces JacobiSVD's truncation.
__device__ __forceinline__ bool lu_solve6(const double* H, const double* b, double* x) {
  double A[6][7];
  double amax = 0;
  bool finite = true;
#pragma unroll
  for (int r = 0; r < 6; r++) {
#pragma unroll
    for (int c = 0; c < 6; c++) {
      A[r][c] = H[r * 6 + c];
      double a = fabs(A[r][c]);
      finite = finite && (a <= 1.7e308);
      amax = fmax(amax, a);
    }
    A[r][6] = b[r];
  }
  if (!finite) {
#pragma unroll
    for (int i = 0; i < 6; i++) x[i] = NAN;
    return true;  // NaN/inf propagate like the SVD would (delta_p_norm != delta_p_norm branch, :134-139)
  }
  if (!(amax > 0)) return false;
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 6; k++) {
    int piv = k;
    double pm = fabs(A[k][k]);
#pragma unroll
    for (int r = k + 1; r < 6; r++) {
      double v = fabs(A[r][k]);
      if (v > pm) {
        pm = v;
        piv = r;
      }
    }
    if (pm <= 1e-13 * amax) ok = false;
#pragma unroll
    for (int r = k + 1; r < 6; r++) {
      const bool sw = (r == piv);
#pragma unroll
      for (int c = k; c < 7; c++) {
        double t0 = A[k][c], t1 = A[r][c];
        A[k][c] = sw ? t1 : t0;
        A[r][c] = sw ? t0 : t1;
      }
    }
    const double inv = 1.0 / A[k][k];
#pragma unroll
    for (int r = k + 1; r < 6; r++) {
      const double f = A[r][k] * inv;
#pragma unroll
      for (int c = k + 1; c < 7; c++) A[r][c] -= f * A[k][c];
    }
  }
  if (!ok) return false;
#pragma unroll
  for (int k = 5; k >= 0; k--) {
    double s = A[k][6];
#pragma unroll
    for (int c = k + 1; c < 6; c++) s -= A[k][c] * x[c];
    x[k] = s / A[k][k];
  }
  return true;
}

struct CtlShared {
  NdtState st;
  NdtControl next;  // control block under construction (then copied to global by the whole warp)
  double tot[SLOT_COUNT];
  int done;
  int build;          // 1: the controller asks the warp to build the control block for st.x_t
  int build_hessian;  // compute_hessian flag of that evaluation
  int build_f64;      // also keep the f64 angle tables (needed by a later K2 pass)
  double fac[8];      // sx, cx, sy, cy, sz, cz, 1, 0 of the pose being built (f64, with the 1e-4 snap)
  float facf[8];      // f32 sin/cos of the same angles (for the transform)
  unsigned code[72];  // shared-memory copy of kAngleTableCode
  int ready;          // per-round: bit w set once reducing warp w has summed all its partial rows
  // the registration this controller is working on (batch launches take new ones from NdtSolverWork::next_job)
  int cur_job;     // index into NdtLaunch::jobs (0 for a single launch)
  int cur_n_src;   // its source size (trans_probability = score / n_src)
  int n_rows;      // evaluator CTAs that own points of it = partial rows to reduce
  int job_done;    // batch: finish() ran this round — hand the result over and start the next registration
  NdtResult result;  // batch: result under construction (copied to the mapped host array by the warp)
  int trace_phase;   // traced launches: st.phase before this round's controller step ...
  int trace_fast;    // ... and 1 when controller_fast handled it
};

// evaluator CTAs that get points of a scan of n_src points: as soon as each gets at least four warps of points, all of
// them (the evaluation is issue-bound per SM, so spreading thin beats filling CTAs)
__host__ __device__ __forceinline__ int rows_for(int n_src, int n_eval_grid) {
  const int want = (n_src + 127) / 128;
  return max(1, min(want, n_eval_grid));
}

// ---- compact f64 helpers ------------------------------------------------------------------------------------
// The controller runs ONCE per evaluation in ONE warp: its cost is the length of its dependent instruction chain
// (measured ~10 cycles per instruction; neither instruction-cache warming nor rolled-vs-unrolled code changed it).
// The per-evaluation path is therefore organised to minimise the number of sequential steps: data-parallel across
// the lanes wherever the mathematics allows it.
__device__ __noinline__ double ddiv(double a, double b) { return a / b; }
__device__ __noinline__ double dsqrt(double a) { return sqrt(a); }

__device__ __noinline__ void dsincos(double x, double* s_out, double* c_out) { sincos_compact(x, s_out, c_out); }

// next pose -> transform + angle tables, by the whole warp: lanes 0..2 evaluate sin/cos of the three angles, then
// every lane evaluates up to three of the 69 table entries from their coded form (ndt_math.cuh) and stores them; lane 0
// forms the 3x4 transform. Nothing here read-modify-writes shared state, so lanes need not run in lockstep.
__device__ __noinline__ void build_control(CtlShared& cs, int lane) {
  const double* x_t = cs.st.x_t;
  const bool want_f64 = cs.build_f64 != 0;
  if (lane < 6) {
    // lanes 0..2: f64 sin/cos of the angle (tables); lanes 3..5: of the angle cast to float — the transform uses
    // cos/sin in float (Eigen::AngleAxis<float>, :811-814): correctly rounded from the f64 value at the float argument
    const int a = lane < 3 ? lane : lane - 3;
    const double ang = x_t[3 + a];
    double sd, cd;
    dsincos(lane < 3 ? ang : (double)(float)ang, &sd, &cd);
    if (lane < 3) {
      if (fabs(ang) < 10e-5) {  // ndt_omp_impl.hpp:292-325
        sd = 0.0;
        cd = 1.0;
      }
      cs.fac[2 * a] = sd;
      cs.fac[2 * a + 1] = cd;
    } else {
      cs.facf[2 * a] = (float)sd;
      cs.facf[2 * a + 1] = (float)cd;
    }
  } else if (lane == 6) {
    cs.fac[6] = 1.0;
    cs.fac[7] = 0.0;
  }
  __syncwarp();
  NdtControl& c = cs.next;
#pragma unroll
  for (int it = 0; it < 3; it++) {  // unrolled: the three entries of a lane are independent chains
    const int e = lane + 32 * it;
    if (e < 69) {
      const double v = angle_table_entry(cs.code[e], cs.fac);  // f64 value (H row d1 carries -sy, :359)
      float fv = (float)v;
      if (e == 24 + 20) fv = -fv;  // the live f32 table keeps +sy (:381)
      if (e < 24) c.jang[e] = fv;
      else c.hang[e - 24] = fv;
      if (want_f64) {
        if (e < 24) cs.st.jd[e] = v;
        else cs.st.hd[e - 24] = v;
      }
    }
  }
  if (lane >= 5 && lane < 8) {
    // T = Translation * Rx * Ry * Rz in float (ndt_omp_impl.hpp:811-814), same product order as pose_to_matrix();
    // lane 5 + r forms row r (lanes 0..4 carry three table entries, the others two)
    const int row = lane - 5;
    const float fsx = cs.facf[0], fcx = cs.facf[1], fsy = cs.facf[2], fcy = cs.facf[3], fsz = cs.facf[4], fcz = cs.facf[5];
    const float a0 = row == 0 ? fcy : (row == 1 ? fsx * fsy : -fcx * fsy);
    const float a1 = row == 0 ? 0.0f : (row == 1 ? fcx : fsx);
    const float a2 = row == 0 ? fsy : (row == 1 ? -fsx * fcy : fcx * fcy);
    const float t0 = __fadd_rn(__fmul_rn(a0, fcz), __fmul_rn(a1, fsz));
    const float t1 = __fadd_rn(__fmul_rn(a0, -fsz), __fmul_rn(a1, fcz));
    const float t3 = (float)x_t[row];
    float* F = cs.st.final_T;  // final_transformation_
    c.T[row * 4 + 0] = t0; c.T[row * 4 + 1] = t1; c.T[row * 4 + 2] = a2; c.T[row * 4 + 3] = t3;
    F[row * 4 + 0] = t0; F[row * 4 + 1] = t1; F[row * 4 + 2] = a2; F[row * 4 + 3] = t3;
    F[12 + row] = 0.0f;
    if (row == 0) {
      F[15] = 1.0f;
      c.mode = EVAL_DERIV;
      c.compute_hessian = cs.build_hessian;
    }
  }
}

// Warp-parallel fast path of the controller for the case every shipped configuration takes: step_max > step_min
// (so computeStepLengthMT performs exactly one evaluation, ndt_omp_impl.hpp:803) and the state is PH_INITIAL or
// PH_LS_FIRST. It performs  [p += dir * a_t; convergence test; ++nr_iterations]  (:143-164), the Newton solve
// (:127-129) by 3x3 block elimination with one matrix element per lane, and the prologue of computeStepLengthMT
// (:761-809). Anything unusual (convergence, ill-conditioned or non-finite Hessian, zero step) returns false BEFORE any
// solver state is written, and the scalar controller() redoes the round from scratch. Scalars are computed redundantly by every lane; lane 0 alone writes the state.
__device__ __noinline__ bool controller_fast(const NdtLaunch& L, CtlShared& cs, int lane) {
  NdtState& st = cs.st;
  const double step_max = L.step_size, step_min = L.trans_eps / 2;
  if (L.mode != NDT_MODE_ALIGN || L.scalar_controller || !((step_max - step_min) > 0)) return false;
  const int phase = st.phase;
  if (phase != PH_INITIAL && phase != PH_LS_FIRST) return false;
  const double* tot = cs.tot;
  int nr_it = st.nr_iterations;
  const double a_prev = st.a_t;
  if (phase == PH_LS_FIRST && (nr_it > L.max_iterations || (nr_it && (fabs(a_prev) < L.trans_eps)))) return false;
  if (phase == PH_LS_FIRST) nr_it += 1;
  // Every lane solves the 6x6 Newton system H x = -g redundantly IN REGISTERS: symmetric elimination (LDL^T, no
  // pivoting — H is definite wherever Newton is meaningful) on the upper triangle, straight-line code with plenty of
  // independent FMAs and not a single shared-memory round trip or warp synchronisation between the dependent steps.
  // A pivot that collapses relative to the largest diagonal entry (or a NaN) hands the round to the scalar controller,
  // whose pivoted LU / SVD reproduce JacobiSVD::solve's behaviour for rank-deficient systems.
  double A[6][6], rhs[6], x[6];  // (the gradient and the pose are re-read from shared memory later: registers are capped at 80)
#pragma unroll
  for (int r = 0; r < 6; r++) {
#pragma unroll
    for (int c = r; c < 6; c++) A[r][c] = tot[SLOT_H + tri_index(r, c)];
    rhs[r] = -tot[SLOT_G + r];
  }
  if (!ldlt_solve6_upper(A, rhs, x)) return false;
  double n2 = 0.0;
#pragma unroll
  for (int i = 0; i < 6; i++) n2 = fma(x[i], x[i], n2);
  const double norm = sqrt(n2);
  if (norm == 0 || norm != norm) return false;
  const double rn = 1.0 / norm;
  double dir[6], dd = 0.0;
#pragma unroll
  for (int k = 0; k < 6; k++) {
    dir[k] = x[k] * rn;
    dd = fma(tot[SLOT_G + k], dir[k], dd);
  }
  double d_phi_0 = -dd;
  double sgn = 1.0;
  if (d_phi_0 >= 0) {
    if (d_phi_0 == 0) return false;
    d_phi_0 *= -1;
    sgn = -1.0;
  }
  double a_t = norm;
  a_t = fmin(a_t, step_max);
  a_t = fmax(a_t, step_min);
  // ---- write phase (nothing of the solver state was touched before this point) ----
  const double score = tot[SLOT_SCORE];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    if (lane == k) {  // static register indexing: lane k owns component k
      const double d = dir[k] * sgn;
      const double pk = (phase == PH_LS_FIRST) ? st.p[k] + st.dir[k] * a_prev : st.p[k];
      st.p[k] = pk;
      st.g[k] = tot[SLOT_G + k];
      st.dir[k] = d;
      st.x_t[k] = pk + d * a_t;
    }
  }
  if (lane == 6) {
    const long long hits = (long long)(tot[SLOT_HITS] + 0.5);
    st.score = score;
    st.hits_last = hits;
    st.hits_total += hits;
    st.evaluations += 1;
    st.nr_iterations = nr_it;
    st.phi_0 = -score;
    st.d_phi_0 = d_phi_0;
    st.a_t = a_t;
    st.step_iterations = 0;
    st.interval_converged = 1;
    st.open_interval = 1;
    st.phase = PH_LS_FIRST;
    cs.build = 1;
    cs.build_hessian = 1;
    cs.build_f64 = 0;
  }
  return true;
}

__device__ __forceinline__ void load_totals(NdtState& st, const double* tot, bool with_hessian) {
  st.score = tot[SLOT_SCORE];
#pragma unroll
  for (int k = 0; k < 6; k++) st.g[k] = tot[SLOT_G + k];
#pragma unroll
  for (int i = 0; i < 6; i++)
#pragma unroll
    for (int j = i; j < 6; j++) {
      double v = with_hessian ? tot[SLOT_H + tri_index(i, j)] : 0.0;
      st.H[i * 6 + j] = v;
      st.H[j * 6 + i] = v;
    }
  st.hits_last = (long long)(tot[SLOT_HITS] + 0.5);
  st.hits_total += st.hits_last;
  st.evaluations += 1;
}

__device__ void finish(const NdtLaunch& L, CtlShared& cs, NdtSolverWork* W, int lane) {
  NdtState& st = cs.st;
  const bool batch = L.jobs != nullptr;
  if (lane == 0) {
    NdtResult& r = batch ? cs.result : W->result;
    for (int k = 0; k < 16; k++) r.final_T[k] = st.final_T[k];
    r.score = st.score;
    r.trans_probability = st.score / (double)cs.cur_n_src;  // ndt_omp_impl.hpp:136,170
    for (int k = 0; k < 6; k++) r.g[k] = st.g[k];
    for (int k = 0; k < 36; k++) r.H[k] = st.H[k];
    r.hits_last = st.hits_last;
    r.hits_total = st.hits_total;
    r.converged = st.converged;
    r.iterations = st.nr_iterations;
    r.evaluations = st.evaluations;
    r.error = 0;
  }
  if (batch) {  // the warp hands the result over and takes the next registration (controller_cta)
    cs.job_done = 1;
    return;
  }
  cs.next.mode = EVAL_DONE;
  cs.done = 1;
}

// batch launches, warp 0 of a controller CTA: take the next unassigned registration. Fills the solver state and
// cs.next (the control block of its first evaluation); when the batch is exhausted the slot is retired (EVAL_DONE).
__device__ __noinline__ void start_next_job(const NdtLaunch& L, CtlShared& cs, int lane, int n_eval_grid) {
  unsigned job = 0;
  if (lane == 0) job = atomicAdd(&L.work->next_job, 1u);
  job = __shfl_sync(0xffffffffu, job, 0);
  if ((int)job >= L.n_jobs) {
    if (lane == 0) {
      cs.next.mode = EVAL_DONE;
      cs.done = 1;
    }
    __syncwarp();
    return;
  }
  const NdtJob* J = L.jobs + job;
  if (J->ready) {  // the scan may still be on its way to the device: wait for the tag the copy stream writes behind it
    const unsigned tag = J->ready_tag;
    const long long t0 = clock64();
    bool ok = true;
    if (lane == 0) {
      while (ld_relaxed_gpu(J->ready) != tag) {
        if (clock64() - t0 > 4 * SPIN_TIMEOUT_CYCLES) {
          ok = false;
          break;
        }
      }
      fence_acq_rel_gpu();
    }
    ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
    if (!ok) {  // the upload never arrived: retire the slot, the host reports the unfinished registrations
      if (lane == 0) {
        cs.next.mode = EVAL_DONE;
        cs.done = 3;
      }
      __syncwarp();
      return;
    }
  }
  {
    const unsigned* src = reinterpret_cast<const unsigned*>(&J->init);
    unsigned* dst = reinterpret_cast<unsigned*>(&cs.next);
    for (int k = lane; k < NDT_CONTROL_WORDS; k += 32) dst[k] = __ldg(src + k);
  }
  if (lane < 6) cs.st.p[lane] = J->p0[lane];
  if (lane < 16) cs.st.final_T[lane] = J->init_final[lane];
  __syncwarp();
  if (lane == 0) {
    NdtState& st = cs.st;
    st.phase = PH_INITIAL;
    st.nr_iterations = 0;
    st.evaluations = 0;
    st.converged = 0;
    st.hits_total = 0;
    st.hits_last = 0;
    st.step_iterations = 0;
    st.a_t = 0;
    cs.next.mode = EVAL_DERIV;
    cs.next.compute_hessian = 1;
    cs.next.job = (int)job;
    cs.cur_job = (int)job;
    cs.cur_n_src = J->n_src;
    cs.n_rows = rows_for(J->n_src, n_eval_grid);
  }
  __syncwarp();
}

// One controller step, executed by ONE thread (lane 0 of warp 0 of the controller CTA): consumes the totals of the
// evaluation that just finished and either requests the control block of the next pose (cs.build) or finishes.
__device__ __noinline__ void controller(const NdtLaunch& L, CtlShared& cs, NdtSolverWork* W) {
  const int lane = 0;
  cs.build = 0;
  NdtState& st = cs.st;
  const double* tot = cs.tot;
  const double mu = 1.e-4, nu = 0.9;  // ndt_omp_impl.hpp:788-790
  const double step_max = L.step_size, step_min = L.trans_eps / 2;
  enum { ACT_NEWTON_BEGIN, ACT_NEWTON_END, ACT_LS_CHECK };
  int act;
  double phi_t = 0, d_phi_t = 0, psi_t = 0, d_psi_t = 0;

  if (L.mode != NDT_MODE_ALIGN) {  // single derivative pass requested through the C-ABI
    load_totals(st, tot, L.init.compute_hessian != 0);
    st.converged = 0;
    finish(L, cs, W, lane);
    return;
  }

  auto eval_point_values = [&]() {
    phi_t = -st.score;
    double dd = 0;  // un-fused like the More-Thuente helpers (ndt_math.cuh): the decisions below are the reference's
#pragma unroll
    for (int k = 0; k < 6; k++) dd = B200_ADDD(dd, B200_MULD(st.g[k], st.dir[k]));
    d_phi_t = -dd;
    psi_t = mt_psi(st.a_t, phi_t, st.phi_0, st.d_phi_0, mu);
    d_psi_t = mt_dpsi(d_phi_t, st.d_phi_0, mu);
  };

  switch (st.phase) {
    case PH_INITIAL:  // result of the initial computeDerivatives (:119)
      load_totals(st, tot, true);
      act = ACT_NEWTON_BEGIN;
      break;
    case PH_LS_FIRST:  // first evaluation inside computeStepLengthMT (:821)
      load_totals(st, tot, true);
      eval_point_values();
      act = ACT_LS_CHECK;
      break;
    case PH_LS_ITER:  // More-Thuente inner evaluation (:865), compute_hessian = false zeroes the Hessian
      load_totals(st, tot, false);
      eval_point_values();
      if (st.open_interval && (psi_t <= 0 && d_psi_t >= 0)) {  // :878-889
        st.open_interval = 0;
        st.f_l = B200_SUBD(B200_ADDD(st.f_l, st.phi_0), B200_MULD(B200_MULD(mu, st.d_phi_0), st.a_l));
        st.g_l = B200_ADDD(st.g_l, B200_MULD(mu, st.d_phi_0));
        st.f_u = B200_SUBD(B200_ADDD(st.f_u, st.phi_0), B200_MULD(B200_MULD(mu, st.d_phi_0), st.a_u));
        st.g_u = B200_ADDD(st.g_u, B200_MULD(mu, st.d_phi_0));
      }
      {
        double a_l = st.a_l, f_l = st.f_l, g_l = st.g_l, a_u = st.a_u, f_u = st.f_u, g_u = st.g_u;
        if (st.open_interval) st.interval_converged = mt_update_interval(a_l, f_l, g_l, a_u, f_u, g_u, st.a_t, psi_t, d_psi_t);
        else st.interval_converged = mt_update_interval(a_l, f_l, g_l, a_u, f_u, g_u, st.a_t, phi_t, d_phi_t);
        st.a_l = a_l; st.f_l = f_l; st.g_l = g_l; st.a_u = a_u; st.f_u = f_u; st.g_u = g_u;
      }
      st.step_iterations++;
      act = ACT_LS_CHECK;
      break;
    default:  // PH_LS_HESSIAN: the K2 pass has written st.H (:912-913)
      act = ACT_NEWTON_END;
      break;
  }

  for (int guard = 0; guard < 8; guard++) {
    if (act == ACT_LS_CHECK) {
      // :834
      if (!st.interval_converged && st.step_iterations < 10 && !(psi_t <= 0 && d_phi_t <= -nu * st.d_phi_0)) {
        double a_t;
        if (st.open_interval) a_t = mt_trial_value(st.a_l, st.f_l, st.g_l, st.a_u, st.f_u, st.g_u, st.a_t, psi_t, d_psi_t);
        else a_t = mt_trial_value(st.a_l, st.f_l, st.g_l, st.a_u, st.f_u, st.g_u, st.a_t, phi_t, d_phi_t);
        a_t = fmin(a_t, step_max);
        a_t = fmax(a_t, step_min);
        st.a_t = a_t;
#pragma unroll
        for (int k = 0; k < 6; k++) st.x_t[k] = st.p[k] + st.dir[k] * a_t;
        cs.build = 1;
        cs.build_hessian = 0;
        cs.build_f64 = 1;
        st.phase = PH_LS_ITER;
        return;
      }
      if (st.step_iterations) {  // :912-913 — needs the f64 radius-neighbourhood Hessian (K2): leave the kernel
        st.phase = PH_LS_HESSIAN;
        cs.next.mode = EVAL_NEED_HESSIAN;
        cs.done = 2;
        return;
      }
      act = ACT_NEWTON_END;
    }
    if (act == ACT_NEWTON_END) {
      // :143-164
#pragma unroll
      for (int k = 0; k < 6; k++) st.p[k] = st.p[k] + st.dir[k] * st.a_t;
      if (st.nr_iterations > L.max_iterations || (st.nr_iterations && (fabs(st.a_t) < L.trans_eps))) st.converged = 1;
      st.nr_iterations++;
      if (st.converged) {
        finish(L, cs, W, lane);
        return;
      }
      act = ACT_NEWTON_BEGIN;
    }
    if (act == ACT_NEWTON_BEGIN) {
      // :127-142 and the prologue of computeStepLengthMT :761-821
      double neg_g[6], dp[6];
#pragma unroll
      for (int k = 0; k < 6; k++) neg_g[k] = -st.g[k];
      if (!lu_solve6(st.H, neg_g, dp)) solve6_svd(st.H, neg_g, dp);
      double n2 = 0;
#pragma unroll
      for (int k = 0; k < 6; k++) n2 += dp[k] * dp[k];
      const double norm = sqrt(n2);
      if (norm == 0 || norm != norm) {
        st.converged = (norm == norm) ? 1 : 0;
        finish(L, cs, W, lane);
        return;
      }
      double dir[6];
#pragma unroll
      for (int k = 0; k < 6; k++) dir[k] = dp[k] / norm;
      st.phi_0 = -st.score;
      double dd = 0;
#pragma unroll
      for (int k = 0; k < 6; k++) dd += st.g[k] * dir[k];
      double d_phi_0 = -dd;
      bool zero_step = false;
      if (d_phi_0 >= 0) {
        if (d_phi_0 == 0) {
          zero_step = true;  // :771-772: zero step, no evaluation
        } else {
          d_phi_0 *= -1;
#pragma unroll
          for (int k = 0; k < 6; k++) dir[k] *= -1;
        }
      }
#pragma unroll
      for (int k = 0; k < 6; k++) st.dir[k] = dir[k];
      st.d_phi_0 = d_phi_0;
      if (zero_step) {
        st.a_t = 0;
        act = ACT_NEWTON_END;
        continue;
      }
      st.step_iterations = 0;
      st.a_l = 0;
      st.a_u = 0;
      st.f_l = mt_psi(0.0, st.phi_0, st.phi_0, d_phi_0, mu);
      st.g_l = mt_dpsi(d_phi_0, d_phi_0, mu);
      st.f_u = st.f_l;
      st.g_u = st.g_l;
      st.interval_converged = (step_max - step_min) > 0 ? 1 : 0;  // :803 (sic)
      st.open_interval = 1;
      double a_t = norm;
      a_t = fmin(a_t, step_max);
      a_t = fmax(a_t, step_min);
      st.a_t = a_t;
#pragma unroll
      for (int k = 0; k < 6; k++) st.x_t[k] = st.p[k] + dir[k] * a_t;
      cs.build = 1;
      cs.build_hessian = 1;
      cs.build_f64 = st.interval_converged ? 0 : 1;
      st.phase = PH_LS_FIRST;
      return;
    }
  }
  st.converged = 0;  // unreachable in practice (two consecutive zero-step iterations terminate); fail safe
  finish(L, cs, W, lane);
}

// Traced align() launches (L.trace != nullptr), whole warp 0 after the step and build_control: one record of the round.
// Kept out of line so that the untraced controller loop is the code it was. Tables and a transform the round did not
// build, and st.H outside the first round of a resumed launch, are written as zeros.
__device__ __noinline__ void trace_round(const NdtLaunch& L, const CtlShared& cs, int lane, int round) {
  unsigned idx = 0;
  if (lane == 0) idx = atomicAdd(&L.work->trace_count, 1u);
  idx = __shfl_sync(0xffffffffu, idx, 0);
  if (idx >= (unsigned)L.trace_cap) return;
  b200reg_ndt_trace_record& R = L.trace[idx];
  const NdtState& st = cs.st;
  const bool resumed = L.resume && round == 0;
  const bool built = cs.build != 0, f64 = built && cs.build_f64 != 0;
  R.tot[lane] = cs.tot[lane];
  for (int k = lane; k < 36; k += 32) R.H[k] = resumed ? st.H[k] : 0.0;
  if (lane < 24) R.jd[lane] = f64 ? st.jd[lane] : 0.0;
  for (int k = lane; k < 45; k += 32) R.hd[k] = f64 ? st.hd[k] : 0.0;
  if (lane < 24) R.jang[lane] = built ? cs.next.jang[lane] : 0.0f;
  for (int k = lane; k < 45; k += 32) R.hang[k] = built ? cs.next.hang[k] : 0.0f;
  if (lane < 12) R.T[lane] = built ? cs.next.T[lane] : 0.0f;
  if (lane < 16) R.final_T[lane] = st.final_T[lane];
  if (lane < 6) {
    R.g[lane] = st.g[lane];
    R.p[lane] = st.p[lane];
    R.dir[lane] = st.dir[lane];
    R.x_t[lane] = st.x_t[lane];
  }
  if (lane == 0) {
    R.round = round;
    R.launch = L.trace_launch;
    R.phase_before = cs.trace_phase;
    R.phase_after = st.phase;
    R.fast = cs.trace_fast;
    R.evaluated = resumed ? 0 : 1;
    R.built = built ? 1 : 0;
    R.build_f64 = f64 ? 1 : 0;
    R.mode = cs.next.mode;
    R.compute_hessian = built ? cs.next.compute_hessian : 0;
    R.interval_converged = st.interval_converged;
    R.open_interval = st.open_interval;
    R.step_iterations = st.step_iterations;
    R.nr_iterations = st.nr_iterations;
    R.evaluations = st.evaluations;
    R.converged = st.converged;
    R.done = cs.done;
    R.pad0 = 0;
    R.hits_total = st.hits_total;
    R.score = st.score;
    R.a_t = st.a_t;
    R.phi_0 = st.phi_0;
    R.d_phi_0 = st.d_phi_0;
    R.a_l = st.a_l;
    R.f_l = st.f_l;
    R.g_l = st.g_l;
    R.a_u = st.a_u;
    R.f_u = st.f_u;
    R.g_u = st.g_u;
    R.pad1 = 0.0f;
  }
}

// Traced launches that start an align(): clear the controller state first, so that fields a solve never writes (the
// fast path keeps no More-Thuente interval) read as zeros in the trace instead of what shared memory held before.
__device__ __noinline__ void trace_clear_state(CtlShared& cs, int tid) {
  int* s = reinterpret_cast<int*>(&cs.st);
  for (int k = tid; k < (int)(sizeof(NdtState) / 4); k += SOLVER_THREADS) s[k] = 0;
  __syncthreads();
}

// =====================================================================================================
// controller CTA
// =====================================================================================================
__device__ __noinline__ void controller_cta(const NdtLaunch& L, CtlShared& cs, double (*warp_part)[SLOT_COUNT], int n_eval_i,
                                            int slot) {
  NdtSolverWork* W = L.work;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool batch = L.jobs != nullptr;
  // sequence number of the control block published at the end of round r: single launches hand round 0's block over
  // in the launch parameters, batch launches publish it (index 0) before the first reduction
  const int pub_shift = batch ? 1 : 0;
  if (L.trace && !L.resume) trace_clear_state(cs, tid);
  // state: fresh, or restored from global after a K2 pass
  if (L.resume) {
    const int* src = reinterpret_cast<const int*>(&W->state);
    int* dst = reinterpret_cast<int*>(&cs.st);
    for (int k = tid; k < (int)(sizeof(NdtState) / 4); k += SOLVER_THREADS) dst[k] = __ldcg(src + k);
  } else if (tid == 0 && !batch) {
    NdtState& st = cs.st;
    for (int k = 0; k < 6; k++) st.p[k] = L.p0[k];
    for (int k = 0; k < 16; k++) st.final_T[k] = L.init_final[k];
    st.phase = PH_INITIAL;
    st.nr_iterations = 0;
    st.evaluations = 0;
    st.converged = 0;
    st.hits_total = 0;
    st.hits_last = 0;
    st.step_iterations = 0;
    st.a_t = 0;
    W->result.error = 2;  // "not finished"; finish() sets 0, the watchdog 1, a K2 request 100
  }
  if (tid == 0) {
    cs.done = 0;
    cs.ready = 0;
    cs.job_done = 0;
    cs.cur_job = 0;
    cs.cur_n_src = L.n_src;
    cs.n_rows = n_eval_i;
  }
  if (tid < 69) cs.code[tid] = kAngleTableCode[tid];
  __syncthreads();
  unsigned long long* ctl_ll = &W->ctl_ll[slot][0][0];
  auto publish = [&](int index) {  // warp 0: {payload, sequence} words, every replica
    const unsigned* src = reinterpret_cast<const unsigned*>(&cs.next);
    const unsigned long long seq = (unsigned long long)ctl_sequence(L.epoch, index) << 32;
    for (int k = lane; k < NDT_CONTROL_WORDS; k += 32) {
      const unsigned long long v = seq | src[k];
#pragma unroll
      for (int c = 0; c < NDT_CTL_COPIES; c++) st_relaxed_gpu_u64(ctl_ll + c * NDT_CTL_LL_WORDS + k, v);
    }
  };
  if (batch) {  // first registration of this slot
    if (warp == 0) {
      if (slot == 0 && L.board.world > 0 && lane < L.board.world)  // header of this rank's rows on every board: {count, tag}
        st_relaxed_sys_u64(L.board.peer[lane] + pose_board_word(L.board, L.board.tag, L.board.rank, L.board.rows, 0),
                           ((unsigned long long)L.board.tag << 32) | (unsigned)L.n_jobs);
      start_next_job(L, cs, lane, n_eval_i);
      publish(0);
    }
    __syncthreads();
    if (cs.done) return;  // more slots than registrations
  }

  const int all_ready = (1 << SOLVER_WARPS) - 2;
  for (int round = 0;; round++) {
    if (warp != 0) {
      // ---- warps 1..23: fixed-order reduction of the evaluators' partial rows --------------------------------------
      // Warp w owns rows w-1, w-1+23, ... in batches of 16: one 16-byte load instruction covers TWO rows (lanes 0..15
      // the first, lanes 16..31 the second, two slots per lane), 8 in flight; the loads double as the arrival poll — a
      // slot still holding NDT_PARTIAL_EMPTY is simply re-loaded. Consumed rows are re-armed for round + 2.
      double* buf = &W->partials[slot][round & 1][0][0];
      const int half = lane >> 4, c2 = (lane & 15) * 2;
      const int stride = SOLVER_WARPS - 1;
      const int n_rows = cs.n_rows;  // rows of the registration evaluated this round (stable until the end-of-round barrier)
      double s0 = 0, s1 = 0;
      bool failed = false;
      const long long t0 = clock64();
      for (int base = 0; (warp - 1) + stride * base < n_rows && !failed; base += 16) {
        unsigned long long va[8], vb[8];
        unsigned pend = 0;
#pragma unroll
        for (int u = 0; u < 8; u++) {
          const int row = (warp - 1) + stride * (base + 2 * u + half);
          va[u] = 0ull;  // bits of +0.0
          vb[u] = 0ull;
          if (row < n_rows) {
            ld_relaxed_gpu_v2(buf + (size_t)row * SLOT_COUNT + c2, va[u], vb[u]);
            if (va[u] == NDT_PARTIAL_EMPTY || vb[u] == NDT_PARTIAL_EMPTY) pend |= 1u << u;
          }
        }
        while (__any_sync(0xffffffffu, pend != 0)) {
#pragma unroll
          for (int u = 0; u < 8; u++) {
            if ((pend >> u) & 1u) {
              const int row = (warp - 1) + stride * (base + 2 * u + half);
              ld_relaxed_gpu_v2(buf + (size_t)row * SLOT_COUNT + c2, va[u], vb[u]);
              if (va[u] != NDT_PARTIAL_EMPTY && vb[u] != NDT_PARTIAL_EMPTY) pend &= ~(1u << u);
            }
          }
          if (clock64() - t0 > SPIN_TIMEOUT_CYCLES) {
            failed = true;
            break;
          }
        }
        if (failed) break;
#pragma unroll
        for (int u = 0; u < 8; u++) {
          s0 += __longlong_as_double((long long)va[u]);
          s1 += __longlong_as_double((long long)vb[u]);
        }
      }
      // even rows (half 0) + odd rows (half 1), fixed order
      const double o0 = __shfl_down_sync(0xffffffffu, s0, 16), o1 = __shfl_down_sync(0xffffffffu, s1, 16);
      if (half == 0) {
        warp_part[warp][c2] = s0 + o0;
        warp_part[warp][c2 + 1] = s1 + o1;
      }
      if (__any_sync(0xffffffffu, failed) && lane == 0) {
        W->result.error = 1;
        cs.done = 3;
      }
      __threadfence_block();
      __syncwarp();
      if (lane == 0) atomicOr(&cs.ready, 1 << warp);
      // re-arm the consumed rows for round + 2 — after the flag, so that no fence of the signalling path has to wait
      // for these stores; they are performed before this warp meets the end-of-round barrier
      for (int i = half; (warp - 1) + stride * i < n_rows; i += 2) {
        const int row = (warp - 1) + stride * i;
        st_relaxed_gpu_v2(buf + (size_t)row * SLOT_COUNT + c2, NDT_PARTIAL_EMPTY, NDT_PARTIAL_EMPTY);
      }
      fence_acq_rel_gpu();
    } else {
      // ---- warp 0: wait for the reducing warps (a shared-memory word), then run the controller step ------------
      // (On its own SM the step costs the same whether or not the warp pre-executes it while waiting — measured — so
      // it simply spins.)
      const long long t0 = clock64();
      while (__shfl_sync(0xffffffffu, *(volatile int*)&cs.ready, 0) != all_ready) {
        if (clock64() - t0 > 2 * SPIN_TIMEOUT_CYCLES) {  // the reducing warps time out first and set cs.done
          if (lane == 0) cs.done = 3;
          break;
        }
      }
      __threadfence_block();
      {
        double t = 0;
#pragma unroll
        for (int w = 1; w < SOLVER_WARPS; w++) t += warp_part[w][lane];
        cs.tot[lane] = t;
      }
      __syncwarp();
      if (lane == 0) cs.build = 0;
      __syncwarp();
      if (cs.done == 3 || round >= NDT_MAX_ROUNDS) {  // watchdog: tell the evaluators to leave
        if (lane == 0) {
          W->result.error = 1;
          cs.done = 3;
          cs.next.mode = EVAL_DONE;
        }
      } else {
        if (L.trace && lane == 0) cs.trace_phase = cs.st.phase;
        const bool handled = controller_fast(L, cs, lane);  // warp-uniform result
        if (L.trace && lane == 0) cs.trace_fast = handled ? 1 : 0;
        if (!handled && lane == 0) controller(L, cs, W);
        __syncwarp();
        if (cs.build) build_control(cs, lane);
        __syncwarp();
        if (L.trace) {
          trace_round(L, cs, lane, round);
          __syncwarp();
        }
        if (batch && cs.job_done) {
          // this registration is finished: its result goes straight to the mapped host array, the slot takes the next one
          const int* src = reinterpret_cast<const int*>(&cs.result);
          int* dst = reinterpret_cast<int*>(L.result_host + cs.cur_job);
          for (int k = lane; k < (int)(sizeof(NdtResult) / 4); k += 32) dst[k] = src[k];
          if (L.board.world > 0 && lane < 16) {
            // ... and its pose to every rank's pose board over NVLink, word by word with the launch tag (engine.hpp)
            const unsigned long long w = ((unsigned long long)L.board.tag << 32) | __float_as_uint(cs.result.final_T[lane]);
            const size_t off = pose_board_word(L.board, L.board.tag, L.board.rank, cs.cur_job, lane);
            for (int p = 0; p < L.board.world; p++) st_relaxed_sys_u64(L.board.peer[p] + off, w);
          }
          __syncwarp();
          if (lane == 0) cs.job_done = 0;
          start_next_job(L, cs, lane, n_eval_i);
        } else if (batch && lane == 0) {
          cs.next.job = cs.cur_job;
          if (cs.done == 2) {  // a K2 pass cannot be served inside a batch launch (the host never batches such configurations)
            cs.next.mode = EVAL_DONE;
            cs.done = 3;
          }
        }
      }
      __syncwarp();
      publish(round + pub_shift);
      if (lane == 0) cs.ready = 0;
    }
    __syncthreads();
    if (cs.done) break;
  }
  if (batch) {
    __threadfence_system();
    return;
  }
  if (cs.done == 2) {  // leaving for a K2 pass: the next launch reads the control block from the work area
    const int* src = reinterpret_cast<const int*>(&cs.next);
    int* dst = reinterpret_cast<int*>(&W->control);
    for (int k = tid; k < NDT_CONTROL_WORDS; k += SOLVER_THREADS) dst[k] = src[k];
  }
  if (cs.done == 2) {  // leaving for a K2 pass: park the state in global memory
    const int* src = reinterpret_cast<const int*>(&cs.st);
    int* dst = reinterpret_cast<int*>(&W->state);
    for (int k = tid; k < (int)(sizeof(NdtState) / 4); k += SOLVER_THREADS) dst[k] = src[k];
    if (tid == 0) W->result.error = 100;
  }
  // the result goes straight to the host (pinned memory mapped into the device address space): the host reads it as
  // soon as the stream has drained, no device-to-host copy on the critical path
  __syncthreads();
  {
    const int* src = reinterpret_cast<const int*>(&W->result);
    int* dst = reinterpret_cast<int*>(L.result_host);
    for (int k = tid; k < (int)(sizeof(NdtResult) / 4); k += SOLVER_THREADS) dst[k] = __ldcg(src + k);
    __threadfence_system();
  }
}

// =====================================================================================================
// the persistent kernel
// =====================================================================================================
template <int METHOD>
__global__ void __launch_bounds__(SOLVER_THREADS, SOLVER_MIN_CTAS) ndt_solver_kernel(const __grid_constant__ NdtLaunch L) {
  extern __shared__ __align__(128) unsigned char dyn_smem[];
  __shared__ double warp_part[SOLVER_WARPS][SLOT_COUNT];

  NdtSolverWork* W = L.work;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  const bool batch = L.jobs != nullptr;
  const int n_slots = batch ? L.n_slots : 1;  // registrations in flight = controller CTAs (the last n_slots of the grid)
  const int n_eval_ctas = (int)gridDim.x - n_slots;
  if ((int)blockIdx.x >= n_eval_ctas) {  // ---- a controller CTA ----
    CtlShared& cs = *reinterpret_cast<CtlShared*>(dyn_smem);
    controller_cta(L, cs, warp_part, n_eval_ctas, (int)blockIdx.x - n_eval_ctas);
    return;
  }
  const int my_rank = (int)blockIdx.x;

  // ---- evaluator CTAs --------------------------------------------------------------------------------------
  // Every evaluator serves all slots in turn: while the controller of one registration reduces, solves and publishes,
  // the evaluators are busy with the other registration's evaluation — the SM's issue slots no longer idle through
  // the sequential part of a Newton round.
  __shared__ __align__(16) NdtControl ctl_s[NDT_MAX_SLOTS];
  __shared__ int abort_flag;
  __shared__ unsigned lapped_to;  // batch: the latest control-block sequence a lapped CTA found (0: none)
  __shared__ __align__(8) unsigned long long tma_bar;
  __shared__ const unsigned char* slot_src[NDT_MAX_SLOTS];
  __shared__ int slot_nsrc[NDT_MAX_SLOTS], slot_job[NDT_MAX_SLOTS], slot_stride[NDT_MAX_SLOTS];
  // dynamic shared memory: [rank index, L.acc_offset bytes][per-thread f32 accumulators][staged points, one block per slot]
  float (*acc_s)[ACC_STRIDE] = reinterpret_cast<float (*)[ACC_STRIDE]>(dyn_smem + L.acc_offset);
  constexpr int PTS_ALLOC = SMEM_POINTS > 0 ? SMEM_POINTS : 1;
  float4 (*pts_s)[PTS_ALLOC] = reinterpret_cast<float4 (*)[PTS_ALLOC]>(dyn_smem + L.pts_offset);
  const RankWord* idx = L.index_in_smem ? reinterpret_cast<const RankWord*>(dyn_smem) : L.index;

  // stage the voxel rank index into shared memory with TMA bulk copies (once per launch)
  if (L.index_in_smem) {
    const unsigned bytes = ((unsigned)L.geom.n_words * 8u + 15u) & ~15u;
    if (tid == 0) {
      mbar_init(&tma_bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&tma_bar, bytes);
      for (unsigned off = 0; off < bytes; off += 16384u) {
        unsigned chunk = min(16384u, bytes - off);
        tma_bulk_g2s(dyn_smem + off, reinterpret_cast<const unsigned char*>(L.index) + off, chunk, &tma_bar);
      }
    }
  }

  // This CTA's share of a scan, staged once into shared memory for the whole registration. The scan is dealt out
  // in units of 32 consecutive points (one warp's worth: consecutive points of a LiDAR ring are spatial neighbours and
  // hit the same voxels, so a warp's record loads coalesce), unit u going to evaluator u mod n_rows: every CTA gets a
  // mix of near and far rings, which evens out the per-CTA evaluation time (measured 2.3 .. 5.1 us with contiguous
  // chunks — the evaluation is issue-bound and the barrier waits for the slowest CTA).
  const int n_eval = n_eval_ctas;
  // point gi of a cloud of `stride`-byte records (16: one aligned 16-byte load; anything else: three float loads)
  auto load_point = [](const unsigned char* base, int stride, int gi) {
    const unsigned char* p = base + (size_t)gi * (size_t)stride;
    if (stride == 16) return *reinterpret_cast<const float4*>(p);
    const float* f = reinterpret_cast<const float*>(p);
    return make_float4(f[0], f[1], f[2], 1.0f);
  };
  auto stage_points = [&](int s, const unsigned char* src, int stride, int n_src) {
    const int n_rows = rows_for(n_src, n_eval);
    if (my_rank >= n_rows) return;
    const int n_units = (n_src + 31) >> 5;
    const int my_units = (n_units > my_rank) ? (n_units - my_rank + n_rows - 1) / n_rows : 0;
    const int n_staged = min(my_units * 32, SMEM_POINTS);
    for (int j = tid; j < n_staged; j += SOLVER_THREADS) {  // thread tid later reads exactly the slots it writes here
      const int gi = (((j >> 5) * n_rows + my_rank) << 5) + (j & 31);
      pts_s[s][j] = (gi < n_src) ? load_point(src, stride, gi) : make_float4(0.f, 0.f, 0.f, 0.f);  // padding slot of the ragged last unit
    }
  };
  if (tid < NDT_MAX_SLOTS) slot_job[tid] = -1;
  if (tid == 0) {
    abort_flag = 0;
    lapped_to = 0u;
  }
  __syncthreads();
  if (!batch) stage_points(0, reinterpret_cast<const unsigned char*>(L.src), 16, L.n_src);

  if (L.index_in_smem) {
    long long t0 = clock64();
    while (!mbar_try_wait(&tma_bar, 0)) {
      if (clock64() - t0 > SPIN_TIMEOUT_CYCLES) {  // a partially staged index must never be evaluated
        W->result.error = 1;
        abort_flag = 1;
        break;
      }
    }
  }
  bool skip_eval = L.resume != 0;
  const float gd2 = (float)L.d2;
  const int pub_shift = batch ? 1 : 0;  // see controller_cta

  int rounds[NDT_MAX_SLOTS];
  bool alive[NDT_MAX_SLOTS];
#pragma unroll
  for (int k = 0; k < NDT_MAX_SLOTS; k++) {
    rounds[k] = 0;
    alive[k] = k < n_slots;
  }
  int n_alive = n_slots;
  for (int s = 0; n_alive > 0; s = (s + 1 >= n_slots) ? 0 : s + 1) {
    int round = 0;
    bool live = false;
#pragma unroll
    for (int k = 0; k < NDT_MAX_SLOTS; k++)
      if (k == s) {
        round = rounds[k];
        live = alive[k];
      }
    if (!live) continue;

    // ---- (0) the control block of (slot s, round): from the launch parameters (single launch, round 0) or from the
    // slot's controller CTA — thread k polls word k until it carries the expected sequence number (one 64-bit load
    // brings payload and validity together) -----------------------------------------------------------------------
    // A batch slot's controller waits only for the evaluators that own points of its current registration. The others
    // still step through its rounds, and one busy with a long evaluation for another slot can be lapped: the block it
    // waits for has already been replaced by a later one. Such a CTA owns no points of the rounds it missed, so it takes
    // the latest block instead (lapped_to: the sequence every word of it must carry). A CTA that owns points of a round
    // cannot be lapped there, since the controller waits for its row.
    unsigned want = ctl_sequence(L.epoch, round - 1 + pub_shift);
    for (;;) {
      if (tid < NDT_CONTROL_WORDS) {
        unsigned payload;
        if (!batch && round == 0) {
          const int* src = L.resume ? reinterpret_cast<const int*>(&W->control) : reinterpret_cast<const int*>(&L.init);
          payload = (unsigned)(L.resume ? __ldcg(src + tid) : src[tid]);
        } else {
          const unsigned long long* wsrc = &W->ctl_ll[s][my_rank % NDT_CTL_COPIES][tid];
          const long long t0 = clock64();
          unsigned long long v;
          for (;;) {
            v = ld_relaxed_gpu_u64(wsrc);
            const int ahead = (int)((unsigned)(v >> 32) - want);  // < 0: an older block (this launch's or an earlier one's)
            if (ahead == 0) break;
            if (ahead > 0 && ahead < 65536) {
              atomicMax(&lapped_to, (unsigned)(v >> 32));
              break;
            }
            if (clock64() - t0 > SPIN_TIMEOUT_CYCLES) {
              W->result.error = 1;
              abort_flag = 1;
              break;
            }
          }
          payload = (unsigned)v;
        }
        reinterpret_cast<unsigned*>(&ctl_s[s])[tid] = payload;
      }
      __syncthreads();
      const unsigned to = lapped_to;
      if (to == 0u || abort_flag) break;
      __syncthreads();  // every thread has read lapped_to
      if (tid == 0) lapped_to = 0u;
      __syncthreads();
      round += (int)(to - want);
      want = to;
      // (the words are read again for exactly `to`, or for a later block if the controller moved on once more)
    }
    const NdtControl& ctl = ctl_s[s];
    if (ctl.mode != EVAL_DERIV || abort_flag) {  // this slot is finished (or the watchdog fired)
#pragma unroll
      for (int k = 0; k < NDT_MAX_SLOTS; k++)
        if (k == s) alive[k] = false;
      n_alive--;
      continue;
    }

    // ---- (0b) batch: a new registration on this slot — restage its points ----------------------------------------
    if (batch && ctl.job != slot_job[s]) {
      __syncthreads();  // everybody has compared before the entry changes
      if (tid == 0) {
        const NdtJob* J = L.jobs + ctl.job;
        slot_job[s] = ctl.job;
        slot_src[s] = J->src;
        slot_nsrc[s] = J->n_src;
        slot_stride[s] = J->stride;
      }
      __syncthreads();
      stage_points(s, slot_src[s], slot_stride[s], slot_nsrc[s]);
    }
    const unsigned char* __restrict__ src = batch ? slot_src[s] : reinterpret_cast<const unsigned char*>(L.src);
    const int src_stride = batch ? slot_stride[s] : 16;
    const int n_src = batch ? slot_nsrc[s] : L.n_src;
    const int n_rows = rows_for(n_src, n_eval);
    const bool active = my_rank < n_rows;  // small scans are spread over fewer evaluators (rows_for)
    const int n_units = (n_src + 31) >> 5;
    const int my_units = (active && n_units > my_rank) ? (n_units - my_rank + n_rows - 1) / n_rows : 0;
    const int n_local = my_units * 32;  // local slots (the last unit of the scan may be ragged)
    auto global_index = [&](int j) { return (((j >> 5) * n_rows + my_rank) << 5) + (j & 31); };
    const int n_staged = min(n_local, SMEM_POINTS);
    const float4* pts = pts_s[s];

    if (active) {
      // ---- (1) evaluate this CTA's points ---------------------------------------------------------------
      Accum acc;
      acc.s = acc_s;
      acc.tid = tid;
      acc.first = true;
      acc.score = 0.0;
      acc.hits = 0;
      if (!skip_eval) {
        if (ctl.compute_hessian) {
          for (int j = tid; j < n_staged; j += SOLVER_THREADS) {
            if (global_index(j) < n_src) process_point<METHOD, true>(L, ctl, idx, pts[j], gd2, acc);
          }
          for (int j = SMEM_POINTS + tid; j < n_local; j += SOLVER_THREADS) {
            const int gi = global_index(j);
            if (gi < n_src) process_point<METHOD, true>(L, ctl, idx, load_point(src, src_stride, gi), gd2, acc);
          }
        } else {
          for (int j = tid; j < n_staged; j += SOLVER_THREADS) {
            if (global_index(j) < n_src) process_point<METHOD, false>(L, ctl, idx, pts[j], gd2, acc);
          }
          for (int j = SMEM_POINTS + tid; j < n_local; j += SOLVER_THREADS) {
            const int gi = global_index(j);
            if (gi < n_src) process_point<METHOD, false>(L, ctl, idx, load_point(src, src_stride, gi), gd2, acc);
          }
        }
      }

      // ---- (2) per-warp reduction: lane L sums slot L over the warp's 32 columns in fixed order (f64), CTA partial --
      if (acc.first) {
#pragma unroll
        for (int k = 0; k < ACC_SLOTS; k++) acc_s[k][tid] = 0.f;
      }
      double sc = acc.score;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, d);
      const double hc = (double)__reduce_add_sync(0xffffffffu, acc.hits);
      __syncwarp();
      {
        double v = 0.0;
        if (lane >= SLOT_G && lane < SLOT_G + ACC_SLOTS) {
          // 32 columns of this slot: eight 16-byte loads; the four values of a load (four neighbouring threads' sums, each of
          // <= a few points) are added in f32, the eight results in f64, fixed order. (The reference adds every pair's f32
          // contribution to an f64 accumulator; a 4-term f32 pre-sum adds ~1e-7 relative rounding to terms that already carry
          // the f32 rounding of the per-pair products — and takes 100 of the 160 instructions out of this reduction.)
          const float4* row4 = reinterpret_cast<const float4*>(&acc_s[lane - SLOT_G][warp * 32]);
          double p[8];
#pragma unroll
          for (int t = 0; t < 8; t++) {
            const float4 q = row4[t];
            p[t] = (double)__fadd_rn(__fadd_rn(q.x, q.y), __fadd_rn(q.z, q.w));
          }
          v = ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
        } else if (lane == SLOT_SCORE) {
          v = sc;
        } else if (lane == SLOT_HITS) {
          v = hc;
        }
        warp_part[warp][lane] = v;
      }
      __syncthreads();
      if (tid < SLOT_COUNT) {  // warp 0: one plain 8-byte store per slot; a written slot can never equal NDT_PARTIAL_EMPTY
        double sa = 0, sb = 0, sc2 = 0, sd = 0;  // four independent chains, fixed order
#pragma unroll
        for (int w = 0; w < SOLVER_WARPS; w += 4) {
          sa += warp_part[w][tid];
          sb += warp_part[w + 1][tid];
          sc2 += warp_part[w + 2][tid];
          sd += warp_part[w + 3][tid];
        }
        const double sum = (sa + sb) + (sc2 + sd);
        st_relaxed_gpu_u64(reinterpret_cast<unsigned long long*>(&W->partials[s][round & 1][my_rank][tid]),
                           (unsigned long long)__double_as_longlong(sum));
      }
    }
    skip_eval = false;
#pragma unroll
    for (int k = 0; k < NDT_MAX_SLOTS; k++)
      if (k == s) rounds[k] = round + 1;
  }
}

__global__ void arm_partials_kernel(unsigned long long* p, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = NDT_PARTIAL_EMPTY;
}

using KernelFn = void (*)(const NdtLaunch);
KernelFn kernel_for(int method) {
  switch (method) {
    case 0: return ndt_solver_kernel<0>;
    case 1: return ndt_solver_kernel<1>;
    case 3: return ndt_solver_kernel<3>;
    default: return ndt_solver_kernel<2>;
  }
}

}  // namespace

// =====================================================================================================
// host side
// =====================================================================================================
NdtSolver::~NdtSolver() {
  if (d_work_) cudaFree(d_work_);
  if (d_trace_) cudaFree(d_trace_);
  if (h_result_) cudaFreeHost(h_result_);
  if (d_jobs_) cudaFree(d_jobs_);
  if (h_jobs_) cudaFreeHost(h_jobs_);
  if (h_batch_results_) cudaFreeHost(h_batch_results_);
}

void NdtSolver::init(int device, cudaStream_t s) {
  device_ = device;
  stream_ = s;
  cudaDeviceProp prop;
  B200_CUDA(cudaGetDeviceProperties(&prop, device));
  sm_count_ = prop.multiProcessorCount;
  max_smem_optin_ = (int)prop.sharedMemPerBlockOptin;
  B200_CUDA(cudaMalloc(&d_work_, sizeof(NdtSolverWork)));
  B200_CUDA(cudaMemset(d_work_, 0, sizeof(NdtSolverWork)));
  arm_partials_kernel<<<296, 256>>>(reinterpret_cast<unsigned long long*>(&d_work_->partials[0][0][0][0]),
                                    (size_t)NDT_MAX_SLOTS * 2 * NDT_MAX_CTAS * SLOT_COUNT);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaDeviceSynchronize());
  B200_CUDA(cudaMallocHost(&h_result_, sizeof(NdtResult)));
  std::memset(h_result_, 0, sizeof(NdtResult));
  for (int m = 0; m < 4; m++)
    B200_CUDA(cudaFuncSetAttribute(kernel_for(m), cudaFuncAttributeMaxDynamicSharedMemorySize, SOLVER_MAX_DYN_SMEM));
}

void NdtSolver::set_trace(int capacity) {
  if (d_trace_) cudaFree(d_trace_);
  d_trace_ = nullptr;
  trace_cap_ = 0;
  if (capacity <= 0) return;
  B200_CUDA(cudaMalloc(&d_trace_, (size_t)capacity * sizeof(b200reg_ndt_trace_record)));
  trace_cap_ = capacity;
  B200_CUDA(cudaMemsetAsync(&d_work_->trace_count, 0, sizeof(unsigned), stream_));
  B200_CUDA(cudaStreamSynchronize(stream_));
}
int NdtSolver::read_trace(b200reg_ndt_trace_record* out, int cap) {
  if (!trace_cap_) return 0;
  unsigned n = 0;
  B200_CUDA(cudaMemcpyAsync(&n, &d_work_->trace_count, sizeof(unsigned), cudaMemcpyDeviceToHost, stream_));
  B200_CUDA(cudaStreamSynchronize(stream_));
  const int m = std::min(std::min((int)n, trace_cap_), cap);
  if (out && m > 0)
    B200_CUDA(cudaMemcpyAsync(out, d_trace_, (size_t)m * sizeof(b200reg_ndt_trace_record), cudaMemcpyDeviceToHost, stream_));
  B200_CUDA(cudaStreamSynchronize(stream_));
  return (int)n;
}
const double* NdtSolver::state_jd() const { return d_work_->state.jd; }
const double* NdtSolver::state_hd() const { return d_work_->state.hd; }
const float* NdtSolver::control_T() const { return d_work_->control.T; }

void NdtSolver::fetch_result() {  // slow path: the kernel did not get to write the host copy
  B200_CUDA(cudaMemcpyAsync(h_result_, &d_work_->result, sizeof(NdtResult), cudaMemcpyDeviceToHost, stream_));
  B200_CUDA(cudaStreamSynchronize(stream_));
}

void NdtSolver::reset_barrier() {
  // after a watchdog abort: clear the error word, re-arm every partial slot and the role-election counters
  B200_CUDA(cudaMemsetAsync(d_work_, 0, 16, stream_));
  arm_partials_kernel<<<296, 256, 0, stream_>>>(reinterpret_cast<unsigned long long*>(&d_work_->partials[0][0][0][0]),
                                                (size_t)NDT_MAX_SLOTS * 2 * NDT_MAX_CTAS * SLOT_COUNT);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaStreamSynchronize(stream_));
}

namespace {
// pose parameters and first control block of a registration that starts at the (row-major) guess T:
// final_transformation_ = guess (or identity), p = (t, eulerAngles(0,1,2)) in float -> double
// (ndt_omp_impl.hpp:95-111); the first evaluation transforms the source by the guess matrix itself.
void initial_pose(const float* T, const double* p6, double* p0, float* init_final, NdtControl& init, int compute_hessian) {
  std::memcpy(init_final, T, 16 * sizeof(float));
  for (int k = 0; k < 12; k++) init.T[k] = T[k];
  if (p6) {
    for (int k = 0; k < 6; k++) p0[k] = p6[k];
  } else {
    float R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    float ang[3];
    euler_angles_012(R, ang);
    p0[0] = T[3];
    p0[1] = T[7];
    p0[2] = T[11];
    p0[3] = ang[0];
    p0[4] = ang[1];
    p0[5] = ang[2];
  }
  angle_tables(p0, init.jang, init.hang, nullptr, nullptr);
  init.mode = EVAL_DERIV;
  init.compute_hessian = compute_hessian;
  init.job = 0;
  for (int k = 0; k < 4; k++) init.pad[k] = 0;
}
}  // namespace

void NdtSolver::fill_common(NdtLaunch& L, const VoxelMap& map, const NdtConfig& cfg, int mode, int n_slots, size_t& dyn_smem) {
  L.index = map.index.ptr;
  L.records = map.records.ptr;
  L.icov_d = map.icov_d.ptr;
  L.centroids = map.centroids.ptr;
  L.work = d_work_;
  L.geom = map.geom;
  L.n_voxels = (int)map.n_voxels;
  L.search_method = cfg.search_method;
  L.mode = mode;
  L.scalar_controller = scalar_controller ? 1 : 0;
  L.epoch = epoch_++;
  L.max_iterations = cfg.max_iterations;
  L.resolution = cfg.resolution;
  L.radius2 = static_cast<float>((double)cfg.resolution * (double)cfg.resolution);
  GaussConsts gc = gauss_constants(cfg.outlier_ratio, cfg.resolution);
  L.d1 = gc.d1;
  L.d2 = gc.d2;
  L.d3 = gc.d3;
  L.step_size = cfg.step_size;
  L.trans_eps = cfg.trans_eps;
  // dynamic shared memory: the rank index when it fits (<= 64 KB), then the per-thread accumulators; the controller
  // CTAs overlay their own state on the same bytes
  const size_t index_bytes = ((size_t)map.geom.n_words * 8 + 127) & ~(size_t)127;
  L.index_in_smem = (map.geom.n_words > 0 && index_bytes <= (size_t)SOLVER_MAX_INDEX_SMEM) ? 1 : 0;
  // the index region is rounded up to 8 KB steps: consecutive targets of similar extent (the loop-closure sweep, the
  // frontend's growing map) then launch with the SAME dynamic shared-memory size — a cooperative launch whose size differs
  // from the previous one's costs the driver ~0.1 ms of extra work (measured on the loop-closure pairs)
  L.acc_offset = L.index_in_smem ? (int)((index_bytes + 8191) & ~(size_t)8191) : 0;
  L.pts_offset = L.acc_offset + ACC_BYTES_PAD;
  // (a single registration stages one block of points: the shared-memory carve-out, and with it the L1 left for the
  // voxel-record gathers, stays what it was before batching existed)
  dyn_smem = std::max((size_t)L.pts_offset + (size_t)n_slots * PTS_BYTES, sizeof(CtlShared));
  dyn_smem = (dyn_smem + 127) & ~(size_t)127;
  index_in_smem_ = L.index_in_smem;
  if (!fits_checked_) {  // the largest configuration (64 KB index + accumulators) fits or nothing does
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel_for(cfg.search_method), SOLVER_THREADS,
                                                            SOLVER_MAX_DYN_SMEM));
    if (per_sm < 1) throw CudaError("ndt_solver_kernel does not fit on an SM");
    fits_checked_ = true;
  }
}

int NdtSolver::eval_ctas_for(size_t n_src) const {
  // one CTA per SM, all co-resident (cooperative launch); NDT_MAX_SLOTS SMs are left to controller CTAs in EVERY launch
  // so that single and batched registrations partition a scan identically (bitwise-equal results)
  const int max_ctas = std::min(sm_count_, NDT_MAX_CTAS);
  return rows_for((int)n_src, std::max(1, max_ctas - NDT_MAX_SLOTS));
}

void NdtSolver::launch(const VoxelMap& map, const float4* src, size_t n_src, const NdtConfig& cfg, int mode,
                       const float* T_rowmajor16, const double* p6, int compute_hessian, int resume) {
  NdtLaunch L{};
  size_t dyn_smem = 0;
  fill_common(L, map, cfg, mode, 1, dyn_smem);
  L.src = src;
  L.result_host = h_result_;
  h_result_->error = 3;  // "the kernel never wrote a result"
  L.jobs = nullptr;
  L.n_jobs = 1;
  L.n_slots = 1;
  L.n_src = (int)n_src;
  L.resume = resume;
  initial_pose(T_rowmajor16, p6, L.p0, L.init_final, L.init, compute_hessian);
  if (trace_cap_ > 0 && mode == NDT_MODE_ALIGN) {
    trace_launch_ = resume ? trace_launch_ + 1 : 0;
    if (!resume) B200_CUDA(cudaMemsetAsync(&d_work_->trace_count, 0, sizeof(unsigned), stream_));
    L.trace = d_trace_;
    L.trace_cap = trace_cap_;
    L.trace_launch = trace_launch_;
  }

  grid_ = eval_ctas_for(n_src) + 1;  // + the controller CTA
  block_ = SOLVER_THREADS;
  KernelFn fn = kernel_for(cfg.search_method);
  void* args[] = {&L};
  B200_CUDA(cudaLaunchCooperativeKernel((const void*)fn, dim3(grid_), dim3(SOLVER_THREADS), args, dyn_smem, stream_));
  launches += 1;
}

// Behind a batch launch with a pose board: wait until every rank's rows of this launch have arrived in OUR board and
// copy them to mapped host memory. One thread per (rank, row, word); rows beyond a rank's count leave at once. The
// peers' kernels make progress independently of this one, so the wait is bounded by their batch duration; the timeout
// only guards against a peer that never launches (collective misuse / a crashed rank).
__global__ void pose_board_collect_kernel(PoseBoardView B, float* __restrict__ rows_host, int* __restrict__ counts_host,
                                          unsigned long long timeout_ns) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int k = t & 15, row = (t >> 4) % B.rows, src = (t >> 4) / B.rows;
  if (src >= B.world) return;
  const unsigned long long* own = B.peer[B.rank];
  const unsigned long long t0 = globaltimer_ns();
  auto wait_word = [&](const unsigned long long* p, unsigned& payload) {
    for (;;) {
      const unsigned long long w = ld_relaxed_sys_u64(p);
      if ((unsigned)(w >> 32) == B.tag) {
        payload = (unsigned)w;
        return true;
      }
      if (globaltimer_ns() - t0 > timeout_ns) return false;
      __nanosleep(200);
    }
  };
  unsigned count = 0, bits = 0;
  if (!wait_word(own + pose_board_word(B, B.tag, src, B.rows, 0), count)) {
    counts_host[B.world] = 1;
    return;
  }
  if (row == 0 && k == 0) counts_host[src] = (int)count;
  if (row >= (int)count) return;
  if (!wait_word(own + pose_board_word(B, B.tag, src, row, k), bits)) {
    counts_host[B.world] = 1;
    return;
  }
  rows_host[((size_t)src * B.rows + row) * 16 + k] = __uint_as_float(bits);
}

// K independent registrations against the same voxel map in ONE cooperative launch, NDT_MAX_SLOTS of them in flight:
// while one registration's controller CTA reduces / solves / publishes, the evaluator CTAs work on the other one.
// Results land in the mapped host array batch_results()[0..n) once the stream has drained.
void NdtSolver::launch_batch(const VoxelMap& map, const BatchItem* items, int n, const NdtConfig& cfg, int slots,
                             b200comm_board* board) {
  if (n <= 0) return;
  if ((size_t)n > jobs_cap_) {
    if (d_jobs_) cudaFree(d_jobs_);
    if (h_jobs_) cudaFreeHost(h_jobs_);
    if (h_batch_results_) cudaFreeHost(h_batch_results_);
    d_jobs_ = nullptr;
    h_jobs_ = nullptr;
    h_batch_results_ = nullptr;
    jobs_cap_ = 0;
    const size_t cap = (size_t)n + 16;
    B200_CUDA(cudaMalloc(&d_jobs_, cap * sizeof(NdtJob)));
    B200_CUDA(cudaMallocHost(&h_jobs_, cap * sizeof(NdtJob)));
    B200_CUDA(cudaMallocHost(&h_batch_results_, cap * sizeof(NdtResult)));
    jobs_cap_ = cap;
  }
  size_t n_max = 0;
  for (int k = 0; k < n; k++) {
    NdtJob& J = h_jobs_[k];
    std::memset(&J, 0, sizeof(J));
    J.src = reinterpret_cast<const unsigned char*>(items[k].src);
    J.n_src = (int)items[k].n_src;
    J.stride = items[k].stride ? items[k].stride : 16;
    J.ready = items[k].ready;
    J.ready_tag = items[k].ready_tag;
    initial_pose(items[k].T_rowmajor16, nullptr, J.p0, J.init_final, J.init, 1);
    J.init.job = k;
    n_max = std::max(n_max, items[k].n_src);
    h_batch_results_[k].error = 3;  // "the kernel never wrote a result"
  }
  B200_CUDA(cudaMemcpyAsync(d_jobs_, h_jobs_, (size_t)n * sizeof(NdtJob), cudaMemcpyHostToDevice, stream_));
  B200_CUDA(cudaMemsetAsync(&d_work_->next_job, 0, sizeof(unsigned), stream_));
  NdtLaunch L{};
  size_t dyn_smem = 0;
  const int n_slots = std::max(1, std::min(std::min(slots, NDT_MAX_SLOTS), n));
  fill_common(L, map, cfg, NDT_MODE_ALIGN, n_slots, dyn_smem);
  L.result_host = h_batch_results_;
  L.jobs = d_jobs_;
  L.n_jobs = n;
  L.n_slots = n_slots;
  L.n_src = (int)n_max;
  if (board) L.board = board->view;
  grid_ = eval_ctas_for(n_max) + L.n_slots;
  block_ = SOLVER_THREADS;
  KernelFn fn = kernel_for(cfg.search_method);
  void* args[] = {&L};
  B200_CUDA(cudaLaunchCooperativeKernel((const void*)fn, dim3(grid_), dim3(SOLVER_THREADS), args, dyn_smem, stream_));
  launches += 1;
}

void NdtSolver::launch_board_collect(b200comm_board* board) {
  const PoseBoardView& B = board->view;
  board->h_counts[B.world] = 0;  // the kernel's timeout flag
  const int threads = B.world * B.rows * 16;
  pose_board_collect_kernel<<<(threads + 255) / 256, 256, 0, stream_>>>(B, board->h_rows, board->h_counts,
                                                                       (unsigned long long)(board->timeout_s * 1e9));
  B200_CUDA(cudaGetLastError());
  launches += 1;
}

}  // namespace b200
