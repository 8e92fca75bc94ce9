// TEST INFRASTRUCTURE: compiles the product's host pose-graph optimiser (csrc/pose_graph.hpp) with g++ so that
// tests/test_posegraph_cpu.py can compare it with tests/posegraphref.py on the CPU. Matrices are 4x4 row-major.
#include "../../lidarslam_ros2_b200/csrc/pose_graph.hpp"

using namespace b200::pg;

namespace {
void to_rowmajor16(const Iso& a, double* M) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) M[r * 4 + c] = a.R[r * 3 + c];
    M[r * 4 + 3] = a.t[r];
  }
  M[12] = M[13] = M[14] = 0.0;
  M[15] = 1.0;
}
}  // namespace

extern "C" {
// error and Jacobians (6x6 row-major) of an edge with measurement Z between X_from and X_to
void pg_edge(const double* xf16, const double* xt16, const double* z16, double* e6, double* jf36, double* jt36) {
  const Iso zinv = inverse(iso_from_rowmajor16(z16));
  Iso E;
  edge_error(iso_from_rowmajor16(xf16), iso_from_rowmajor16(xt16), zinv, e6, &E);
  edge_jacobians(E, zinv, jf36, jt36);
}

// doPoseAdjustment on n poses; loops: n_loops (from, to) pairs and their 4x4 relative poses. res4 = chi2_initial,
// chi2_final, iterations, trials; trace: up to trace_cap trials of (iteration, accepted, lambda, chi2). Returns the edges.
int pg_adjust(int n, const double* poses16, int k, int n_loops, const int* loops, const double* loop_rel16, int max_iterations,
              double* out16, double* res4, int trace_cap, double* trace4, int* n_trace) {
  std::vector<Iso> X(n);
  for (int i = 0; i < n; i++) X[i] = iso_from_rowmajor16(poses16 + 16 * i);
  std::vector<Iso> rel(n_loops);
  for (int l = 0; l < n_loops; l++) rel[l] = iso_from_rowmajor16(loop_rel16 + 16 * l);
  const std::vector<Edge> edges = build_edges(X, k, loops, rel.data(), n_loops);
  std::vector<LmTrial> trace;
  const LmResult r = optimize(X, edges, max_iterations, &trace);
  for (int i = 0; i < n; i++) to_rowmajor16(X[i], out16 + 16 * i);
  res4[0] = r.chi2_initial;
  res4[1] = r.chi2_final;
  res4[2] = r.iterations;
  res4[3] = r.trials;
  *n_trace = (int)trace.size();
  for (int t = 0; t < (int)trace.size() && t < trace_cap; t++) {
    trace4[4 * t] = trace[t].iteration;
    trace4[4 * t + 1] = trace[t].accepted;
    trace4[4 * t + 2] = trace[t].lambda;
    trace4[4 * t + 3] = trace[t].chi2;
  }
  return (int)edges.size();
}

// envelope Cholesky solve of a dense (6 n_blocks)^2 row-major system whose off-diagonal nonzero blocks are the given pairs;
// returns 1 on success, 0 when the factorisation fails
int pg_envelope_solve(int n_blocks, int n_pairs, const int* pairs, const double* H, const double* b, double* x) {
  std::vector<std::pair<int, int>> pr;
  for (int p = 0; p < n_pairs; p++) pr.push_back({pairs[2 * p], pairs[2 * p + 1]});
  EnvelopeMatrix M;
  M.init(n_blocks, pr);
  const size_t dim = (size_t)n_blocks * 6;
  for (int r = 0; r < n_blocks; r++)
    for (int c = M.first[r]; c <= r; c++) {
      double* blk = M.block(r, c);
      for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) blk[i * 6 + j] = H[(size_t)(6 * r + i) * dim + 6 * c + j];
    }
  if (!M.factor()) return 0;
  M.solve(b, x);
  return 1;
}

// the envelope's row starts, for the complexity check
void pg_envelope_first(int n_blocks, int n_pairs, const int* pairs, int* first) {
  std::vector<std::pair<int, int>> pr;
  for (int p = 0; p < n_pairs; p++) pr.push_back({pairs[2 * p], pairs[2 * p + 1]});
  EnvelopeMatrix M;
  M.init(n_blocks, pr);
  for (int r = 0; r < n_blocks; r++) first[r] = M.first[r];
}
}
