// CPU harness of lidarslam_ros2_b200/csrc/session_merge.hpp (the host part of b200sm_merge_session) and of the segmented
// build_edges of csrc/pose_graph.hpp, built by tests/test_session_merge_cpu.py with g++ -ffp-contract=off as the library
// builds them. Matrices are 4x4 row-major doubles unless said otherwise.
#include <cstring>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/session_merge.hpp"

using namespace b200;

namespace {
MergeEdge row(const double* Pa, const double* Pb, const double* Z, double da, double db, double fitness) {
  MergeEdge e;
  e.a = e.b = 0;
  e.fitness = fitness;
  e.da = da;
  e.db = db;
  std::memcpy(e.Pa, Pa, sizeof(e.Pa));
  std::memcpy(e.Pb, Pb, sizeof(e.Pb));
  std::memcpy(e.Z, Z, sizeof(e.Z));
  return e;
}
MergeTolerance tolerance(const double* t4) { return MergeTolerance{t4[0], t4[1], t4[2], t4[3]}; }
void to_rowmajor16(const pg::Iso& a, double* M) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) M[r * 4 + c] = a.R[r * 3 + c];
    M[r * 4 + 3] = a.t[r];
  }
  M[12] = M[13] = M[14] = 0.0;
  M[15] = 1.0;
}
}  // namespace

extern "C" {

// one row's selection: out = the first top_k a, returns their count
int smh_select_row(const double* D, int n_cand, double threshold, int top_k, int* out) {
  const std::vector<int> r = merge_select_row(D, n_cand, threshold, top_k);
  for (size_t k = 0; k < r.size(); k++) out[k] = r[k];
  return (int)r.size();
}

// n candidates (D, b, a) in any order: out3 = (b, a, index) of the first max_verifications in (D, b, a) order
int smh_order(int n, const double* D, const int* b, const int* a, int max_verifications, int* out_b, int* out_a) {
  std::vector<MergeCandidate> c(n);
  for (int k = 0; k < n; k++) c[k] = {D[k], b[k], a[k], 0};
  merge_order(c, max_verifications);
  for (size_t k = 0; k < c.size(); k++) {
    out_b[k] = c[k].b;
    out_a[k] = c[k].a;
  }
  return (int)c.size();
}

// Z = P_a^-1 (F P_b) with F column-major float; X = T P_b
void smh_edge(const double* Pa, const float* F_col, const double* Pb, double* Z) {
  double F[16];
  merge_final_rowmajor(F_col, F);
  merge_edge(Pa, F, Pb, Z);
}
void smh_place(const double* T, const double* Pb, double* X) { merge_place(T, Pb, X); }

// cycle error of rows i and j, and the tolerance test on given (e_t, e_r, L)
void smh_cycle_error(const double* Pai, const double* Pbi, const double* Zi, const double* Paj, const double* Pbj, const double* Zj,
                     double* e_t, double* e_r) {
  merge_cycle_error(row(Pai, Pbi, Zi, 0, 0, 0), row(Paj, Pbj, Zj, 0, 0, 0), e_t, e_r);
}
int smh_within(double e_t, double e_r, double L, const double* tol4) { return merge_within(e_t, e_r, L, tolerance(tol4)) ? 1 : 0; }

// n accepted rows (16 doubles each of Pa, Pb, Z; da, db, fitness): out = the consistent set in joining order
int smh_inliers(int n, const double* Pa, const double* Pb, const double* Z, const double* da, const double* db, const double* fitness,
                const double* tol4, int* out) {
  std::vector<MergeEdge> rows;
  for (int k = 0; k < n; k++) rows.push_back(row(Pa + 16 * k, Pb + 16 * k, Z + 16 * k, da[k], db[k], fitness[k]));
  const std::vector<int> in = merge_inliers(rows, tolerance(tol4));
  for (size_t k = 0; k < in.size(); k++) out[k] = in[k];
  return (int)in.size();
}

// the edges of build_edges over n poses: segmented (n_seg > 0) or the one-segment overload (n_seg == 0); (from, to) and
// the kept inverse measurement, row-major. Returns the edge count.
int smh_build_edges(int n, const double* poses16, int k, int n_seg, const int* seg_first, int n_loops, const int* loops,
                    const double* rel16, int* from_to, double* zinv16) {
  std::vector<pg::Iso> X(n), rel(n_loops);
  for (int i = 0; i < n; i++) X[i] = pg::iso_from_rowmajor16(poses16 + 16 * i);
  for (int l = 0; l < n_loops; l++) rel[l] = pg::iso_from_rowmajor16(rel16 + 16 * l);
  const std::vector<pg::Edge> E = n_seg > 0 ? pg::build_edges(X, k, std::vector<int>(seg_first, seg_first + n_seg), loops, rel.data(), n_loops)
                                            : pg::build_edges(X, k, loops, rel.data(), n_loops);
  for (size_t e = 0; e < E.size(); e++) {
    from_to[2 * e] = E[e].from;
    from_to[2 * e + 1] = E[e].to;
    to_rowmajor16(E[e].zinv, zinv16 + 16 * e);
  }
  return (int)E.size();
}

// the joint adjustment: segmented edges, LM; out16 = the adjusted poses, res4 = chi2_initial, chi2_final, iterations, trials
int smh_adjust(int n, const double* poses16, int k, int n_seg, const int* seg_first, int n_loops, const int* loops,
               const double* rel16, int max_iterations, double* out16, double* res4) {
  std::vector<pg::Iso> X(n), rel(n_loops);
  for (int i = 0; i < n; i++) X[i] = pg::iso_from_rowmajor16(poses16 + 16 * i);
  for (int l = 0; l < n_loops; l++) rel[l] = pg::iso_from_rowmajor16(rel16 + 16 * l);
  const std::vector<pg::Edge> E = pg::build_edges(X, k, std::vector<int>(seg_first, seg_first + n_seg), loops, rel.data(), n_loops);
  const pg::LmResult r = pg::optimize(X, E, max_iterations);
  for (int i = 0; i < n; i++) to_rowmajor16(X[i], out16 + 16 * i);
  res4[0] = r.chi2_initial;
  res4[1] = r.chi2_final;
  res4[2] = r.iterations;
  res4[3] = r.trials;
  return (int)E.size();
}
}
