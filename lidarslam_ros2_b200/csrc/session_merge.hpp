// Merging a second mapping session into the session's map (b200sm_merge_session), the host part in double precision:
// the order in which candidate pairs are verified, the cycle error of two accepted pairs, the greedy consistent set, and
// the rigid placement of the second session. Header-only and free of CUDA so that a CPU harness
// (tests/hostmath/session_merge_host.cpp, g++ -ffp-contract=off) compiles it as scanmatcher.cu does.
//
// Session A (dst) keeps its frame; session B (src) is in a frame of its own. A verified pair (b, a) gives F, the
// registration's final transform, which maps B's frame into A's near submap b, and the edge Z = P_a^-1 (F P_b) from a to b.
// Two pairs i and j close a cycle through both sessions' odometry:
//   E_ij = Z_i^-1 (P_{a_i}^-1 P_{a_j}) Z_j (P_{b_j}^-1 P_{b_i}),
// the identity when F_i = F_j. The tolerance on E grows with the distance L the cycle travels along the two chains,
// because odometry drift grows along each chain. DESIGN.md section 7b says why there is no max-clique search, no
// covariance-weighted tolerance and no averaging of the transforms.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>

#include "pose_graph.hpp"

namespace b200 {

constexpr int MERGE_MAX_TOP_K = 32, MERGE_MAX_VERIFICATIONS = 1024;
constexpr unsigned long long MERGE_MAX_PAIRS = 1ull << 28;  // 12 bytes a pair: 3.2 GB of scores

// One candidate pair of the cross-session search: query b (src), candidate a (dst), its distance and best shift.
struct MergeCandidate {
  double D;
  int b, a, shift;
};

// The selection of one query row (the device's selection kernel does the same): the a with D[a] < threshold, ordered by
// (D[a], a), the first top_k of them.
inline std::vector<int> merge_select_row(const double* D, int n_cand, double threshold, int top_k) {
  std::vector<int> rows;
  for (int a = 0; a < n_cand; a++)
    if (D[a] < threshold) rows.push_back(a);
  std::sort(rows.begin(), rows.end(), [&](int x, int y) { return D[x] < D[y] || (D[x] == D[y] && x < y); });
  if ((int)rows.size() > top_k) rows.resize(top_k);
  return rows;
}

// Every row's selection together, ordered by (D, b, a); the first max_verifications are verified.
inline void merge_order(std::vector<MergeCandidate>& c, int max_verifications) {
  std::sort(c.begin(), c.end(), [](const MergeCandidate& x, const MergeCandidate& y) {
    if (x.D != y.D) return x.D < y.D;
    if (x.b != y.b) return x.b < y.b;
    return x.a < y.a;
  });
  if ((int)c.size() > max_verifications) c.resize(max_verifications);
}

// 4x4 row-major products with every entry summed k = 0..3 from 0, and the inverse of an Isometry3d (R^T, -R^T t): the
// arithmetic of loop_evaluate's edge, so that Z and the placement are the same bits wherever they are formed.
inline void merge_mul16(const double* A, const double* B, double* C) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      double a = 0;
      for (int k = 0; k < 4; k++) a += A[r * 4 + k] * B[k * 4 + c];
      C[r * 4 + c] = a;
    }
}
inline void merge_inverse16(const double* P, double* inv) {
  const double R[16] = {P[0], P[4], P[8], 0, P[1], P[5], P[9], 0, P[2], P[6], P[10], 0, 0, 0, 0, 1};
  for (int k = 0; k < 16; k++) inv[k] = R[k];
  for (int r = 0; r < 3; r++) inv[r * 4 + 3] = -(inv[r * 4 + 0] * P[3] + inv[r * 4 + 1] * P[7] + inv[r * 4 + 2] * P[11]);
}

// F (the registration's column-major float result) as a row-major double matrix
inline void merge_final_rowmajor(const float* F_colmajor16, double* F) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) F[r * 4 + c] = (double)F_colmajor16[c * 4 + r];
}

// The edge from a to b: Z = P_a^-1 (F P_b), row-major
inline void merge_edge(const double* P_a, const double* F, const double* P_b, double* Z) {
  double to[16], inv[16];
  merge_mul16(F, P_b, to);
  merge_inverse16(P_a, inv);
  merge_mul16(inv, to, Z);
}

// The rigid placement of submap b: X_b = T* P_b, row-major
inline void merge_place(const double* T, const double* P_b, double* X) { merge_mul16(T, P_b, X); }

// An accepted row of the verification, with what the consistency check reads: the poses of both ends (row-major), the
// travelled distances the sessions store, the edge and the registration's fitness.
struct MergeEdge {
  int a, b;
  double fitness;
  double da, db;
  double Pa[16], Pb[16], Z[16];
};

struct MergeTolerance {
  double translation, rotation;              // metres, radians
  double drift_translation, drift_rotation;  // per metre travelled
};

// e_t = |t(E_ij)| and e_r = acos(clamp((tr R(E_ij) - 1) / 2, -1, 1)), with E_ij composed left to right as written above
inline void merge_cycle_error(const MergeEdge& i, const MergeEdge& j, double* e_t, double* e_r) {
  using namespace pg;
  const Iso E = compose(compose(compose(inverse(iso_from_rowmajor16(i.Z)), compose(inverse(iso_from_rowmajor16(i.Pa)), iso_from_rowmajor16(j.Pa))),
                                iso_from_rowmajor16(j.Z)),
                        compose(inverse(iso_from_rowmajor16(j.Pb)), iso_from_rowmajor16(i.Pb)));
  *e_t = std::sqrt((E.t[0] * E.t[0] + E.t[1] * E.t[1]) + E.t[2] * E.t[2]);
  const double c = (((E.R[0] + E.R[4]) + E.R[8]) - 1.0) / 2.0;
  *e_r = std::acos(std::min(1.0, std::max(-1.0, c)));
}

// L = |d_{a_i} - d_{a_j}| + |d_{b_i} - d_{b_j}|
inline double merge_cycle_length(const MergeEdge& i, const MergeEdge& j) { return std::fabs(i.da - j.da) + std::fabs(i.db - j.db); }

inline bool merge_within(double e_t, double e_r, double L, const MergeTolerance& tol) {
  return e_t <= tol.translation + tol.drift_translation * L && e_r <= tol.rotation + tol.drift_rotation * L;
}

inline bool merge_consistent(const MergeEdge& i, const MergeEdge& j, const MergeTolerance& tol) {
  double e_t, e_r;
  merge_cycle_error(i, j, &e_t, &e_r);
  return merge_within(e_t, e_r, merge_cycle_length(i, j), tol);
}

// The inlier set, greedily: the rows in (fitness, index) order, each kept iff it is consistent with every row kept before
// it. Returns indices into `rows`, in the order they joined.
inline std::vector<int> merge_inliers(const std::vector<MergeEdge>& rows, const MergeTolerance& tol) {
  std::vector<int> order(rows.size());
  for (size_t k = 0; k < rows.size(); k++) order[k] = (int)k;
  std::sort(order.begin(), order.end(),
            [&](int x, int y) { return rows[x].fitness < rows[y].fitness || (rows[x].fitness == rows[y].fitness && x < y); });
  std::vector<int> in;
  for (int r : order) {
    bool ok = true;
    for (int q : in)
      if (!merge_consistent(rows[q], rows[r], tol)) {
        ok = false;
        break;
      }
    if (ok) in.push_back(r);
  }
  return in;
}

}  // namespace b200
