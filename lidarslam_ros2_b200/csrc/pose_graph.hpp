// Pose-graph optimisation of the backend node, on the host in double precision: GraphBasedSlamComponent::doPoseAdjustment
// (graph_based_slam/src/graph_based_slam_component.cpp:262-319) without g2o. Header-only and free of CUDA so that a CPU
// harness (tests/hostmath/posegraph_host.cpp) compiles it with g++.
//
// g2o is not vendored in the reference. Everything marked *g2o* below is restated from upstream g2o (types/slam3d
// EdgeSE3 / VertexSE3 / isometry3d_mappings, core/optimization_algorithm_levenberg.cpp) and cannot be checked against
// source here; the numpy restatement the tests compare with (tests/posegraphref.py) carries the same note.
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

namespace b200 {

// tf2::fromMsg(pose, Affine3d) = Translation3d(p) * Quaterniond(w, x, y, z): Eigen's QuaternionBase::toRotationMatrix
inline void pose_to_matrix_d(const double* p, const double* q, double* M /* row-major 16 */) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  M[0] = 1.0 - (tyy + tzz); M[1] = txy - twz;         M[2] = txz + twy;          M[3] = p[0];
  M[4] = txy + twz;         M[5] = 1.0 - (txx + tzz); M[6] = tyz - twx;          M[7] = p[1];
  M[8] = txz - twy;         M[9] = tyz + twx;         M[10] = 1.0 - (txx + tyy); M[11] = p[2];
  M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
}

// Eigen::Quaterniond(Matrix3d): the trace / largest-diagonal branches of Eigen's quaternionbase_assign_impl (3x3)
inline void matrix_to_quat_d(const double* R /* row-major 9 */, double* q /* x y z w */) {
  auto m = [&](int r, int c) { return R[r * 3 + c]; };
  double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0.0) {
    t = std::sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m(2, 1) - m(1, 2)) * t;
    q[1] = (m(0, 2) - m(2, 0)) * t;
    q[2] = (m(1, 0) - m(0, 1)) * t;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m(k, j) - m(j, k)) * t;
    q[j] = (m(j, i) + m(i, j)) * t;
    q[k] = (m(k, i) + m(i, k)) * t;
  }
}

namespace pg {

// Isometry3d: rotation row-major and translation. Every product is written out left to right, ((a0 b0 + a1 b1) + a2 b2).
struct Iso {
  double R[9], t[3];
};

inline Iso iso_from_rowmajor16(const double* M) {
  Iso a;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) a.R[r * 3 + c] = M[r * 4 + c];
    a.t[r] = M[r * 4 + 3];
  }
  return a;
}
inline Iso iso_from_colmajor16(const double* M) {
  Iso a;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) a.R[r * 3 + c] = M[c * 4 + r];
    a.t[r] = M[12 + r];
  }
  return a;
}
inline void iso_to_colmajor16(const Iso& a, double* M) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) M[c * 4 + r] = a.R[r * 3 + c];
    M[12 + r] = a.t[r];
    M[r * 4 + 3] = 0.0;
  }
  M[15] = 1.0;
}

inline Iso compose(const Iso& a, const Iso& b) {
  Iso c;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) c.R[i * 3 + j] = (a.R[i * 3] * b.R[j] + a.R[i * 3 + 1] * b.R[3 + j]) + a.R[i * 3 + 2] * b.R[6 + j];
    c.t[i] = ((a.R[i * 3] * b.t[0] + a.R[i * 3 + 1] * b.t[1]) + a.R[i * 3 + 2] * b.t[2]) + a.t[i];
  }
  return c;
}

// Isometry3d::inverse(): R^T, -(R^T t). compose(inverse(P), P) then has a translation of exactly zero and an exactly
// symmetric rotation part, whose compact quaternion is exactly zero: an edge whose measurement is X_from^-1 * X_to of the
// current estimates has an error of exactly 0 (see edge_error).
inline Iso inverse(const Iso& a) {
  Iso b;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) b.R[i * 3 + j] = a.R[j * 3 + i];
    b.t[i] = -((a.R[i] * a.t[0] + a.R[3 + i] * a.t[1]) + a.R[6 + i] * a.t[2]);
  }
  return b;
}

// *g2o* internal::fromVectorMQT: translation d[0..2], rotation fromCompactQuaternion(d[3..5]) = Quaternion(w, v) with
// w = sqrt(1 - |v|^2), the identity when 1 - |v|^2 < 0.
inline Iso from_vector_mqt(const double* d) {
  const double* v = d + 3;
  const double w2 = 1.0 - (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  double M[16];
  if (w2 < 0.0) {
    const double ident[4] = {0.0, 0.0, 0.0, 1.0};
    pose_to_matrix_d(d, ident, M);
  } else {
    const double q[4] = {v[0], v[1], v[2], std::sqrt(w2)};
    pose_to_matrix_d(d, q, M);
  }
  return iso_from_rowmajor16(M);
}

// *g2o* internal::toCompactQuaternion: Quaternion(R) normalised, negated when w < 0; returns w >= 0 and the xyz part.
inline void compact_quaternion(const double* R, double* w, double* v) {
  double q[4];
  matrix_to_quat_d(R, q);
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int k = 0; k < 4; k++) q[k] /= n;
  if (q[3] < 0.0)
    for (int k = 0; k < 4; k++) q[k] = -q[k];
  *w = q[3];
  for (int k = 0; k < 3; k++) v[k] = q[k];
}

// *g2o* EdgeSE3 with an identity information matrix: the edge keeps the inverse of its measurement Z.
struct Edge {
  int from, to;
  Iso zinv;
};

// *g2o* EdgeSE3::computeError: e = toVectorMQT(Z^-1 * X_from^-1 * X_to), translation then the compact quaternion. Evaluated
// as Z^-1 * (X_from^-1 * X_to) so that the error of an edge built from the same estimates is exactly zero; g2o associates
// the product the other way, which differs from this in rounding only.
inline void edge_error(const Iso& xf, const Iso& xt, const Iso& zinv, double* e, Iso* E_out = nullptr) {
  const Iso E = compose(zinv, compose(inverse(xf), xt));
  double w;
  for (int k = 0; k < 3; k++) e[k] = E.t[k];
  compact_quaternion(E.R, &w, e + 3);
  if (E_out) *E_out = E;
}

// d e / d delta of both vertices, 6x6 row-major each (columns: translation increment, compact-quaternion increment), at
// delta = 0 for the increments X <- X * fromVectorMQT(delta) of VertexSE3::oplusImpl (*g2o*). With E = Z^-1 X_from^-1 X_to
// = (R_E, t_E), its compact quaternion (w, q), A = Z^-1 = (R_A, t_A) and [a]x the cross-product matrix:
//   X_to:   e_t = t_E + R_E u                     -> [R_E, 0]
//           q(R_E (1, v))  = q + (w I + [q]x) v   -> [0, w I + [q]x]
//   X_from: E = (A D^-1 A^-1) E, the left factor is (I - 2[R_A v]x, 2[R_A v]x t_A - R_A u) to first order:
//           e_t = t_E + 2 [t_E - t_A]x R_A v - R_A u   -> [-R_A, 2 [t_E - t_A]x R_A]
//           q((1, -R_A v) q) = q - (w I - [q]x) R_A v  -> [0, -(w I - [q]x) R_A]
// These are the exact derivatives; tests/test_posegraph_cpu.py checks them against central differences.
inline void edge_jacobians(const Iso& E, const Iso& zinv, double* Jf, double* Jt) {
  double w, q[3];
  compact_quaternion(E.R, &w, q);
  auto skew = [](const double* a, double* S) {
    S[0] = 0;     S[1] = -a[2]; S[2] = a[1];
    S[3] = a[2];  S[4] = 0;     S[5] = -a[0];
    S[6] = -a[1]; S[7] = a[0];  S[8] = 0;
  };
  auto mul3 = [](const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) C[i * 3 + j] = (A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j]) + A[i * 3 + 2] * B[6 + j];
  };
  std::memset(Jf, 0, 36 * sizeof(double));
  std::memset(Jt, 0, 36 * sizeof(double));
  double Q[9], P[9], M[9], d[3], S[9];
  skew(q, Q);
  for (int k = 0; k < 9; k++) {
    P[k] = Q[k];  // w I + [q]x
    M[k] = -Q[k];  // w I - [q]x
  }
  for (int k = 0; k < 3; k++) {
    P[k * 4] += w;
    M[k * 4] += w;
  }
  for (int k = 0; k < 3; k++) d[k] = 2.0 * (E.t[k] - zinv.t[k]);
  skew(d, S);
  double SR[9], MR[9];
  mul3(S, zinv.R, SR);
  mul3(M, zinv.R, MR);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      Jt[i * 6 + j] = E.R[i * 3 + j];
      Jt[(3 + i) * 6 + 3 + j] = P[i * 3 + j];
      Jf[i * 6 + j] = -zinv.R[i * 3 + j];
      Jf[i * 6 + 3 + j] = SR[i * 3 + j];
      Jf[(3 + i) * 6 + 3 + j] = -MR[i * 3 + j];
    }
}

// doPoseAdjustment's graph (gbs.cpp:276-315): for i > k, edges (i-k+j, i), j = 0..k-1, measurement pose_from^-1 * pose_i;
// then the loop edges in the caller's order. Vertex 0 is never the end of an odometry edge (i - k + j >= 1): it is
// reached through loop edges only, exactly as in the reference.
//
// A map merged from several recordings (b200sm_merge_session) applies the rule per segment: seg_first[s] is the first vertex
// of segment s (ascending, seg_first[0] = 0), and local index i of a segment starting at f0 gives the edges
// (f0 + i-k+j, f0 + i). No odometry edge crosses a segment boundary; with one segment the edges are the ones above.
inline std::vector<Edge> build_edges(const std::vector<Iso>& X, int k, const std::vector<int>& seg_first, const int* loop_from_to,
                                     const Iso* loop_rel, int n_loops) {
  std::vector<Edge> E;
  const int n = (int)X.size();
  for (size_t s = 0; s < seg_first.size(); s++) {
    const int f0 = seg_first[s], f1 = s + 1 < seg_first.size() ? seg_first[s + 1] : n;
    for (int i = k + 1; i < f1 - f0; i++)
      for (int j = 0; j < k; j++) {
        const int f = f0 + i - k + j, t = f0 + i;
        E.push_back({f, t, inverse(compose(inverse(X[f]), X[t]))});
      }
  }
  for (int l = 0; l < n_loops; l++) E.push_back({loop_from_to[2 * l], loop_from_to[2 * l + 1], inverse(loop_rel[l])});
  return E;
}
inline std::vector<Edge> build_edges(const std::vector<Iso>& X, int k, const int* loop_from_to, const Iso* loop_rel, int n_loops) {
  return build_edges(X, k, std::vector<int>{0}, loop_from_to, loop_rel, n_loops);
}

// Block (6x6) envelope (profile) Cholesky of a symmetric positive definite matrix. Row r stores its blocks from first[r]
// to r; the factor L has the same envelope, so nothing outside it is ever touched. With odometry edges of k blocks and
// loop edges (a, b) filling row b back to a, factoring costs O(N k + sum_loops (b - a) k) block products, plus a dense
// term where two filled loop rows overlap (at most O(L^2 N) for L loop edges), instead of the dense O(N^3).
struct EnvelopeMatrix {
  int n = 0;
  std::vector<int> first;
  std::vector<size_t> row_off;  // block index of (r, first[r])
  std::vector<double> a;        // 36 doubles per block, row-major

  // pairs: the (i, j) block positions that are nonzero off the diagonal (either order)
  void init(int n_blocks, const std::vector<std::pair<int, int>>& pairs) {
    n = n_blocks;
    first.resize(n);
    for (int r = 0; r < n; r++) first[r] = r;
    for (const auto& p : pairs) {
      const int r = std::max(p.first, p.second), c = std::min(p.first, p.second);
      first[r] = std::min(first[r], c);
    }
    row_off.resize(n + 1);
    size_t off = 0;
    for (int r = 0; r < n; r++) {
      row_off[r] = off;
      off += (size_t)(r - first[r] + 1);
    }
    row_off[n] = off;
    a.assign(off * 36, 0.0);
  }
  double* block(int r, int c) { return a.data() + (row_off[r] + (size_t)(c - first[r])) * 36; }
  const double* block(int r, int c) const { return a.data() + (row_off[r] + (size_t)(c - first[r])) * 36; }

  // in place: the lower blocks become L (A = L L^T). false when a pivot is not positive and finite.
  bool factor() {
    double S[36];
    for (int r = 0; r < n; r++) {
      for (int c = first[r]; c <= r; c++) {
        std::memcpy(S, block(r, c), sizeof(S));
        for (int k = std::max(first[r], first[c]); k < c; k++) {  // S -= L_rk L_ck^T
          const double* Lr = block(r, k);
          const double* Lc = block(c, k);
          for (int i = 0; i < 6; i++)
            for (int j = 0; j < 6; j++) {
              double s = 0.0;
              for (int m = 0; m < 6; m++) s += Lr[i * 6 + m] * Lc[j * 6 + m];
              S[i * 6 + j] -= s;
            }
        }
        double* out = block(r, c);
        if (c < r) {  // L_rc = S L_cc^-T: row i of L_rc solves L_cc x = S_i
          const double* Lcc = block(c, c);
          for (int i = 0; i < 6; i++)
            for (int j = 0; j < 6; j++) {
              double s = S[i * 6 + j];
              for (int m = 0; m < j; m++) s -= out[i * 6 + m] * Lcc[j * 6 + m];
              out[i * 6 + j] = s / Lcc[j * 6 + j];
            }
        } else {  // dense Cholesky of the diagonal block
          for (int j = 0; j < 6; j++) {
            double d = S[j * 6 + j];
            for (int m = 0; m < j; m++) d -= out[j * 6 + m] * out[j * 6 + m];
            if (!(d > 0.0) || !std::isfinite(d)) return false;
            const double l = std::sqrt(d);
            out[j * 6 + j] = l;
            for (int i = j + 1; i < 6; i++) {
              double s = S[i * 6 + j];
              for (int m = 0; m < j; m++) s -= out[i * 6 + m] * out[j * 6 + m];
              out[i * 6 + j] = s / l;
            }
            for (int i = 0; i < j; i++) out[i * 6 + j] = 0.0;
          }
        }
      }
    }
    return true;
  }

  // x = (L L^T)^-1 b after factor(); x and b may alias
  void solve(const double* b, double* x) const {
    std::vector<double> y(b, b + (size_t)n * 6);
    for (int r = 0; r < n; r++) {
      double* yr = y.data() + (size_t)r * 6;
      for (int k = first[r]; k < r; k++) {
        const double* L = block(r, k);
        const double* yk = y.data() + (size_t)k * 6;
        for (int i = 0; i < 6; i++) {
          double s = 0.0;
          for (int m = 0; m < 6; m++) s += L[i * 6 + m] * yk[m];
          yr[i] -= s;
        }
      }
      const double* D = block(r, r);
      for (int i = 0; i < 6; i++) {
        double s = yr[i];
        for (int m = 0; m < i; m++) s -= D[i * 6 + m] * yr[m];
        yr[i] = s / D[i * 6 + i];
      }
    }
    for (int r = n - 1; r >= 0; r--) {
      double* xr = y.data() + (size_t)r * 6;
      const double* D = block(r, r);
      for (int i = 5; i >= 0; i--) {
        double s = xr[i];
        for (int m = i + 1; m < 6; m++) s -= D[m * 6 + i] * xr[m];
        xr[i] = s / D[i * 6 + i];
      }
      for (int k = first[r]; k < r; k++) {  // y_k -= L_rk^T x_r
        const double* L = block(r, k);
        double* yk = y.data() + (size_t)k * 6;
        for (int i = 0; i < 6; i++) {
          double s = 0.0;
          for (int m = 0; m < 6; m++) s += L[m * 6 + i] * xr[m];
          yk[i] -= s;
        }
      }
    }
    std::memcpy(x, y.data(), y.size() * sizeof(double));
  }
};

struct LmTrial {  // one damped solve, for the tests' iteration-by-iteration comparison
  int iteration, accepted;
  double lambda, chi2;  // lambda the solve used, chi2 after the trial (DBL_MAX for a failed solve)
};

struct LmResult {
  double chi2_initial = 0, chi2_final = 0;
  int iterations = 0, trials = 0;
};

inline double total_chi2(const std::vector<Iso>& X, const std::vector<Edge>& edges) {
  double chi = 0.0;
  for (const Edge& ed : edges) {
    double e[6];
    edge_error(X[ed.from], X[ed.to], ed.zinv, e);
    double s = 0.0;
    for (int k = 0; k < 6; k++) s += e[k] * e[k];
    chi += s;
  }
  return chi;
}

// *g2o* SparseOptimizer::optimize(max_iterations) with OptimizationAlgorithmLevenberg::solve. Vertex 0 is fixed; a vertex
// no edge touches is not optimised (initializeOptimization leaves it out). Per iteration: H = sum J^T J, b = -sum J^T e over
// the free vertices; at iteration 0 lambda = 1e-5 max diag(H), nu = 2. Up to 10 trials: solve (H + lambda I) d = b, apply
// X_i <- X_i * fromVectorMQT(d_i), rho = (chi_old - chi_new) / (sum d (lambda d + b) + 1e-3); a failed solve counts as
// chi_new = DBL_MAX with d = 0. rho > 0 and chi_new finite: accept, lambda *= max(1/3, min(2/3, 1 - (2 rho - 1)^3)), nu = 2;
// otherwise restore the estimates bit for bit, lambda *= nu, nu *= 2. The trials stop at the first rho >= 0 (or a
// non-finite lambda); the run stops after an iteration that used all 10 trials, ended with rho == 0, or left lambda
// non-finite. VertexSE3's re-orthogonalisation after 1000 increments is never reached (at most 10 x max_iterations).
inline LmResult optimize(std::vector<Iso>& X, const std::vector<Edge>& edges, int max_iterations, std::vector<LmTrial>* trace = nullptr) {
  const int nv = (int)X.size();
  LmResult res;
  std::vector<int> pos(nv, -1);  // position of a free vertex among the unknowns, in vertex order
  std::vector<char> touched(nv, 0);
  for (const Edge& ed : edges) touched[ed.from] = touched[ed.to] = 1;
  int np = 0;
  for (int i = 1; i < nv; i++)
    if (touched[i]) pos[i] = np++;
  res.chi2_initial = res.chi2_final = total_chi2(X, edges);
  if (np == 0 || max_iterations <= 0) return res;
  std::vector<std::pair<int, int>> pairs;
  for (const Edge& ed : edges)
    if (pos[ed.from] >= 0 && pos[ed.to] >= 0) pairs.push_back({pos[ed.from], pos[ed.to]});
  EnvelopeMatrix H, F;
  H.init(np, pairs);
  std::vector<double> b((size_t)np * 6), dx((size_t)np * 6);
  std::vector<Iso> backup(nv);
  double lambda = 0.0, nu = 2.0, current = res.chi2_initial;
  for (int it = 0; it < max_iterations; it++) {
    current = total_chi2(X, edges);
    std::fill(H.a.begin(), H.a.end(), 0.0);
    std::fill(b.begin(), b.end(), 0.0);
    for (const Edge& ed : edges) {
      double e[6], Jf[36], Jt[36];
      Iso E;
      edge_error(X[ed.from], X[ed.to], ed.zinv, e, &E);
      edge_jacobians(E, ed.zinv, Jf, Jt);
      const int pv[2] = {pos[ed.from], pos[ed.to]};
      const double* J[2] = {Jf, Jt};
      for (int u = 0; u < 2; u++) {
        if (pv[u] < 0) continue;
        double* bu = b.data() + (size_t)pv[u] * 6;
        for (int i = 0; i < 6; i++) {
          double s = 0.0;
          for (int m = 0; m < 6; m++) s += J[u][m * 6 + i] * e[m];
          bu[i] -= s;
        }
        for (int w = 0; w < 2; w++) {  // the lower block (row >= column) of every vertex pair, once per ordered pair
          if (pv[w] < 0 || pv[w] > pv[u] || (pv[w] == pv[u] && w != u)) continue;
          double* blk = H.block(pv[u], pv[w]);
          for (int i = 0; i < 6; i++)
            for (int j = 0; j < 6; j++) {
              double s = 0.0;
              for (int m = 0; m < 6; m++) s += J[u][m * 6 + i] * J[w][m * 6 + j];
              blk[i * 6 + j] += s;
            }
        }
      }
    }
    if (it == 0) {
      double maxd = 0.0;
      for (int p = 0; p < np; p++) {
        const double* D = H.block(p, p);
        for (int i = 0; i < 6; i++) maxd = std::max(maxd, std::fabs(D[i * 7]));
      }
      lambda = 1e-5 * maxd;
      nu = 2.0;
    }
    int q = 0;
    double rho = 0.0;
    do {
      for (int i = 0; i < nv; i++)
        if (pos[i] >= 0) backup[i] = X[i];
      F = H;
      for (int p = 0; p < np; p++) {
        double* D = F.block(p, p);
        for (int i = 0; i < 6; i++) D[i * 7] += lambda;
      }
      const bool ok = F.factor();
      double chi_new = DBL_MAX;
      if (ok) {
        F.solve(b.data(), dx.data());
        for (int i = 0; i < nv; i++)
          if (pos[i] >= 0) X[i] = compose(X[i], from_vector_mqt(dx.data() + (size_t)pos[i] * 6));
        chi_new = total_chi2(X, edges);
      } else {
        std::fill(dx.begin(), dx.end(), 0.0);
      }
      double scale = 0.0;
      for (size_t j = 0; j < dx.size(); j++) scale += dx[j] * (lambda * dx[j] + b[j]);
      rho = (current - chi_new) / (scale + 1e-3);
      const double used_lambda = lambda;
      const bool accept = rho > 0 && std::isfinite(chi_new);
      if (accept) {
        const double alpha = std::min(1.0 - std::pow(2.0 * rho - 1.0, 3), 2.0 / 3.0);
        lambda *= std::max(1.0 / 3.0, alpha);
        nu = 2.0;
        current = chi_new;
      } else {
        lambda *= nu;
        nu *= 2.0;
        for (int i = 0; i < nv; i++)
          if (pos[i] >= 0) X[i] = backup[i];
      }
      res.trials++;
      if (trace) trace->push_back({it, accept ? 1 : 0, used_lambda, chi_new});
      if (!accept && !std::isfinite(lambda)) break;
      q++;
    } while (rho < 0 && q < 10);
    res.iterations++;
    if (q == 10 || rho == 0 || !std::isfinite(lambda)) break;
  }
  res.chi2_final = current;
  return res;
}

}  // namespace pg
}  // namespace b200
