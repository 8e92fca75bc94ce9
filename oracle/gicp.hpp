// ORACLE — TEST INFRASTRUCTURE ONLY. PARITY UNPINNED (no reference tests; PCL/Eigen/FLANN absent).
// CPU restatement of pclomp::GeneralizedIterativeClosestPoint
// (Thirdparty/ndt_omp_ros2/include/pclomp/gicp_omp.h, gicp_omp_impl.hpp):
//   computeCovariances              gicp_omp_impl.hpp:48-122
//   computeRDerivative              gicp_omp_impl.hpp:125-177
//   estimateRigidTransformationBFGS gicp_omp_impl.hpp:180-241
//   functor operator() / df / fdf   gicp_omp_impl.hpp:244-366
//   computeTransformation           gicp_omp_impl.hpp:369-515
//   applyState                      gicp_omp_impl.hpp:517-528
//   defaults                        gicp_omp.h:108-128
//
// NOTE on the inner-solver stop test (gicp_omp_impl.hpp:229 `bfgs.testGradient()`): with PCL >= 1.11 the
// zero-argument form forwards to `functor.checkGradient(g)`, which pclomp's functor does not override;
// the original ndt_omp code (and PCL <= 1.10) used `testGradient(gradient_tol = 1e-2)` = "|g| < 1e-2".
// The README's pclomp::GICP fitness (0.220388 vs pcl::GICP 0.220382) was produced by a converging solver,
// so this restatement keeps the |g| < 1e-2 test. PCL is not available to settle it: parity unpinned.
#pragma once
#include <omp.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

#include "bfgs.hpp"
#include "kdtree.hpp"
#include "linalg.hpp"
#include "ndt.hpp"

namespace oracle {

// opt-in record of the optimiser (same layout as the engine's b200reg_gicp_trace_record, include/b200reg.h): type 0 per
// functor call, 1 per minimizeOneStep, 2 per outer iteration
struct GicpTraceRec {
  int type, outer, inner, evaluation, want_grad, status, m, nr_iterations, converged, last;
  double x[6], f, g[6], x0[6], delta;
  float T[12], final_T[16];
};

class GICP {
 public:
  // gicp_omp.h:108-128
  int k_correspondences = 20;
  double gicp_epsilon = 0.001;
  double rotation_epsilon = 2e-3;
  int max_inner_iterations = 20;
  int max_iterations = 200;
  double transformation_epsilon = 5e-4;
  double corr_dist_threshold = 5.0;
  double gradient_tol = 1e-2;

  float final_transformation[16];
  bool converged = false;
  int nr_iterations = 0;
  bool trace_on = false;
  std::vector<GicpTraceRec> trace;

  std::vector<P3> target, input;
  KdTree tree, tree_reciprocal;
  bool tree_dirty = true, rtree_dirty = true;
  std::vector<double> target_covariances, input_covariances;  // 9 doubles per point, row-major
  std::vector<float> mahalanobis;                              // 9 floats per source point (3x3 block of the 4x4)
  std::vector<int> src_idx, tgt_idx;                           // correspondences of the last outer iteration
  float base_transformation[16];
  std::vector<P3> out_cloud;  // "output" (source transformed by guess)

  GICP() {
    NDT::set_identity(final_transformation);
    NDT::set_identity(base_transformation);
  }

  void setInputTarget(const std::vector<P3>& c) {  // gicp_omp.h:156-170
    if (c.empty()) return;
    target = c;
    tree_dirty = true;
    target_covariances.clear();
  }
  void setInputSource(const std::vector<P3>& c) {  // gicp_omp.h:133-149
    if (c.empty()) return;
    input = c;
    rtree_dirty = true;
    input_covariances.clear();
  }

  // gicp_omp_impl.hpp:48-122
  void computeCovariances(const std::vector<P3>& cloud, const KdTree& kd, std::vector<double>& covs) const {
    if (k_correspondences > (int)cloud.size()) return;
    covs.assign(cloud.size() * 9, 0.0);
#pragma omp parallel
    {
      std::vector<int> nn;
      std::vector<float> d2;
#pragma omp for
      for (long i = 0; i < (long)cloud.size(); i++) {
        double mean[3] = {0, 0, 0};
        double* cov = &covs[(size_t)i * 9];
        for (int k = 0; k < 9; k++) cov[k] = 0;
        kd.knn(cloud[i], k_correspondences, nn, d2);
        for (int j = 0; j < k_correspondences; j++) {
          const P3& pt = cloud[nn[j]];
          mean[0] += pt.x;
          mean[1] += pt.y;
          mean[2] += pt.z;
          cov[0] += pt.x * pt.x;
          cov[3] += pt.y * pt.x;
          cov[4] += pt.y * pt.y;
          cov[6] += pt.z * pt.x;
          cov[7] += pt.z * pt.y;
          cov[8] += pt.z * pt.z;
        }
        for (int a = 0; a < 3; a++) mean[a] /= static_cast<double>(k_correspondences);
        for (int k = 0; k < 3; k++)
          for (int l = 0; l <= k; l++) {
            cov[k * 3 + l] /= static_cast<double>(k_correspondences);
            cov[k * 3 + l] -= mean[k] * mean[l];
            cov[l * 3 + k] = cov[k * 3 + l];
          }
        JacobiSVD<3> svd(cov);
        for (int k = 0; k < 9; k++) cov[k] = 0;
        for (int k = 0; k < 3; k++) {
          double col[3] = {svd.U[0 * 3 + k], svd.U[1 * 3 + k], svd.U[2 * 3 + k]};
          double v = (k == 2) ? gicp_epsilon : 1.0;
          for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) cov[a * 3 + b] += v * col[a] * col[b];
        }
      }
    }
  }

  // gicp_omp_impl.hpp:517-528 (t row-major 4x4 float)
  static void applyState(float* t, const double* x) {
    float cx = std::cos((float)x[3]), sx = std::sin((float)x[3]);
    float cy = std::cos((float)x[4]), sy = std::sin((float)x[4]);
    float cz = std::cos((float)x[5]), sz = std::sin((float)x[5]);
    float Rz[9] = {cz, -sz, 0, sz, cz, 0, 0, 0, 1}, Ry[9] = {cy, 0, sy, 0, 1, 0, -sy, 0, cy}, Rx[9] = {1, 0, 0, 0, cx, -sx, 0, sx, cx};
    float A[9], R[9], N[9];
    mul3f(Rz, Ry, A);
    mul3f(A, Rx, R);
    float old[9];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) old[r * 3 + c] = t[r * 4 + c];
    mul3f(R, old, N);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) t[r * 4 + c] = N[r * 3 + c];
    t[3] += (float)x[0];
    t[7] += (float)x[1];
    t[11] += (float)x[2];
  }

  // gicp_omp_impl.hpp:125-177. R row-major 3x3
  static void computeRDerivative(const double* x, const double* R, double* g) {
    double phi = x[3], theta = x[4], psi = x[5];
    double cphi = std::cos(phi), sphi = std::sin(phi), ctheta = std::cos(theta), stheta = std::sin(theta);
    double cpsi = std::cos(psi), spsi = std::sin(psi);
    double dPhi[9] = {0, sphi * spsi + cphi * cpsi * stheta, cphi * spsi - cpsi * sphi * stheta,
                      0, -cpsi * sphi + cphi * spsi * stheta, -cphi * cpsi - sphi * spsi * stheta,
                      0, cphi * ctheta, -ctheta * sphi};
    double dTheta[9] = {-cpsi * stheta, cpsi * ctheta * sphi, cphi * cpsi * ctheta,
                        -spsi * stheta, ctheta * sphi * spsi, cphi * ctheta * spsi,
                        -ctheta, -sphi * stheta, -cphi * stheta};
    double dPsi[9] = {-ctheta * spsi, -cphi * cpsi - sphi * spsi * stheta, cpsi * sphi - cphi * spsi * stheta,
                      cpsi * ctheta, -cphi * spsi + cpsi * sphi * stheta, sphi * spsi + cphi * cpsi * stheta,
                      0, 0, 0};
    auto inner = [&](const double* m1) {  // tr(m1^T R) as written at gicp_omp.h:316-326: sum m1(j,i)*R(i,j)
      double r = 0;
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r += m1[j * 3 + i] * R[i * 3 + j];
      return r;
    };
    g[3] = inner(dPhi);
    g[4] = inner(dTheta);
    g[5] = inner(dPsi);
  }

  // functor operator()  (gicp_omp_impl.hpp:244-274)
  double f_only(const double* x) const {
    float T[16];
    std::memcpy(T, base_transformation, sizeof(T));
    applyState(T, x);
    const int m = (int)src_idx.size();
    double f = 0;
#pragma omp parallel for reduction(+ : f)
    for (int i = 0; i < m; i++) {
      const P3& ps = out_cloud[src_idx[i]];
      const P3& pt = target[tgt_idx[i]];
      float res[3] = {T[0] * ps.x + T[1] * ps.y + T[2] * ps.z + T[3] - pt.x,
                      T[4] * ps.x + T[5] * ps.y + T[6] * ps.z + T[7] - pt.y,
                      T[8] * ps.x + T[9] * ps.y + T[10] * ps.z + T[11] - pt.z};
      const float* M = &mahalanobis[(size_t)src_idx[i] * 9];
      float mr[3];
      for (int r = 0; r < 3; r++) mr[r] = M[r * 3] * res[0] + M[r * 3 + 1] * res[1] + M[r * 3 + 2] * res[2];
      f += (double)(res[0] * mr[0] + res[1] * mr[1] + res[2] * mr[2]);
    }
    return f / m;
  }

  // functor fdf / df (gicp_omp_impl.hpp:277-366); f returned as well
  void fdf(const double* x, double& f, double* g) const {
    float T[16];
    std::memcpy(T, base_transformation, sizeof(T));
    applyState(T, x);
    const int m = (int)src_idx.size();
    double fs = 0, gt[3] = {0, 0, 0}, R[9] = {0};
    for (int i = 0; i < m; i++) {
      const P3& ps = out_cloud[src_idx[i]];
      const P3& pt = target[tgt_idx[i]];
      float pp[3] = {T[0] * ps.x + T[1] * ps.y + T[2] * ps.z + T[3], T[4] * ps.x + T[5] * ps.y + T[6] * ps.z + T[7],
                     T[8] * ps.x + T[9] * ps.y + T[10] * ps.z + T[11]};
      double res[3] = {(double)(pp[0] - pt.x), (double)(pp[1] - pt.y), (double)(pp[2] - pt.z)};
      const float* M = &mahalanobis[(size_t)src_idx[i] * 9];
      double temp[3];
      for (int r = 0; r < 3; r++) temp[r] = (double)M[r * 3] * res[0] + (double)M[r * 3 + 1] * res[1] + (double)M[r * 3 + 2] * res[2];
      fs += res[0] * temp[0] + res[1] * temp[1] + res[2] * temp[2];
      for (int r = 0; r < 3; r++) gt[r] += temp[r];
      const float* B = base_transformation;
      float pb[3] = {B[0] * ps.x + B[1] * ps.y + B[2] * ps.z + B[3], B[4] * ps.x + B[5] * ps.y + B[6] * ps.z + B[7],
                     B[8] * ps.x + B[9] * ps.y + B[10] * ps.z + B[11]};
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) R[r * 3 + c] += (double)pb[r] * temp[c];
    }
    f = fs / double(m);
    for (int r = 0; r < 3; r++) g[r] = gt[r] * double(2.0 / m);
    for (int k = 0; k < 9; k++) R[k] *= 2.0 / m;
    computeRDerivative(x, R, g);
  }

  // gicp_omp_impl.hpp:180-241. Returns false where the reference throws.
  bool estimateRigidTransformationBFGS(float* transformation_matrix) {
    if (src_idx.size() < 4) {
      if (trace_on) {
        GicpTraceRec r{};
        r.type = 2;
        r.outer = nr_iterations;
        r.status = -2;  // BFGS not started
        r.m = (int)src_idx.size();
        r.nr_iterations = nr_iterations;
        trace.push_back(r);
      }
      return false;
    }
    double x[6];
    const float* t = transformation_matrix;
    x[0] = t[3];
    x[1] = t[7];
    x[2] = t[11];
    x[3] = std::atan2(t[9], t[10]);   // (2,1),(2,2)
    x[4] = std::asin(-t[8]);          // -(2,0)
    x[5] = std::atan2(t[4], t[0]);    // (1,0),(0,0)
    double x0[6];
    std::memcpy(x0, x, sizeof(x0));
    int inner_iterations = 0, calls = 0;
    auto record = [&](int type, int want_grad, const double* xx, double f, const double* gg) {
      GicpTraceRec r{};
      r.type = type;
      r.outer = nr_iterations;
      r.inner = inner_iterations;
      r.evaluation = calls;
      r.want_grad = want_grad;
      std::memcpy(r.x, xx, sizeof(r.x));
      r.f = f;
      if (gg) std::memcpy(r.g, gg, sizeof(r.g));
      if (type == 0) {
        float T[16];
        std::memcpy(T, base_transformation, sizeof(T));
        applyState(T, xx);
        std::memcpy(r.T, T, sizeof(r.T));
      }
      trace.push_back(r);
      return &trace.back();
    };
    BfgsFunctor6 fn;
    fn.f = [&](const double* xx) {
      const double f = f_only(xx);
      if (trace_on) record(0, 0, xx, f, nullptr);
      calls++;
      return f;
    };
    fn.df = [&](const double* xx, double* gg) { double f; fn.fdf(xx, f, gg); };
    fn.fdf = [&](const double* xx, double& f, double* gg) {
      fdf(xx, f, gg);
      if (trace_on) record(0, 1, xx, f, gg);
      calls++;
    };
    BFGS6 bfgs(fn);
    int result = bfgs.minimizeInit(x);
    result = BFGS_Running;
    do {
      inner_iterations++;
      result = bfgs.minimizeOneStep(x);
      if (trace_on) record(1, 0, x, bfgs.f, bfgs.gradient)->status = result;
      if (result) break;
      result = bfgs.testGradient(gradient_tol);
    } while (result == BFGS_Running && inner_iterations < max_inner_iterations);
    if (trace_on) {
      GicpTraceRec* r = record(2, 0, x, 0.0, nullptr);
      r->f = 0;
      r->status = result;
      r->m = (int)src_idx.size();
      r->nr_iterations = nr_iterations;
      std::memcpy(r->x0, x0, sizeof(x0));
    }
    if (result == BFGS_NoProgress || result == BFGS_Success || inner_iterations == max_inner_iterations) {
      NDT::set_identity(transformation_matrix);
      applyState(transformation_matrix, x);
      return true;
    }
    return false;
  }

  // pcl::Registration::align + gicp_omp_impl.hpp:369-515. guess row-major or nullptr.
  void align(const float* guess_in) {
    converged = false;
    NDT::set_identity(final_transformation);
    trace.clear();
    if (target.empty() || input.empty()) return;
    float guess[16];
    if (guess_in) std::memcpy(guess, guess_in, sizeof(guess));
    else NDT::set_identity(guess);
    if (tree_dirty) { tree.build(target); tree_dirty = false; }
    if (rtree_dirty) { tree_reciprocal.build(input); rtree_dirty = false; }
    const size_t N = input.size();
    mahalanobis.assign(N * 9, 0.0f);
    for (size_t i = 0; i < N; i++) mahalanobis[i * 9] = mahalanobis[i * 9 + 4] = mahalanobis[i * 9 + 8] = 1.0f;
    if (target_covariances.empty()) computeCovariances(target, tree, target_covariances);
    if (input_covariances.empty()) computeCovariances(input, tree_reciprocal, input_covariances);
    NDT::set_identity(base_transformation);
    nr_iterations = 0;
    double dist_threshold = corr_dist_threshold * corr_dist_threshold;
    NDT::transform_cloud(input, out_cloud, guess);
    float transformation[16], previous[16];
    NDT::set_identity(transformation);
    NDT::set_identity(previous);
    while (!converged) {
      double transform_R[16] = {0};
      for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
          for (int k = 0; k < 4; k++) transform_R[i * 4 + j] += double(transformation[i * 4 + k]) * double(guess[k * 4 + j]);
      double R[9], Rt[9];
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) R[r * 3 + c] = transform_R[r * 4 + c];
      mat3_transpose(R, Rt);
      std::vector<int> nn_of(N, -1);
#pragma omp parallel
      {
        std::vector<int> nn;
        std::vector<float> d2;
#pragma omp for
        for (long i = 0; i < (long)N; i++) {
          const P3& o = out_cloud[i];
          const float* T = transformation;
          P3 q = {T[0] * o.x + T[1] * o.y + T[2] * o.z + T[3], T[4] * o.x + T[5] * o.y + T[6] * o.z + T[7],
                  T[8] * o.x + T[9] * o.y + T[10] * o.z + T[11]};
          if (tree.knn(q, 1, nn, d2) < 1) continue;
          if (d2[0] < dist_threshold) {
            const double* C1 = &input_covariances[(size_t)i * 9];
            const double* C2 = &target_covariances[(size_t)nn[0] * 9];
            double M[9], temp[9];
            mat3_mul(R, C1, M);
            mat3_mul(M, Rt, temp);
            for (int k = 0; k < 9; k++) temp[k] += C2[k];
            mat3_inverse(temp, M);
            for (int k = 0; k < 9; k++) mahalanobis[(size_t)i * 9 + k] = (float)M[k];
            nn_of[i] = nn[0];
          }
        }
      }
      src_idx.clear();
      tgt_idx.clear();
      for (size_t i = 0; i < N; i++)  // == sort by source index (gicp_omp_impl.hpp:460-471)
        if (nn_of[i] >= 0) {
          src_idx.push_back((int)i);
          tgt_idx.push_back(nn_of[i]);
        }
      std::memcpy(previous, transformation, sizeof(previous));
      double delta = 0.;
      if (!estimateRigidTransformationBFGS(transformation)) break;  // exception path: gicp_omp_impl.hpp:494-498
      for (int k = 0; k < 4; k++)
        for (int l = 0; l < 4; l++) {
          double ratio = (k < 3 && l < 3) ? 1. / rotation_epsilon : 1. / transformation_epsilon;
          double c_delta = ratio * std::fabs(previous[k * 4 + l] - transformation[k * 4 + l]);
          if (c_delta > delta) delta = c_delta;
        }
      nr_iterations++;
      if (nr_iterations >= max_iterations || delta < 1) {
        converged = true;
        std::memcpy(previous, transformation, sizeof(previous));
      }
      if (trace_on) {
        GicpTraceRec& r = trace.back();
        std::memcpy(r.T, transformation, sizeof(r.T));
        r.delta = delta;
        r.nr_iterations = nr_iterations;
        r.converged = converged ? 1 : 0;
      }
    }
    // final = previous * guess (float)
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) {
        float s = 0;
        for (int k = 0; k < 4; k++) s += previous[i * 4 + k] * guess[k * 4 + j];
        final_transformation[i * 4 + j] = s;
      }
    if (trace_on && !trace.empty() && trace.back().type == 2) {
      trace.back().last = 1;
      std::memcpy(trace.back().final_T, final_transformation, sizeof(final_transformation));
    }
  }

  double getFitnessScore(double max_range = std::numeric_limits<double>::max()) {
    if (tree_dirty) { tree.build(target); tree_dirty = false; }
    std::vector<P3> tr;
    NDT::transform_cloud(input, tr, final_transformation);
    double sum = 0;
    int nr = 0;
    std::vector<int> idx;
    std::vector<float> d2;
    for (const P3& p : tr) {
      if (tree.knn(p, 1, idx, d2) < 1) continue;
      if (d2[0] <= max_range) { sum += d2[0]; nr++; }
    }
    return nr > 0 ? sum / nr : std::numeric_limits<double>::max();
  }

 private:
  static void mul3f(const float* a, const float* b, float* c) {
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        float s = 0;
        for (int k = 0; k < 3; k++) s += a[i * 3 + k] * b[k * 3 + j];
        c[i * 3 + j] = s;
      }
  }
};

}  // namespace oracle
