// ORACLE — TEST INFRASTRUCTURE ONLY. extern "C" surface over the CPU restatement so that tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs can drive it through
// ctypes. Nothing under lidarslam_ros2_b200/ may load this library.
// 4x4 matrices cross this boundary COLUMN-MAJOR (Eigen::Matrix4f::data() order), like include/b200reg.h.
#include <cstring>
#include <string>
#include <vector>

#include "gicp.hpp"
#include "ndt.hpp"

using namespace oracle;

namespace {
void col_to_row(const float* c, float* r) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) r[i * 4 + j] = c[j * 4 + i];
}
void row_to_col(const float* r, float* c) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) c[j * 4 + i] = r[i * 4 + j];
}
std::vector<P3> gather(const float* base, size_t n, size_t stride_bytes) {
  std::vector<P3> v(n);
  const char* b = reinterpret_cast<const char*>(base);
  for (size_t i = 0; i < n; i++) {
    const float* f = reinterpret_cast<const float*>(b + i * stride_bytes);
    v[i] = {f[0], f[1], f[2]};
  }
  return v;
}
}  // namespace

extern "C" {

int oracle_max_threads() { return omp_get_max_threads(); }

// ---------------- VoxelGrid ----------------
// in: n points, xyz at byte offset 0, intensity at intensity_off bytes (<0: none → 0). out: 4 floats/pt.
size_t oracle_voxelgrid(const float* in, size_t n, size_t stride_bytes, long intensity_off, float leaf, float* out,
                        size_t out_capacity) {
  std::vector<P4> cloud(n), res;
  const char* b = reinterpret_cast<const char*>(in);
  for (size_t i = 0; i < n; i++) {
    const float* f = reinterpret_cast<const float*>(b + i * stride_bytes);
    float inten = intensity_off >= 0 ? *reinterpret_cast<const float*>(b + i * stride_bytes + intensity_off) : 0.0f;
    cloud[i] = {f[0], f[1], f[2], inten};
  }
  voxelgrid_filter(cloud, leaf, res);
  size_t m = std::min(res.size(), out_capacity);
  for (size_t i = 0; i < m; i++) {
    out[i * 4 + 0] = res[i].x;
    out[i * 4 + 1] = res[i].y;
    out[i * 4 + 2] = res[i].z;
    out[i * 4 + 3] = res[i].i;
  }
  return res.size();
}

// ---------------- NDT ----------------
void* oracle_ndt_create() { return new NDT(); }
void oracle_ndt_destroy(void* h) { delete static_cast<NDT*>(h); }

int oracle_ndt_set(void* h, const char* key, double v) {
  NDT* n = static_cast<NDT*>(h);
  std::string k(key);
  if (k == "resolution") n->setResolution((float)v);
  else if (k == "step_size") n->step_size = v;
  else if (k == "outlier_ratio") n->outlier_ratio = v;
  else if (k == "transformation_epsilon") n->transformation_epsilon = v;
  else if (k == "max_iterations") n->max_iterations = (int)v;
  else if (k == "search_method") n->search_method = (int)v;
  else if (k == "num_threads") n->num_threads = (int)v;
  else if (k == "min_points_per_voxel") n->target_cells.min_points_per_voxel = (int)v;
  else return -1;
  return 0;
}

void oracle_ndt_set_target(void* h, const float* base, size_t n, size_t stride_bytes) {
  static_cast<NDT*>(h)->setInputTarget(gather(base, n, stride_bytes));
}
void oracle_ndt_set_source(void* h, const float* base, size_t n, size_t stride_bytes) {
  static_cast<NDT*>(h)->setInputSource(gather(base, n, stride_bytes));
}

void oracle_ndt_align(void* h, const float* guess_colmajor, float* T_out_colmajor, int* converged, int* iters,
                      double* trans_prob, int* n_evals) {
  NDT* n = static_cast<NDT*>(h);
  float g[16];
  if (guess_colmajor) col_to_row(guess_colmajor, g);
  n->align(guess_colmajor ? g : nullptr);
  row_to_col(n->final_transformation, T_out_colmajor);
  if (converged) *converged = n->converged ? 1 : 0;
  if (iters) *iters = n->nr_iterations;
  if (trans_prob) *trans_prob = n->trans_probability;
  if (n_evals) *n_evals = n->n_evaluations;
}

double oracle_ndt_fitness(void* h, double max_range) { return static_cast<NDT*>(h)->getFitnessScore(max_range); }

// score/gradient/Hessian of the source transformed by T (col-major), angle tables from p[3..5].
double oracle_ndt_derivatives(void* h, const float* T_colmajor, const double* p6, int compute_hessian, double* g6,
                              double* H36) {
  NDT* n = static_cast<NDT*>(h);
  float T[16];
  col_to_row(T_colmajor, T);
  n->init_gauss();
  std::vector<P3> tr;
  NDT::transform_cloud(n->input, tr, T);
  return n->computeDerivatives(g6, H36, tr, p6, compute_hessian != 0);
}

void oracle_ndt_hessian(void* h, const float* T_colmajor, const double* p6, double* H36) {
  NDT* n = static_cast<NDT*>(h);
  float T[16];
  col_to_row(T_colmajor, T);
  n->init_gauss();
  n->computeAngleDerivatives(p6);
  std::vector<P3> tr;
  NDT::transform_cloud(n->input, tr, T);
  n->computeHessian(H36, tr);
}

double oracle_ndt_calculate_score(void* h, const float* T_colmajor) {
  NDT* n = static_cast<NDT*>(h);
  float T[16];
  col_to_row(T_colmajor, T);
  std::vector<P3> tr;
  NDT::transform_cloud(n->input, tr, T);
  return n->calculateScore(tr);
}

// voxels with nr_points >= min_points_per_voxel, ascending leaf index
size_t oracle_ndt_num_voxels(void* h) {
  NDT* n = static_cast<NDT*>(h);
  size_t c = 0;
  for (auto& kv : n->target_cells.leaves)
    if (kv.second.nr_points >= n->target_cells.min_points_per_voxel) c++;
  return c;
}
size_t oracle_ndt_num_leaves(void* h) { return static_cast<NDT*>(h)->target_cells.leaves.size(); }

void oracle_ndt_get_voxels(void* h, int* idx, int* npts, double* mean3, double* cov9, double* icov9,
                           float* centroid3) {
  NDT* n = static_cast<NDT*>(h);
  size_t c = 0;
  for (auto& kv : n->target_cells.leaves) {
    const Leaf& l = kv.second;
    if (l.nr_points < n->target_cells.min_points_per_voxel) continue;
    if (idx) idx[c] = (int)kv.first;
    if (npts) npts[c] = l.nr_points;
    if (mean3) std::memcpy(mean3 + 3 * c, l.mean, 3 * sizeof(double));
    if (cov9) std::memcpy(cov9 + 9 * c, l.cov, 9 * sizeof(double));
    if (icov9) std::memcpy(icov9 + 9 * c, l.icov, 9 * sizeof(double));
    if (centroid3) std::memcpy(centroid3 + 3 * c, l.centroid, 3 * sizeof(float));
    c++;
  }
}

void oracle_ndt_grid_geom(void* h, int* min_b3, int* div_b3) {
  NDT* n = static_cast<NDT*>(h);
  for (int a = 0; a < 3; a++) {
    min_b3[a] = n->target_cells.geom.min_b[a];
    div_b3[a] = n->target_cells.geom.div_b[a];
  }
}

void oracle_ndt_gauss(void* h, double* d123) {
  NDT* n = static_cast<NDT*>(h);
  n->init_gauss();
  d123[0] = n->gauss_d1;
  d123[1] = n->gauss_d2;
  d123[2] = n->gauss_d3;
}

// ---------------- small known-answer hooks ----------------
void oracle_euler_angles_012(const float* R_rowmajor9, float* out3) { euler_angles_012(R_rowmajor9, out3); }
void oracle_pose_to_matrix(const double* p6, float* T_colmajor) {
  float T[16];
  pose_to_matrix_f(p6, T);
  row_to_col(T, T_colmajor);
}
void oracle_sym_eigen3(const double* A9, double* evals3, double* evecs9) { sym_eigen3(A9, evals3, evecs9); }
void oracle_svd6_solve(const double* A36, const double* b6, double* x6) {
  JacobiSVD<6> sv(A36);
  sv.solve(b6, x6);
}
void oracle_mat3_inverse(const double* A9, double* out9) { mat3_inverse(A9, out9); }
double oracle_mt_trial(const double* v9) {
  return NDT::trialValueSelectionMT(v9[0], v9[1], v9[2], v9[3], v9[4], v9[5], v9[6], v9[7], v9[8]);
}
int oracle_mt_update(double* v6, const double* t3) {
  return NDT::updateIntervalMT(v6[0], v6[1], v6[2], v6[3], v6[4], v6[5], t3[0], t3[1], t3[2]) ? 1 : 0;
}
void oracle_angle_tables(const double* p6, float* jang24, float* hang45) {
  NDT n;
  n.computeAngleDerivatives(p6);
  for (int r = 0; r < 8; r++)
    for (int c = 0; c < 3; c++) jang24[r * 3 + c] = n.j_ang[r][c];
  for (int r = 0; r < 15; r++)
    for (int c = 0; c < 3; c++) hang45[r * 3 + c] = n.h_ang[r][c];
}

// ---------------- exact NN (fitness building block) ----------------
// for each query the (d2, index) of the nearest target point
void oracle_nn1(const float* tgt, size_t nt, size_t tstride, const float* qry, size_t nq, size_t qstride, int* idx,
                float* d2) {
  std::vector<P3> t = gather(tgt, nt, tstride), q = gather(qry, nq, qstride);
  KdTree tree;
  tree.build(t);
#pragma omp parallel
  {
    std::vector<int> i1;
    std::vector<float> d1;
#pragma omp for
    for (long k = 0; k < (long)nq; k++) {
      tree.knn(q[k], 1, i1, d1);
      idx[k] = i1.empty() ? -1 : i1[0];
      d2[k] = d1.empty() ? -1.0f : d1[0];
    }
  }
}

// ---------------- GICP ----------------
void* oracle_gicp_create() { return new GICP(); }
void oracle_gicp_destroy(void* h) { delete static_cast<GICP*>(h); }
int oracle_gicp_set(void* h, const char* key, double v) {
  GICP* g = static_cast<GICP*>(h);
  std::string k(key);
  if (k == "max_correspondence_distance") g->corr_dist_threshold = v;
  else if (k == "transformation_epsilon") g->transformation_epsilon = v;
  else if (k == "rotation_epsilon") g->rotation_epsilon = v;
  else if (k == "max_iterations") g->max_iterations = (int)v;
  else if (k == "k_correspondences") g->k_correspondences = (int)v;
  else if (k == "gicp_epsilon") g->gicp_epsilon = v;
  else if (k == "max_inner_iterations") g->max_inner_iterations = (int)v;
  else return -1;
  return 0;
}
void oracle_gicp_set_target(void* h, const float* base, size_t n, size_t stride_bytes) {
  static_cast<GICP*>(h)->setInputTarget(gather(base, n, stride_bytes));
}
void oracle_gicp_set_source(void* h, const float* base, size_t n, size_t stride_bytes) {
  static_cast<GICP*>(h)->setInputSource(gather(base, n, stride_bytes));
}
void oracle_gicp_align(void* h, const float* guess_colmajor, float* T_out_colmajor, int* converged, int* iters) {
  GICP* g = static_cast<GICP*>(h);
  float gr[16];
  if (guess_colmajor) col_to_row(guess_colmajor, gr);
  g->align(guess_colmajor ? gr : nullptr);
  row_to_col(g->final_transformation, T_out_colmajor);
  if (converged) *converged = g->converged ? 1 : 0;
  if (iters) *iters = g->nr_iterations;
}
double oracle_gicp_fitness(void* h, double max_range) { return static_cast<GICP*>(h)->getFitnessScore(max_range); }
// per-point covariances (row-major 3x3 doubles); which: 0 = source, 1 = target. Requires align() first
size_t oracle_gicp_get_covariances(void* h, int which, double* out9) {
  GICP* g = static_cast<GICP*>(h);
  const auto& v = which ? g->target_covariances : g->input_covariances;
  if (out9) std::memcpy(out9, v.data(), v.size() * sizeof(double));
  return v.size() / 9;
}
// cost / gradient of the fixed-correspondence objective at state x (gicp_omp_impl.hpp:332-366)
double oracle_gicp_fdf(void* h, const double* x6, double* g6) {
  GICP* g = static_cast<GICP*>(h);
  double f;
  g->fdf(x6, f, g6);
  return f;
}
int oracle_gicp_num_correspondences(void* h) { return (int)static_cast<GICP*>(h)->src_idx.size(); }
// functor operator(), the f32 path (gicp_omp_impl.hpp:244-274), at state x on the last correspondences
double oracle_gicp_f_only(void* h, const double* x6) { return static_cast<GICP*>(h)->f_only(x6); }
// base_transformation_ with the state applied (applyState, gicp_omp_impl.hpp:517-528), column-major
void oracle_gicp_apply_state(void* h, const double* x6, float* T_colmajor) {
  GICP* g = static_cast<GICP*>(h);
  float T[16];
  std::memcpy(T, g->base_transformation, sizeof(T));
  GICP::applyState(T, x6);
  row_to_col(T, T_colmajor);
}
// opt-in trace of align()'s optimiser (GicpTraceRec); get returns the record count and copies up to cap records
void oracle_gicp_set_trace(void* h, int on) { static_cast<GICP*>(h)->trace_on = on != 0; }
int oracle_gicp_get_trace(void* h, void* out, int cap) {
  const auto& t = static_cast<GICP*>(h)->trace;
  const size_t k = std::min(t.size(), (size_t)std::max(cap, 0));
  if (out && k) std::memcpy(out, t.data(), k * sizeof(GicpTraceRec));
  return (int)t.size();
}
// correspondences of the last outer iteration: source / target indices and the source point's Mahalanobis matrix
// (row-major 3x3 floats), m of each
void oracle_gicp_correspondences(void* h, int* src_idx, int* tgt_idx, float* maha9) {
  GICP* g = static_cast<GICP*>(h);
  const size_t m = g->src_idx.size();
  for (size_t i = 0; i < m; i++) {
    src_idx[i] = g->src_idx[i];
    tgt_idx[i] = g->tgt_idx[i];
    std::memcpy(maha9 + i * 9, &g->mahalanobis[(size_t)g->src_idx[i] * 9], 9 * sizeof(float));
  }
}

}  // extern "C"
