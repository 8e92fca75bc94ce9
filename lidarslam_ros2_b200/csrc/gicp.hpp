// GICP engine behind the C-ABI: K5 kNN covariances, K6 correspondences + Mahalanobis matrices, K7 cost / gradient
// reductions, and the host-side BFGS driver (pclomp::GeneralizedIterativeClosestPoint, gicp_omp_impl.hpp).
#pragma once
#include "engine.hpp"

namespace b200 {

constexpr int GICP_MAX_K = 32;

struct GicpConfig {  // gicp_omp.h:108-128
  int k_correspondences = 20;
  double gicp_epsilon = 0.001;
  double rotation_eps = 2e-3;
  int max_inner_iterations = 20;
  int max_iterations = 200;
  double trans_eps = 5e-4;
  double corr_dist = 5.0;
  double gradient_tol = 1e-2;  // see oracle/gicp.hpp header note on testGradient
};

struct GicpOutcome {
  float final_T[16];
  int converged, iterations, evaluations;
};

struct GicpInnerWork;     // device work area of the persistent inner-loop kernel (gicp.cu)
struct GicpInnerResult {  // written by the kernel into pinned host memory
  double x[6];
  double f;
  double g[6];  // gradient at x: the BFGS's last one, or the evaluate-once call's (zero for an f-only call)
  float T[12];  // row-major 3x4 transform apply_state_dev builds from x
  int status, inner, evaluations, error;
  int trace_n;  // trace records produced so far in the align(), when traced
};

class GicpSolver {
 public:
  ~GicpSolver() {
    if (h_trace_) cudaFreeHost(h_trace_);
  }
  void init(int device, cudaStream_t s);
  void invalidate_target() {
    target_cov_valid_ = false;
    corr_current_ = false;
  }
  void invalidate_source() {
    source_cov_valid_ = false;
    source_grid_valid_ = false;
    corr_current_ = false;
  }
  // the correspondences of the last K6 pass still refer to the clouds set now (no setInput* since)
  bool correspondences_current() const { return corr_current_; }
  // traced: record the trace set up by set_trace (single aligns; batch calls pass false)
  GicpOutcome align(const NnGrid& target_grid, const float4* target, size_t n_target, const float4* source,
                    size_t n_source, const GicpConfig& cfg, const float* guess_rowmajor16, cudaStream_t s,
                    bool traced = false);
  // the two halves of align()'s work, public for the read-back tests:
  // prelude: lazy covariances (K5), the source grid, moved = guess * source
  void prepare(const NnGrid& target_grid, const float4* target, size_t n_target, const float4* source, size_t n_source,
               const GicpConfig& cfg, const float* guess_rowmajor16, cudaStream_t s);
  // one K6 pass at transformation_ = transformation_rowmajor16: nearest neighbours, distance gate, Mahalanobis
  // matrices; returns (and keeps) the correspondence count m
  int correspondences(const NnGrid& target_grid, const GicpConfig& cfg, const float* guess_rowmajor16,
                      const float* transformation_rowmajor16, cudaStream_t s);
  // one functor evaluation at state x on the current correspondences, by the path align() uses: the persistent kernel in
  // evaluate-once mode (device_bfgs) or one gicp_cost_kernel launch. g6 is written when want_grad; T12 (row-major 3x4) is
  // the f32 transform that path built from x. Requires m >= 4 (align() never evaluates with fewer).
  void evaluate(const double* x, bool want_grad, double* f, double* g6, float* T12);
  // read-back of the last K6 pass: corr n_source ints (-1 = none), maha n_source x 9 floats (meaningful where corr >= 0)
  void read_correspondences(int* corr, float* maha9, cudaStream_t s);
  // read-back for parity tests (row-major 3x3 doubles per point); which: 0 source, 1 target
  size_t covariances(int which, std::vector<double>& out, cudaStream_t s);
  int last_correspondences() const { return last_m_; }
  size_t n_source() const { return n_source_; }
  int launches = 0;
  // true: estimateRigidTransformationBFGS runs as ONE persistent cooperative kernel per outer iteration (BFGS on the
  // device); false: host-side BFGS, one K7 launch + synchronisation per functor evaluation
  bool device_bfgs = true;
  // accounting of the last align(): device time of the persistent inner kernel(s), their launches, and the
  // (correspondence, evaluation) products they processed (algorithmic bytes = that times 72, DESIGN.md section 4)
  float inner_ms = 0;
  int inner_launches = 0;
  double inner_pair_evaluations = 0;
  // opt-in trace of align() (b200reg_gicp_set_trace / b200reg_gicp_get_trace): functor calls, BFGS steps, outer iterations
  void set_trace(int capacity);
  int read_trace(b200reg_gicp_trace_record* out, int cap) const;  // copies up to cap records, returns the records counted

 private:
  void fdf(const float* T_rowmajor16, bool want_grad, double* f, double* g_t3, double* R9);
  // returns the BFGS status; x is updated in place. eval_once: 0 runs the BFGS; 1 (f only) or 2 (f and g) makes exactly
  // one functor call at x instead, its result left in *h_inner_result_
  int inner_loop_device(double* x, const GicpConfig& cfg, int* inner_iterations, int eval_once = 0);
  GicpInnerWork* d_inner_work_ = nullptr;
  GicpInnerResult* h_inner_result_ = nullptr;  // pinned
  unsigned inner_epoch_ = 0;
  cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
  int sm_count_ = 0;
  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  bool target_cov_valid_ = false, source_cov_valid_ = false, source_grid_valid_ = false, corr_current_ = false;
  int cov_k_ = 0;
  double cov_eps_ = 0;
  NnGrid source_grid_;
  DeviceBuffer<double> target_cov_, source_cov_;  // 6 doubles per point (xx xy xz yy yz zz)
  DeviceBuffer<float> maha_;                      // 9 floats per source point
  DeviceBuffer<int> corr_;                        // target index per source point, -1 = none
  DeviceBuffer<int> nn_idx_;
  DeviceBuffer<float> nn_d2_;
  DeviceBuffer<float4> moved_;                    // source transformed by the guess ("output" cloud)
  DeviceBuffer<double> partials_;                 // per-CTA partial sums (16 doubles each)
  DeviceBuffer<double> result_;                   // 16 doubles
  DeviceBuffer<unsigned> counter_;
  double* h_result_ = nullptr;                    // pinned
  size_t n_source_ = 0, n_target_ = 0;
  const float4* target_ = nullptr;
  int last_m_ = 0;
  int evaluations_ = 0;
  // pinned, device-visible: the inner kernel's controller writes its call and step records there directly
  b200reg_gicp_trace_record* h_trace_ = nullptr;
  int trace_cap_ = 0;
  int trace_n_ = 0;      // records produced by the current / last align()
  int trace_outer_ = 0;  // outer iteration being traced
  bool tracing_ = false; // the current align() is traced
  b200reg_gicp_trace_record* trace_slot(int type);  // next record, zeroed (nullptr past the capacity); counts it
};

// k-NN based point covariances of a cloud against its own grid (gicp_omp_impl.hpp:48-122)
void gicp_covariances(const NnGrid& grid, const float4* pts, size_t n, int k, double gicp_epsilon, double* d_cov6,
                      cudaStream_t s);

}  // namespace b200
