/* b200reg.h — C-ABI of the H100-native scan-registration engine.
 *
 * Drop-in boundary: the pcl::Registration<PointXYZI,PointXYZI> surface that lidarslam_ros2's nodes hold
 * (scanmatcher/include/scanmatcher/scanmatcher_component.h:93, graph_based_slam/include/graph_based_slam/
 * graph_based_slam_component.h:106) and through which they drive pclomp::NormalDistributionsTransform and
 * pclomp::GeneralizedIterativeClosestPoint. Every entry point below names the reference interface it
 * replaces (paths relative to the reference root; "ndt.h" = Thirdparty/ndt_omp_ros2/include/pclomp/ndt_omp.h,
 * "gicp.h" = .../gicp_omp.h, "sm.cpp" = scanmatcher/src/scanmatcher_component.cpp,
 * "gbs.cpp" = graph_based_slam/src/graph_based_slam_component.cpp).
 *
 * Conventions
 *  - plain C, opaque handle, no exceptions; every call returns 0 (B200REG_OK) or a negative error code,
 *    b200reg_last_error() gives the text. PCL-style soft failure: an empty cloud is rejected and ignored.
 *  - 4x4 matrices are 16 floats COLUMN-MAJOR — exactly Eigen::Matrix4f::data().
 *  - clouds are (const float* base, size_t n, size_t stride_bytes) with x,y,z at byte offsets 0,4,8 of every
 *    point: pass pcl::PointCloud<PointXYZI>::points.data() with stride 32 (PointXYZ: 16).
 *  - a record layout (stride_bytes[, intensity_offset_bytes]) is valid when stride_bytes >= 12 and is a multiple of 4,
 *    and the intensity offset is either negative (no intensity) or a multiple of 4 with offset + 4 <= stride_bytes (the
 *    intensity float lies inside the record: PointXYZI's 16, a PointCloud2 intensity field's offset). Any other layout
 *    is refused with B200REG_ERR_ARG before anything is copied or launched, and the handle or session is unchanged.
 *  - the library copies what it needs to the GPU inside set_input_*; caller memory (host or device) may be freed or
 *    overwritten on return. A device buffer must be complete (its producer stream synchronised) at the call.
 *  - one handle = one CUDA stream + its device buffers; a handle is used from one host thread at a time,
 *    different handles may be used concurrently from different threads (lidarslam/src/lidarslam.cpp:12-17).
 *  - there is NO CPU fallback: without a CUDA device b200reg_create fails with B200REG_ERR_CUDA.
 */
#ifndef B200REG_H_
#define B200REG_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200reg_engine* b200reg_t;

enum b200reg_kind { B200REG_NDT = 0, B200REG_GICP = 1 };

/* pclomp::NeighborSearchMethod (ndt.h:52-57), same numeric order */
enum b200reg_search { B200REG_KDTREE = 0, B200REG_DIRECT26 = 1, B200REG_DIRECT7 = 2, B200REG_DIRECT1 = 3 };

enum b200reg_status {
  B200REG_OK = 0,
  B200REG_ERR_ARG = -1,       /* bad argument / wrong engine kind                                    */
  B200REG_ERR_NO_TARGET = -2, /* align/fitness without setInputTarget (PCL: initCompute() fails)      */
  B200REG_ERR_NO_SOURCE = -3, /* align without setInputSource                                          */
  B200REG_ERR_CUDA = -4,      /* CUDA runtime error, or no device                                      */
  B200REG_ERR_TIMEOUT = -5,   /* device-side watchdog fired inside the persistent solver               */
  B200REG_ERR_GRID = -6,      /* voxel grid would overflow int32 (voxel_grid_covariance_omp_impl.hpp:79) */
  B200REG_ERR_IO = -7,        /* a file could not be opened, read or written                           */
  B200REG_ERR_FORMAT = -8     /* a PCD file the reader does not accept (b200reg_load_pcd)              */
};

/* ---- lifetime --------------------------------------------------------------------------------------- */
/* replaces `new pclomp::NormalDistributionsTransform<...>()` / `new pclomp::GeneralizedIterativeClosestPoint
 * <...>()` (sm.cpp:105-106,116-117; gbs.cpp:64-65,74-75). Defaults are the reference constructors'
 * (ndt_omp_impl.hpp:47-76: resolution 1.0, step 0.1, outlier 0.55, eps 0.1, 35 iterations, DIRECT7;
 * gicp.h:108-128: k=20, gicp_eps 1e-3, rot_eps 2e-3, 20 inner, 200 outer, eps 5e-4, corr-dist 5). */
int b200reg_create(int kind, int device, b200reg_t* out);
int b200reg_destroy(b200reg_t h);
const char* b200reg_last_error(b200reg_t h);

/* ---- pcl::Registration setters (sm.cpp:109,118-119; gbs.cpp:66-69,76-81) ---------------------------- */
int b200reg_set_transformation_epsilon(b200reg_t h, double eps);      /* setTransformationEpsilon      */
int b200reg_set_maximum_iterations(b200reg_t h, int n);               /* setMaximumIterations          */
int b200reg_set_max_correspondence_distance(b200reg_t h, double d);   /* setMaxCorrespondenceDistance  */
int b200reg_set_euclidean_fitness_epsilon(b200reg_t h, double eps);   /* stored; unused by both engines */
int b200reg_set_ransac_iterations(b200reg_t h, int n);                /* stored; unused by both engines */

/* ---- pclomp::NormalDistributionsTransform setters / getters (ndt.h:110-233) ------------------------- */
int b200reg_ndt_set_resolution(b200reg_t h, float resolution);        /* ndt.h:127-137                 */
int b200reg_ndt_set_step_size(b200reg_t h, double step);              /* ndt.h:162-166                 */
int b200reg_ndt_set_outlier_ratio(b200reg_t h, double ratio);         /* ndt.h:180-184 (setOulierRatio) */
int b200reg_ndt_set_neighborhood_search_method(b200reg_t h, int m);   /* ndt.h:186-188                 */
int b200reg_ndt_set_num_threads(b200reg_t h, int n);                  /* ndt.h:110-112; accepted, no-op */
int b200reg_ndt_get_transformation_probability(b200reg_t h, double* out); /* ndt.h:193-197             */
int b200reg_ndt_get_final_num_iteration(b200reg_t h, int* out);       /* ndt.h:202-206                 */
/* ndt.h:233 calculateScore(cloud): cloud is an already-transformed source */
int b200reg_ndt_calculate_score(b200reg_t h, const float* base, size_t n, size_t stride_bytes, double* out);

/* ---- pclomp::GeneralizedIterativeClosestPoint setters (gicp.h:156-252) ------------------------------- */
int b200reg_gicp_set_rotation_epsilon(b200reg_t h, double eps);       /* setRotationEpsilon            */
int b200reg_gicp_set_correspondence_randomness(b200reg_t h, int k);   /* setCorrespondenceRandomness   */
int b200reg_gicp_set_maximum_optimizer_iterations(b200reg_t h, int n);/* setMaximumOptimizerIterations */
int b200reg_gicp_set_epsilon(b200reg_t h, double gicp_epsilon);       /* gicp_epsilon_ (gicp.h:110)    */

/* ---- clouds ----------------------------------------------------------------------------------------- */
/* setInputTarget (ndt.h:117-122 → init() ndt.h:271-278 → VoxelGridCovariance::filter; gicp.h:156-170):
 * uploads the cloud and, for NDT, builds the voxel map (mean / regularised inverse covariance) on the GPU. */
int b200reg_set_input_target(b200reg_t h, const float* base, size_t n, size_t stride_bytes);
/* setInputSource (pcl::Registration; gicp.h:133-149) */
int b200reg_set_input_source(b200reg_t h, const float* base, size_t n, size_t stride_bytes);
/* Same, from a DEVICE buffer of n float4 (x,y,z,ignored) already resident in HBM on the handle's device. */
int b200reg_set_input_target_device(b200reg_t h, const void* dev_float4, size_t n);
int b200reg_set_input_source_device(b200reg_t h, const void* dev_float4, size_t n);

/* ---- align ------------------------------------------------------------------------------------------ */
/* pcl::Registration::align(output, guess) (sm.cpp:353, gbs.cpp:230, apps/align.cpp:27,33) →
 * computeTransformation (ndt_omp_impl.hpp:80-171 / gicp_omp_impl.hpp:369-515). guess == NULL means identity.
 * Synchronous: on return final_out (may be NULL) holds getFinalTransformation(). */
int b200reg_align(b200reg_t h, const float* guess, float* final_out);
int b200reg_get_final_transformation(b200reg_t h, float* out16);      /* sm.cpp:356; gbs.cpp:244,253   */
int b200reg_has_converged(b200reg_t h, int* out);                     /* sm.cpp:375                    */
/* getFitnessScore(max_range) (gbs.cpp:231, sm.cpp:376): mean squared 1-NN distance of the aligned source
 * to the target, over points with d^2 <= max_range; DBL_MAX if none. */
int b200reg_get_fitness_score(b200reg_t h, double max_range, double* out);
/* the `output` cloud of align(): source transformed by the final transformation; out has n_source points */
int b200reg_get_aligned(b200reg_t h, float* out, size_t stride_bytes);

/* align() on `count` independent handles (each with its own target and source already set), one after the other — a
 * convenience loop: every solve is a persistent kernel that owns all SMs, so solves never overlap; what overlaps between
 * pairs is done by b200reg_ndt_sweep below (uploads, map builds, fitness passes). guesses may be NULL (identity);
 * finals = 16*count floats. Results are those of b200reg_align on each handle. */
int b200reg_align_batch(b200reg_t* handles, int count, const float* guesses, float* finals);

/* K independent NDT registrations against the handle's CURRENT target in ONE persistent launch — repeated
 * align() calls of apps/align.cpp:32-36 ("10times"), multi-hypothesis initial guesses, or the candidate scans of a
 * loop-closure sweep sharing one map. Up to three registrations are in flight inside the kernel: while one registration's
 * Newton step (fixed-order reduction, 6x6 solve, next pose) runs on its controller SM, the evaluator SMs compute the
 * other registrations' derivatives, so the sequential part of ndt_omp_impl.hpp:121-166 no longer idles the GPU.
 * Every result is BITWISE the result b200reg_align gives for the same (source, guess).
 * guesses: 16*count floats column-major, or NULL (identity). results[k].status is B200REG_OK or an error code.
 * After the call the handle's getters (final transformation, converged, ...) describe the LAST registration;
 * b200reg_get_stats reports evaluations / hits_total / solve_ms summed over the batch. */
typedef struct b200reg_batch_result {
  float final_T[16];         /* getFinalTransformation(), column-major                                     */
  double trans_probability;  /* getTransformationProbability()                                              */
  int converged, iterations, evaluations, status;
  long long hits_total;
} b200reg_batch_result;
/* sources in HOST memory: (base, n, stride) clouds as in b200reg_set_input_source, one bulk copy + unpack each, no
 * synchronisation in between */
int b200reg_ndt_align_batch(b200reg_t h, int count, const float* const* sources, const size_t* n_points,
                            size_t stride_bytes, const float* guesses, b200reg_batch_result* results);
/* sources already in HBM as float4 (x, y, z, ignored) on the handle's device; read in place (no copy) — they must
 * be complete when the call is made and stay untouched until it returns */
int b200reg_ndt_align_batch_device(b200reg_t h, int count, const void* const* dev_sources, const size_t* n_points,
                                   const float* guesses, b200reg_batch_result* results);
/* The loop-closure candidate sweep on one GPU (generalises gbs.cpp:187-233 from the arg-min candidate to all of them):
 * `count` independent (source, target) pairs, each through the node's own sequence setInputTarget (gbs.cpp:227) ->
 * setInputSource (:181) -> align (:230) -> getFitnessScore (:231) with the handle's parameters. Two internal engines
 * (stream + buffers each) driven by two host threads take the pairs in turn, so that the upload and voxel-map build of
 * one pair overlap the solve and fitness pass of the other. Results equal those of the sequential calls.
 * guesses: 16*count floats column-major or NULL (identity). Sharding pairs across GPUs is the caller's (one process per
 * GPU, include/b200comm.h for the all-gather of the result rows). */
typedef struct b200reg_sweep_result {
  float final_T[16];         /* column-major */
  double fitness;            /* getFitnessScore(fitness_max_range) */
  double trans_probability;
  int converged, iterations, status, pad;
} b200reg_sweep_result;
int b200reg_ndt_sweep(b200reg_t h, int count, const float* const* sources, const size_t* n_src,
                      const float* const* targets, const size_t* n_tgt, size_t stride_bytes, const float* guesses,
                      double fitness_max_range, b200reg_sweep_result* results);
/* Multi-GPU form of the batch calls (SURVEY.md section 8e: the shards are independent, the only exchange is the 4x4 poses):
 * attach a pose board (include/b200comm.h, b200comm_board_create) and every b200reg_ndt_align_batch[_device] call on this
 * handle also publishes its poses to all ranks FROM INSIDE the solver kernel — peer-memory stores over NVLink as each
 * registration converges — and returns when all ranks' poses of the call have arrived here. Such calls are collective:
 * all ranks of the board make the same sequence of them (counts may differ; 1 <= count <= the board's max_rows).
 * b200reg_ndt_gathered_poses then copies them out: poses[(r * max_rows + k) * 16 ..] = column-major pose of rank r's
 * registration k, counts[r] = how many rank r registered. board = NULL detaches. */
struct b200comm_board;
int b200reg_ndt_attach_pose_board(b200reg_t h, struct b200comm_board* board);
int b200reg_ndt_gathered_poses(b200reg_t h, float* poses, int* counts, int max_rows);
/* registrations in flight per batch launch (1..3; default 3). Developer / measurement switch. */
int b200reg_ndt_set_batch_slots(b200reg_t h, int slots);

/* ---- pcl::VoxelGrid<PointXYZI>::filter (sm.cpp:266-269,311-314,325-328,444-447; gbs.cpp:225-226) ------ */
/* Centroid downsample of all fields (x,y,z,intensity). intensity_offset_bytes < 0: no intensity field.
 * out: same point layout as in (stride_bytes), capacity in points; *m = number of output points (ascending
 * leaf index). Each output record gets x, y, z, the intensity (when there is one) and, for strides >= 16 whose bytes
 * 12-15 are not the intensity, PointXYZ's padding float data[3] = 1; its other bytes are not written.
 * If the grid would overflow int32 the input records are returned unchanged (PCL behaviour). */
int b200reg_voxelgrid(int device, const float* in, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                      float leaf, float* out, size_t out_capacity, size_t* m);

/* ---- introspection (parity tests, roofline accounting) ---------------------------------------------- */
typedef struct b200reg_stats {
  int evaluations;        /* computeDerivatives passes of the last align (ndt_omp_impl.hpp:179)          */
  int iterations;         /* nr_iterations_                                                              */
  long long hits;         /* (point, voxel) pairs visited in the last evaluation                         */
  long long hits_total;   /* ... summed over all evaluations of the last align                           */
  float solve_ms;         /* device time of the last align's solver kernel (CUDA events, handle stream)  */
  float target_build_ms;  /* device time of the last setInputTarget                                      */
  int kernel_launches;    /* kernels launched by this handle since creation                              */
  int grid_ctas, block_threads, index_in_smem;
  long long n_voxels, n_cells, n_source, n_target;
  /* GICP: the persistent inner-loop kernel(s) of the last align (estimateRigidTransformationBFGS on the device)      */
  float gicp_inner_ms;             /* their summed device time (CUDA events on the handle's stream)                  */
  int gicp_inner_launches;         /* = outer iterations                                                            */
  double gicp_pair_evaluations;    /* sum over cost / gradient evaluations of the number of correspondences          */
} b200reg_stats;
int b200reg_get_stats(b200reg_t h, b200reg_stats* out);

/* one fused derivative pass (ndt_omp_impl.hpp:179-284) at a given transform T (col-major) with the angle
 * tables taken at p6[3..5]; out: score, g[6], H[36] row-major. */
int b200reg_ndt_derivatives(b200reg_t h, const float* T, const double* p6, int compute_hessian, double* score,
                            double* g6, double* H36);
/* NDT score of `count` rigid poses of the handle's current source against its current target, in one launch.
 * scores[k] = the score of computeDerivatives (ndt_omp_impl.hpp:179-284) at poses[k] (16 floats, column-major): over the
 * source points and the voxels of their neighbourhood (the handle's search method: KDTREE, DIRECT26, DIRECT7, DIRECT1), the
 * sum of -d1 * exp(-d2 * q / 2), with a pair dropped, score included, by the test of :504-505. hits[k] (may be NULL) =
 * pairs kept. The per-pair arithmetic is the solver's; each point's pairs are summed in f32 in probe order and added to an
 * f64 sum, so scores[k] agrees with b200reg_ndt_derivatives' score to rounding and hits[k] equals its hit count.
 * Deterministic: scores[k] and hits[k] depend bit for bit only on poses[k], the two clouds, the resolution, the outlier
 * ratio and the search method — not on count, on k or on the other poses.
 * count == 0: B200REG_OK, nothing launched. A GICP handle, count < 0 or a non-finite pose entry: B200REG_ERR_ARG (checked
 * before anything is launched). No target / no source: B200REG_ERR_NO_TARGET / B200REG_ERR_NO_SOURCE. A target with no
 * valid voxel: every score and hit count is 0. An ordinary (not cooperative) launch on the handle's stream. The handle
 * keeps device buffers for the largest count it has scored (80 bytes per pose, grown geometrically) until it is destroyed. */
int b200reg_ndt_score_poses(b200reg_t h, int count, const float* poses_colmajor16, double* scores, long long* hits);
/* Hessian-only pass over the radius neighbourhood in f64 (ndt_omp_impl.hpp:538-629) */
int b200reg_ndt_hessian_radius(b200reg_t h, const float* T, const double* p6, double* H36);
/* voxel map read-back, voxels with >= 6 points in ascending leaf index (voxel_grid_covariance_omp_impl.hpp:
 * 282-367). Any pointer may be NULL. mean3/icov9 doubles, centroid3 floats. */
int b200reg_ndt_num_voxels(b200reg_t h, size_t* out);
int b200reg_ndt_get_voxels(b200reg_t h, int* leaf_idx, int* npts, double* mean3, double* icov9, float* centroid3);
/* GICP read-back for parity tests: per-point 3x3 covariances (row-major doubles, gicp_omp_impl.hpp:48-122) of the
 * source (which = 0) or target (which = 1) cloud after an align(); *n = number of points (out9 may be NULL). */
int b200reg_gicp_get_covariances(b200reg_t h, int which, double* out9, size_t* n);
int b200reg_gicp_num_correspondences(b200reg_t h, int* out);
/* GICP read-back for the kernel tests: the prelude of align() (lazy covariances, source grid, output = guess * source)
 * and one correspondence pass (gicp_omp_impl.hpp:412-456) at transformation_ = T. guess and T are column-major, NULL =
 * identity. corr: n_source ints, the target index or -1 (may be NULL); maha9: n_source x 9 floats, row-major
 * (meaningful where corr >= 0; may be NULL); *m = number of correspondences. The state stays in place for
 * b200reg_gicp_objective. */
int b200reg_gicp_correspondences(b200reg_t h, const float* guess, const float* T, int* corr, float* maha9, int* m);
/* one evaluation of the fixed-correspondence objective (operator() when want_grad == 0, else fdf;
 * gicp_omp_impl.hpp:244-366) at state x6 on the correspondences of the last align() / b200reg_gicp_correspondences, by
 * the persistent inner-loop kernel align() uses, run for this one call.
 * g6 is written when want_grad; T12 (may be NULL) = the f32 row-major 3x4 transform the kernel built from x6.
 * B200REG_ERR_ARG when there are fewer than 4 correspondences or the clouds changed since they were found. */
int b200reg_gicp_objective(b200reg_t h, const double* x6, int want_grad, double* f, double* g6, float* T12);
/* NDT read-back for the controller tests: an opt-in per-round trace of b200reg_align (batch calls are never traced).
 * Each round of the solver's Newton / More-Thuente controller (ndt_omp_impl.hpp:80-171, 756-916) appends one record:
 * the totals it consumed, its state after the step and the control block it published. Launches that resume after a K2
 * pass continue the trace of their align(). b200reg_ndt_set_trace(h, capacity) keeps room for `capacity` records
 * (0 turns tracing off); b200reg_ndt_get_trace copies min(*n, capacity, cap) records of the last align() and sets *n to
 * the number of rounds it ran, which exceeds the capacity when the trace overflowed.
 * phase: 0 initial evaluation, 1 first evaluation of a line search, 2 More-Thuente iteration, 3 K2 Hessian pending. */
typedef struct b200reg_ndt_trace_record {
  int round;              /* round within its launch                                                              */
  int launch;             /* 0 for the first launch of the align(), +1 for each launch resumed after a K2 pass     */
  int phase_before, phase_after;
  int fast;               /* 1: the warp-parallel Newton step handled the round, 0: the scalar controller          */
  int evaluated;          /* 1: the round consumed a fresh evaluation (0: the first round of a resumed launch)     */
  int built;              /* 1: the round built a control block: T, jang, hang, compute_hessian are valid           */
  int build_f64;          /* 1: ... and the f64 angle tables jd, hd                                                */
  int mode;               /* control word published: 0 evaluate, 1 done, 2 leave for a K2 pass                    */
  int compute_hessian;
  int interval_converged, open_interval, step_iterations, nr_iterations, evaluations, converged;
  int done;               /* 0 continue, 1 finished, 2 leave for a K2 pass                                        */
  int pad0;
  long long hits_total;
  double tot[32];         /* totals consumed: [0] score, [1..6] g, [7..27] upper H row-major, [28] hits, rest 0    */
  double score, g[6];     /* score and gradient the controller holds after the step                               */
  double p[6], dir[6], x_t[6];
  double a_t, phi_0, d_phi_0;
  double a_l, f_l, g_l, a_u, f_u, g_u;  /* More-Thuente interval; 0 on fast rounds, which keep none                */
  double H[36];           /* first round of a resumed launch: the Hessian the K2 pass injected; 0 otherwise       */
  double jd[24], hd[45];  /* f64 angle tables at x_t (hd row d1 carries -sy) when build_f64, 0 otherwise         */
  float T[12];            /* 3x4 row-major transform of the published control block                               */
  float jang[24], hang[45];
  float final_T[16];      /* final_transformation_ after the step, row-major                                      */
  float pad1;
} b200reg_ndt_trace_record;
int b200reg_ndt_set_trace(b200reg_t h, int capacity);
int b200reg_ndt_get_trace(b200reg_t h, b200reg_ndt_trace_record* out, int capacity, int* n);
/* GICP read-back for the optimiser tests: an opt-in trace of b200reg_align (batch calls are never traced), one stream of
 * records in the order they happen. estimateRigidTransformationBFGS (gicp_omp_impl.hpp:180-241) appends a type 0 record
 * per functor call and a type 1 record per minimizeOneStep; each outer iteration of computeTransformation (:369-515)
 * ends with a type 2 record. The type 0 and 1 records come from the persistent inner-loop kernel's controller: each of
 * the twelve T words is written by the controller thread that published it.
 * b200reg_gicp_set_trace(h, capacity) keeps room for `capacity` records (0 turns tracing off); b200reg_gicp_get_trace
 * copies min(*n, capacity, cap) records of the last align() and sets *n to the number of records it produced, which
 * exceeds the capacity when the trace overflowed. Fields a record type does not use are 0. */
typedef struct b200reg_gicp_trace_record {
  int type;               /* 0 functor call, 1 minimizeOneStep, 2 outer iteration                                    */
  int outer;              /* outer iteration, from 0                                                                 */
  int inner;              /* 0, 1: the inner iteration (0 = minimizeInit's call); 2: inner iterations the BFGS ran   */
  int evaluation;         /* 0: index of the call in its BFGS run, from 0; 1, 2: calls made so far in the run        */
  int want_grad;          /* 0: 0 operator() (f only), 1 fdf / df                                                    */
  int status;             /* 1: minimizeOneStep's status; 2: the BFGS result, -2 when m < 4 stopped the loop         */
  int m;                  /* 2: correspondences of the iteration                                                     */
  int nr_iterations;      /* 2: after the iteration                                                                  */
  int converged;          /* 2: after the iteration                                                                  */
  int last;               /* 2: 1 on the last record of the align(), which carries final_T                           */
  double x[6];            /* 0: the state the call was made at; 1: x after the step; 2: x the BFGS returned          */
  double f;               /* 0: f returned to the BFGS; 1: f after the step                                          */
  double g[6];            /* 0: g returned to the BFGS (0 for f-only calls); 1: the gradient after the step          */
  double x0[6];           /* 2: the state extracted from transformation_                                             */
  double delta;           /* 2: the convergence delta                                                                */
  float T[12];            /* 0: the row-major 3x4 transform published for the call; 2: transformation_ after applyState */
  float final_T[16];      /* 2, last record: final_transformation_, row-major                                        */
} b200reg_gicp_trace_record;
int b200reg_gicp_set_trace(b200reg_t h, int capacity);
int b200reg_gicp_get_trace(b200reg_t h, b200reg_gicp_trace_record* out, int capacity, int* n);
/* exact 1-NN of n query points against the target cloud (building block of getFitnessScore / GICP) */
int b200reg_nn1(b200reg_t h, const float* base, size_t n, size_t stride_bytes, int* idx, float* d2);

/* ---- scan-matcher frontend session: device-resident map maintenance (SURVEY.md section 8f, rows 1 and 3) --------
 * The callers either side of align() in scanmatcher/src/scanmatcher_component.cpp, rebuilt so that a frame costs ONE
 * host-to-device copy: the submaps (voxel-filtered, sensor frame) and the targeted cloud stay in HBM.
 * Poses are position (x, y, z) + quaternion (x, y, z, w) in double, like geometry_msgs/Pose.                       */
typedef struct b200sm_session* b200sm_t;
int b200sm_create(int device, b200sm_t* out);
void b200sm_destroy(b200sm_t s);
const char* b200sm_last_error(b200sm_t s);
int b200reg_get_kind(b200reg_t h, int* kind);
/* node parameters: vg_size_for_input, vg_size_for_map, num_targeted_cloud, trans_for_mapupdate, use_min_max_filter,
 * scan_min_range, scan_max_range (sm.cpp:34-50; defaults 0.2, 0.1, 10, 1.5, false, 0.1, 100)                        */
int b200sm_set_params(b200sm_t s, float vg_size_for_input, float vg_size_for_map, int num_targeted_cloud,
                      double trans_for_mapupdate, int use_min_max_filter, double scan_min_range, double scan_max_range);
int b200sm_set_initial_pose(b200sm_t s, const double* position3, const double* quat_xyzw); /* sm.cpp:57-69, 127-141 */
/* cloud_callback range filter (sm.cpp:211-219) + receiveCloud's VoxelGrid(vg_size_for_input) and
 * registration->setInputSource (sm.cpp:323-328): uploads the frame once and keeps it on the device for a later
 * b200sm_update_map. *n_filtered = points of the filtered source.                                                    */
int b200sm_set_scan(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes,
                    long intensity_offset_bytes, size_t* n_filtered);
/* updateMap (sm.cpp:438-491; the first call is initializeMap, sm.cpp:257-297) on the frame given to the last
 * b200sm_set_scan / b200sm_receive_cloud: VoxelGrid(vg_size_for_map) -> new submap (kept untransformed with its
 * pose); targeted cloud = transformPointCloud(filtered, final_T [float]) followed by the previous
 * num_targeted_cloud-1 submaps, newest first, each through its pose matrix [double]. adopt_now != 0 also performs
 * receiveCloud's registration->setInputTarget(targeted) (sm.cpp:300-322; GICP: VoxelGrid(vg_size_for_input) first). */
int b200sm_update_map(b200sm_t s, b200reg_t reg, const float* final_T_colmajor16, const double* position3,
                      const double* quat_xyzw, int adopt_now);
/* One frame of the frontend: cloud_callback + initializeMap (first frame) + receiveCloud + publishMapAndPose
 * (sm.cpp:201-235, 299-434): adopt a pending target, filter, setInputSource, align(guess = current pose), pose
 * bookkeeping, and updateMap when the sensor moved >= trans_for_mapupdate (performed immediately; the new target is
 * adopted at the start of the next frame — the reference's mapping thread finishing before the next scan).
 * pose7_out = position + quaternion after the frame; *map_updated = 1 if updateMap ran.                             */
int b200sm_receive_cloud(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes,
                         long intensity_offset_bytes, double* pose7_out, float* final_T_colmajor16_out, int* map_updated);
/* cloud_callback's tf2::doTransform(*msg, transformed_msg, transform) (sm.cpp:188-199): transform =
 * lookupTransform(robot_frame_id_, msg->header.frame_id, stamp). Every later frame given to b200sm_set_scan /
 * b200sm_receive_cloud is moved into the robot frame by the upload's unpack pass, before the de-skew, the range filter and
 * both VoxelGrids, so the caller passes msg->data as it arrived. The matrix is tf2_sensor_msgs' Translation3f *
 * Quaternionf(w, x, y, z) in float, the quaternion used as given (not normalised); each point is
 * ((r0 x + r1 y) + r2 z) + t, intensity copied. A caller whose TF varies calls this before each frame. Both pointers
 * NULL: off (the points are used as given). Non-finite values or a zero quaternion: B200REG_ERR_ARG.                 */
int b200sm_set_sensor_transform(b200sm_t s, const double* translation3, const double* quat_xyzw);
/* use_odom (sm.cpp:333-348) for the NEXT b200sm_receive_cloud: the odometry = lookupTransform(odom_frame_id_,
 * robot_frame_id_, stamp). That frame's guess becomes sim_trans * previous_odom_mat_^-1 * odom_mat (all float; nothing
 * changes while previous_odom_mat_ is exactly Identity, as on the first armed frame), then previous_odom_mat_ = odom_mat.
 * A frame without an armed odometry keeps the current pose as its guess and leaves previous_odom_mat_ unchanged.
 * Non-finite values or a zero quaternion: B200REG_ERR_ARG.                                                          */
int b200sm_odom_next_scan(b200sm_t s, const double* translation3, const double* quat_xyzw);
/* read-back (parity tests; the node's map / map_array publishers). Clouds are x, y, z, intensity floats. */
int b200sm_num_submaps(b200sm_t s, size_t* out);
int b200sm_get_targeted(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n);
int b200sm_get_submap(b200sm_t s, size_t index, float* out_xyzi, size_t capacity, size_t* n, double* pose_colmajor16,
                      double* distance);
int b200sm_get_filtered_scan(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n);
/* GraphBasedSlamComponent::searchLoop (gbs.cpp:144-258) on the session's submaps, device-resident: the newest submap is the
 * source; among the older submaps with (travelled-distance gap > distance_loop_closure) and (position distance <
 * range_of_searching_loop_closure) the closest one, id_min, is the candidate; target = VoxelGrid(voxel_leaf_size) of the
 * submaps id_min +- search_submap_num, each moved by its pose cast to float; align() without guess, getFitnessScore();
 * accepted iff fitness < threshold_loop_closure_score, then relative_pose = from^-1 * (final * init) as in the LoopEdge.
 * `reg` is the backend's registration object (gbs.cpp:47-64 sets its parameters). 4x4 matrices are column-major.       */
typedef struct b200sm_loop_result {
  int is_candidate, id_min, accepted, pad;
  double min_dist, fitness;
  float final_T[16];
  double relative_pose[16];
  size_t n_source, n_target;
} b200sm_loop_result;
int b200sm_search_loop(b200sm_t s, b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score,
                       double distance_loop_closure, double range_of_searching_loop_closure, int search_submap_num,
                       b200sm_loop_result* out);
/* ---- IMU de-skew (use_imu; sm.cpp:205-209, 222-235): LidarUndistortion of scanmatcher/include/scanmatcher/
 * lidar_undistortion.hpp. getImu (:52-106) is the per-message ring-buffer update (host state); adjustDistortion
 * (:110-226) runs as kernels on the uploaded scan: the half-turn switch is a first-index reduction, the carried IMU
 * ring pointer an exclusive prefix-max scan, interpolation + rigid correction per point.                          */
int b200sm_imu_set_scan_period(b200sm_t s, double scan_period);                        /* setScanPeriod :228  */
int b200sm_imu_push(b200sm_t s, const float* angular_velocity3, const float* linear_acceleration3,
                    const float* orientation_xyzw, double stamp_sec);                  /* getImu :52-106      */
/* arm the de-skew for the NEXT frame given to b200sm_set_scan / b200sm_receive_cloud: it then runs on the device right
 * after the upload, before the range filter — cloud_callback's order (sm.cpp:205-219)                              */
int b200sm_deskew_next_scan(b200sm_t s, double scan_time_sec);
/* adjustDistortion (:110-226) on a HOST cloud, in place (x, y, z rewritten; points in firing order)               */
int b200sm_imu_adjust_distortion(b200sm_t s, float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                                 double scan_time_sec);
/* read-back for the parity tests: imu_ptr_front_, imu_ptr_last_, imu_ptr_last_iter_; one ring entry                */
int b200sm_imu_get_state(b200sm_t s, int* ptr_front, int* ptr_last, int* ptr_last_iter);
int b200sm_imu_get_sample(b200sm_t s, int index, double* stamp, float* rpy3, float* shift3, float* velo3);
/* read-back of the last adjustDistortion's per-point scratch for the de-skew tests: copies min(capacity, n) entries of
 * rel_time (float), t = scan_time + rel_time (double), imu_ptr_front_ after the walk (ring index) and the skip flag
 * (1: the point was `continue`d), and sets *n to the number of points; k_first is the first index that set half_passed
 * (n if none), rounds the passes of the skipped-set fix point (0 when the clock stepped back and the walk ran
 * literally). *n is 0 when no kernel ran (an empty cloud, or imu_ptr_last_ <= 0). Any output pointer may be NULL.    */
int b200sm_imu_get_trace(b200sm_t s, size_t capacity, size_t* n, float* rel_time, double* t, int* front,
                         unsigned char* skip, int* k_first, int* rounds);

/* A backend in its OWN process gets the submaps as lidarslam_msgs/SubMap (voxel-filtered cloud in the sensor frame, pose,
 * travelled distance; gbs.cpp:91-101): append one to the session (uploaded once, then device-resident like the
 * frontend's own). pose: 4x4 column-major double (Eigen::Affine3d::matrix().data()).                                 */
int b200sm_import_submap(b200sm_t s, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                         const double* pose_colmajor16, double distance);

/* Every candidate instead of the closest one (SURVEY.md section 8f row 2): all older submaps that pass the two gates of
 * gbs.cpp:187-204 are registered against the newest submap, each exactly like b200sm_search_loop does its single one
 * (id_min = the candidate's submap id, min_dist = its distance), on the device-resident submaps — nothing is uploaded.
 * out[0..*n_out) in ascending submap id. shard_rank / shard_world (0 / 1 on one GPU) deal the candidates out across
 * processes (candidate k -> rank k mod shard_world; *n_candidates_total = all of them); the rows are then all-gathered
 * with include/b200comm.h.                                                                                          */
int b200sm_search_loop_all(b200sm_t s, b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score,
                           double distance_loop_closure, double range_of_searching_loop_closure, int search_submap_num,
                           int shard_rank, int shard_world, b200sm_loop_result* out, size_t capacity, size_t* n_out,
                           size_t* n_candidates_total);

/* ---- place recognition: a loop search that does not trust the drifted poses (Scan Context, Kim & Kim, IROS 2018) ------
 * Each submap's cloud (sensor frame) is described by a num_rings x num_sectors grid of the horizontal plane around the
 * sensor out to max_radius: bin (ring, sector) holds the largest z + lidar_height of its points, 0 when it has none. The
 * newest descriptor is compared with every older submap's at every column shift, so a revisit is found however far the
 * odometry has drifted, and the best shift gives the heading to start the registration from. The exact definitions
 * (bins, norms, distance, guess) are in csrc/scan_context.hpp; DESIGN.md section 7b describes the search.
 * Descriptors are built on the device at the first b200sm_search_loop_place / b200sm_get_scan_context after submaps were
 * added, and stay there: num_rings * num_sectors * 4 + num_sectors * 8 bytes per submap.                                */
typedef struct b200sm_scan_context_params {
  int num_rings;        /* 1..128, default 20                                                    */
  int num_sectors;      /* 1..720, default 60; num_rings * num_sectors <= 8192                    */
  double max_radius;    /* finite, > 0, default 80 (metres, horizontal)                          */
  double lidar_height;  /* finite, default 2.0: added to z (as a float) before the max           */
} b200sm_scan_context_params;
/* NULL: the defaults. B200REG_ERR_ARG for a value out of range (nothing changes). Every cached descriptor is dropped. */
int b200sm_set_scan_context_params(b200sm_t s, const b200sm_scan_context_params* p);
/* descriptor of submap `index`, num_rings * num_sectors floats, ring-major (ring i, sector j at i * num_sectors + j);
 * capacity (floats) must hold all of it */
int b200sm_get_scan_context(b200sm_t s, size_t index, float* out, size_t capacity);

typedef struct b200sm_place_result {
  b200sm_loop_result loop;  /* filled exactly as b200sm_search_loop_all fills a row (min_dist = position distance) */
  double sc_distance;       /* D(newest, candidate)                                                                */
  int shift;                /* s*: the newest sensor is turned by about 2 pi shift / num_sectors counter-clockwise
                               relative to the candidate's                                                         */
  int pad;
  float guess[16];          /* the initial guess the verification aligned from, column-major                       */
} b200sm_place_result;
/* The newest submap against every older one with (travelled-distance gap > distance_loop_closure); there is no position
 * gate. Those with D < sc_threshold are ranked by (D, id) and the first min(top_k, capacity) are verified exactly like a
 * b200sm_search_loop_all row, except that align() starts from guess = P_cand * Rz(2 pi s* / num_sectors) * P_new^-1.
 * An accepted row is the loop edge (loop.id_min, newest, loop.relative_pose) of b200sm_pose_adjust. *n_out = rows
 * written, *n_scored (may be NULL) = eligible submaps. Fewer than two submaps: B200REG_OK with *n_out = 0.
 * B200REG_ERR_ARG for top_k outside 1..1024, a non-finite sc_threshold, voxel_leaf_size <= 0, search_submap_num < 0 or
 * out == NULL with capacity > 0. NDT and GICP handles alike.                                                        */
int b200sm_search_loop_place(b200sm_t s, b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score,
                             double distance_loop_closure, int search_submap_num, double sc_threshold, int top_k,
                             b200sm_place_result* out, size_t capacity, size_t* n_out, size_t* n_scored);
/* the last place search's per-submap scores: *n = submaps at that search; min(capacity, n) rows of D (NaN for a submap
 * that was not eligible) and s* (-1 there). Either array may be NULL.                                               */
int b200sm_get_place_scores(b200sm_t s, size_t capacity, size_t* n, double* distances, int* shifts);

/* ---- backend pose adjustment: GraphBasedSlamComponent::doPoseAdjustment (gbs.cpp:262-371) ----------------------------
 * LoopEdge of graph_based_slam_component.h: pair_id = (from, to), relative_pose = from^-1 * to (gbs.cpp:240-247).
 * A b200sm_search_loop result with accepted = 1 gives from = id_min, relative_pose = relative_pose and
 * to = the newest submap index at the time of the search (b200sm_num_submaps - 1), exactly as gbs.cpp:241 does.     */
typedef struct b200sm_loop_edge {
  int from, to;
  double relative_pose[16]; /* column-major */
} b200sm_loop_edge;
typedef struct b200sm_pose_adjust_result {
  double chi2_initial, chi2_final; /* sum of e^T e over all edges before / after                       */
  int iterations;                  /* LM iterations run (<= max_iterations; fewer when g2o would stop)  */
  int trials;                      /* damped solves tried, accepted and rejected                       */
  int n_vertices, n_edges;
} b200sm_pose_adjust_result;
/* doPoseAdjustment's graph and solve (gbs.cpp:262-319) on the session's submap poses, on the host in double precision:
 * one SE3 vertex per submap (vertex 0 fixed), for i > num_adjacent_pose_cnstraints (k) the odometry edges
 * (i-k+j, i), j = 0..k-1, then the loop edges; identity information; g2o's Levenberg-Marquardt for max_iterations
 * (the node uses 10), with an exact block-envelope Cholesky solve. poses_out = 16 * n_submaps doubles, column-major
 * (the adjusted Isometry3d of every vertex; vertex 0 is fixed). The session's own submap poses are NOT changed:
 * searchLoop, updateMap and the targeted cloud keep using the frontend's poses, as in the reference.
 * B200REG_ERR_ARG for a loop edge id outside [0, n_submaps) or from == to, a non-finite relative_pose,
 * num_adjacent_pose_cnstraints < 1 or max_iterations < 0. optimizer.save("pose_graph.g2o") (:319) is written by
 * b200sm_save_session, with the session's submaps, from the same graph. */
int b200sm_pose_adjust(b200sm_t s, int num_adjacent_pose_cnstraints, const b200sm_loop_edge* loop_edges, int n_loop_edges,
                       int max_iterations, double* poses_out, b200sm_pose_adjust_result* result);

/* ---- merging a second mapping session into the session's map ---------------------------------------------------------
 * A session's submaps form segments: one recording's contiguous run each. A session starts with one; every successful
 * b200sm_merge_session appends the other session's submaps as a new one. On a session of more than one segment
 * b200sm_set_scan, b200sm_receive_cloud and b200sm_update_map return B200REG_ERR_ARG and change nothing (it is a backend's
 * map); b200sm_import_submap appends to the last segment; b200sm_pose_adjust puts its odometry edges inside each segment
 * (with one segment: exactly the edges above); the loop searches, the map assembly, PCD saving, the occupancy grid and the
 * static map work on all the submaps. Definitions: csrc/session_merge.hpp; DESIGN.md section 7b.                       */
typedef struct b200sm_merge_params {
  double sc_threshold;                  /* candidates need D < sc_threshold; finite, default 0.4                   */
  int top_k;                            /* candidates kept per src submap, 1..32, default 3                          */
  int max_verifications;                /* candidates verified, best (D, b, a) first, 1..1024, default 64            */
  float voxel_leaf_size;                /* VoxelGrid of the verification's target window, > 0, default 0.3           */
  double threshold_loop_closure_score;  /* a verified pair is accepted iff fitness < this; not NaN, default 1.0       */
  int search_submap_num;                /* target window a +- search_submap_num (inside a's segment), >= 0, default 1 */
  double consistency_translation;       /* cycle-error tolerance |t(E)| <= t + drift_t * L, metres, default 1.5      */
  double consistency_rotation;          /* acos((tr R(E) - 1) / 2) <= r + drift_r * L, radians, default 0.1           */
  double consistency_drift_translation; /* per metre travelled around the cycle, default 0.02                         */
  double consistency_drift_rotation;    /* radians per metre, default 0.003; the four: finite, >= 0                   */
  int min_inliers;                      /* the merge succeeds iff the consistent set has this many rows, >= 1, def. 2 */
  int num_adjacent_pose_cnstraints;     /* odometry edges of the joint adjustment, >= 1, default 5                    */
  int max_iterations;                   /* LM iterations of the joint adjustment, >= 0, default 10                    */
} b200sm_merge_params;
typedef struct b200sm_merge_row {
  b200sm_place_result place;  /* loop.id_min = a (dst), loop.relative_pose = Z = P_a^-1 (F P_b) when accepted,
                                 loop.min_dist = |t(P_a) - t(F P_b)|; guess = P_a Rz(2 pi s* / S) P_b^-1; sc_distance, shift */
  int src_id;                 /* b (src)                                                                                  */
  int inlier;                 /* rank in the consistent set (the order of the inter-session edges), -1 when not in it    */
} b200sm_merge_row;
typedef struct b200sm_merge_result {
  int merged;                       /* 1: src was appended to dst as a new segment                                        */
  int query_tile;                   /* src descriptors per block of the score launch                                     */
  unsigned long long pairs_scored;  /* n_A * n_B                                                                          */
  int candidates, verified, accepted, inliers;
  int first_submap;                 /* the new segment's first submap (n_A), -1 when not merged                          */
  double T[16];                     /* T*, the first inlier's F (column-major): the rigid placement X_b = T* P_b        */
  b200sm_pose_adjust_result adjust; /* the joint adjustment (zero when not merged)                                        */
} b200sm_merge_result;
/* Merge session src (B, any frame) into dst (A): (1) D(b, a) and s* of every src submap b against every dst submap a, on
 * the device in one launch (Scan Context, bitwise b200sm_search_loop_place's for the same pair); (2) per b the first
 * top_k a with D < sc_threshold in (D, a) order, selected on the device; all of them ordered by (D, b, a), the first
 * max_verifications verified; (3) a verification is b200sm_search_loop_place's with source = src submap b moved by its
 * pose, target = VoxelGrid(voxel_leaf_size) of dst submaps a +- search_submap_num inside a's segment and guess
 * sc_guess(P_a, P_b, s*); (4) the accepted rows in (fitness, row) order each join the consistent set iff their cycle error
 * with every row already in it is within tolerance; (5) with at least min_inliers rows: X_b = T* P_b, the joint pose
 * adjustment over dst's submaps then src's at X_b (numbered n_A + b), odometry edges per segment, then loop_edges (merged
 * numbering), then (a, n_A + b, Z) per inlier in rank order; vertex 0 fixed; poses_out (may be NULL) = (n_A + n_B) * 16
 * doubles column-major; (6) src's submaps (clouds device to device, intensity included) are appended to dst at X_b with
 * distance d_{A,last} + d_b, as a new segment (as several when src is itself a merged map: its segments are kept). The
 * odometry rule leaves the first submap of every segment without an odometry edge, as the reference leaves vertex 0: an
 * appended segment's first submap moves in the adjustment only through a loop edge of its own (an inlier with b = 0, or a
 * caller's edge), and otherwise stays at X_b. A candidate with an empty src submap or an empty target window is reported
 * as a row that is not accepted (fitness = HUGE_VAL) and registers nothing. b200sm_pose_adjust(dst) with loop_edges followed by the inter-session edges
 * gives poses_out bit for bit. src is only read. Otherwise (no candidate, or fewer inliers) B200REG_OK with merged = 0:
 * the rows are reported, poses_out is untouched and dst's submaps, poses, segments and descriptors are as they were.
 * rows[0 .. *n_rows) = min(verified, capacity) rows in verification order. params NULL: the defaults. B200REG_ERR_ARG,
 * with nothing changed, for a NULL handle, dst == src, sessions on different devices or with different Scan Context
 * parameters, an empty session, n_A * n_B > 2^28, a parameter out of range, a loop edge id outside [0, n_A + n_B) or with
 * from == to (or a non-finite relative_pose), or rows == NULL with capacity > 0. NDT and GICP handles alike.         */
int b200sm_merge_session(b200sm_t dst, b200sm_t src, b200reg_t reg, const b200sm_merge_params* params,
                         const b200sm_loop_edge* loop_edges, int n_loop_edges, b200sm_merge_row* rows, size_t capacity,
                         size_t* n_rows, double* poses_out, b200sm_merge_result* result);
/* the last merge's score matrix: *n_query = n_B, *n_cand = n_A; min(capacity, n_B * n_A) entries of D and s*, row-major
 * by src submap (entry b * n_A + a). Either array may be NULL. */
int b200sm_get_merge_scores(b200sm_t dst, size_t capacity, size_t* n_query, size_t* n_cand, double* distances, int* shifts);
/* the first submap of every segment: *n = segments (0 for a session without submaps), min(capacity, n) copied */
int b200sm_get_segments(b200sm_t s, size_t* first, size_t capacity, size_t* n);

/* ---- saving a mapping session to disk and loading it back ------------------------------------------------------------
 * A directory: session.txt (the manifest: Scan Context parameters, segments, every submap's point count, distance and
 * pose, and the caller's graph: num_adjacent_pose_cnstraints, loop edges, adjusted poses or none; every double printed
 * with %.17g, so it reads back bitwise), pose_graph.g2o (the graph as the reference's optimizer.save writes it,
 * gbs.cpp:319; an export, never read back) and submaps/%06zu.pcd (one binary PCD per submap as pcl::io::savePCDFileBinary
 * writes a dense PointXYZI cloud: the sensor-frame rows, intensity included; an empty submap is a header with POINTS 0).
 * Definitions: csrc/session_io.hpp; DESIGN.md section 7b. */
typedef struct b200sm_session_io_info {
  size_t n_submaps, n_segments, n_points;
  int n_loop_edges, num_adjacent_pose_cnstraints, adjusted;
  unsigned long long n_bytes; /* bytes written / read, all files */
} b200sm_session_io_info;
/* Save the session into dir (created when missing, as is dir/submaps; files of an earlier save that this one does not name
 * are left alone). loop_edges / num_adjacent_pose_cnstraints are b200sm_pose_adjust's; adjusted_poses_colmajor16 (may be
 * NULL) = 16 * n_submaps doubles, e.g. its output. The submap bodies come to the host through two pinned buffers, the
 * next copy overlapping the current write. An existing session.txt is removed before the first submap file is opened;
 * the new one is written to session.txt.tmp and renamed into place only after every other file closed without error, so
 * a failed save never leaves a manifest that names a partial file. B200REG_ERR_ARG before any file is touched for an
 * empty session, num_adjacent_pose_cnstraints < 1, a loop edge id outside [0, n_submaps) or with from == to, or a
 * non-finite relative or adjusted pose; B200REG_ERR_IO for a file or directory that cannot be created or written. */
int b200sm_save_session(b200sm_t s, const char* dir, int num_adjacent_pose_cnstraints, const b200sm_loop_edge* loop_edges,
                        int n_loop_edges, const double* adjusted_poses_colmajor16, b200sm_session_io_info* info);
/* Load dir into an empty session (no submaps, frames or imports; otherwise B200REG_ERR_ARG). The manifest is parsed whole
 * first; every submap file is read by b200reg_load_pcd's reader (a binary body unpacked on the device) and its POINTS must
 * be the manifest's count. The result is the session b200sm_import_submap of every saved submap in order gives, with the
 * saved segments and Scan Context parameters (descriptors are rebuilt lazily, bitwise). A loaded session is a backend's
 * map: b200sm_set_scan, b200sm_receive_cloud and b200sm_update_map return B200REG_ERR_ARG on it; b200sm_import_submap
 * appends to its last segment. B200REG_ERR_IO: a file cannot be opened or read. B200REG_ERR_FORMAT: the manifest
 * deviates from its format (b200sm_last_error names the line) or a submap file is not what it says. After either, and
 * after B200REG_ERR_ARG, the session is as it was: empty, with its Scan Context parameters, holding no submap memory.
 * After B200REG_ERR_CUDA it holds no submaps. */
int b200sm_load_session(b200sm_t s, const char* dir, b200sm_session_io_info* info);
/* The graph the loaded session was saved with: *n_loop_edges = L, min(capacity, L) loop edges copied;
 * adjusted_poses_colmajor16 (may be NULL) receives 16 * n doubles (n: submaps at the save) when it was saved with adjusted
 * poses; *num_adjacent_pose_cnstraints (may be NULL). A session that was not loaded: B200REG_ERR_ARG. */
int b200sm_get_session_graph(b200sm_t s, b200sm_loop_edge* loop_edges, size_t capacity, size_t* n_loop_edges,
                             double* adjusted_poses_colmajor16, int* num_adjacent_pose_cnstraints);
/* The map of every submap moved by a pose cast to float (modified map gbs.cpp:321-368; publishMap sm.cpp:529-552 when
 * poses == NULL, i.e. the submaps' own poses), assembled on the device in one launch. Output is x, y, z, intensity
 * floats in submap order. *n = total points; min(*n, capacity) points are copied, so capacity 0 is a size query (it
 * launches nothing). offsets (may be NULL) = n_submaps + 1 prefix sums: submap i is out[offsets[i] .. offsets[i+1]),
 * which is the cloud of modified_map_array's i-th SubMap.                                                            */
int b200sm_assemble_map(b200sm_t s, const double* poses_colmajor16, float* out_xyzi, size_t capacity, size_t* n,
                        size_t* offsets);
/* pcl::io::savePCDFileASCII(path, map) (gbs.cpp:369, the map_save service gbs.cpp:90-103) where map is what
 * b200sm_assemble_map(s, poses_colmajor16, ...) returns (poses == NULL: the submaps' own poses): the PCD v0.7 header of a
 * PointXYZI cloud and one "x y z intensity" line per point, every float as PCL prints it (ostream precision 8, "nan").
 * The map is assembled and its text formatted on the device; the text comes to the host in chunks of a fixed number of
 * points through two pinned buffers, the calling thread writing one chunk while the device encodes and copies the next.
 * No point of the map is read back. The file is written in place. n_points, n_bytes (may be NULL) = points and file size.
 * B200REG_ERR_ARG for an empty map (no file is created), B200REG_ERR_IO when the file cannot be opened or written.      */
int b200sm_save_map_pcd_ascii(b200sm_t s, const double* poses_colmajor16, const char* path, size_t* n_points, size_t* n_bytes);
/* ---- 2D occupancy grid of the map, for a navigation stack (nav2's map_server, AMCL) -------------------------------------
 * No counterpart in the reference. Every submap's points are rays from its sensor origin: the endpoint is the point
 * b200sm_assemble_map(s, poses_colmajor16, ...) returns for it, the origin the same float pose applied to (float)
 * sensor_origin. A ray marks its endpoint's cell HIT when the endpoint lies in the height band [z_min, z_max] (map frame),
 * and every cell its segment crosses inside the band FREE (a 4-connected Amanatides-Woo walk in 2^16-per-cell fixed
 * point); within one submap a hit cell is not free (OctoMap's per-scan update). Each cell counts the submaps that hit it
 * and those that freed it; its value is -1 when both are 0, else round-half-up of 100 * hits / (hits + frees). The exact
 * definitions (skipped points, fixed point, band clip, walk and its tie rule, extent, image) are in
 * csrc/occupancy_grid.hpp; DESIGN.md section 7b describes the build. Counts of per-submap booleans do not depend on the
 * order of the work, so the grid is bitwise deterministic. A pose adjustment moves every submap, so each call rebuilds the
 * grid from all submaps. NDT and GICP sessions alike; no registration handle is involved. */
typedef struct b200sm_occupancy_params {
  double resolution;        /* metres per cell, finite, > 0; default 0.05                                             */
  double z_min, z_max;      /* map-frame height band, finite, z_min < z_max; defaults 0.2 and 2.0 (ground at z = 0)  */
  double max_range;         /* finite, > 0: rays longer than this (horizontally) are skipped; default 100;
                               max_range / resolution <= 2^14                                                         */
  double sensor_origin[3];  /* LiDAR position in the robot frame (the translation given to b200sm_set_sensor_transform,
                               or 0 when the clouds are in the sensor frame); default 0                               */
  double occupied_thresh, free_thresh; /* 0 <= free_thresh < occupied_thresh <= 1; defaults 0.65, 0.25                */
} b200sm_occupancy_params;
typedef struct b200sm_occupancy_info {
  unsigned width, height;            /* cells                                                                      */
  double origin[2], resolution;      /* map-frame corner of cell (0, 0), as map_server's YAML origin               */
  unsigned long long n_rays, n_skipped; /* points cast as rays / skipped (non-finite, or beyond max_range)          */
  int n_batches;                     /* launches of the walks (submaps batched by a fixed 64 MiB bitmap budget)    */
  unsigned long long n_occupied, n_free, n_unknown; /* cells the image marks 0 / 254, and cells of value -1         */
} b200sm_occupancy_info;
/* Build the grid from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps doubles (the
 * output of b200sm_pose_adjust). params NULL: the defaults. A parameter out of range, a non-finite pose entry, a sensor
 * origin beyond 2^30 cells or farther than 2^16 cells from the band, no submaps, or a grid of more than 2^28 cells (the
 * message gives width and height): B200REG_ERR_ARG, checked before the grid is allocated (the extent is measured on the
 * device first, with 144 bytes per submap of tables); the previous grid stays. The
 * session keeps the grid until the next build or destroy: 10 bytes per cell (hits and frees uint32, value, image byte;
 * 2.7 GB at the 2^28-cell cap), plus the walks' bitmap scratch (the largest batch: at most 64 MiB, or the bitmaps of
 * the largest submap when they are larger: 2 bits per cell of its window) and 144 bytes per submap of tables. info may
 * be NULL. */
int b200sm_build_occupancy_grid(b200sm_t s, const double* poses_colmajor16, const b200sm_occupancy_params* params,
                                b200sm_occupancy_info* info);
/* The last grid, row-major from cell (0, 0) (nav_msgs/OccupancyGrid.data): min(capacity, width * height) cells of each
 * non-NULL array (values -1..100, hits, frees). No grid built yet: B200REG_ERR_ARG. */
int b200sm_get_occupancy_grid(b200sm_t s, signed char* data, unsigned* hits, unsigned* frees, size_t capacity);
/* The map_server pair of the last grid: pgm_path gets "P5", a comment line, "width height", "255", then the trinary image
 * (0 occupied, 254 free, 205 unknown; top row first); yaml_path gets image (the PGM's basename), mode: trinary,
 * resolution, origin: [x, y, 0], negate: 0, occupied_thresh, free_thresh (numbers that read back bitwise; the image name
 * double-quoted, so that any file name reads back as itself). The rule is
 * nav2's map_saver's as its documentation states it; csrc/occupancy_grid.hpp's text is the contract. No grid built yet:
 * B200REG_ERR_ARG. A file that cannot be opened or written: B200REG_ERR_IO. */
int b200sm_save_occupancy_map(b200sm_t s, const char* pgm_path, const char* yaml_path);
/* ---- 2.5D elevation and traversability map, for a navigation stack on non-flat ground ---------------------------------
 * No counterpart in the reference. The occupancy grid's band is fixed in the map frame, so a ramp rising into it reads as
 * an obstacle and a drop below it as free; this map follows the ground instead. Every submap's points are the points
 * b200sm_assemble_map(s, poses_colmajor16, ...) returns, skipped by the occupancy grid's rule (non-finite, or horizontally
 * beyond max_range from the submap's sensor origin), on the occupancy grid's lattice. Each cell keeps its point count n,
 * its lowest height lo and its surface height h: the highest point no more than `clearance` above lo (points higher up
 * are overhangs: canopy, a bridge deck). A cell with n >= min_points is observed. Over the observed cells within
 * window_cells of an observed cell: step = max h - min h, the least-squares plane's slope and the RMS of the residuals to
 * it (roughness). The cell is unknown (-1) with fewer than min_cells such cells or collinear ones; lethal (100) when the
 * step, slope or roughness passes its limit; otherwise round-half-up of 99 * the largest of the three ratios to their
 * limits. Integer statistics, exact int64 moment sums and a fixed double formula make it bitwise deterministic; the exact
 * definitions are in csrc/elevation_map.hpp, DESIGN.md section 7b describes the build. NDT and GICP sessions alike; no
 * registration handle is involved. */
typedef struct b200sm_elevation_params {
  double resolution;        /* metres per cell, finite, > 0; default 0.1                                               */
  double max_range;         /* finite, > 0: points farther (horizontally) from the sensor are skipped; default 100;
                               max_range / resolution <= 2^14                                                         */
  double sensor_origin[3];  /* LiDAR position in the robot frame, as for b200sm_build_occupancy_grid; default 0         */
  double clearance;         /* metres above a cell's lowest point that still count as its surface, >= 0; default 2    */
  int min_points;           /* points that make a cell observed, >= 1; default 2                                      */
  int window_cells;         /* window radius r in cells, 1..8; default 3 (a 7 x 7 window)                              */
  int min_cells;            /* observed cells a window needs, 3..(2r + 1)^2; default 6                                */
  double max_slope;         /* degrees, in (0, 90); default 20                                                         */
  double max_step;          /* metres, > 0; default 0.15                                                               */
  double max_roughness;     /* metres (RMS), > 0; default 0.05                                                         */
  double occupied_thresh, free_thresh; /* image: value >= rint(100 occupied_thresh) -> 0, <= rint(100 free_thresh) -> 254,
                               else 205; 0 <= free_thresh < occupied_thresh <= 1; defaults 0.65, 0.25                  */
} b200sm_elevation_params;
typedef struct b200sm_elevation_info {
  unsigned width, height;            /* cells                                                                      */
  double origin[2], resolution;      /* map-frame corner of cell (0, 0), as map_server's YAML origin               */
  unsigned long long n_points, n_skipped, n_overhang; /* points used / skipped / above a cell's clearance            */
  unsigned long long n_observed;     /* cells with n >= min_points                                                  */
  unsigned long long n_lethal, n_traversable, n_unknown; /* cells of value 100 / 0..99 / -1                         */
} b200sm_elevation_info;
/* Build the map from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps doubles. params
 * NULL: the defaults. A parameter out of range, a non-finite pose entry, a sensor origin beyond 2^30 cells, no submaps,
 * no non-skipped point or a grid of more than 2^28 cells: B200REG_ERR_ARG, checked before the grid is allocated (the
 * extent is measured on the device first). A height extent (highest minus lowest non-skipped point) of 2^24 cells or
 * more: B200REG_ERR_ARG, checked after the statistics pass, before the window pass. After any refusal the previous map
 * stays. The session keeps the map until the next build or destroy: 34 bytes per cell (n, lo, h, step, tan_slope,
 * roughness, value, image byte; 9.1 GB at the 2^28-cell cap), and a build holds the new map beside the old one until it
 * succeeds. info may be NULL. */
int b200sm_build_elevation_map(b200sm_t s, const double* poses_colmajor16, const b200sm_elevation_params* params,
                               b200sm_elevation_info* info);
/* The last map, row-major from cell (0, 0): min(capacity, width * height) cells of each non-NULL array. n: points per
 * cell; h and lo: surface and lowest height in fixed point (metres * 2^16 / resolution, floor), 0x8080808080808080 and
 * 0x7f7f7f7f7f7f7f7f in a cell without points; step (metres), tan_slope, roughness (metres): NaN in an unknown cell;
 * value: -1, 0..99 or 100. No map built yet: B200REG_ERR_ARG. */
int b200sm_get_elevation_map(b200sm_t s, unsigned* n, long long* h, long long* lo, float* step, float* tan_slope, float* roughness,
                             signed char* value, size_t capacity);
/* The map_server pair of the last map, in b200sm_save_occupancy_map's format: 0 where the value is lethal or at least
 * occupied_thresh, 254 where it is at most free_thresh, 205 elsewhere and where unknown. No map built yet:
 * B200REG_ERR_ARG. A file that cannot be opened or written: B200REG_ERR_IO. */
int b200sm_save_traversability_map(b200sm_t s, const char* pgm_path, const char* yaml_path);
/* ---- static map: the map without what moved while it was recorded ---------------------------------------------------
 * No counterpart in the reference. Every submap's points are rays from its sensor origin through a 3D voxel grid: the
 * endpoint is the point b200sm_assemble_map(s, poses_colmajor16, ...) returns for it, the origin the same float pose
 * applied to (float) sensor_origin. A ray HITS its endpoint's voxel and FREES the voxels of the first ray_fraction of its
 * length (a 6-connected Amanatides-Woo walk in 2^16-per-voxel fixed point; the rest of the ray is not freed, because rays
 * that graze a surface cross its voxels just before their ends). Only voxels some endpoint lies in are counted; within one
 * submap a hit voxel is not free (OctoMap's per-scan update). Each voxel counts the submaps that hit it and those that
 * freed it; it is DYNAMIC when frees >= min_frees and round-half-up of 100 * hits / (hits + frees) <= rint(100 *
 * dynamic_thresh). The static map is the assembled map, in its order, without the points whose voxel is dynamic; points
 * that are not rays (non-finite, or beyond max_range) are kept. The exact definitions are in csrc/static_map.hpp;
 * DESIGN.md section 7b describes the build. Counts of per-submap booleans do not depend on the order of the work, so the
 * result is bitwise deterministic. Each call rebuilds from all submaps; the session's submaps are not changed. NDT and GICP
 * sessions alike; no registration handle is involved. */
typedef struct b200sm_static_map_params {
  double resolution;        /* metres per voxel, finite, > 0; default 0.2                                             */
  double max_range;         /* finite, > 0: rays longer than this are not cast (their points are kept); default 100;
                               max_range / resolution <= 2^14                                                         */
  double sensor_origin[3];  /* LiDAR position in the robot frame (as for b200sm_build_occupancy_grid); default 0       */
  double ray_fraction;      /* the part of each ray that frees voxels, (0, 1] (rint(ray_fraction * 2^16) >= 1);
                               default 0.85                                                                           */
  unsigned min_frees;       /* >= 1; default 2                                                                        */
  double dynamic_thresh;    /* [0, 1]; default 0.4                                                                    */
} b200sm_static_map_params;
typedef struct b200sm_static_map_info {
  int box_origin[3];                 /* voxel (i, j, k) of the box's lower corner: map x in [i, i + 1) * resolution */
  unsigned box_dims[3];              /* voxels; the box bounds every ray's endpoint voxel (0 when there is no ray)   */
  unsigned long long n_rays, n_skipped; /* points cast as rays / not cast (non-finite, or beyond max_range)          */
  unsigned long long n_voxels, n_dynamic_voxels; /* voxels some endpoint lies in; of those, the dynamic ones         */
  unsigned long long n_points, n_static_points;  /* the assembled map; the static map                               */
  int n_batches;                     /* launches of the walks (submaps batched by a fixed 64 MiB bitmap budget)      */
} b200sm_static_map_info;
/* Build the static map from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps doubles
 * (the output of b200sm_pose_adjust). params NULL: the defaults. A parameter out of range, a non-finite pose entry, a
 * sensor origin beyond 2^30 voxels, no submaps, a map of 2^32 points or more, or a box of more than 2^31 - 1 voxels:
 * B200REG_ERR_ARG, checked before anything is sized from the box (the box is measured on the device first, with 120
 * bytes per submap of tables); the previous build stays. The session keeps the build until the next one or destroy:
 * the rank index (8 bytes per 32 box voxels), 9 bytes per occupied voxel (hits, frees, flag), the static map (16 bytes per
 * point), the walks' bitmap scratch (the largest batch: at most 64 MiB, or two bits per occupied voxel when that is
 * more) and 4 bytes per 1024 points of tile counts. info may be NULL. */
int b200sm_build_static_map(b200sm_t s, const double* poses_colmajor16, const b200sm_static_map_params* params,
                            b200sm_static_map_info* info);
/* The last static map: x, y, z, intensity floats. *n = its points; min(*n, capacity) points are copied, so capacity 0 is
 * a size query. offsets (may be NULL) = n_submaps at the build + 1 prefix sums: submap i's kept points are
 * out[offsets[i] .. offsets[i+1]) (modified_map_array's i-th SubMap without its dynamic points). No build yet:
 * B200REG_ERR_ARG. */
int b200sm_get_static_map(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n, size_t* offsets);
/* The occupied voxels of the last build in rank order (ascending (k, j, i) within the box): *n = their number;
 * min(*n, capacity) rows of each non-NULL array: ijk3 (3 ints, the voxel), hits, frees, dynamic (0 / 1). For tuning the
 * parameters. No build yet: B200REG_ERR_ARG. */
int b200sm_get_map_voxels(b200sm_t s, int* ijk3, unsigned* hits, unsigned* frees, unsigned char* dynamic, size_t capacity,
                          size_t* n);
/* pcl::io::savePCDFileASCII(path, static map): the text of b200sm_save_map_pcd_ascii for the last static map, formatted
 * on the device and written by the same double-buffered chunks. n_points, n_bytes (may be NULL) = points and file size.
 * No build yet, or a static map without points (no file is created): B200REG_ERR_ARG. A file that cannot be opened or
 * written: B200REG_ERR_IO. */
int b200sm_save_static_map_pcd_ascii(b200sm_t s, const char* path, size_t* n_points, size_t* n_bytes);
/* ---- map consistency: how crisp the map is, without ground truth ------------------------------------------------------
 * No counterpart in the reference. The points are those b200sm_assemble_map(s, poses_colmajor16, ...) returns, in map
 * order; non-finite ones are skipped. Every point whose map index is a multiple of query_stride is a query: its
 * neighbours are the points within `radius` of it (itself included, 2^16-per-radius fixed point, the radius test exact).
 * From their covariance Sigma (m^2) come h = 1/2 ln det(2 pi e Sigma), the differential entropy, and plane_var, the
 * smallest eigenvalue of Sigma. A query is valid with n >= min_neighbors and det Sigma >= (radius / 2^16)^6. MME (Mean
 * Map Entropy, Razlaw et al. 2015) and MPV (Mean Plane Variance) are their means over the valid queries, per submap and
 * for the whole map: a crisp map has thin, flat neighbourhoods, and double walls or blur from a bad pose or a wrong loop
 * edge raise both, so a build before and after b200sm_pose_adjust, or with and without a loop edge, tells which map is
 * better. Exact integer moment sums, a fixed double formula and integer aggregates make every value bitwise
 * deterministic; the exact definitions are in csrc/map_consistency.hpp, DESIGN.md section 7b describes the build. The
 * session's submaps, poses and other products are not changed. NDT and GICP sessions alike. */
typedef struct b200sm_map_consistency_params {
  double radius;      /* metres, [0.01, 100]; default 0.5                                                              */
  int min_neighbors;  /* neighbours (the query included) a valid query needs, >= 4; default 10                          */
  int query_stride;   /* every query_stride-th point of the map is a query, >= 1; default 1                              */
} b200sm_map_consistency_params;
typedef struct b200sm_map_consistency_info {
  int box_origin[3];                     /* cell (i, j, k) of the box's lower corner; cells are radius on a side      */
  unsigned box_dims[3];                  /* cells; 0 when no point is finite                                            */
  unsigned long long n_points, n_skipped; /* the assembled map; its non-finite points                                  */
  unsigned long long n_cells;            /* occupied cells                                                              */
  unsigned long long n_queries, n_valid; /* queries; valid ones                                                         */
  unsigned long long n_neighbors;        /* neighbours over all queries                                                 */
  unsigned long long n_candidates;       /* points of the 27 cells around each query, summed: the candidates tested    */
  long long sum_h_q, sum_plane_q;        /* over the valid queries: sum rint(h 2^24), sum rint(plane_var / radius^2 2^30) */
  double mme, mpv;                       /* Mean Map Entropy (nats), Mean Plane Variance (m^2); NaN without a valid query */
} b200sm_map_consistency_info;
typedef struct b200sm_submap_consistency {
  unsigned long long n_points, n_queries, n_valid, n_neighbors; /* the submap's points; its queries ...                 */
  long long sum_h_q, sum_plane_q;                               /* as in b200sm_map_consistency_info                    */
  double mme, mpv;                                              /* its queries' means; NaN without a valid query        */
} b200sm_submap_consistency;
/* Build the map's consistency from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps
 * doubles. params NULL: the defaults. A parameter out of range, a non-finite pose entry, no submaps, a map of 2^31 points
 * or more, a point whose fixed-point coordinate is 2^46 or more in magnitude (about 2^30 radii), or a box of more than
 * 2^31 - 1 cells (its dims in the message; at 0.3 m that is about 2 km x 2 km x 50 m): B200REG_ERR_ARG, checked before
 * anything is sized from the map (the box is measured on the device first, with 72 bytes per submap of tables); the
 * previous build stays. The session keeps the build until the next one or destroy: 20 bytes per point (n, h, plane_var),
 * the rank index (8 bytes per 32 box cells), 32 bytes per occupied cell (counts, chunk offsets, the cell list) and 40
 * bytes per submap; a build also reuses 12 bytes per point of cell-ordered scratch, kept with the session. info may be
 * NULL. */
int b200sm_build_map_consistency(b200sm_t s, const double* poses_colmajor16, const b200sm_map_consistency_params* params,
                                 b200sm_map_consistency_info* info);
/* The per-point layers of the last build, in map order: min(n_points, capacity) rows of each non-NULL array. n: the
 * neighbours of a query (0 for other points); h (nats) and plane_var (m^2): NaN (0x7ff8000000000000) for an invalid
 * query and for every other point. No build yet: B200REG_ERR_ARG. */
int b200sm_get_map_consistency(b200sm_t s, unsigned* n, double* h, double* plane_var, size_t capacity);
/* The per-submap rows of the last build: min(n_submaps at the build, capacity) rows. No build yet: B200REG_ERR_ARG. */
int b200sm_get_submap_consistency(b200sm_t s, b200sm_submap_consistency* rows, size_t capacity);
/* pcl::io::savePCDFileASCII(path, map) of the assembled map at the build's poses with its intensity replaced by
 * (float) h, NaN where h is: a heat map of the entropy for a viewer, formatted on the device and written as
 * b200sm_save_static_map_pcd_ascii writes. n_points, n_bytes (may be NULL) = points and file size. No build yet, a map
 * without points, or submaps added since the build: B200REG_ERR_ARG. A file that cannot be opened or written:
 * B200REG_ERR_IO. */
int b200sm_save_map_consistency_pcd_ascii(b200sm_t s, const char* path, size_t* n_points, size_t* n_bytes);
/* ---- map changes: what changed between two recordings, and the map brought up to date --------------------------------
 * No counterpart in the reference. The submaps are split into two epochs: BEFORE, submaps [0, split), and AFTER,
 * [split, n_submaps). The rays, voxels and walks are those of b200sm_build_static_map with the same parameters, but each
 * voxel counts the submaps that hit and freed it in each epoch separately. In an epoch a voxel is FREE when the static map
 * would call it dynamic from that epoch's counts, and OCCUPIED when that epoch hit it and it is not free. A voxel is
 * APPEARED when it is occupied AFTER and free BEFORE, VANISHED when occupied BEFORE and free AFTER, else UNCHANGED. A point
 * of an AFTER submap in an APPEARED voxel is APPEARED, a point of a BEFORE submap in a VANISHED voxel is VANISHED, every
 * other point (skipped ones included) UNCHANGED. The updated map is the assembled map without the VANISHED points: save it
 * and hand it to b200sm_set_prior_map_pcd to localise in the map as it is now. Something that only moves through one
 * recording is dynamic in that recording, not occupied, so it is never reported as a change. The exact definitions are
 * in csrc/map_changes.hpp; DESIGN.md section 7b describes the build. Bitwise deterministic; the session's submaps, poses
 * and other products (the static map included) are not changed. NDT and GICP sessions alike. */
#define B200SM_CHANGE_UNCHANGED 0
#define B200SM_CHANGE_APPEARED 1
#define B200SM_CHANGE_VANISHED 2
typedef struct b200sm_map_change_info {
  int box_origin[3];                 /* as in b200sm_static_map_info: the box of both epochs' endpoint voxels           */
  unsigned box_dims[3];
  long long split_submap;            /* the first AFTER submap (split_submap -1 resolved)                              */
  unsigned long long n_rays, n_skipped; /* points cast as rays / not cast                                               */
  unsigned long long n_voxels, n_appeared_voxels, n_vanished_voxels; /* voxels some endpoint lies in; changed ones      */
  unsigned long long n_points, n_appeared_points, n_vanished_points; /* the assembled map; its changed points           */
  unsigned long long n_updated_points; /* the updated map: n_points - n_vanished_points                                 */
  int n_batches;                     /* launches of the walks; no batch holds submaps of both epochs                    */
} b200sm_map_change_info;
/* Build the changes from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps doubles.
 * params NULL: the static map's defaults. split_submap: the first AFTER submap, in [1, n_submaps); -1 = the first submap
 * of the session's last segment (after b200sm_merge_session, the merged recording). Refused with B200REG_ERR_ARG, before
 * anything is sized, the previous build staying: split_submap -1 on a session of one segment, any other value outside
 * [1, n_submaps), and everything b200sm_build_static_map refuses. The session keeps the build until the next one or
 * destroy, beside (not in place of) the static map's: the rank index (8 bytes per 32 box voxels), 17 bytes per occupied
 * voxel (four counts and a label), 1 byte per point (its label) and 16 per point of the updated map; the walks' bitmap
 * scratch is the static map's. info may be NULL. */
int b200sm_build_map_changes(b200sm_t s, const double* poses_colmajor16, const b200sm_static_map_params* params, long long split_submap,
                             b200sm_map_change_info* info);
/* The label of every point of the last build (B200SM_CHANGE_*), in map order: *n = n_points; min(*n, capacity) bytes are
 * copied (capacity 0: a size query). No build yet: B200REG_ERR_ARG. */
int b200sm_get_map_changes(b200sm_t s, unsigned char* labels, size_t capacity, size_t* n);
/* The occupied voxels of the last build in rank order (as b200sm_get_map_voxels): *n = their number; min(*n, capacity) rows
 * of each non-NULL array: ijk3 (3 ints), the counts of each epoch, label (B200SM_CHANGE_*). No build yet: B200REG_ERR_ARG. */
int b200sm_get_change_voxels(b200sm_t s, int* ijk3, unsigned* hits_before, unsigned* frees_before, unsigned* hits_after,
                             unsigned* frees_after, unsigned char* label, size_t capacity, size_t* n);
/* The updated map of the last build: x, y, z, intensity floats, in the assembled map's order. *n = its points; min(*n,
 * capacity) points are copied. offsets (may be NULL) = n_submaps at the build + 1 prefix sums per submap. No build yet:
 * B200REG_ERR_ARG. */
int b200sm_get_updated_map(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n, size_t* offsets);
/* pcl::io::savePCDFileASCII(path, updated map), written as b200sm_save_static_map_pcd_ascii writes. n_points, n_bytes (may
 * be NULL) = points and file size. No build yet, or an updated map without points (no file is created): B200REG_ERR_ARG.
 * A file that cannot be opened or written: B200REG_ERR_IO. */
int b200sm_save_updated_map_pcd_ascii(b200sm_t s, const char* path, size_t* n_points, size_t* n_bytes);

/* ---- surface mesh: a TSDF fused from every submap's rays, extracted by surface nets, saved as binary PLY --------------
 * No counterpart in the reference. The rays are those of b200sm_build_static_map (its fixed point, origins and skip rule;
 * the whole ray, no ray_fraction). Each ray walks a band of 2 * truncation around its endpoint through a voxel grid and
 * adds to every voxel it crosses the signed distance from the voxel's centre to the endpoint along the ray (positive on
 * the sensor's side, clamped to +-truncation) and one to its weight. A voxel with at least min_weight rays is observed; a
 * cell of eight observed voxels whose signs differ gets one vertex (the mean of its edges' zero crossings), and every
 * sign-changing edge between observed voxels whose four cells all have vertices gives two triangles, oriented so their
 * normals point towards free space. The exact definitions are in csrc/mesh.hpp; DESIGN.md section 7b describes the build.
 * Bitwise deterministic; the session's submaps, poses and other products are not changed. NDT and GICP sessions alike. */
typedef struct b200sm_mesh_params {
  double resolution;        /* metres per voxel, finite, > 0; default 0.2                                             */
  double truncation;        /* metres, 1 <= truncation / resolution <= 16; default 0.6                                */
  double max_range;         /* as b200sm_static_map_params.max_range: longer rays are not cast; default 100            */
  double sensor_origin[3];  /* LiDAR position in the robot frame; default 0                                           */
  unsigned min_weight;      /* rays a voxel needs to count as observed, >= 1; default 2                               */
} b200sm_mesh_params;
typedef struct b200sm_mesh_info {
  int box_origin[3];                 /* lowest voxel of the band box: the endpoint voxels' box widened on every side   */
  unsigned box_dims[3];
  unsigned long long n_points;       /* the assembled map                                                             */
  unsigned long long n_rays, n_skipped; /* points cast as rays / not cast (as the static map's)                        */
  unsigned long long n_walked;       /* voxel visits of the band walks                                                */
  unsigned long long n_band_voxels, n_observed_voxels; /* voxels some walk crosses; those with weight >= min_weight    */
  unsigned long long n_vertices, n_faces;
} b200sm_mesh_info;
/* Build the mesh from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps doubles (e.g.
 * b200sm_pose_adjust's output). params NULL: the defaults. Refused with B200REG_ERR_ARG, the previous build staying
 * readable: a parameter out of range, a non-finite pose, a sensor origin beyond 2^30 voxels, no submaps, a map of 2^32
 * points or more, a band box of more than 2^31 - 1 voxels (all before anything is sized), and 2^32 faces or more (after
 * they are counted). The session keeps the build until the next successful one or destroy, beside every other product:
 * the rank index (8 bytes per 32 box voxels), 29 bytes per band voxel (voxel, sum, weight, flag, vertex id), 12 bytes per
 * vertex and 12 per face, and 4 bytes per 256 band voxels of tile counts. info may be NULL. */
int b200sm_build_mesh(b200sm_t s, const double* poses_colmajor16, const b200sm_mesh_params* params, b200sm_mesh_info* info);
/* The last build's mesh: *n_vertices, *n_faces = its sizes; min(*n_vertices, vertex_capacity) vertices (x, y, z floats,
 * map frame) and min(*n_faces, face_capacity) faces (three vertex ids each, counter-clockwise seen from free space) are
 * copied (capacity 0: a size query). No build yet: B200REG_ERR_ARG. */
int b200sm_get_mesh(b200sm_t s, float* xyz, size_t vertex_capacity, size_t* n_vertices, unsigned* faces3, size_t face_capacity,
                    size_t* n_faces);
/* The band voxels of the last build in rank order (ascending linear index in the box): *n = their number; min(*n,
 * capacity) rows of each non-NULL array: ijk3 (3 ints), sdf_sum (the fused signed distances, 2^-16 voxel units), weight
 * (rays). No build yet: B200REG_ERR_ARG. */
int b200sm_get_mesh_voxels(b200sm_t s, int* ijk3, long long* sdf_sum, unsigned* weight, size_t capacity, size_t* n);
/* The last build's mesh as binary little-endian PLY (csrc/mesh.hpp gives the bytes), written in pieces through pinned
 * staging buffers. n_bytes (may be NULL) = the file size. No build yet, or a mesh without faces (no file is created):
 * B200REG_ERR_ARG. A file that cannot be opened or written: B200REG_ERR_IO. */
int b200sm_save_mesh_ply(b200sm_t s, const char* path, size_t* n_bytes);

/* ---- OctoMap: free and occupied voxels from every submap's rays, pruned into an octree, saved as a .bt file ------------
 * No counterpart in the reference. The rays, walks and parameters are exactly those of b200sm_build_static_map. The box
 * bounds every ray's endpoint voxel and the origin voxel of every submap with a ray, so every freed walk lies in it. A box
 * voxel is OCCUPIED (2) when the static map at the same parameters counts it as an occupied voxel that is not dynamic,
 * FREE (1) when it is not OCCUPIED and some ray's freed walk crosses it or some ray ends in it (a dynamic voxel is FREE:
 * what moved leaves free space behind), UNKNOWN (0) otherwise. The known voxels form OctoMap's depth-16 key tree (key =
 * voxel index + 32768), pruned where 8 leaf children share a state, and the file is the bytes octomap 1.9's
 * OcTree::writeBinary writes for that tree (octomap_server, MoveIt and rviz load it). The counts are per-submap booleans;
 * there are no clamped log-odds. The exact definitions are in csrc/octomap.hpp; DESIGN.md section 7b describes the
 * build. Bitwise deterministic; the session's submaps, poses and other products are not changed. */
typedef struct b200sm_octomap_info {
  int box_origin[3];                 /* voxel (i, j, k) of the box's lower corner (0 when there is no ray)            */
  unsigned box_dims[3];              /* voxels (0 when there is no ray)                                                */
  unsigned long long n_rays, n_skipped; /* points cast as rays / not cast (as the static map's)                        */
  unsigned long long n_occupied_voxels, n_dynamic_voxels, n_free_voxels; /* box voxels by state; the static map's
                                        dynamic voxels, all of them FREE                                               */
  unsigned long long n_inner_nodes, n_occupied_leaves, n_free_leaves; /* the pruned tree's nodes by kind              */
  unsigned long long tree_size;      /* its nodes, the .bt header's size: inner nodes + leaves                        */
  unsigned long long n_bytes;        /* the .bt file: header + 2 bytes per inner node                                  */
  int n_batches;                     /* launches of the static map's walks                                             */
} b200sm_octomap_info;
/* Build the OctoMap from every submap at its own pose (poses_colmajor16 NULL) or at the given 16 * n_submaps doubles
 * (e.g. b200sm_pose_adjust's output). params NULL: the static map's defaults. Refused with B200REG_ERR_ARG, the previous
 * build staying readable: everything b200sm_build_static_map refuses, a resolution that printf("%g") does not give back
 * exactly (the header's res), and a box of more than 2^31 - 1 voxels or with a voxel index outside [-32768, 32767] on
 * some axis (all before anything is sized from the box). The session keeps the build until the next successful one or
 * destroy, beside every other product: 1 byte per box voxel (its state) and 2 bytes per inner node (the .bt data). The
 * call's scratch: the static map's (its rank index, 9 bytes per occupied voxel and the walks' bitmaps), 1 bit per box
 * voxel (the freed walks) and 5 bytes per pyramid cell (about a seventh of the box's voxels). info may be NULL. */
int b200sm_build_octomap(b200sm_t s, const double* poses_colmajor16, const b200sm_static_map_params* params,
                         b200sm_octomap_info* info);
/* The last build's box voxel states (0 UNKNOWN, 1 FREE, 2 OCCUPIED) in linear order, x fastest, then y, then z: *n = the
 * box's voxels; min(*n, capacity) are copied (capacity 0: a size query). No build yet: B200REG_ERR_ARG. */
int b200sm_get_octomap_states(b200sm_t s, unsigned char* states, size_t capacity, size_t* n);
/* The last build's .bt file bytes: *n_bytes = its size; min(*n_bytes, capacity) bytes are copied (capacity 0: a size
 * query). An empty tree is the header with size 0. No build yet: B200REG_ERR_ARG. */
int b200sm_get_octomap_bt(b200sm_t s, unsigned char* bytes, size_t capacity, size_t* n_bytes);
/* The last build's .bt file written to path through pinned staging buffers. n_bytes (may be NULL) = the file size. No
 * build yet, or an empty tree (no file is created): B200REG_ERR_ARG. A file that cannot be opened or written:
 * B200REG_ERR_IO. */
int b200sm_save_octomap_bt(b200sm_t s, const char* path, size_t* n_bytes);
/* The same text for a HOST PointXYZI cloud (records as in b200sm_import_submap; intensity_offset_bytes >= 0), formatted
 * on `device`. *n_bytes = size of the whole file content (header and data); min(*n_bytes, capacity) bytes are copied to
 * out, so capacity 0 is a size query. B200REG_ERR_ARG for n == 0, a negative intensity offset, or a stride or offset that
 * is not a multiple of 4. */
int b200reg_encode_pcd_ascii(int device, const float* base, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                             char* out, size_t capacity, size_t* n_bytes);

/* ---- pcl::io::loadPCDFile (apps/align.cpp:54-61; a localisation or resume node reading the map.pcd saved above) ---
 * The header is parsed on the host, PCD v0.7 as PCL reads it: '#' comment lines, VERSION, FIELDS, SIZE, TYPE, COUNT,
 * WIDTH, HEIGHT, VIEWPOINT, POINTS, DATA (COUNT may be absent: 1 each; WIDTH * HEIGHT must equal POINTS). Organised clouds
 * (HEIGHT > 1) come out flat, WIDTH * HEIGHT points. Fields x, y, z are required and intensity is optional, each TYPE F,
 * SIZE 4, COUNT 1; every other field is skipped whatever its type and count. Output rows are float4 (x, y, z, intensity),
 * intensity 0 when the file has none (the PointXYZI default).
 * DATA ascii, as PCDReader::readBodyASCII / copyStringValue<float> of PCL 1.12: lines from getline, empty lines skipped,
 * tokens split on ' ', '\t' and '\r' with runs of separators compressed; a token equal to "nan" in any case is quiet_NaN,
 * every other token reads as `istringstream >> float` in the classic locale (glibc strtof, correctly rounded, subnormals,
 * overflow to +-inf), and the signed nan and inf / infinity spellings take the value of PCL's atof fallback. Reading
 * stops after POINTS points (the file is read at most one piece further). The text is parsed on the device, piece by piece (B200REG_PCD_LOAD_PIECE_BYTES of the body at
 * a time, each ending at its last '\n', read into two pinned buffers in turn while the device parses the previous one).
 * B200REG_ERR_FORMAT: a POINTS the body cannot hold (checked against the file size before anything is allocated), fewer
 * data lines than POINTS, a line whose token count is not the sum of COUNT (a line of
 * separators only included), an x / y / z / intensity token outside the grammar [+-](digits[.[digits]] | .digits)
 * [(e|E)[+-]digits] | [+-](nan | inf | infinity), a line longer than a piece before the POINTS-th line. Deliberate divergences from PCL: PCL takes
 * atof's value of a malformed token silently, and its handling of a bad token count differs between releases.
 * DATA binary: POINTS records of sum(SIZE * COUNT) bytes, unpacked on the device by the upload path of set_input_*; x, y,
 * z must be consecutive, intensity (if any) after x, the record size and the offsets multiples of 4; a body shorter than
 * the header says is B200REG_ERR_FORMAT. DATA binary_compressed (one sequential LZF block) is B200REG_ERR_FORMAT. */
#define B200REG_PCD_LOAD_PIECE_BYTES ((size_t)64 << 20)
/* The file's points into out_xyzi (4 floats per point): *n_points = POINTS, min(POINTS, capacity) rows copied; capacity 0
 * is a size query from the header alone. B200REG_ERR_IO when the file cannot be opened or read. */
int b200reg_load_pcd(int device, const char* path, float* out_xyzi, size_t capacity, size_t* n_points);
/* setInputTarget(cloud) of a loadPCDFile(path, cloud): the file is parsed into device scratch and handed over device to
 * device as b200reg_set_input_target_device does; no point of it exists as floats on the host, and the scratch copy of
 * the cloud is freed after the hand-over. On B200REG_ERR_IO, B200REG_ERR_FORMAT, B200REG_ERR_ARG (no points) and, for
 * NDT, B200REG_ERR_GRID (the new map's voxel grid would overflow int32 at the current resolution; checked before the
 * hand-over) the handle's previous target is unchanged, and b200reg_last_error names the reason (and the line of the
 * file, for a bad line). After B200REG_ERR_CUDA the handle has no valid target. The handle keeps the reader's fixed-size
 * buffers for later calls: two pinned pieces of B200REG_PCD_LOAD_PIECE_BYTES and one device piece; a binary file also
 * keeps a pinned and a device buffer of its body's size. n_points (may be NULL) = points of the new target. */
int b200reg_set_input_target_pcd(b200reg_t h, const char* path, size_t* n_points);

/* ---- localisation in a prior map: drive in the map.pcd saved above ---------------------------------------------------
 * The reference has no localisation mode; this is the session's own contract. The prior map stays on the device as float4
 * (x, y, z, intensity) and is never modified. The registration target of a frame is a CUT of it: the rows with
 *   dx = (double)x - cx, dy = (double)y - cy, dx * dx + dy * dy <= crop_radius * crop_radius
 * (cx, cy the session's position when the cut is made; every operation one IEEE double operation, nothing fused; NaN
 * coordinates fail; z is not tested — a cylinder, like the range filter), in MAP ORDER: bitwise map[mask] of that boolean
 * mask. The cut is a two-pass stream compaction (per-tile counts, scan, write at tile offset + rank), so target indices
 * (GICP's correspondences, its "lower index wins a tie") mean rows of the map in order. Each cut reads the map twice and
 * writes the kept rows once: 32 * n_map + 16 * n_cut bytes. At most 2^32 - 1 points; larger maps are B200REG_ERR_ARG.
 *
 * b200sm_set_prior_map_pcd reads the file with the reader of b200reg_load_pcd (the session keeps that reader's fixed-size
 * buffers); on B200REG_ERR_IO / B200REG_ERR_FORMAT / B200REG_ERR_ARG (no points) the previous prior map and cut stay and
 * b200sm_last_error names the reason. *n_points (may be NULL) = POINTS of the file; non-finite rows stay in the map and
 * are never kept by a cut. b200sm_set_prior_map takes host records as b200sm_import_submap does (no intensity field:
 * intensity 0). Both replace the previous map, return with the session's stream synchronised and make the current cut
 * stale: the next frame cuts anew. */
int b200sm_set_prior_map_pcd(b200sm_t s, const char* path, size_t* n_points);
int b200sm_set_prior_map(b200sm_t s, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes);
/* crop_radius: horizontal radius (metres, finite, > 0) of the cut; recrop_distance (finite, >= 0): the target is cut again
 * once the pose is this far (horizontally) from the centre of the current cut. Defaults 120 and 20. The caller keeps
 * crop_radius >= scan_max_range + recrop_distance, so that a scan never reaches past the edge of its target; this is not
 * enforced. Makes the current cut stale. Anything else: B200REG_ERR_ARG, nothing changes. */
int b200sm_set_localization_params(b200sm_t s, double crop_radius, double recrop_distance);
typedef struct b200sm_localize_stats {
  size_t n_map, n_cut, n_target;     /* prior map, current cut, what the engine was given (GICP: after VoxelGrid) */
  double cut_centre[2];              /* x, y the current cut was made around                                   */
  double dist_from_centre;           /* horizontal distance of the pose from the cut's centre as the last frame compared it
                                        with recrop_distance (before any re-cut that frame made)              */
  int n_cuts;                        /* cuts made since the prior map was set                                   */
  int cut_pending;                   /* a new cut waits to become the target at the next frame                  */
} b200sm_localize_stats;
/* One frame of a localising frontend: b200sm_receive_cloud without a map of its own. (1) The frame is uploaded exactly as
 * there (sensor transform, armed de-skew, range filter). (2) If there is no cut yet or it is stale (new prior map, new
 * parameters, b200sm_set_initial_pose since), the map is cut around the current position now; a pending cut then becomes
 * the engine's target (NDT: the cut; GICP: VoxelGrid(vg_size_for_input) of it, as for the targeted cloud). (3)
 * VoxelGrid(vg_size_for_input) + setInputSource, guess = current pose (or the armed use_odom guess), align, and the pose of
 * publishMapAndPose. No submap is made and latest_distance does not move. (4) dist_from_centre = sqrt(dx * dx + dy * dy)
 * in double from the new position to cut_centre; when dist_from_centre >= recrop_distance the map is cut again around the
 * new position at once, *target_recut = 1, and that cut becomes the target at the start of the next frame.
 * B200REG_ERR_NO_TARGET: no prior map, or the cut of step 2 keeps no row (the pose is outside the map; the message gives
 * centre and radius) — the pose, the previous cut and the engine's target are unchanged. A re-cut of step 4 that keeps no
 * row does not fail the frame: *target_recut = 0, the old cut and target stay, the next frame tries again.
 * B200REG_ERR_GRID (NDT): the cut's voxel grid would overflow int32 at the engine's resolution; the engine's target is
 * unchanged and the cut stays pending. Frames of b200sm_receive_cloud and of this call may be mixed on one session: each
 * uses its own buffers (the targeted cloud there, the cut here). */
int b200sm_localize_cloud(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes,
                          long intensity_offset_bytes, double* pose7_out, float* final_T_colmajor16_out, int* target_recut);
/* The initial pose from several hypotheses (NDT only; a GICP handle is B200REG_ERR_ARG). Steps 1 and 2 as above (the cut
 * is made around the current position, e.g. a rough b200sm_set_initial_pose), then the filtered scan is registered from
 * `count` >= 1 initial guesses (16 * count floats, column-major) in ONE b200reg_ndt_align_batch_device call, the scan read
 * in place `count` times. Every results[k] is bitwise what b200reg_align gives for that scan, target and guess. The
 * converged row with the highest trans_probability (the lowest index on a tie) becomes the session's pose; *best = its
 * index, or -1 when none converged (pose unchanged, B200REG_OK). An armed use_odom guess is left for the next frame. */
int b200sm_localize_init(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes,
                         long intensity_offset_bytes, const float* guesses, int count, b200reg_batch_result* results,
                         int* best);
/* Global localisation: the pose found in the prior map without a precise guess (NDT only; a GICP handle is
 * B200REG_ERR_ARG). (1) The frame is uploaded and the map cut around the current position as in b200sm_localize_init
 * (upload, cut, VoxelGrid + setInputSource). (2) A grid of (x, y, yaw) hypotheses is built on the host around the current
 * pose: with K = floor(radius / step), positions (i, j) for j = -K-1 .. K+1 (outer) and i = -K-1 .. K+1 (inner) are kept
 * when a * a + b * b <= radius * radius (a = (double)i * step, b = (double)j * step, every operation rounded on its own);
 * hypothesis k = position_index * yaw_steps + m has translation (cx + a, cy + b, z0) (the current position), rotation
 * Rz(2 pi m / yaw_steps) * R0 (R0: the rotation of the current pose, as sim_trans builds it in double; std::cos / std::sin,
 * products summed left to right in double), cast to float. z, roll and pitch are not searched: they come from the current
 * pose and the refinement corrects what remains. (3) Every hypothesis is scored by b200reg_ndt_score_poses on the filtered
 * scan. (4) The top_k highest scores, in descending score and the lower index first on equal scores, are refined in ONE
 * batch launch exactly as b200sm_localize_init refines its guesses: candidates[r] = the hypothesis of row r, results[r] =
 * bitwise what b200sm_localize_init returns for that guess (both arrays need min(top_k, n_hypotheses) rows). The converged
 * row with the highest trans_probability (the lowest row on a tie) becomes the session's pose; out->best = that row, or -1
 * (pose unchanged, B200REG_OK). out may be NULL. The caller keeps crop_radius >= radius + scan_max_range (not enforced).
 * An invalid spec, floor(radius / step) > 4096 or more than 2^24 hypotheses: B200REG_ERR_ARG before anything changes. No
 * prior map: B200REG_ERR_NO_TARGET. A node with no initial pose, or one that has lost track, calls this once and then
 * b200sm_localize_cloud frame by frame. */
typedef struct b200sm_global_search {
  double radius;   /* finite, >= 0: positions within this horizontal distance of the current position          */
  double step;     /* finite, > 0: grid spacing                                                                */
  int yaw_steps;   /* 1..4096: yaw offsets 2*pi*m / yaw_steps, m = 0..yaw_steps-1                              */
  int top_k;       /* 1..1024: best-scored hypotheses refined in one batch launch                              */
} b200sm_global_search;
typedef struct b200sm_global_result {
  long long n_hypotheses, hits_total;
  int n_refined;   /* min(top_k, n_hypotheses)                                                                 */
  int best;        /* refined row adopted as the session's pose, -1 when none converged (pose unchanged)        */
  float score_ms;  /* device time of the scoring launch (CUDA events around it on the engine's stream)         */
} b200sm_global_result;
int b200sm_localize_global(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes,
                           long intensity_offset_bytes, const b200sm_global_search* spec, int* candidates,
                           b200reg_batch_result* results, b200sm_global_result* out);
/* the grid of the last b200sm_localize_global that reached its scoring: *n = its hypotheses; min(capacity, n) rows of poses
 * (16 floats, column-major), scores and hits; any pointer may be NULL. The session keeps this grid in host memory (80 bytes per
 * hypothesis, about 1.3 GB at the 2^24 cap) until the next such call or until it is destroyed. */
int b200sm_get_global_search(b200sm_t s, size_t capacity, size_t* n, float* poses_colmajor16, double* scores, long long* hits);
/* Relocalisation anywhere in the prior map ("kidnapped robot"): no position is assumed (NDT and GICP handles). The map's
 * rows in the height band [z_min, z_max] are projected into a 2D occupancy grid of `resolution` cells over the map's whole
 * extent, with a max-pyramid of num_levels levels (kept in the session until the prior map, resolution, the band or
 * num_levels changes). The frame's filtered scan (upload, sensor transform, armed de-skew, range filter,
 * VoxelGrid(vg_size_for_input) + setInputSource, as b200sm_localize_init) is rotated to each of yaw_steps headings about the
 * current pose's rotation and height, and an exact branch-and-bound search over (heading, cell) counts the scan points
 * that land in occupied cells (csrc/relocalize.hpp states every definition). The answer is the first top_k tiles (the
 * 2^(num_levels-1)-cell squares of the grid, over all headings) ranked by their best leaf (score descending, leaf index
 * ascending) among those scoring >= max(1, ceil(min_score * m)), m the projected scan points. For each row in rank order:
 * the map is cut around the leaf's cell corner, handed over as target (NDT: the grid check first), align(guess) and
 * getFitnessScore() (no max range): bitwise setInputTarget(cut) / setInputSource(filtered) / align(guess) /
 * getFitnessScore(). The row with status OK, converged and fitness < accept_fitness that has the lowest fitness (the lowest
 * row on a tie) becomes the pose; out->best = that row or -1 (pose unchanged). The cut is then stale, so the next
 * b200sm_localize_cloud cuts around the pose. rows needs capacity >= top_k.
 * params NULL: the defaults below. A bad parameter, capacity < top_k, or a limit (W * H > 2^28 cells, the pyramid over 2^32
 * bytes, yaw_steps * W * H >= 2^40, over 2^32 roots, m >= 2^24 or yaw_steps * m > 2^26, a level's stored nodes over 2^26):
 * B200REG_ERR_ARG, found before the refinement, with the pose, the cut and the engine's target unchanged. No prior map:
 * B200REG_ERR_NO_TARGET. m = 0, no projected map row or no tile reaching the threshold: B200REG_OK, no rows, best = -1.
 * The limits that depend on yaw_steps (leaves, roots) are checked by every call, before its search launches anything.
 * Memory the session keeps: the pyramid, (W + 2^h - 1) * (H + 2^h - 1) bytes for each level h < num_levels (the margins
 * grow as 4^h: 6 W H + 57 (W + H) + 1245 bytes at 6 levels, but about 1.4 GB at 16 levels even for a 1 x 1 grid); the
 * offsets table (8 * yaw_steps * m bytes); 8 bytes per tile on the device (TW * TH tiles, every cell a tile at num_levels
 * = 1: 2 GB at the 2^28-cell limit); the largest frontier (16 bytes per stored node, its score included) and the roots'
 * scores (4 bytes per root, kept when there are at most 2^26 roots). A call also holds 8 host bytes per tile, 16 when
 * num_levels > 1. A node calls this at start-up, or when b200sm_localize_cloud's fitness says it is lost, then
 * b200sm_localize_cloud frame by frame. */
typedef struct b200sm_relocalize_params {
  double resolution;      /* > 0, metres per cell (default 0.25)                                                    */
  double z_min, z_max;    /* finite, z_min < z_max: the height band of map rows and rotated scan points (0.3, 3.0)   */
  int yaw_steps;          /* 1..4096 headings 2 pi k / yaw_steps about the current rotation (360)                    */
  int num_levels;         /* 1..16 pyramid levels; 1 is the exhaustive search (6)                                    */
  double min_score;       /* [0, 1]: a tile's best must score >= ceil(min_score * m) (0.3)                           */
  int top_k;              /* 1..64 tiles refined (4)                                                                 */
  double accept_fitness;  /* > 0: a refined row is adopted only below this fitness (1.0)                             */
} b200sm_relocalize_params;
typedef struct b200sm_relocalize_row {
  int yaw_index, cell_i, cell_j;  /* the tile's best leaf: heading, cell relative to the grid's origin cell          */
  int score;                      /* its score (projected scan points on occupied cells)                             */
  float guess[16];                /* R_k and the cell's lower corner at the current z, column-major                  */
  float final_T[16];              /* align()'s result, column-major                                                   */
  double fitness;                 /* getFitnessScore()                                                                */
  double trans_probability;       /* NDT: getTransformationProbability(); GICP: 0                                     */
  int converged, iterations, status, pad;
} b200sm_relocalize_row;
typedef struct b200sm_relocalize_result {
  long long width, height;        /* W, H cells                                                                       */
  int origin_cell[2];             /* i0, j0: cell (0, 0) covers [i0, i0 + 1) * resolution x [j0, j0 + 1) * resolution */
  long long m, t0, t;             /* projected scan points, the score threshold T0, the search's threshold T           */
  unsigned long long leaves;      /* yaw_steps * W * H                                                                */
  long long nodes[16];            /* nodes scored per level by the expansion; level num_levels - 1: the roots          */
  int n_rows, best;
  int pyramid_builds;             /* pyramids the session has built                                                   */
  float search_ms;                /* device time of the search's launches (CUDA events around each run of launches
                                     between two host waits, summed; the waits and the pyramid build excluded)        */
} b200sm_relocalize_result;
int b200sm_relocalize(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                      const b200sm_relocalize_params* params, b200sm_relocalize_row* rows, size_t capacity,
                      b200sm_relocalize_result* out);
/* Level `level` of the last pyramid: the byte of cell (i, j), i, j in [1 - 2^level, W) x [1 - 2^level, H), at
 * (j + 2^level - 1) * width + (i + 2^level - 1); *width = W + 2^level - 1, *height likewise (0 x 0 for an empty grid);
 * min(capacity, width * height) bytes into out (may be NULL). No pyramid or level outside it: B200REG_ERR_ARG. */
int b200sm_get_relocalize_grid(b200sm_t s, int level, unsigned char* out, size_t capacity, long long* width, long long* height);
/* score_level of `count` nodes (heading, i, j triples, any i, j) with the last relocalize search's discretised scan. No
 * search since the pyramid was built, a heading outside it or a level outside the pyramid: B200REG_ERR_ARG. */
int b200sm_relocalize_score_nodes(b200sm_t s, int level, long long count, const int* k_i_j, int* scores);
int b200sm_get_localize_stats(b200sm_t s, b200sm_localize_stats* out);
/* read-back of the current cut (the newest one, pending or adopted), like b200sm_get_targeted */
int b200sm_get_cut(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n);

typedef struct b200sm_stats {
  size_t n_scan, n_filtered, n_targeted, n_submaps;
  int kernel_launches;
  double trans, latest_distance;
} b200sm_stats;
int b200sm_get_stats(b200sm_t s, b200sm_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* B200REG_H_ */
