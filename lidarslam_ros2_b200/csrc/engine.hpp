// Host-side engine classes behind the C-ABI (include/b200reg.h). C++17, CUDA runtime only — no torch types.
#pragma once
#include <algorithm>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200reg.h"
#include "common.cuh"
#include "ndt_math.cuh"
#include "pcd_parse.cuh"

namespace b200 {

// Persistent cooperative kernels (NDT solver, GICP inner loop) need every CTA of their grid resident at once and spin on
// one another. Two of them launched from different host threads / streams of one device must never be interleaved by
// the block scheduler (each holding part of the SMs while waiting for the rest): whoever launches one holds this
// per-device mutex from the launch until the kernel has completed. Uploads, map builds and NN passes of other handles
// still overlap it.
std::mutex& cooperative_launch_mutex(int device);

// ---- RAII device / pinned buffers -------------------------------------------------------------------
template <typename T>
struct DeviceBuffer {
  T* ptr = nullptr;
  size_t cap = 0;
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
  ~DeviceBuffer() { release(); }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    cap = 0;
  }
  // grow-only; contents are NOT preserved. Geometric growth: a buffer that creeps up (the targeted cloud of the
  // frontend session, the per-frame scratch) must not pay a cudaFree + cudaMalloc pair on every call.
  void ensure(size_t n) {
    if (n <= cap) return;
    const size_t want = std::max(n + n / 8 + 64, cap + cap / 2);
    release();
    B200_CUDA(cudaMalloc(&ptr, want * sizeof(T)));
    cap = want;
  }
};

template <typename T>
struct PinnedBuffer {
  T* ptr = nullptr;
  size_t cap = 0;
  PinnedBuffer() = default;
  PinnedBuffer(const PinnedBuffer&) = delete;
  PinnedBuffer& operator=(const PinnedBuffer&) = delete;
  ~PinnedBuffer() {
    if (ptr) cudaFreeHost(ptr);
  }
  void ensure(size_t n) {
    if (n <= cap) return;
    if (ptr) cudaFreeHost(ptr);
    ptr = nullptr;
    size_t want = n + n / 8 + 64;
    B200_CUDA(cudaMallocHost(&ptr, want * sizeof(T)));
    cap = want;
  }
};

// ---- rank index (occupancy bitmap + popcount prefix), see common.cuh; grid_index.cu -------------------
struct RankIndexScratch {
  DeviceBuffer<unsigned> block_sums;
  DeviceBuffer<unsigned> total;  // 1 element
};
// zero-fills table[0..n_words)
void rank_index_clear(RankWord* table, int n_words, cudaStream_t s);
// fills .prefix from .bits, enqueue only: the number of set bits is left in *d_total (device memory)
void rank_index_scan_async(RankWord* table, size_t n_words, RankIndexScratch& scratch, unsigned* d_total, cudaStream_t s);
// exclusive scan of data[0..n) in place, enqueue only; data[n] receives the total
void counter_scan_async(unsigned* data, size_t n, DeviceBuffer<unsigned>& tile_sums, cudaStream_t s);
// cell_of_point[i] = leaf index of point i in g (-1 if not finite); marks cell >> shift occupied in table
void mark_grid_cells(const float4* pts, size_t n, const GridGeom& g, RankWord* table, int* cell_of_point, int shift,
                     cudaStream_t s);

// min/max of the finite points of a cloud
struct Bounds {
  float mn[3], mx[3];
  bool any;
};
// the six order-preserving uints {min xyz, max xyz} the bounds kernels leave → Bounds
Bounds decode_bounds(const unsigned* res6);
// min/max of the finite points of a float4 cloud → host (synchronises the stream)
Bounds cloud_bounds(const float4* pts, size_t n, unsigned* d_scratch8, cudaStream_t s);
// the bounds a builder grids a cloud by: known_bounds when the caller has them, else measured by cloud_bounds (counted
// in `launches`)
Bounds grid_bounds(const float4* pts, size_t n, const Bounds* known_bounds, DeviceBuffer<unsigned>& scratch, int& launches,
                   cudaStream_t s);
// PCL grid geometry from bounds (voxel_grid_covariance_omp_impl.hpp:67-103); returns false on int32 overflow
bool make_grid_geom(const Bounds& b, float leaf, GridGeom& g);

// upload an arbitrary-stride host cloud into a float4 device buffer (w = 1)
// strided host records -> float4 on the device: one bulk H2D copy of the raw bytes + an unpack kernel (cloud_codec.cu)
struct CloudUploader {
  DeviceBuffer<unsigned char> raw;
  PinnedBuffer<unsigned char> staging;  // only used when the caller's buffer is pageable
  int launches = 0;
  // w_off >= 0: byte offset of the float that goes to .w (intensity); otherwise .w = w_default
  void upload(const void* host, size_t n, size_t stride, long w_off, float w_default, float4* dst, cudaStream_t s);
  // upload + min/max of the finite points in the same pass; finish_bounds() is valid once the stream has been synchronised.
  // T (3x4 row-major, optional): every point's x, y, z is moved by T before the store and the bounds are the moved points'.
  DeviceBuffer<unsigned> bounds_dev;
  PinnedBuffer<unsigned> bounds_host;
  void upload_with_bounds(const void* host, size_t n, size_t stride, long w_off, float w_default, float4* dst, cudaStream_t s,
                          const Mat34f* T = nullptr);
  Bounds finish_bounds() const;
  // batched form (no synchronisation between clouds): reserve once, then upload_at per cloud at its byte offset
  void reserve(size_t raw_bytes, bool need_staging);
  static bool is_pinned(const void* host);
  void upload_at(const void* host, bool pinned, size_t n, size_t stride, long w_off, float w_default, float4* dst,
                 size_t byte_offset, cudaStream_t s);
  void copy_at(const void* host, bool pinned, size_t bytes, size_t byte_offset, cudaStream_t s);
};
void upload_cloud(const float* base, size_t n, size_t stride_bytes, DeviceBuffer<float4>& dst, CloudUploader& up, cudaStream_t s);

// ---- NDT voxel map (K3) -------------------------------------------------------------------------------
struct VoxelMap {
  GridGeom geom{};
  size_t n_voxels = 0;    // voxels with >= min_points (valid), ascending leaf index
  size_t n_occupied = 0;  // all occupied leaves
  DeviceBuffer<RankWord> index;      // rank index over VALID voxels (what the solver probes)
  DeviceBuffer<VoxelRecord> records; // n_voxels
  DeviceBuffer<double> icov_d;       // n_voxels x 9 (f64 inverse covariance, for the f64 paths)
  DeviceBuffer<float4> centroids;    // n_voxels: f32 centroid xyz, w = leaf index (int bits)
  DeviceBuffer<int> npts;            // n_voxels
  // build scratch
  DeviceBuffer<RankWord> index_all;
  DeviceBuffer<int> cell_of_point;
  DeviceBuffer<double> acc;          // n_occupied x 10
  DeviceBuffer<int> leaf_of_rank;
  DeviceBuffer<VoxelRecord> tmp_records;
  DeviceBuffer<double> tmp_icov;
  DeviceBuffer<float4> tmp_centroids;
  DeviceBuffer<int> tmp_npts;
  DeviceBuffer<unsigned char> tmp_valid;
  DeviceBuffer<unsigned> bounds_scratch;
  DeviceBuffer<unsigned> counts;   // [0] occupied leaves, [1] valid voxels (device side of the build)
  PinnedBuffer<unsigned> h_counts;
  RankIndexScratch scan_scratch;
  int launches = 0;

  // returns false if the grid overflows int32 (map left empty, like voxel_grid_covariance_omp_impl.hpp:79-84).
  // known_bounds: min/max of the cloud when the caller already has them (measured during the upload).
  // One host synchronisation (the final counts), none when... see voxel_map.cu.
  bool build(const float4* pts, size_t n, float leaf, int min_points_per_voxel, double min_covar_eigvalue_mult,
             cudaStream_t s, const Bounds* known_bounds = nullptr);
};

// ---- exact nearest-neighbour grid over a cloud (K8 fitness, GICP) ---------------------------------------
struct NnGrid {
  float h = 0, inv_h = 0;
  float origin[3] = {0, 0, 0};
  int dims[3] = {0, 0, 0};
  long long n_cells = 0;
  int n_words = 0;
  size_t n_points = 0, n_cells_occupied = 0;
  DeviceBuffer<RankWord> index;
  DeviceBuffer<unsigned> coarse;      // 6 ordered uints per 8x8x8 block of cells: bounding box of its points (far queries)
  int cdims[3] = {0, 0, 0};
  int n_coarse = 0;
  DeviceBuffer<unsigned> cell_start;  // n_cells_occupied + 1
  DeviceBuffer<float4> sorted;        // xyz + original index (int bits) in w
  DeviceBuffer<int> cell_of_point;
  DeviceBuffer<unsigned> cursor;
  DeviceBuffer<unsigned> bounds_scratch;
  RankIndexScratch scan_scratch;
  DeviceBuffer<unsigned> scan_tmp;
  DeviceBuffer<int> unresolved;             // query scratch: indices of queries left to the brute-force pass
  DeviceBuffer<unsigned> unresolved_count;
  int launches = 0;
  bool valid = false;
  void build(const float4* pts, size_t n, cudaStream_t s, const Bounds* known_bounds = nullptr);
};
// 1-NN of n queries (optionally transformed by T, 3x4 row-major; nullptr = none). d2 accumulated in f32 as
// ((dx*dx + dy*dy) + dz*dz); ties → lower index. idx = -1 when the target is empty.
// max_d2: only neighbours closer than this matter to the caller (FLT_MAX = unbounded). Queries whose neighbourhood is
// not resolved within a few cell rings are finished by a brute-force pass (exact either way).
void nn1_query(const NnGrid& grid, const float4* queries, size_t n, const float* T12_host, int* d_idx, float* d_d2,
               cudaStream_t s, float max_d2 = 3.402823466e+38f);
// mean of d2 over queries with d2 <= max_range → (sum, count) on device, returned to host (synchronises)
void fitness_reduce(const float* d_d2, const int* d_idx, size_t n, double max_range, double* d_scratch2, double* sum,
                    long long* count, cudaStream_t s);

// ---- NDT solver (K1 fused derivative kernel inside a persistent cooperative Newton loop) ----------------
struct NdtSolverWork;  // device-side work area, defined in ndt_solver.cu
struct NdtJob;
struct NdtLaunch;

struct NdtResult {
  float final_T[16];  // row-major 4x4
  double score;
  double trans_probability;
  double g[6];
  double H[36];
  long long hits_last, hits_total;
  int converged, iterations, evaluations, error;
};

struct NdtConfig {
  float resolution = 1.0f;
  double step_size = 0.1, outlier_ratio = 0.55, trans_eps = 0.1;
  int max_iterations = 35;
  int search_method = 2;  // DIRECT7
};

// ---- pose board: the poses of a sharded batch exchanged by the solver kernel itself over NVLink peer memory ----------
// Every rank owns one board in its HBM; all ranks map all boards (CUDA IPC, include/b200comm.h). When a registration of
// a batch launch finishes, its controller CTA stores the 4x4 pose into row [own rank][registration] of EVERY board —
// sixteen 64-bit words {float bits, launch tag}, so a word is valid exactly when its tag is the current launch's (the
// same flag-in-data convention as the kernel's internal signalling: no fence, no second message). The exchange rides
// on the kernel's own progress: by the time the last registration converges all earlier poses have already crossed
// NVSwitch. A small collect kernel behind the solver waits for the remaining words and copies the rows to mapped host
// memory. Boards are double-buffered by tag parity: a rank can be at most one launch ahead of its slowest peer.
constexpr int POSE_BOARD_MAX_PEERS = 8;
struct PoseBoardView {
  unsigned long long* peer[POSE_BOARD_MAX_PEERS];  // peer[r]: rank r's board as mapped on THIS device (peer[rank] = own)
  int world, rank;
  int rows;      // registrations per rank and launch the board has room for; row `rows` is the header {count, tag}
  unsigned tag;  // this launch's sequence number (> 0; the same on every rank: attached batch calls are collective)
};
__host__ __device__ inline size_t pose_board_word(const PoseBoardView& b, unsigned tag, int src_rank, int row, int k) {
  return ((((size_t)(tag & 1u) * (size_t)b.world + (size_t)src_rank) * (size_t)(b.rows + 1)) + (size_t)row) * 16 + (size_t)k;
}
inline size_t pose_board_words(int world, int rows) { return (size_t)2 * world * (rows + 1) * 16; }

}  // namespace b200
// the opaque object of include/b200comm.h (created by b200comm_board_create in comm.cu, consumed by capi.cu)
struct b200comm_board {
  b200::PoseBoardView view{};
  unsigned long long* own = nullptr;
  void* opened[b200::POSE_BOARD_MAX_PEERS] = {};
  float* h_rows = nullptr;   // pinned + mapped: world x rows x 16 floats (row-major poses), written by the collect kernel
  int* h_counts = nullptr;   // pinned + mapped: world counts, then [world] = error flag of the collect kernel
  int device = 0;
  double timeout_s = 20.0;  // a peer that never makes the collective batch call is reported, not waited for for ever
};
namespace b200 {

enum NdtMode : int { NDT_MODE_ALIGN = 0, NDT_MODE_DERIVATIVES = 1, NDT_MODE_HESSIAN_RADIUS = 2, NDT_MODE_SCORE = 3 };

class NdtSolver {
 public:
  NdtSolver() = default;
  ~NdtSolver();
  void init(int device, cudaStream_t s);
  // enqueue one solver launch on the stream; result lands in pinned host memory after the stream syncs
  // resume = 1 continues a solve that left the kernel for a K2 (radius Hessian) pass
  void launch(const VoxelMap& map, const float4* src, size_t n_src, const NdtConfig& cfg, int mode,
              const float* T_rowmajor16, const double* p6, int compute_hessian, int resume = 0);
  // one registration of a batch: device-resident source (float4) and the row-major 4x4 guess
  struct BatchItem {
    const void* src;       // device memory: float4 points (stride 0 or 16) or raw records of `stride` bytes (x, y, z first)
    size_t n_src;
    float T_rowmajor16[16];
    int stride = 0;
    const unsigned* ready = nullptr;  // device flag that reads ready_tag once the points have arrived (nullptr: they are there)
    unsigned ready_tag = 0;
  };
  // enqueue ONE launch that performs n independent registrations against `map`, `slots` (<= NDT_MAX_SLOTS) in flight;
  // after the stream has drained batch_results()[k] holds registration k (error != 0: the kernel never finished it)
  // board (optional): the finished poses also go to every peer's pose board (board->view.tag = this launch's number);
  // launch_board_collect() then enqueues the kernel that gathers all ranks' rows of the launch into board->h_rows / h_counts
  void launch_batch(const VoxelMap& map, const BatchItem* items, int n, const NdtConfig& cfg, int slots,
                    b200comm_board* board = nullptr);
  void launch_board_collect(b200comm_board* board);
  const NdtResult* batch_results() const { return h_batch_results_; }
  // rounds one slot can run inside a launch (sequence numbers are 16 bits per launch)
  static constexpr int kMaxRoundsPerLaunch = 60000;
  NdtSolverWork* work() const { return d_work_; }
  // device addresses of the controller's f64 angle tables / current transform (inputs of the K2 pass)
  const double* state_jd() const;
  const double* state_hd() const;
  const float* control_T() const;
  const NdtResult& result() const { return *h_result_; }
  int grid_ctas() const { return grid_; }
  int block_threads() const { return block_; }
  int index_in_smem() const { return index_in_smem_; }
  int launches = 0;
  bool scalar_controller = false;  // developer switch (env B200REG_SCALAR_CTL=1)
  // per-round trace of align-mode single launches (b200reg_ndt_set_trace / b200reg_ndt_get_trace)
  void set_trace(int capacity);
  int read_trace(b200reg_ndt_trace_record* out, int cap);  // copies up to cap records, returns the rounds counted
  void reset_barrier();
  void fetch_result();

 private:
  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  int sm_count_ = 0;
  int grid_ = 0, block_ = 0, index_in_smem_ = 0;
  int max_smem_optin_ = 0;
  unsigned epoch_ = 0;
  bool fits_checked_ = false;
  NdtSolverWork* d_work_ = nullptr;
  NdtResult* h_result_ = nullptr;  // pinned
  NdtJob* d_jobs_ = nullptr;       // batch launches: job table on the device ...
  NdtJob* h_jobs_ = nullptr;       // ... and its pinned host image
  NdtResult* h_batch_results_ = nullptr;  // pinned + device-visible: the controllers write the results there
  size_t jobs_cap_ = 0;
  b200reg_ndt_trace_record* d_trace_ = nullptr;
  int trace_cap_ = 0;
  int trace_launch_ = 0;
  void fill_common(NdtLaunch& L, const VoxelMap& map, const NdtConfig& cfg, int mode, int n_slots, size_t& dyn_smem);
  int eval_ctas_for(size_t n_src) const;
};

// off-hot-path f64 kernels (ndt_aux.cu)
// d_T12: DEVICE pointer to the 3x4 row-major transform applied to src
void ndt_hessian_radius(const VoxelMap& map, const float4* src, size_t n, const NdtConfig& cfg, const float* d_T12,
                        const double* d_jd, const double* d_hd, double* d_out21, cudaStream_t s);
void ndt_hessian_into_state(const double* d_upper21, NdtSolverWork* work, cudaStream_t s);
void ndt_score(const VoxelMap& map, const float4* cloud, size_t n, const NdtConfig& cfg, double* d_out1, cudaStream_t s);
// K12 (ndt_score.cu): d_scores[k] / d_hits[k] = NDT score and kept pairs of `count` column-major poses (d_poses, 16 floats
// each, device memory) of src against map; enqueue only. The map must hold at least one voxel.
void ndt_score_poses(const VoxelMap& map, const float4* src, size_t n_src, const NdtConfig& cfg, const float* d_poses, int count,
                     double* d_scores, long long* d_hits, cudaStream_t s);
// out = T * in, xyz in f32 (transform_point), w copied
void transform_cloud_device(const float4* in, size_t n, float4* out, const Mat34f& T, cudaStream_t s);

// ---- VoxelGrid downsample (K4) --------------------------------------------------------------------------
struct VoxelGridFilter {
  DeviceBuffer<float4> in;   // xyz + intensity
  DeviceBuffer<float4> out;
  DeviceBuffer<RankWord> index;     // dense rank index, or level 1 (pages) of the sparse one
  DeviceBuffer<RankWord> index_l2;  // sparse form: 32 words per occupied page
  DeviceBuffer<int> cell_of_point;
  DeviceBuffer<double> acc;  // n_vox x 5
  DeviceBuffer<unsigned> bounds_scratch;
  DeviceBuffer<unsigned> count_dev;
  PinnedBuffer<unsigned> count_host;
  RankIndexScratch scan_scratch;
  PinnedBuffer<float4> staging;
  int launches = 0;
  // the dense occupancy bitmap is used up to this many 8-byte words (32 MB); larger bounding boxes take the two-level
  // sparse index whose memory is O(points), like pcl::VoxelGrid's (voxelgrid.cu)
  size_t dense_word_budget = (size_t)4 << 20;
  bool last_sparse = false;
  // device-resident core: returns number of output points, or -1 on grid overflow (output = input).
  // known_bounds: min/max of d_in when the caller already has them. One host synchronisation at the end (the count).
  long long filter_device(const float4* d_in, size_t n, float leaf, cudaStream_t s, const Bounds* known_bounds = nullptr);
};

// ---- ASCII PCD text of a float4 (x, y, z, intensity) cloud (pcd_codec.cu) ------------------------------------------
// The text is produced in chunks of PCD_CHUNK_POINTS points, so that a writer can hold two chunks in host memory and one
// on the device whatever the size of the map.
constexpr size_t PCD_CHUNK_POINTS = (size_t)1 << 22;
// the header savePCDFileASCII writes for n PointXYZI points, "DATA ascii\n" included
std::string pcd_ascii_header(size_t n);
struct PcdEncoder {
  DeviceBuffer<unsigned> counts;  // per chunk: tile byte counts, scanned in place into tile offsets, then the chunk's total
  DeviceBuffer<unsigned> scan_tmp;
  DeviceBuffer<char> text;        // the text of one chunk
  PinnedBuffer<unsigned> h_counts;
  std::vector<size_t> chunk_bytes;  // text bytes of every chunk, known after measure()
  int launches = 0;
  // pass 1 over the whole cloud and the per-chunk scans; fills chunk_bytes and sizes `text` (synchronises the stream)
  void measure(const float4* pts, size_t n, cudaStream_t s);
  // pass 2: the text of chunk c into `text` (enqueue only; the offsets are those of the last measure() of the same cloud)
  void encode_chunk(const float4* pts, size_t n, size_t c, cudaStream_t s);
};

// ---- PCD file -> float4 (x, y, z, intensity) on the device (pcd_load.cu; the contract is b200reg_load_pcd's) ---------
// the header of an open file, read up to and including its DATA line: B200REG_OK, B200REG_ERR_IO or B200REG_ERR_FORMAT
int read_pcd_header(FILE* fp, PcdHeader& h, std::string& err);
struct PcdLoader {
  PinnedBuffer<char> pieces[2];            // the ASCII body, B200REG_PCD_LOAD_PIECE_BYTES at a time
  DeviceBuffer<char> text;                 // one piece, plus the parse kernel's staging slack
  DeviceBuffer<unsigned> counts, scan_tmp; // non-empty lines per tile, scanned in place into tile offsets
  DeviceBuffer<unsigned long long> state;  // [0] non-empty lines so far, [1] first failing line: file offset << 2 | kind
  PinnedBuffer<unsigned long long> h_state;
  PinnedBuffer<unsigned char> body;        // a binary body, read whole
  CloudUploader uploader;
  int launches = 0;
  // The points of `path` into dst (grown to POINTS rows); *n = POINTS. B200REG_OK, B200REG_ERR_IO or B200REG_ERR_FORMAT
  // (reason in err); CUDA errors throw. The stream is synchronised on return.
  int load(const char* path, DeviceBuffer<float4>& dst, size_t* n, std::string& err, cudaStream_t s);
};

}  // namespace b200
