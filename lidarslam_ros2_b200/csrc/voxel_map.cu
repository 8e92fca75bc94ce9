// K3 — NDT target voxel map on the GPU, plus the shared rank-index / bounds / upload utilities.
//
// Replaces pclomp::VoxelGridCovariance::applyFilter (Thirdparty/ndt_omp_ros2/include/pclomp/
// voxel_grid_covariance_omp_impl.hpp:48-370) reached from NormalDistributionsTransform::setInputTarget →
// init() (ndt_omp.h:117-122, 271-278). The reference walks a std::map<size_t, Leaf> serially; here the leaf
// index is hashed perfectly by an occupancy bitmap + popcount prefix ("rank index"), per-leaf moments are
// reduced with f64 atomics, and one thread per leaf does the covariance regularisation in f64.
//
// Algorithmic HBM bytes (DESIGN.md §kernels):  N_tgt*16 (points) + V*(48+8) (records + index share).
#include <cfloat>
#include <cmath>

#include "engine.hpp"

namespace b200 {

std::mutex& cooperative_launch_mutex(int device) {
  static std::mutex m[64];
  return m[(device >= 0 && device < 64) ? device : 0];
}

// =====================================================================================================
// rank index
// =====================================================================================================
void rank_index_clear(RankWord* table, int n_words, cudaStream_t s) {
  B200_CUDA(cudaMemsetAsync(table, 0, sizeof(RankWord) * (size_t)n_words, s));
}

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;  // words per thread
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// block-local exclusive scan of popc(bits); per-block totals to block_sums
__global__ void __launch_bounds__(SCAN_THREADS) rank_scan_local_kernel(RankWord* table, int n_words,
                                                                       unsigned* block_sums) {
  __shared__ unsigned warp_tot[SCAN_THREADS / 32];
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  unsigned cnt[SCAN_ITEMS];
  unsigned local = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    int w = base + k;
    cnt[k] = (w < n_words) ? __popc(table[w].bits) : 0u;
    local += cnt[k];
  }
  // warp inclusive scan of `local`
  unsigned incl = local;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    unsigned v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned warp_off = 0;
  for (int w = 0; w < warp; w++) warp_off += warp_tot[w];
  unsigned run = warp_off + incl - local;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    int w = base + k;
    if (w < n_words) table[w].prefix = run;
    run += cnt[k];
  }
  if (threadIdx.x == SCAN_THREADS - 1) block_sums[blockIdx.x] = run;
}

// single block: exclusive scan of block_sums in place, grand total to *total
__global__ void __launch_bounds__(1024) rank_scan_blocks_kernel(unsigned* block_sums, int n_blocks, unsigned* total) {
  __shared__ unsigned warp_tot[32];
  __shared__ unsigned carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n_blocks; base += 1024) {
    int i = base + threadIdx.x;
    unsigned v = (i < n_blocks) ? block_sums[i] : 0u;
    unsigned incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      unsigned t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    unsigned off = 0;
    for (int w = 0; w < warp; w++) off += warp_tot[w];
    unsigned carry = carry_s;
    if (i < n_blocks) block_sums[i] = carry + off + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + off + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry_s;
}

__global__ void __launch_bounds__(SCAN_THREADS) rank_scan_apply_kernel(RankWord* table, int n_words,
                                                                       const unsigned* block_sums) {
  const unsigned off = block_sums[blockIdx.x];
  const int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    int w = base + k;
    if (w < n_words) table[w].prefix += off;
  }
}

// fills .prefix from .bits and leaves the number of set bits in *d_total (device memory); nothing waits
void rank_index_scan_async(RankWord* table, int n_words, RankIndexScratch& scratch, unsigned* d_total, cudaStream_t s) {
  const int n_blocks = (n_words + SCAN_TILE - 1) / SCAN_TILE;
  scratch.block_sums.ensure((size_t)n_blocks + 1);
  rank_scan_local_kernel<<<n_blocks, SCAN_THREADS, 0, s>>>(table, n_words, scratch.block_sums.ptr);
  rank_scan_blocks_kernel<<<1, 1024, 0, s>>>(scratch.block_sums.ptr, n_blocks, d_total);
  if (n_blocks > 1) rank_scan_apply_kernel<<<n_blocks, SCAN_THREADS, 0, s>>>(table, n_words, scratch.block_sums.ptr);
}

unsigned rank_index_scan(RankWord* table, int n_words, RankIndexScratch& scratch, cudaStream_t s) {
  scratch.total.ensure(1);
  rank_index_scan_async(table, n_words, scratch, scratch.total.ptr, s);
  unsigned total = 0;
  B200_CUDA(cudaMemcpyAsync(&total, scratch.total.ptr, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  return total;
}

// =====================================================================================================
// bounds, geometry, upload
// =====================================================================================================
__global__ void __launch_bounds__(256) bounds_kernel(const float4* __restrict__ pts, size_t n, unsigned* out6) {
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float4 p = pts[i];
    if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) continue;
    mn[0] = fminf(mn[0], p.x); mn[1] = fminf(mn[1], p.y); mn[2] = fminf(mn[2], p.z);
    mx[0] = fmaxf(mx[0], p.x); mx[1] = fmaxf(mx[1], p.y); mx[2] = fmaxf(mx[2], p.z);
  }
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], d));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], d));
    }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; a++) {
      atomicMin(&out6[a], float_to_ordered(mn[a]));
      atomicMax(&out6[3 + a], float_to_ordered(mx[a]));
    }
  }
}

Bounds cloud_bounds(const float4* pts, size_t n, unsigned* d_scratch8, cudaStream_t s) {
  unsigned init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
  B200_CUDA(cudaMemcpyAsync(d_scratch8, init, sizeof(init), cudaMemcpyHostToDevice, s));
  int blocks = (int)std::min<size_t>((n + 255) / 256, H100_SMS * 8);
  if (blocks < 1) blocks = 1;
  bounds_kernel<<<blocks, 256, 0, s>>>(pts, n, d_scratch8);
  unsigned res[6];
  B200_CUDA(cudaMemcpyAsync(res, d_scratch8, sizeof(res), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  Bounds b;
  b.any = !(res[0] == 0xffffffffu && res[3] == 0u);
  for (int a = 0; a < 3; a++) {
    b.mn[a] = ordered_to_float(res[a]);
    b.mx[a] = ordered_to_float(res[3 + a]);
  }
  return b;
}

bool make_grid_geom(const Bounds& b, float leaf, GridGeom& g) {
  g.leaf = leaf;
  g.inv_leaf = 1.0f / leaf;
  // voxel_grid_covariance_omp_impl.hpp:75-84 — float products, int64 casts
  long long dx = static_cast<long long>((b.mx[0] - b.mn[0]) * g.inv_leaf) + 1;
  long long dy = static_cast<long long>((b.mx[1] - b.mn[1]) * g.inv_leaf) + 1;
  long long dz = static_cast<long long>((b.mx[2] - b.mn[2]) * g.inv_leaf) + 1;
  if (dx * dy * dz > static_cast<long long>(INT32_MAX)) return false;
  for (int a = 0; a < 3; a++) {
    g.min_b[a] = static_cast<int>(std::floor(b.mn[a] * g.inv_leaf));
    g.max_b[a] = static_cast<int>(std::floor(b.mx[a] * g.inv_leaf));
    g.div_b[a] = g.max_b[a] - g.min_b[a] + 1;
  }
  g.mul[0] = 1;
  g.mul[1] = g.div_b[0];
  g.mul[2] = g.div_b[0] * g.div_b[1];
  g.n_cells = (long long)g.div_b[0] * g.div_b[1] * g.div_b[2];
  if (g.n_cells > static_cast<long long>(INT32_MAX)) return false;
  g.n_words = (int)((g.n_cells + 31) / 32);
  return true;
}

// =====================================================================================================
// voxel map build
// =====================================================================================================
__global__ void __launch_bounds__(256) vm_mark_kernel(const float4* __restrict__ pts, size_t n, GridGeom g,
                                                      RankWord* table, int* cell_of_point) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = pts[i];
  int cell = -1;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    cell = build_leaf_index(g, p.x, p.y, p.z);
    if (cell < 0 || cell >= g.n_cells) cell = -1;  // cannot happen for finite points inside the bounds
  }
  cell_of_point[i] = cell;
  // a 1 M-point map has ~10^4 occupied leaves: almost every point finds its bit already set — look before the atomic
  // (a stale read can only cause a redundant atomicOr, never a missing one)
  if (cell >= 0 && !((__ldcg(&table[cell >> 5].bits) >> (cell & 31)) & 1u)) atomicOr(&table[cell >> 5].bits, 1u << (cell & 31));
}

__device__ __forceinline__ unsigned rank_of(const RankWord* __restrict__ table, int cell) {
  RankWord w = table[cell >> 5];
  return w.prefix + __popc(w.bits & ((1u << (cell & 31)) - 1u));
}

// per-leaf moments: acc[r*10 + {0..2}] = sum x, {3..8} = sum xx^T (upper: xx xy xz yy yz zz), {9} = count
__global__ void __launch_bounds__(256) vm_accumulate_kernel(const float4* __restrict__ pts, size_t n,
                                                            const int* __restrict__ cell_of_point,
                                                            const RankWord* __restrict__ table, double* acc,
                                                            int* leaf_of_rank) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cell = cell_of_point[i];
  if (cell < 0) return;
  unsigned r = rank_of(table, cell);
  float4 p = pts[i];
  double x = p.x, y = p.y, z = p.z;
  double* a = acc + (size_t)r * 10;
  atomicAdd(a + 0, x);
  atomicAdd(a + 1, y);
  atomicAdd(a + 2, z);
  atomicAdd(a + 3, x * x);
  atomicAdd(a + 4, x * y);
  atomicAdd(a + 5, x * z);
  atomicAdd(a + 6, y * y);
  atomicAdd(a + 7, y * z);
  atomicAdd(a + 8, z * z);
  atomicAdd(a + 9, 1.0);
  leaf_of_rank[r] = cell;  // every writer stores the same value
}

// ---- 3x3 f64 helpers (device) ----
__device__ void d_inverse3(const double* m, double* o) {
  double c00 = m[4] * m[8] - m[5] * m[7];
  double c01 = m[5] * m[6] - m[3] * m[8];
  double c02 = m[3] * m[7] - m[4] * m[6];
  double id = 1.0 / (m[0] * c00 + m[1] * c01 + m[2] * c02);
  o[0] = c00 * id;
  o[1] = (m[2] * m[7] - m[1] * m[8]) * id;
  o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  o[3] = c01 * id;
  o[4] = (m[0] * m[8] - m[2] * m[6]) * id;
  o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  o[6] = c02 * id;
  o[7] = (m[1] * m[6] - m[0] * m[7]) * id;
  o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// cyclic Jacobi on a symmetric 3x3; eigenvalues ascending in ev[], eigenvectors as columns of V (row-major)
__device__ void d_sym_eigen3(const double* ain, double* ev, double* V) {
  double a00 = ain[0], a01 = ain[3], a02 = ain[6], a11 = ain[4], a12 = ain[7], a22 = ain[8];  // lower triangle
  double v[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int sweep = 0; sweep < 64; sweep++) {
    double off = a01 * a01 + a02 * a02 + a12 * a12;
    double diag = a00 * a00 + a11 * a11 + a22 * a22;
    if (off == 0.0 || off <= 1e-34 * diag) break;
    // rotation (p,q) = (0,1)
#define B200_JACOBI_ROT(app, aqq, apq, apr, aqr, P, Q)                                   \
  if (apq != 0.0) {                                                                      \
    double theta = (aqq - app) / (2.0 * apq);                                            \
    double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));    \
    double c = 1.0 / sqrt(t * t + 1.0), s = t * c;                                       \
    double napp = app - t * apq, naqq = aqq + t * apq;                                   \
    double napr = c * apr - s * aqr, naqr = s * apr + c * aqr;                           \
    app = napp; aqq = naqq; apq = 0.0; apr = napr; aqr = naqr;                           \
    for (int k = 0; k < 3; k++) {                                                        \
      double vp = v[k * 3 + P], vq = v[k * 3 + Q];                                       \
      v[k * 3 + P] = c * vp - s * vq;                                                    \
      v[k * 3 + Q] = s * vp + c * vq;                                                    \
    }                                                                                    \
  }
    B200_JACOBI_ROT(a00, a11, a01, a02, a12, 0, 1)
    B200_JACOBI_ROT(a00, a22, a02, a01, a12, 0, 2)
    B200_JACOBI_ROT(a11, a22, a12, a01, a02, 1, 2)
#undef B200_JACOBI_ROT
  }
  double d[3] = {a00, a11, a22};
  int o0 = 0, o1 = 1, o2 = 2;
  if (d[o0] > d[o1]) { int t = o0; o0 = o1; o1 = t; }
  if (d[o1] > d[o2]) { int t = o1; o1 = o2; o2 = t; }
  if (d[o0] > d[o1]) { int t = o0; o0 = o1; o1 = t; }
  ev[0] = d[o0]; ev[1] = d[o1]; ev[2] = d[o2];
  for (int r = 0; r < 3; r++) {
    V[r * 3 + 0] = v[r * 3 + o0];
    V[r * 3 + 1] = v[r * 3 + o1];
    V[r * 3 + 2] = v[r * 3 + o2];
  }
}

// one thread per occupied leaf (voxel_grid_covariance_omp_impl.hpp:282-367)
__global__ void __launch_bounds__(128) vm_finalize_kernel(const double* __restrict__ acc, const int* __restrict__ leaf_of_rank,
                                                          const unsigned* __restrict__ n_occ_ptr, int min_points, double eig_mult,
                                                          VoxelRecord* rec, double* icov_d, float4* centroids, int* npts,
                                                          unsigned char* valid, RankWord* valid_table) {
  size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (r >= (size_t)*n_occ_ptr) return;  // the occupied-leaf count stays on the device: no host round trip mid-build
  const double* a = acc + r * 10;
  const int n_i = (int)(a[9] + 0.5);
  valid[r] = 0;
  if (n_i < min_points) return;
  const double n = (double)n_i;
  double pt_sum[3] = {a[0], a[1], a[2]};
  double mean[3] = {pt_sum[0] / n, pt_sum[1] / n, pt_sum[2] / n};
  // cov_ started at Identity (voxel_grid_covariance_omp.h:101) and accumulated x x^T on top of it
  double sxx[9] = {a[3] + 1.0, a[4], a[5], a[4], a[6] + 1.0, a[7], a[5], a[7], a[8] + 1.0};
  double cov[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      cov[i * 3 + j] = (sxx[i * 3 + j] - 2 * (pt_sum[i] * mean[j])) / n + mean[i] * mean[j];
  const double f = (n - 1.0) / n;
  for (int k = 0; k < 9; k++) cov[k] *= f;
  double ev[3], V[9];
  d_sym_eigen3(cov, ev, V);
  if (ev[0] < 0 || ev[1] < 0 || ev[2] <= 0) return;  // reference flags nr_points = -1
  double min_ev = eig_mult * ev[2];
  if (ev[0] < min_ev) {
    ev[0] = min_ev;
    if (ev[1] < min_ev) ev[1] = min_ev;
    double Vinv[9], VD[9];
    d_inverse3(V, Vinv);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) VD[i * 3 + j] = V[i * 3 + j] * ev[j];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        cov[i * 3 + j] = VD[i * 3 + 0] * Vinv[0 * 3 + j] + VD[i * 3 + 1] * Vinv[1 * 3 + j] + VD[i * 3 + 2] * Vinv[2 * 3 + j];
  }
  double ic[9];
  d_inverse3(cov, ic);
  double mxv = ic[0], mnv = ic[0];
  for (int k = 1; k < 9; k++) {
    mxv = fmax(mxv, ic[k]);
    mnv = fmin(mnv, ic[k]);
  }
  if (isinf(mxv) || isinf(mnv) || isnan(mxv) || isnan(mnv)) return;
  VoxelRecord o;
  o.mhx = (float)mean[0]; o.mlx = (float)(mean[0] - (double)o.mhx);
  o.mhy = (float)mean[1]; o.mly = (float)(mean[1] - (double)o.mhy);
  o.mhz = (float)mean[2]; o.mlz = (float)(mean[2] - (double)o.mhz);
  o.c00 = (float)ic[0]; o.c01 = (float)ic[1]; o.c02 = (float)ic[2];
  o.c11 = (float)ic[4]; o.c12 = (float)ic[5]; o.c22 = (float)ic[8];
  rec[r] = o;
  for (int k = 0; k < 9; k++) icov_d[r * 9 + k] = ic[k];
  const int leaf = leaf_of_rank[r];
  const float nf = (float)n_i;
  centroids[r] = make_float4((float)pt_sum[0] / nf, (float)pt_sum[1] / nf, (float)pt_sum[2] / nf, __int_as_float(leaf));
  npts[r] = n_i;
  valid[r] = 1;
  atomicOr(&valid_table[leaf >> 5].bits, 1u << (leaf & 31));
}

__global__ void __launch_bounds__(128) vm_compact_kernel(const unsigned* __restrict__ n_occ_ptr, const unsigned char* __restrict__ valid,
                                                         const int* __restrict__ leaf_of_rank,
                                                         const RankWord* __restrict__ valid_table,
                                                         const VoxelRecord* __restrict__ rec_in, const double* __restrict__ icov_in,
                                                         const float4* __restrict__ cen_in, const int* __restrict__ npts_in,
                                                         VoxelRecord* rec, double* icov_d, float4* centroids, int* npts) {
  size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (r >= (size_t)*n_occ_ptr || !valid[r]) return;
  unsigned q = rank_of(valid_table, leaf_of_rank[r]);
  rec[q] = rec_in[r];
  for (int k = 0; k < 9; k++) icov_d[(size_t)q * 9 + k] = icov_in[r * 9 + k];
  centroids[q] = cen_in[r];
  npts[q] = npts_in[r];
}

bool VoxelMap::build(const float4* pts, size_t n, float leaf, int min_points_per_voxel, double min_covar_eigvalue_mult,
                     cudaStream_t s, const Bounds* known_bounds) {
  n_voxels = 0;
  n_occupied = 0;
  Bounds b;
  if (known_bounds) {  // the caller measured the cloud while uploading it (cloud_codec.cu): no extra pass, no round trip
    b = *known_bounds;
  } else {
    bounds_scratch.ensure(8);
    b = cloud_bounds(pts, n, bounds_scratch.ptr, s);
    launches += 1;
  }
  if (!b.any) return true;
  if (!make_grid_geom(b, leaf, geom)) {
    geom.n_cells = 0;
    geom.n_words = 0;
    return false;
  }
  // Everything below is enqueued without a single host round trip: buffers are sized by the upper bound
  // min(points, cells) on the occupied leaves, the kernels read the actual counts from device memory, and both counts
  // come back in ONE copy at the end.
  const size_t occ_max = (size_t)std::min<long long>((long long)n, geom.n_cells);
  index_all.ensure((size_t)geom.n_words);
  index.ensure((size_t)geom.n_words);
  cell_of_point.ensure(n);
  counts.ensure(2);
  h_counts.ensure(2);
  acc.ensure(occ_max * 10);
  leaf_of_rank.ensure(occ_max);
  tmp_records.ensure(occ_max);
  tmp_icov.ensure(occ_max * 9);
  tmp_centroids.ensure(occ_max);
  tmp_npts.ensure(occ_max);
  tmp_valid.ensure(occ_max);
  records.ensure(occ_max + 1);
  icov_d.ensure(occ_max * 9 + 9);
  centroids.ensure(occ_max + 1);
  npts.ensure(occ_max + 1);
  rank_index_clear(index_all.ptr, geom.n_words, s);
  rank_index_clear(index.ptr, geom.n_words, s);
  B200_CUDA(cudaMemsetAsync(acc.ptr, 0, sizeof(double) * occ_max * 10, s));
  const int blocks = (int)((n + 255) / 256);
  vm_mark_kernel<<<blocks, 256, 0, s>>>(pts, n, geom, index_all.ptr, cell_of_point.ptr);
  rank_index_scan_async(index_all.ptr, geom.n_words, scan_scratch, counts.ptr, s);
  vm_accumulate_kernel<<<blocks, 256, 0, s>>>(pts, n, cell_of_point.ptr, index_all.ptr, acc.ptr, leaf_of_rank.ptr);
  const int vblocks = (int)((occ_max + 127) / 128);
  vm_finalize_kernel<<<vblocks, 128, 0, s>>>(acc.ptr, leaf_of_rank.ptr, counts.ptr, min_points_per_voxel,
                                             min_covar_eigvalue_mult, tmp_records.ptr, tmp_icov.ptr, tmp_centroids.ptr,
                                             tmp_npts.ptr, tmp_valid.ptr, index.ptr);
  rank_index_scan_async(index.ptr, geom.n_words, scan_scratch, counts.ptr + 1, s);
  vm_compact_kernel<<<vblocks, 128, 0, s>>>(counts.ptr, tmp_valid.ptr, leaf_of_rank.ptr, index.ptr, tmp_records.ptr,
                                            tmp_icov.ptr, tmp_centroids.ptr, tmp_npts.ptr, records.ptr, icov_d.ptr,
                                            centroids.ptr, npts.ptr);
  launches += 11;
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(h_counts.ptr, counts.ptr, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  n_occupied = h_counts.ptr[0];
  n_voxels = h_counts.ptr[1];
  return true;
}

}  // namespace b200
