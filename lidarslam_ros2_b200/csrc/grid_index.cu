// The pipeline the target-side builders share — the voxel map (K3, voxel_map.cu), VoxelGrid (K4, voxelgrid.cu) and the
// NN grid (K6/K8, nn_grid.cu): bounds of the cloud, PCL grid geometry, the occupancy bitmap and its exclusive scan into a
// rank index. The device helpers they share are in grid_index.cuh.
#include <cfloat>
#include <cmath>

#include "engine.hpp"
#include "grid_index.cuh"

namespace b200 {

namespace {

// ---- exclusive scan -------------------------------------------------------------------------------------------------
// Three launches: tile-local scans, one block scans the tile sums (and writes the total), then the tile offsets are
// added back (skipped for a single tile). Io says what is scanned: count(i) is element i's value, out(i) where its
// exclusive prefix goes.
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;  // elements per thread
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

struct RankWordIo {  // popc(bits) -> prefix
  RankWord* t;
  __device__ unsigned count(size_t i) const { return __popc(t[i].bits); }
  __device__ unsigned& out(size_t i) const { return t[i].prefix; }
};
struct CounterIo {  // u32 counters, scanned in place
  unsigned* d;
  __device__ unsigned count(size_t i) const { return d[i]; }
  __device__ unsigned& out(size_t i) const { return d[i]; }
};

template <typename Io>
__global__ void __launch_bounds__(SCAN_THREADS) scan_local_kernel(Io io, size_t n, unsigned* tile_sums) {
  __shared__ unsigned warp_tot[SCAN_THREADS / 32];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  unsigned v[SCAN_ITEMS], local = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    v[k] = (base + k < n) ? io.count(base + k) : 0u;
    local += v[k];
  }
  // warp inclusive scan of `local`
  unsigned incl = local;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    unsigned t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned off = 0;
  for (int w = 0; w < warp; w++) off += warp_tot[w];
  unsigned run = off + incl - local;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    if (base + k < n) io.out(base + k) = run;
    run += v[k];
  }
  if (threadIdx.x == SCAN_THREADS - 1) tile_sums[blockIdx.x] = run;
}

// single block: exclusive scan of tile_sums in place, grand total to *total
__global__ void __launch_bounds__(1024) scan_tile_sums_kernel(unsigned* tile_sums, int n_tiles, unsigned* total) {
  __shared__ unsigned warp_tot[32];
  __shared__ unsigned carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n_tiles; base += 1024) {
    int i = base + threadIdx.x;
    unsigned v = (i < n_tiles) ? tile_sums[i] : 0u;
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
    if (i < n_tiles) tile_sums[i] = carry + off + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + off + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry_s;
}

template <typename Io>
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(Io io, size_t n, const unsigned* tile_sums) {
  const unsigned off = tile_sums[blockIdx.x];
  const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++)
    if (base + k < n) io.out(base + k) += off;
}

template <typename Io>
void exclusive_scan_async(Io io, size_t n, DeviceBuffer<unsigned>& tile_sums, unsigned* d_total, cudaStream_t s) {
  const int n_tiles = (int)((n + SCAN_TILE - 1) / SCAN_TILE);
  tile_sums.ensure((size_t)n_tiles + 1);
  scan_local_kernel<<<n_tiles, SCAN_THREADS, 0, s>>>(io, n, tile_sums.ptr);
  scan_tile_sums_kernel<<<1, 1024, 0, s>>>(tile_sums.ptr, n_tiles, d_total);
  if (n_tiles > 1) scan_apply_kernel<<<n_tiles, SCAN_THREADS, 0, s>>>(io, n, tile_sums.ptr);
}

// ---- bounds, marking ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bounds_kernel(const float4* __restrict__ pts, size_t n, unsigned* out6) {
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float4 p = pts[i];
    if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) continue;
    mn[0] = fminf(mn[0], p.x); mn[1] = fminf(mn[1], p.y); mn[2] = fminf(mn[2], p.z);
    mx[0] = fmaxf(mx[0], p.x); mx[1] = fmaxf(mx[1], p.y); mx[2] = fmaxf(mx[2], p.z);
  }
  block_bounds_merge(mn, mx, out6);
}

__global__ void __launch_bounds__(256) mark_cells_kernel(const float4* __restrict__ pts, size_t n, GridGeom g, RankWord* table,
                                                         int* cell_of_point, int shift) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = pts[i];
  int cell = -1;
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    cell = build_leaf_index(g, p.x, p.y, p.z);
    if (cell < 0 || cell >= g.n_cells) cell = -1;  // cannot happen for finite points inside the bounds
  }
  cell_of_point[i] = cell;
  if (cell >= 0) mark_occupied(table, cell >> shift);
}

}  // namespace

void rank_index_clear(RankWord* table, int n_words, cudaStream_t s) {
  B200_CUDA(cudaMemsetAsync(table, 0, sizeof(RankWord) * (size_t)n_words, s));
}

void rank_index_scan_async(RankWord* table, size_t n_words, RankIndexScratch& scratch, unsigned* d_total, cudaStream_t s) {
  exclusive_scan_async(RankWordIo{table}, n_words, scratch.block_sums, d_total, s);
}

void counter_scan_async(unsigned* data, size_t n, DeviceBuffer<unsigned>& tile_sums, cudaStream_t s) {
  exclusive_scan_async(CounterIo{data}, n, tile_sums, data + n, s);
}

void mark_grid_cells(const float4* pts, size_t n, const GridGeom& g, RankWord* table, int* cell_of_point, int shift,
                     cudaStream_t s) {
  mark_cells_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(pts, n, g, table, cell_of_point, shift);
}

Bounds decode_bounds(const unsigned* res6) {
  Bounds b;
  for (int a = 0; a < 3; a++) {
    b.mn[a] = ordered_to_float(res6[a]);
    b.mx[a] = ordered_to_float(res6[3 + a]);
  }
  // no finite point: either initial value is still there — the upload's {0xffffffff, 0} (both decode to NaN) or
  // cloud_bounds' inverted {FLT_MAX, -FLT_MAX} — and min <= max fails
  b.any = b.mn[0] <= b.mx[0];
  return b;
}

Bounds cloud_bounds(const float4* pts, size_t n, unsigned* d_scratch8, cudaStream_t s) {
  // min = FLT_MAX, max = -FLT_MAX: a cloud without a finite point comes back with exactly these (inverted) bounds
  unsigned init[6];
  for (int a = 0; a < 3; a++) {
    init[a] = 0xff7fffffu;      // float_to_ordered(FLT_MAX)
    init[3 + a] = 0x00800000u;  // float_to_ordered(-FLT_MAX)
  }
  B200_CUDA(cudaMemcpyAsync(d_scratch8, init, sizeof(init), cudaMemcpyHostToDevice, s));
  int blocks = (int)std::min<size_t>((n + 255) / 256, H100_SMS * 8);
  if (blocks < 1) blocks = 1;
  bounds_kernel<<<blocks, 256, 0, s>>>(pts, n, d_scratch8);
  unsigned res[6];
  B200_CUDA(cudaMemcpyAsync(res, d_scratch8, sizeof(res), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  return decode_bounds(res);
}

Bounds grid_bounds(const float4* pts, size_t n, const Bounds* known_bounds, DeviceBuffer<unsigned>& scratch, int& launches,
                   cudaStream_t s) {
  if (known_bounds) return *known_bounds;  // measured while the cloud was uploaded (cloud_codec.cu): no pass, no round trip
  scratch.ensure(8);
  launches += 1;
  return cloud_bounds(pts, n, scratch.ptr, s);
}

bool make_grid_geom(const Bounds& b, float leaf, GridGeom& g) {
  g.leaf = leaf;
  g.inv_leaf = 1.0f / leaf;
  // voxel_grid_covariance_omp_impl.hpp:75-84 — float products, int64 casts, dx * dy * dz > INT32_MAX refused. A float
  // product of 2^31 or more (inf for a range near FLT_MAX), or a bound whose leaf index is not an int, already means
  // overflow: refusing it first keeps the casts defined (the reference's would not be), and dx * dy cannot wrap.
  constexpr float kIntLimit = 2147483648.0f;
  long long d[3];
  for (int a = 0; a < 3; a++) {
    const float p = (b.mx[a] - b.mn[a]) * g.inv_leaf;
    if (!(p < kIntLimit) || !(std::fabs(b.mn[a] * g.inv_leaf) < kIntLimit) || !(std::fabs(b.mx[a] * g.inv_leaf) < kIntLimit))
      return false;
    d[a] = static_cast<long long>(p) + 1;
  }
  if (d[0] * d[1] > static_cast<long long>(INT32_MAX) || d[0] * d[1] * d[2] > static_cast<long long>(INT32_MAX)) return false;
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

}  // namespace b200
