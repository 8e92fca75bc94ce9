// K14: the occupancy grid of the session's submaps (b200sm_build_occupancy_grid). Every decision follows
// csrc/occupancy_grid.hpp, which a host compile also builds, so the counts, values and image are bitwise the host's. Counts
// are integers of per-submap booleans: neither the order of the atomics nor the batching changes them.
#include "common.cuh"
#include "occupancy.cuh"

namespace b200 {
namespace {

__device__ __forceinline__ OgConst og_const(double S, long long R, long long zlo, long long zhi) {
  OgConst c;
  c.S = S;
  c.R = R;
  c.zlo = zlo;
  c.zhi = zhi;
  c.occ_value = c.free_value = 0;
  return c;
}

// K14a. Block b serves tile b; a thread takes OG_PER_THREAD points of it. Each warp reduces its endpoint cells and counts,
// then one lane per warp widens the entry's bounds with atomicMin / atomicMax.
__global__ void __launch_bounds__(OG_THREADS) og_bounds_kernel(const OgEntry* __restrict__ table, int n_entries, double S, long long R,
                                                               long long zlo, long long zhi, int* __restrict__ bounds,
                                                               unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &OgEntry::first_tile);
  const OgEntry& e = table[k];
  const OgConst c = og_const(S, R, zlo, zhi);
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)OG_TILE + threadIdx.x;
  int x0 = INT_MAX, y0 = INT_MAX, x1 = INT_MIN, y1 = INT_MIN;
  unsigned rays = 0, skipped = 0;
  for (int j = 0; j < OG_PER_THREAD; j++) {
    const unsigned i = base + j * OG_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int hx, hy;
    OgSeg s;
    if (og_ray(c, e.xo, e.yo, e.zo, q[0], q[1], q[2], &hx, &hy, &s) < 0) {
      skipped++;
      continue;
    }
    rays++;
    x0 = min(x0, hx);
    y0 = min(y0, hy);
    x1 = max(x1, hx);
    y1 = max(y1, hy);
  }
  x0 = __reduce_min_sync(0xffffffffu, x0);
  y0 = __reduce_min_sync(0xffffffffu, y0);
  x1 = __reduce_max_sync(0xffffffffu, x1);
  y1 = __reduce_max_sync(0xffffffffu, y1);
  rays = __reduce_add_sync(0xffffffffu, rays);
  skipped = __reduce_add_sync(0xffffffffu, skipped);
  if ((threadIdx.x & 31) == 0) {
    if (rays) {
      atomicMin(&bounds[4 * k + 0], x0);
      atomicMin(&bounds[4 * k + 1], y0);
      atomicMax(&bounds[4 * k + 2], x1);
      atomicMax(&bounds[4 * k + 3], y1);
      atomicAdd(&counters[OG_CTR_RAYS], (unsigned long long)rays);
    }
    if (skipped) atomicAdd(&counters[OG_CTR_SKIPPED], (unsigned long long)skipped);
  }
}

// set bit (cx, cy) of a bitmap, reading first: most rays of a submap cross the same cells near its origin, and a bit that
// is already set needs no atomic
__device__ __forceinline__ void og_mark(uint32_t* words, unsigned stride, int x0, int y0, unsigned width, unsigned height, int cx,
                                        int cy, unsigned* tripped) {
  const unsigned wx = (unsigned)(cx - x0), wy = (unsigned)(cy - y0);
  if (wx >= width || wy >= height) {
    *tripped = 1u;
    return;
  }
  uint32_t* w = words + (size_t)wy * stride + (wx >> 5);
  const uint32_t bit = 1u << (wx & 31u);
  if (!(*w & bit)) atomicOr(w, bit);
}

// K14b. Block b serves tile b; thread t casts the rays of OG_PER_THREAD points: the endpoint's cell into the hit bitmap when
// it is in the band, every cell of the clipped segment's walk into the free bitmap.
__global__ void __launch_bounds__(OG_THREADS) og_walk_kernel(const OgEntry* __restrict__ table, int n_entries, double S, long long R,
                                                             long long zlo, long long zhi, uint32_t* __restrict__ scratch,
                                                             unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &OgEntry::first_tile);
  const OgEntry& e = table[k];
  const OgConst c = og_const(S, R, zlo, zhi);
  const int x0 = e.x0, y0 = e.y0;
  const unsigned width = e.width, height = e.height, stride = e.stride;
  uint32_t* hit = scratch + e.words_at;
  uint32_t* fre = hit + (size_t)stride * e.rows;
  unsigned tripped = 0;
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)OG_TILE + threadIdx.x;
  for (int j = 0; j < OG_PER_THREAD; j++) {
    const unsigned i = base + j * OG_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int hx, hy;
    OgSeg s;
    const int f = og_ray(c, e.xo, e.yo, e.zo, q[0], q[1], q[2], &hx, &hy, &s);
    if (f < 0) continue;
    if (f & 1) og_mark(hit, stride, x0, y0, width, height, hx, hy, &tripped);
    if (f & 2) og_walk(s, [&](int cx, int cy) { og_mark(fre, stride, x0, y0, width, height, cx, cy, &tripped); });
  }
  if (tripped) atomicAdd(&counters[OG_CTR_TRIPPED], 1ull);
}

// K14c. Thread g takes hit-bitmap word g of the batch (entry: the last with fold_first <= g) and the free word beside it;
// each hit bit adds one to `hits`, each free bit without a hit one to `frees`.
__global__ void __launch_bounds__(OG_THREADS) og_fold_kernel(const OgEntry* __restrict__ table, int n_entries, unsigned long long fold_words,
                                                             const uint32_t* __restrict__ scratch, int gx0, int gy0, unsigned width,
                                                             uint32_t* __restrict__ hits, uint32_t* __restrict__ frees) {
  const unsigned long long g = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (g >= fold_words) return;
  const OgEntry& e = table[entry_of(table, n_entries, g, &OgEntry::fold_first)];
  const unsigned long long w = g - e.fold_first;
  const uint32_t h = scratch[e.words_at + w];
  const uint32_t f = scratch[e.words_at + (unsigned long long)e.stride * e.rows + w] & ~h;
  if (!(h | f)) return;
  const unsigned row = (unsigned)(w / e.stride), col = (unsigned)(w % e.stride) * 32u;
  const size_t line = (size_t)(e.y0 + (int)row - gy0) * width + (size_t)(e.x0 - gx0) + col;
  for (uint32_t m = h; m; m &= m - 1) atomicAdd(&hits[line + __ffs(m) - 1], 1u);
  for (uint32_t m = f; m; m &= m - 1) atomicAdd(&frees[line + __ffs(m) - 1], 1u);
}

// K14d. One thread per cell (grid-stride): value, the image byte at the flipped row, and the three counts (warp sums, one
// atomic per warp and count).
__global__ void __launch_bounds__(OG_THREADS) og_classify_kernel(const uint32_t* __restrict__ hits, const uint32_t* __restrict__ frees,
                                                                 unsigned width, unsigned height, int occ_value, int free_value,
                                                                 signed char* __restrict__ values, unsigned char* __restrict__ image,
                                                                 unsigned long long* __restrict__ counters) {
  const unsigned long long cells = (unsigned long long)width * height;
  unsigned occ = 0, fre = 0, unk = 0;
  for (unsigned long long q = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; q < cells;
       q += (unsigned long long)gridDim.x * blockDim.x) {
    const int v = og_value(hits[q], frees[q]);
    const unsigned char px = og_pixel(v, occ_value, free_value);
    const unsigned long long y = q / width, x = q - y * width;
    values[q] = (signed char)v;
    image[(height - 1 - y) * width + x] = px;
    unk += v < 0;
    occ += v >= 0 && px == 0;
    fre += v >= 0 && px == 254;
  }
  occ = __reduce_add_sync(0xffffffffu, occ);
  fre = __reduce_add_sync(0xffffffffu, fre);
  unk = __reduce_add_sync(0xffffffffu, unk);
  if ((threadIdx.x & 31) == 0) {
    if (occ) atomicAdd(&counters[OG_CTR_OCCUPIED], (unsigned long long)occ);
    if (fre) atomicAdd(&counters[OG_CTR_FREE], (unsigned long long)fre);
    if (unk) atomicAdd(&counters[OG_CTR_UNKNOWN], (unsigned long long)unk);
  }
}

}  // namespace

void og_bounds_launch(const OgEntry* table, int n_entries, unsigned tiles, const OgConst& c, int* bounds, unsigned long long* counters,
                      cudaStream_t stream) {
  if (tiles == 0) return;
  og_bounds_kernel<<<tiles, OG_THREADS, 0, stream>>>(table, n_entries, c.S, c.R, c.zlo, c.zhi, bounds, counters);
  B200_CUDA(cudaGetLastError());
}

void og_walk_launch(const OgEntry* table, int n_entries, unsigned tiles, const OgConst& c, uint32_t* scratch,
                    unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  og_walk_kernel<<<tiles, OG_THREADS, 0, stream>>>(table, n_entries, c.S, c.R, c.zlo, c.zhi, scratch, counters);
  B200_CUDA(cudaGetLastError());
}

void og_fold_launch(const OgEntry* table, int n_entries, unsigned long long fold_words, const uint32_t* scratch, int gx0, int gy0,
                    unsigned width, uint32_t* hits, uint32_t* frees, cudaStream_t stream) {
  if (fold_words == 0) return;
  const unsigned long long blocks = (fold_words + OG_THREADS - 1) / OG_THREADS;
  og_fold_kernel<<<(unsigned)blocks, OG_THREADS, 0, stream>>>(table, n_entries, fold_words, scratch, gx0, gy0, width, hits, frees);
  B200_CUDA(cudaGetLastError());
}

void og_classify_launch(const uint32_t* hits, const uint32_t* frees, unsigned width, unsigned height, int occ_value, int free_value,
                        signed char* values, unsigned char* image, unsigned long long* counters, cudaStream_t stream) {
  const unsigned long long cells = (unsigned long long)width * height;
  const unsigned long long want = (cells + OG_THREADS - 1) / OG_THREADS;
  const unsigned blocks = (unsigned)(want < 16ull * H100_SMS ? want : 16ull * H100_SMS);
  og_classify_kernel<<<blocks, OG_THREADS, 0, stream>>>(hits, frees, width, height, occ_value, free_value, values, image, counters);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
