// K18: the elevation / traversability map of the session's submaps (b200sm_build_elevation_map). Every decision follows
// csrc/elevation_map.hpp, which a host compile also builds, so every layer is bitwise the host's. The cell statistics are
// integer minima, maxima and counts: the order of the atomics does not change them.
#include "common.cuh"
#include "elevation.cuh"

namespace b200 {
namespace {

constexpr int EL_THREADS = OG_THREADS, EL_PER_THREAD = OG_PER_THREAD;
constexpr int EL_HALO_PITCH = EL_TILE_X + 2 * EL_MAX_WINDOW;
constexpr int EL_HALO_ROWS = EL_TILE_Y + 2 * EL_MAX_WINDOW;

// the grid index of point i of entry e, false when the point is skipped; *bad when its cell lies outside the grid
__device__ __forceinline__ bool el_locate(const OgEntry& e, unsigned i, const ElConst& c, int gx0, int gy0, unsigned W, unsigned H,
                                          size_t* q, long long* Z, unsigned* bad) {
  const float4 p = e.cloud[i];
  float t[3];
  og_transform(e.T, p.x, p.y, p.z, t);
  int cx, cy;
  if (!el_point(c, e.xo, e.yo, t, &cx, &cy, Z)) return false;
  const unsigned x = (unsigned)(cx - gx0), y = (unsigned)(cy - gy0);
  if (x >= W || y >= H) {
    *bad = 1u;
    return false;
  }
  *q = (size_t)y * W + x;
  return true;
}

// K18a. Block b serves tile b (OgEntry::first_tile); a thread takes EL_PER_THREAD points of it.
__global__ void __launch_bounds__(EL_THREADS) el_lowest_kernel(const OgEntry* __restrict__ table, int n_entries, ElConst c, int gx0,
                                                               int gy0, unsigned W, unsigned H, uint32_t* __restrict__ n,
                                                               long long* __restrict__ lo, unsigned long long* __restrict__ counters) {
  const OgEntry& e = table[entry_of(table, n_entries, blockIdx.x, &OgEntry::first_tile)];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)OG_TILE + threadIdx.x;
  unsigned bad = 0;
  for (int j = 0; j < EL_PER_THREAD; j++) {
    const unsigned i = base + j * EL_THREADS;
    if (i >= e.n) break;
    size_t q;
    long long Z;
    if (!el_locate(e, i, c, gx0, gy0, W, H, &q, &Z, &bad)) continue;
    atomicAdd(&n[q], 1u);
    if (Z < lo[q]) atomicMin(&lo[q], Z);  // a stale read only costs an atomic: lo never rises
  }
  if (bad) atomicAdd(&counters[EL_CTR_TRIPPED], 1ull);
}

__device__ __forceinline__ long long warp_min64(long long v) {
  for (int o = 16; o; o >>= 1) {
    const long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w < v ? w : v;
  }
  return v;
}
__device__ __forceinline__ long long warp_max64(long long v) {
  for (int o = 16; o; o >>= 1) {
    const long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// K18b. The same tiles: the surface candidates raise top, the others are overhangs (one atomic per warp); the height extent
// is reduced per warp.
__global__ void __launch_bounds__(EL_THREADS) el_top_kernel(const OgEntry* __restrict__ table, int n_entries, ElConst c, int gx0,
                                                            int gy0, unsigned W, unsigned H, const long long* __restrict__ lo,
                                                            long long* __restrict__ top, unsigned long long* __restrict__ counters,
                                                            long long* __restrict__ zrange) {
  const OgEntry& e = table[entry_of(table, n_entries, blockIdx.x, &OgEntry::first_tile)];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)OG_TILE + threadIdx.x;
  unsigned bad = 0, over = 0;
  long long zmin = EL_LO_EMPTY, zmax = EL_TOP_EMPTY;
  for (int j = 0; j < EL_PER_THREAD; j++) {
    const unsigned i = base + j * EL_THREADS;
    if (i >= e.n) break;
    size_t q;
    long long Z;
    if (!el_locate(e, i, c, gx0, gy0, W, H, &q, &Z, &bad)) continue;
    zmin = Z < zmin ? Z : zmin;
    zmax = Z > zmax ? Z : zmax;
    if (Z > lo[q] + c.C) {
      over++;
    } else if (Z > top[q]) {
      atomicMax(&top[q], Z);
    }
  }
  over = __reduce_add_sync(0xffffffffu, over);
  zmin = warp_min64(zmin);
  zmax = warp_max64(zmax);
  if ((threadIdx.x & 31) == 0) {
    if (over) atomicAdd(&counters[EL_CTR_OVERHANG], (unsigned long long)over);
    if (zmin != EL_LO_EMPTY) {
      atomicMin(&zrange[0], zmin);
      atomicMax(&zrange[1], zmax);
    }
  }
  if (bad) atomicAdd(&counters[EL_CTR_TRIPPED], 1ull);
}

// K18c. Block b serves a 32 x 8 tile of cells (blocks row-major over the tiles); the tile and its window_cells halo of
// surface heights (EL_NONE where a cell is not observed or lies beyond the grid) are staged in shared memory, then each
// thread evaluates the window of its cell.
__global__ void __launch_bounds__(EL_TILE_X* EL_TILE_Y) el_window_kernel(ElConst c, unsigned W, unsigned H, unsigned tiles_x,
                                                                         const uint32_t* __restrict__ n,
                                                                         const long long* __restrict__ top, float* __restrict__ step,
                                                                         float* __restrict__ tan_slope, float* __restrict__ roughness,
                                                                         signed char* __restrict__ value, unsigned char* __restrict__ image,
                                                                         unsigned long long* __restrict__ counters) {
  __shared__ long long sh[EL_HALO_ROWS * EL_HALO_PITCH];
  const int r = c.r, pitch = EL_TILE_X + 2 * r, rows = EL_TILE_Y + 2 * r;
  const long long x0 = (long long)(blockIdx.x % tiles_x) * EL_TILE_X, y0 = (long long)(blockIdx.x / tiles_x) * EL_TILE_Y;
  const int tid = threadIdx.y * EL_TILE_X + threadIdx.x;
  for (int k = tid; k < pitch * rows; k += EL_TILE_X * EL_TILE_Y) {
    const long long gx = x0 - r + k % pitch, gy = y0 - r + k / pitch;
    long long h = EL_NONE;
    if (gx >= 0 && gy >= 0 && gx < W && gy < H) {
      const size_t q = (size_t)gy * W + (size_t)gx;
      if (n[q] >= (unsigned)c.min_points) h = top[q];
    }
    sh[k] = h;
  }
  __syncthreads();
  const long long x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  unsigned obs = 0, lethal = 0, trav = 0, unk = 0;
  if (x < W && y < H) {
    const long long* centre = sh + (threadIdx.y + r) * pitch + threadIdx.x + r;
    float s, t, g;
    const int v = el_window(c, [&](int du, int dv) { return centre[dv * pitch + du]; }, &s, &t, &g);
    const size_t q = (size_t)y * W + (size_t)x;
    step[q] = s;
    tan_slope[q] = t;
    roughness[q] = g;
    value[q] = (signed char)v;
    image[(size_t)(H - 1 - y) * W + (size_t)x] = og_pixel(v, c.og.occ_value, c.og.free_value);
    obs = centre[0] != EL_NONE;
    lethal = v == 100;
    trav = v >= 0 && v < 100;
    unk = v < 0;
  }
  obs = __reduce_add_sync(0xffffffffu, obs);
  lethal = __reduce_add_sync(0xffffffffu, lethal);
  trav = __reduce_add_sync(0xffffffffu, trav);
  unk = __reduce_add_sync(0xffffffffu, unk);
  if (threadIdx.x == 0) {
    if (obs) atomicAdd(&counters[EL_CTR_OBSERVED], (unsigned long long)obs);
    if (lethal) atomicAdd(&counters[EL_CTR_LETHAL], (unsigned long long)lethal);
    if (trav) atomicAdd(&counters[EL_CTR_TRAVERSABLE], (unsigned long long)trav);
    if (unk) atomicAdd(&counters[EL_CTR_UNKNOWN], (unsigned long long)unk);
  }
}

}  // namespace

void el_lowest_launch(const OgEntry* table, int n_entries, unsigned tiles, const ElConst& c, int gx0, int gy0, unsigned W, unsigned H,
                      uint32_t* n, long long* lo, unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  el_lowest_kernel<<<tiles, EL_THREADS, 0, stream>>>(table, n_entries, c, gx0, gy0, W, H, n, lo, counters);
  B200_CUDA(cudaGetLastError());
}

void el_top_launch(const OgEntry* table, int n_entries, unsigned tiles, const ElConst& c, int gx0, int gy0, unsigned W, unsigned H,
                   const long long* lo, long long* top, unsigned long long* counters, long long* zrange, cudaStream_t stream) {
  if (tiles == 0) return;
  el_top_kernel<<<tiles, EL_THREADS, 0, stream>>>(table, n_entries, c, gx0, gy0, W, H, lo, top, counters, zrange);
  B200_CUDA(cudaGetLastError());
}

void el_window_launch(const ElConst& c, unsigned W, unsigned H, const uint32_t* n, const long long* top, float* step, float* tan_slope,
                      float* roughness, signed char* value, unsigned char* image, unsigned long long* counters, cudaStream_t stream) {
  const unsigned tiles_x = (W + EL_TILE_X - 1) / EL_TILE_X;
  const unsigned long long blocks = (unsigned long long)tiles_x * ((H + EL_TILE_Y - 1) / EL_TILE_Y);
  if (blocks == 0) return;
  el_window_kernel<<<(unsigned)blocks, dim3(EL_TILE_X, EL_TILE_Y), 0, stream>>>(c, W, H, tiles_x, n, top, step, tan_slope, roughness,
                                                                               value, image, counters);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
