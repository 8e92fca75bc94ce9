// K15: the static map of the session's submaps (b200sm_build_static_map). Every decision follows csrc/static_map.hpp,
// which a host compile also builds, so the counts, flags and the static map are bitwise the host's. Counts are integers
// of per-submap booleans: neither the order of the atomics nor the batching changes them.
#include <climits>

#include "grid_index.cuh"
#include "static_map.cuh"

namespace b200 {
namespace {

// set bit r of a bitmap of n_voxels bits, reading first: the rays of a submap cross the voxels near its origin over and over,
// and a bit that is already set needs no atomic
__device__ __forceinline__ void sm_set(uint32_t* bits, unsigned r, unsigned n_voxels, unsigned* tripped) {
  if (r >= n_voxels) {
    *tripped = 1u;
    return;
  }
  uint32_t* w = bits + (r >> 5);
  const uint32_t bit = 1u << (r & 31u);
  if (!(*w & bit)) atomicOr(w, bit);
}

// K15a. Block b serves tile b; a thread takes SM_PER_THREAD points of it. Each warp reduces its endpoint voxels and counts,
// then one lane per warp widens the entry's bounds with atomicMin / atomicMax.
__global__ void __launch_bounds__(SM_THREADS) sm_bounds_kernel(const SmEntry* __restrict__ table, int n_entries, SmConst c,
                                                               int* __restrict__ bounds, unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  unsigned rays = 0, skipped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int v[3];
    long long f[3];
    if (!sm_ray(c, e.o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) {
      skipped++;
      continue;
    }
    rays++;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      lo[a] = min(lo[a], v[a]);
      hi[a] = max(hi[a], v[a]);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
    hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
  }
  rays = __reduce_add_sync(0xffffffffu, rays);
  skipped = __reduce_add_sync(0xffffffffu, skipped);
  if ((threadIdx.x & 31) == 0) {
    if (rays) {
#pragma unroll
      for (int a = 0; a < 3; a++) {
        atomicMin(&bounds[6 * k + a], lo[a]);
        atomicMax(&bounds[6 * k + 3 + a], hi[a]);
      }
      atomicAdd(&counters[SM_CTR_RAYS], (unsigned long long)rays);
    }
    if (skipped) atomicAdd(&counters[SM_CTR_SKIPPED], (unsigned long long)skipped);
  }
}

// K15b. The endpoint voxel of every ray into the rank index.
__global__ void __launch_bounds__(SM_THREADS) sm_mark_kernel(const SmEntry* __restrict__ table, int n_entries, SmConst c, SmBox box,
                                                             RankWord* __restrict__ index, unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  unsigned tripped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int v[3];
    long long f[3];
    if (!sm_ray(c, e.o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) continue;
    unsigned lin;
    if (!sm_lin(box, v[0], v[1], v[2], &lin)) {
      tripped = 1u;
      continue;
    }
    mark_occupied(index, (int)lin);
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

// K15c. Block b serves tile b of the batch; thread t casts the rays of SM_PER_THREAD points: the endpoint's rank into its
// submap's hit bitmap, the rank of every occupied voxel of the box on the freed segment's walk into the free bitmap.
__global__ void __launch_bounds__(SM_THREADS) sm_walk_kernel(const SmEntry* __restrict__ table, int n_entries, SmConst c, SmBox box,
                                                             const RankWord* __restrict__ index, unsigned n_voxels,
                                                             unsigned long long words_per, uint32_t* __restrict__ scratch,
                                                             unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::batch_tile);
  const SmEntry& e = table[k];
  uint32_t* hit = scratch + 2ull * (unsigned long long)k * words_per;
  uint32_t* fre = hit + words_per;
  unsigned tripped = 0;
  const unsigned base = (blockIdx.x - e.batch_tile) * (unsigned)SM_TILE + threadIdx.x;
  const long long* o = e.o;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int v[3];
    long long f[3];
    if (!sm_ray(c, o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) continue;
    unsigned r;
    if (sm_rank(index, box, v[0], v[1], v[2], &r)) sm_set(hit, r, n_voxels, &tripped);
    else tripped = 1u;
    sm_walk(o[0], o[1], o[2], f[0], f[1], f[2], [&](int x, int y, int z) {
      unsigned rw;
      if (sm_rank(index, box, x, y, z, &rw)) sm_set(fre, rw, n_voxels, &tripped);
    });
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

// K15d. One thread per bitmap word (32 voxels): the word of every submap of the batch, read once (a warp reads 128
// consecutive bytes per bitmap), added into bit-sliced counters — plane p holds bit p of each of the 32 voxels' counts,
// and adding a word is a ripple carry through the planes. Every SM_FOLD_CHUNK submaps (the most SM_FOLD_PLANES planes
// can count) the counts are added to hits / frees and the planes cleared. A voxel's counts are touched by this thread
// only, so there are no atomics.
constexpr int SM_FOLD_PLANES = 10, SM_FOLD_CHUNK = (1 << SM_FOLD_PLANES) - 1;

__device__ __forceinline__ void sm_fold_add(uint32_t (&plane)[SM_FOLD_PLANES], uint32_t x) {
#pragma unroll
  for (int p = 0; p < SM_FOLD_PLANES; p++) {
    const uint32_t carry = plane[p] & x;
    plane[p] ^= x;
    x = carry;
  }
}

__device__ __forceinline__ void sm_fold_flush(uint32_t (&plane)[SM_FOLD_PLANES], uint32_t* __restrict__ counts, unsigned v0,
                                              unsigned n_voxels) {
  uint32_t any = 0;
#pragma unroll
  for (int p = 0; p < SM_FOLD_PLANES; p++) any |= plane[p];
  for (uint32_t m = any; m; m &= m - 1) {
    const unsigned b = (unsigned)__ffs(m) - 1u;
    unsigned c = 0;
#pragma unroll
    for (int p = 0; p < SM_FOLD_PLANES; p++) c |= ((plane[p] >> b) & 1u) << p;
    if (v0 + b < n_voxels) counts[v0 + b] += c;  // bits beyond n_voxels are never set; the guard bounds the store
  }
#pragma unroll
  for (int p = 0; p < SM_FOLD_PLANES; p++) plane[p] = 0;
}

__global__ void __launch_bounds__(SM_THREADS) sm_fold_kernel(const uint32_t* __restrict__ scratch, int n_entries,
                                                             unsigned long long words_per, unsigned n_voxels, uint32_t* __restrict__ hits,
                                                             uint32_t* __restrict__ frees) {
  const unsigned long long w = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (w >= words_per) return;
  uint32_t hp[SM_FOLD_PLANES], fp[SM_FOLD_PLANES];
#pragma unroll
  for (int p = 0; p < SM_FOLD_PLANES; p++) hp[p] = fp[p] = 0;
  const unsigned v0 = (unsigned)(w * 32ull);
  for (int k0 = 0; k0 < n_entries; k0 += SM_FOLD_CHUNK) {
    const int k1 = min(n_entries, k0 + SM_FOLD_CHUNK);
    for (int k = k0; k < k1; k++) {
      const uint32_t h = __ldg(scratch + 2ull * (unsigned long long)k * words_per + w);
      const uint32_t f = __ldg(scratch + (2ull * (unsigned long long)k + 1ull) * words_per + w) & ~h;
      if (h) sm_fold_add(hp, h);
      if (f) sm_fold_add(fp, f);
    }
    sm_fold_flush(hp, hits, v0, n_voxels);
    sm_fold_flush(fp, frees, v0, n_voxels);
  }
}

// K15e. One thread per voxel (grid-stride): the flag, and the dynamic count (a warp sum, one atomic per warp).
__global__ void __launch_bounds__(SM_THREADS) sm_classify_kernel(const uint32_t* __restrict__ hits, const uint32_t* __restrict__ frees,
                                                                 unsigned n_voxels, unsigned min_frees, int dyn_value,
                                                                 unsigned char* __restrict__ dynamic,
                                                                 unsigned long long* __restrict__ counters) {
  unsigned n = 0;
  for (unsigned long long v = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; v < n_voxels;
       v += (unsigned long long)gridDim.x * blockDim.x) {
    const bool d = sm_dynamic(hits[v], frees[v], min_frees, dyn_value);
    dynamic[v] = d ? 1 : 0;
    n += d;
  }
  n = __reduce_add_sync(0xffffffffu, n);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(&counters[SM_CTR_DYNAMIC], (unsigned long long)n);
}

// whether the static map keeps point p of entry e; *out = the point moved by the entry's pose (assemble_map's point)
__device__ __forceinline__ bool sm_keep(const SmEntry& e, const SmConst& c, const SmBox& box, const RankWord* __restrict__ index,
                                        const unsigned char* __restrict__ dynamic, unsigned n_voxels, float4 p, float4* out) {
  float q[3];
  og_transform(e.T, p.x, p.y, p.z, q);
  *out = make_float4(q[0], q[1], q[2], p.w);
  int v[3];
  long long f[3];
  if (!sm_ray(c, e.o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) return true;
  unsigned r;
  if (!sm_rank(index, box, v[0], v[1], v[2], &r) || r >= n_voxels) return true;
  return !dynamic[r];
}

// K15f / K15g share the walk over a tile: round j of a tile is its points j * SM_THREADS .. + SM_THREADS - 1, one per thread
// in thread order, so (round, warp, lane) is the assembled map's order within the tile.
template <bool kWrite>
__global__ void __launch_bounds__(SM_THREADS) sm_compact_kernel(const SmEntry* __restrict__ table, int n_entries, SmConst c, SmBox box,
                                                                const RankWord* __restrict__ index, const unsigned char* __restrict__ dynamic,
                                                                unsigned n_voxels, unsigned* __restrict__ counts,
                                                                const unsigned* __restrict__ tile_offsets, unsigned total,
                                                                float4* __restrict__ out, unsigned long long* __restrict__ counters) {
  constexpr int W = SM_THREADS / 32;
  __shared__ unsigned warp_count[SM_PER_THREAD][W];
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  float4 q[SM_PER_THREAD];
  unsigned mask[SM_PER_THREAD];
#pragma unroll
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    bool keep = false;
    q[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < e.n) keep = sm_keep(e, c, box, index, dynamic, n_voxels, e.cloud[i], &q[j]);
    mask[j] = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_count[j][warp] = (unsigned)__popc(mask[j]);
  }
  __syncthreads();
  if (!kWrite) {
    if (threadIdx.x == 0) {
      unsigned t = 0;
      for (int j = 0; j < SM_PER_THREAD; j++)
        for (int w = 0; w < W; w++) t += warp_count[j][w];
      counts[blockIdx.x] = t;
    }
    return;
  }
  unsigned dst = tile_offsets[blockIdx.x];
  unsigned tripped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    unsigned before = 0, round = 0;
    for (int w = 0; w < W; w++) {
      before += w < warp ? warp_count[j][w] : 0u;
      round += warp_count[j][w];
    }
    if ((mask[j] >> lane) & 1u) {
      const unsigned at = dst + before + (unsigned)__popc(mask[j] & ((1u << lane) - 1u));
      if (at < total) out[at] = q[j];
      else tripped = 1u;
    }
    dst += round;
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

__global__ void __launch_bounds__(SM_THREADS) sm_voxel_list_kernel(const RankWord* __restrict__ index, unsigned long long n_words, SmBox box,
                                                                   unsigned n_voxels, int* __restrict__ ijk) {
  const unsigned long long w = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  const RankWord rw = index[w];
  const unsigned long long plane = (unsigned long long)box.dims[0] * box.dims[1];
  for (uint32_t m = rw.bits; m; m &= m - 1) {
    const unsigned bit = (unsigned)__ffs(m) - 1u;
    const unsigned r = rw.prefix + (unsigned)__popc(rw.bits & ((1u << bit) - 1u));
    if (r >= n_voxels) return;
    const unsigned long long lin = w * 32ull + bit;
    const unsigned long long z = lin / plane, rem = lin - z * plane, y = rem / box.dims[0], x = rem - y * box.dims[0];
    ijk[3ull * r + 0] = box.lo[0] + (int)x;
    ijk[3ull * r + 1] = box.lo[1] + (int)y;
    ijk[3ull * r + 2] = box.lo[2] + (int)z;
  }
}

unsigned blocks_for(unsigned long long n) { return (unsigned)((n + SM_THREADS - 1) / SM_THREADS); }

}  // namespace

void sm_bounds_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, int* bounds, unsigned long long* counters,
                      cudaStream_t stream) {
  if (tiles == 0) return;
  sm_bounds_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, bounds, counters);
  B200_CUDA(cudaGetLastError());
}

void sm_mark_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, RankWord* index,
                    unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  sm_mark_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, counters);
  B200_CUDA(cudaGetLastError());
}

void sm_walk_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                    unsigned n_voxels, unsigned long long words_per, uint32_t* scratch, unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  sm_walk_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, n_voxels, words_per, scratch, counters);
  B200_CUDA(cudaGetLastError());
}

void sm_fold_launch(const uint32_t* scratch, int n_entries, unsigned long long words_per, unsigned n_voxels, uint32_t* hits,
                    uint32_t* frees, cudaStream_t stream) {
  if (n_voxels == 0 || n_entries == 0) return;
  sm_fold_kernel<<<blocks_for(words_per), SM_THREADS, 0, stream>>>(scratch, n_entries, words_per, n_voxels, hits, frees);
  B200_CUDA(cudaGetLastError());
}

void sm_classify_launch(const uint32_t* hits, const uint32_t* frees, unsigned n_voxels, const SmConst& c, unsigned char* dynamic,
                        unsigned long long* counters, cudaStream_t stream) {
  if (n_voxels == 0) return;
  const unsigned want = blocks_for(n_voxels);
  const unsigned blocks = want < 16u * H100_SMS ? want : 16u * H100_SMS;
  sm_classify_kernel<<<blocks, SM_THREADS, 0, stream>>>(hits, frees, n_voxels, c.min_frees, c.dyn_value, dynamic, counters);
  B200_CUDA(cudaGetLastError());
}

void sm_count_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                     const unsigned char* dynamic, unsigned n_voxels, unsigned* counts, cudaStream_t stream) {
  if (tiles == 0) return;
  sm_compact_kernel<false><<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, dynamic, n_voxels, counts, nullptr, 0u,
                                                            nullptr, nullptr);
  B200_CUDA(cudaGetLastError());
}

void sm_write_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                     const unsigned char* dynamic, unsigned n_voxels, const unsigned* tile_offsets, unsigned total, float4* out,
                     unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  sm_compact_kernel<true><<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, dynamic, n_voxels, nullptr,
                                                           tile_offsets, total, out, counters);
  B200_CUDA(cudaGetLastError());
}

void sm_voxel_list_launch(const RankWord* index, unsigned long long n_words, const SmBox& box, unsigned n_voxels, int* ijk,
                          cudaStream_t stream) {
  if (n_words == 0 || n_voxels == 0) return;
  sm_voxel_list_kernel<<<blocks_for(n_words), SM_THREADS, 0, stream>>>(index, n_words, box, n_voxels, ijk);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
