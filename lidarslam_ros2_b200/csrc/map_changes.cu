// K20: the map changes of the session's submaps (b200sm_build_map_changes). Every decision follows csrc/map_changes.hpp,
// which a host compile also builds; the per-epoch counts they read are K15d's integers of per-submap booleans, so the
// labels, counts and the updated map are bitwise the host's whatever the order of the work.
#include "map_changes.cuh"

namespace b200 {
namespace {

// K20a. One thread per voxel (grid-stride): the label, and the appeared / vanished counts (warp sums, one atomic per warp).
__global__ void __launch_bounds__(SM_THREADS) ch_classify_kernel(const uint32_t* __restrict__ hits_b, const uint32_t* __restrict__ frees_b,
                                                                 const uint32_t* __restrict__ hits_a, const uint32_t* __restrict__ frees_a,
                                                                 unsigned n_voxels, unsigned min_frees, int dyn_value,
                                                                 unsigned char* __restrict__ label,
                                                                 unsigned long long* __restrict__ counters) {
  unsigned app = 0, van = 0;
  for (unsigned long long v = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; v < n_voxels;
       v += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned char l = ch_voxel_label(hits_b[v], frees_b[v], hits_a[v], frees_a[v], min_frees, dyn_value);
    label[v] = l;
    app += l == CH_APPEARED;
    van += l == CH_VANISHED;
  }
  app = __reduce_add_sync(0xffffffffu, app);
  van = __reduce_add_sync(0xffffffffu, van);
  if ((threadIdx.x & 31) == 0) {
    if (app) atomicAdd(&counters[CH_CTR_APPEARED_VOXELS], (unsigned long long)app);
    if (van) atomicAdd(&counters[CH_CTR_VANISHED_VOXELS], (unsigned long long)van);
  }
}

// K20b. Block b serves tile b of the whole map; thread t labels SM_PER_THREAD points of it (round j: points j SM_THREADS +
// t). The tile's kept points are summed over the warps' ballots in shared memory.
__global__ void __launch_bounds__(SM_THREADS) ch_label_kernel(const SmEntry* __restrict__ table, int n_entries, SmConst c, SmBox box,
                                                              const RankWord* __restrict__ index, const unsigned char* __restrict__ label,
                                                              unsigned n_voxels, int split_entry, const unsigned* __restrict__ map_first,
                                                              unsigned char* __restrict__ point_label, unsigned* __restrict__ counts,
                                                              unsigned long long* __restrict__ counters) {
  __shared__ unsigned block_kept;
  if (threadIdx.x == 0) block_kept = 0;
  __syncthreads();
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const int epoch = k >= split_entry ? CH_AFTER : CH_BEFORE;
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  unsigned char* out = point_label + map_first[k];
  unsigned kept = 0, app = 0, van = 0, tripped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int v[3];
    long long f[3];
    unsigned char l = CH_UNCHANGED;
    if (sm_ray(c, e.o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) {
      unsigned r;
      if (sm_rank(index, box, v[0], v[1], v[2], &r) && r < n_voxels) l = ch_point_label(label[r], epoch);
      else tripped = 1u;
    }
    out[i] = l;
    kept += l != CH_VANISHED;
    app += l == CH_APPEARED;
    van += l == CH_VANISHED;
  }
  kept = __reduce_add_sync(0xffffffffu, kept);
  app = __reduce_add_sync(0xffffffffu, app);
  van = __reduce_add_sync(0xffffffffu, van);
  if ((threadIdx.x & 31) == 0) {
    if (kept) atomicAdd(&block_kept, kept);
    if (app) atomicAdd(&counters[CH_CTR_APPEARED_POINTS], (unsigned long long)app);
    if (van) atomicAdd(&counters[CH_CTR_VANISHED_POINTS], (unsigned long long)van);
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
  __syncthreads();
  if (threadIdx.x == 0) counts[blockIdx.x] = block_kept;
}

// K20c. The same tiles and rounds as K20b: (round, warp, lane) is the assembled map's order within the tile, so a kept
// point's destination is the tile's offset plus the kept points of the earlier rounds, of the earlier warps of its round
// and of the lower lanes of its warp.
__global__ void __launch_bounds__(SM_THREADS) ch_write_kernel(const SmEntry* __restrict__ table, int n_entries,
                                                              const unsigned* __restrict__ map_first,
                                                              const unsigned char* __restrict__ point_label,
                                                              const unsigned* __restrict__ tile_offsets, unsigned total,
                                                              float4* __restrict__ out, unsigned long long* __restrict__ counters) {
  constexpr int W = SM_THREADS / 32;
  __shared__ unsigned warp_count[SM_PER_THREAD][W];
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  const unsigned char* lab = point_label + map_first[k];
  unsigned mask[SM_PER_THREAD];
#pragma unroll
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    mask[j] = __ballot_sync(0xffffffffu, i < e.n && lab[i] != CH_VANISHED);
    if (lane == 0) warp_count[j][warp] = (unsigned)__popc(mask[j]);
  }
  __syncthreads();
  unsigned dst = tile_offsets[blockIdx.x];
  unsigned tripped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    unsigned before = 0, round = 0;
    for (int w = 0; w < W; w++) {
      before += w < warp ? warp_count[j][w] : 0u;
      round += warp_count[j][w];
    }
    if ((mask[j] >> lane) & 1u) {
      const unsigned i = base + j * SM_THREADS;
      const float4 p = e.cloud[i];
      float q[3];
      og_transform(e.T, p.x, p.y, p.z, q);
      const unsigned at = dst + before + (unsigned)__popc(mask[j] & ((1u << lane) - 1u));
      if (at < total) out[at] = make_float4(q[0], q[1], q[2], p.w);
      else tripped = 1u;
    }
    dst += round;
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

}  // namespace

void ch_classify_launch(const uint32_t* hits_b, const uint32_t* frees_b, const uint32_t* hits_a, const uint32_t* frees_a,
                        unsigned n_voxels, const SmConst& c, unsigned char* label, unsigned long long* counters, cudaStream_t stream) {
  if (n_voxels == 0) return;
  const unsigned want = (n_voxels + SM_THREADS - 1) / SM_THREADS;
  const unsigned blocks = want < 16u * H100_SMS ? want : 16u * H100_SMS;
  ch_classify_kernel<<<blocks, SM_THREADS, 0, stream>>>(hits_b, frees_b, hits_a, frees_a, n_voxels, c.min_frees, c.dyn_value, label,
                                                        counters);
  B200_CUDA(cudaGetLastError());
}

void ch_label_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                     const unsigned char* label, unsigned n_voxels, int split_entry, const unsigned* map_first,
                     unsigned char* point_label, unsigned* counts, unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  ch_label_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, label, n_voxels, split_entry, map_first,
                                                    point_label, counts, counters);
  B200_CUDA(cudaGetLastError());
}

void ch_write_launch(const SmEntry* table, int n_entries, unsigned tiles, const unsigned* map_first, const unsigned char* point_label,
                     const unsigned* tile_offsets, unsigned total, float4* out, unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  ch_write_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, map_first, point_label, tile_offsets, total, out, counters);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
