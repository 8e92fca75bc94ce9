// The static map of the scan-matcher session (b200sm_build_static_map): the K15 kernels of static_map.cu. The arithmetic
// is csrc/static_map.hpp's; these are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "grid_index.cuh"
#include "static_map.hpp"

namespace b200 {

// One submap with points: its cloud and float pose, its ray origin in fixed point, its first tile in the launches over
// the whole map (K15a, K15b, K15f, K15g) and in its walk batch (K15c).
struct SmEntry {
  const float4* cloud;
  unsigned n, first_tile, batch_tile;
  float T[12];
  long long o[3];
};
constexpr int SM_THREADS = 256, SM_PER_THREAD = 4, SM_TILE = SM_THREADS * SM_PER_THREAD;

// The box of the occupied voxels: its lower corner and dimensions
struct SmBox {
  int lo[3];
  unsigned dims[3];
};

// the linear index of voxel (x, y, z) in the box; false outside it (the differences in int64: voxel indices reach 2^30 + 2^14)
__device__ __forceinline__ bool sm_lin(const SmBox& b, int x, int y, int z, unsigned* lin) {
  const long long wx = (long long)x - b.lo[0], wy = (long long)y - b.lo[1], wz = (long long)z - b.lo[2];
  if (wx < 0 || wy < 0 || wz < 0 || wx >= b.dims[0] || wy >= b.dims[1] || wz >= b.dims[2]) return false;
  *lin = (unsigned)(((unsigned long long)wz * b.dims[1] + (unsigned long long)wy) * b.dims[0] + (unsigned long long)wx);
  return true;
}

// the rank of an occupied voxel; false when it is outside the box or not occupied
__device__ __forceinline__ bool sm_rank(const RankWord* __restrict__ index, const SmBox& b, int x, int y, int z, unsigned* r) {
  unsigned lin;
  if (!sm_lin(b, x, y, z, &lin)) return false;
  return rank_probe(__ldg(reinterpret_cast<const uint2*>(index + (lin >> 5))), lin & 31u, *r);
}

// counters[] slots
enum : int { SM_CTR_RAYS = 0, SM_CTR_SKIPPED, SM_CTR_DYNAMIC, SM_CTR_TRIPPED, SM_CTR_COUNT };

// K15a: bounds[6 k .. 6 k + 5] (min x, y, z, max x, y, z voxel; the host initialises them to INT_MAX / INT_MIN) of entry k
// widened by every ray's endpoint voxel; counters[RAYS / SKIPPED] += the launch's rays and skipped points.
void sm_bounds_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, int* bounds, unsigned long long* counters,
                      cudaStream_t stream);
// K15b: every ray's endpoint voxel marked in the rank index over the box (zero beforehand); counters[TRIPPED] is raised
// for an endpoint outside the box (never, by construction) instead of a store.
void sm_mark_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, RankWord* index,
                    unsigned long long* counters, cudaStream_t stream);
// K15c: the rays of the entries (one walk batch) set, in entry k's two bitmaps of `words_per` words each (hit at
// scratch + 2 k words_per, free right after it; zero beforehand), the bit of their endpoint voxel's rank and of the rank of
// every occupied voxel of the box their walk crosses. A rank at or beyond n_voxels raises counters[TRIPPED] instead.
void sm_walk_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                    unsigned n_voxels, unsigned long long words_per, uint32_t* scratch, unsigned long long* counters, cudaStream_t stream);
// K15d: hits[v] += the batch's submaps whose hit bit v is set, frees[v] += those whose free bit is set without the hit bit
// (one thread per bitmap word, bit-sliced counters).
void sm_fold_launch(const uint32_t* scratch, int n_entries, unsigned long long words_per, unsigned n_voxels, uint32_t* hits,
                    uint32_t* frees, cudaStream_t stream);
// K15e: dynamic[v] = sm_dynamic(hits[v], frees[v]); counters[DYNAMIC] += the dynamic voxels.
void sm_classify_launch(const uint32_t* hits, const uint32_t* frees, unsigned n_voxels, const SmConst& c, unsigned char* dynamic,
                        unsigned long long* counters, cudaStream_t stream);
// K15f: counts[tile] = the points of the tile the static map keeps (tiles of the whole map, in assembly order).
void sm_count_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                     const unsigned char* dynamic, unsigned n_voxels, unsigned* counts, cudaStream_t stream);
// K15g: the kept points, moved by their submap's float pose, at tile_offsets[tile] + their rank among the tile's kept
// points: the assembled map's order. A destination at or beyond `total` (the count the host read back after K15f) is not
// stored; counters[TRIPPED] is raised instead.
void sm_write_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                     const unsigned char* dynamic, unsigned n_voxels, const unsigned* tile_offsets, unsigned total, float4* out,
                     unsigned long long* counters, cudaStream_t stream);
// The voxel list for the read-back: ijk[3 r .. 3 r + 2] = the voxel of rank r, for every occupied voxel of the box
// (ranks at or beyond n_voxels are not stored).
void sm_voxel_list_launch(const RankWord* index, unsigned long long n_words, const SmBox& box, unsigned n_voxels, int* ijk,
                          cudaStream_t stream);

}  // namespace b200
