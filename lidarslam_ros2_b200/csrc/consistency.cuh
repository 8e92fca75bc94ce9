// The map consistency of the scan-matcher session (b200sm_build_map_consistency): the K19 kernels of consistency.cu. The
// arithmetic is csrc/map_consistency.hpp's; the box and its rank index are the static map's (sm_box, RankWord, the cell
// list of sm_voxel_list_launch). These are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "map_consistency.hpp"
#include "static_map.cuh"

namespace b200 {

// One submap with points: its cloud, float pose, first map index and first tile in the launches over the whole map.
struct McEntry {
  const float4* cloud;
  unsigned n, first_tile, map_offset;
  float T[12];
};
constexpr int MC_THREADS = 256, MC_PER_THREAD = 4, MC_TILE = MC_THREADS * MC_PER_THREAD;
constexpr int MC_CHUNK = 256;  // queries of one cell per K19c block, and candidates per shared-memory tile

// counters[] slots
enum : int { MC_CTR_SKIPPED = 0, MC_CTR_RANGE, MC_CTR_CANDIDATES, MC_CTR_TRIPPED, MC_CTR_COUNT };
// per-submap row slots (rows[MC_ROW_COUNT k + slot])
enum : int { MC_ROW_QUERIES = 0, MC_ROW_VALID, MC_ROW_NEIGHBORS, MC_ROW_SUM_H, MC_ROW_SUM_PLANE, MC_ROW_COUNT };

// K19a: bounds[6 k .. 6 k + 5] (min x, y, z, max x, y, z cell; INT_MAX / INT_MIN beforehand) of entry k widened by every
// non-skipped point's cell; counters[SKIPPED] += the skipped points, counters[RANGE] += the points beyond 2^46.
void mc_bounds_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, int* bounds, unsigned long long* counters,
                      cudaStream_t stream);
// K19b, first pass: every non-skipped point's cell marked in the rank index over the box (zero beforehand).
void mc_mark_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, const SmBox& box, RankWord* index,
                    unsigned long long* counters, cudaStream_t stream);
// K19b, second pass: count[r] += 1 for every non-skipped point of occupied cell r, queries[r] += 1 for every query (both
// zero beforehand).
void mc_count_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, const SmBox& box, const RankWord* index,
                     unsigned* count, unsigned* queries, cudaStream_t stream);
// chunks[r] = the K19c blocks of cell r: ceil(queries[r] / MC_CHUNK)
void mc_chunks_launch(const unsigned* queries, unsigned n_cells, unsigned* chunks, cudaStream_t stream);
// K19b, third pass: every non-skipped point into cell order — cell r's queries at start[r] .. start[r] + queries[r], its
// other points after them, in any order (cursors zero beforehand): its position within the cell (X, Y, Z & 0xffff) in
// offs and its map index in idx. Every point's layers are reset (n 0, h and plane_var MC_NAN_BITS). A slot beyond the
// cell raises counters[TRIPPED] instead of a store.
void mc_scatter_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, const SmBox& box, const RankWord* index,
                       const unsigned* start, const unsigned* queries, unsigned* qcursor, unsigned* ocursor, ushort4* offs,
                       unsigned* idx, unsigned* n_out, double* h_out, double* plane_out, unsigned long long* counters,
                       cudaStream_t stream);
// K19c + K19d: one block per chunk of up to MC_CHUNK queries of one cell (chunk_start: the exclusive scan of chunks,
// n_chunks blocks), the 27 cells' points staged through shared memory; per query n, h and plane_var at its map index and
// the per-submap rows (sub_first: the first map index of each of the n_sub submaps); counters[CANDIDATES] += the points
// of the 27 cells times the chunk's queries.
void mc_neighbour_launch(const unsigned* chunk_start, unsigned n_chunks, unsigned n_cells, const unsigned* start, const unsigned* queries,
                         const int* cell_ijk, const SmBox& box, const RankWord* index, const ushort4* offs, const unsigned* idx,
                         const unsigned* sub_first, int n_sub, const McConst& c, unsigned* n_out, double* h_out, double* plane_out,
                         unsigned long long* rows, unsigned long long* counters, cudaStream_t stream);
// The per-point intensity of the saved PCD: pts[i].w = (float)h[i] (NaN where h is NaN), n points.
void mc_intensity_launch(float4* pts, const double* h, size_t n, cudaStream_t stream);

}  // namespace b200
