// Place recognition on the scan-matcher session (b200sm_search_loop_place): the Scan Context kernels of
// place_recognition.cu. The arithmetic is csrc/scan_context.hpp's; these are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace b200 {

// One submap to describe: its cloud (sensor frame), its points, the first tile of the launch that serves it, and the slot
// of the descriptor store it is written to.
struct ScBuildEntry {
  const float4* cloud;
  unsigned n, first_tile, slot, pad;
};
constexpr int SC_BUILD_THREADS = 256, SC_BUILD_PER_THREAD = 16, SC_BUILD_TILE = SC_BUILD_THREADS * SC_BUILD_PER_THREAD;

// K13a: keys[slot * R * S + bin] = max order key of the bin's points over the submaps of `table` (n_entries rows, sorted by
// first_tile, `tiles` tiles in all). The keys of those slots must be zero beforehand. tables = R ring bounds then S sector
// directions (scan_context.hpp's sc_tables).
void sc_build_launch(const ScBuildEntry* table, int n_entries, unsigned tiles, uint32_t* keys, const double* tables, int num_rings,
                     int num_sectors, float lidar_height, cudaStream_t stream);
// The finishing pass of K13a over slots [first_slot, first_slot + n_slots): keys become the descriptor's floats in place
// (an empty bin 0), and norms[slot * S + j] the column norms.
void sc_finish_launch(uint32_t* keys, double* norms, size_t first_slot, size_t n_slots, int num_rings, int num_sectors,
                      cudaStream_t stream);
// K13b: for r < n_ids, (distance[r], shift[r]) = (D, s*) of descriptor `query_slot` against descriptor ids[r].
void sc_search_launch(const float* desc, const double* norms, size_t query_slot, const int* ids, int n_ids, double* distance,
                      int* shift, int num_rings, int num_sectors, cudaStream_t stream);

// K16 (b200sm_merge_session): queries per block of the score launch, from the descriptor's size and the device's opt-in
// shared memory shared by MERGE_BLOCKS_PER_SM blocks, 1..MERGE_QUERY_TILE_MAX.
constexpr int MERGE_QUERY_TILE_MAX = 32, MERGE_BLOCKS_PER_SM = 5;
int merge_query_tile(int num_rings, int num_sectors);
// distance[b * n_cand + a], shift[b * n_cand + a] = (D, s*) of query descriptor b (q_desc) against candidate a (c_desc),
// bitwise K13b's for the same pair; one launch.
void merge_scores_launch(const float* q_desc, const double* q_norms, int n_query, const float* c_desc, const double* c_norms,
                         int n_cand, double* distance, int* shift, int num_rings, int num_sectors, cudaStream_t stream);
// per query row b: the first top_k candidates with D < threshold in (D, a) order, at sel_*[b * top_k + r]; sel_a = -1
// past the row's last candidate.
void merge_select_launch(const double* distance, const int* shift, int n_query, int n_cand, double threshold, int top_k, int* sel_a,
                         double* sel_d, int* sel_s, cudaStream_t stream);

}  // namespace b200
