// The map changes of the scan-matcher session (b200sm_build_map_changes): the K20 kernels of map_changes.cu. The
// arithmetic is csrc/map_changes.hpp's; the rays, box, rank index and per-epoch counts come from the static map's K15a-K15d
// (static_map.cuh), run once per epoch. These are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "map_changes.hpp"
#include "static_map.cuh"

namespace b200 {

// counters[] slots: the static map's, then the changes'
enum : int {
  CH_CTR_APPEARED_VOXELS = SM_CTR_COUNT,
  CH_CTR_VANISHED_VOXELS,
  CH_CTR_APPEARED_POINTS,
  CH_CTR_VANISHED_POINTS,
  CH_CTR_COUNT
};

// K20a: label[v] = ch_voxel_label of the four counts of voxel v; counters[APPEARED / VANISHED_VOXELS] += those voxels.
void ch_classify_launch(const uint32_t* hits_b, const uint32_t* frees_b, const uint32_t* hits_a, const uint32_t* frees_a,
                        unsigned n_voxels, const SmConst& c, unsigned char* label, unsigned long long* counters, cudaStream_t stream);
// K20b: over the tiles of the whole map (the static map's table; entries from split_entry on are AFTER), point_label[
// map_first[k] + i] = ch_point_label of point i of entry k, and counts[tile] = the tile's points the updated map keeps;
// counters[APPEARED / VANISHED_POINTS] += those points. A ray whose endpoint has no rank below n_voxels (never, by
// construction) raises counters[TRIPPED] and keeps its label UNCHANGED.
void ch_label_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, const RankWord* index,
                     const unsigned char* label, unsigned n_voxels, int split_entry, const unsigned* map_first,
                     unsigned char* point_label, unsigned* counts, unsigned long long* counters, cudaStream_t stream);
// K20c: the kept points (label not VANISHED), moved by their submap's float pose, at tile_offsets[tile] + their rank among
// the tile's kept points: the assembled map's order. A destination at or beyond `total` (the count the host read back
// after K20b) is not stored; counters[TRIPPED] is raised instead.
void ch_write_launch(const SmEntry* table, int n_entries, unsigned tiles, const unsigned* map_first, const unsigned char* point_label,
                     const unsigned* tile_offsets, unsigned total, float4* out, unsigned long long* counters, cudaStream_t stream);

}  // namespace b200
