// The surface mesh of the scan-matcher session (b200sm_build_mesh): the K21 kernels of mesh.cu. The arithmetic is
// csrc/mesh.hpp's; the rays, the endpoint bounds (K15a), the rank index's helpers and the voxel list are the static map's
// (static_map.cuh). These are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "mesh.hpp"
#include "static_map.cuh"

namespace b200 {

constexpr int MS_THREADS = 256;  // K21c-e: one band voxel per thread, a tile of MS_THREADS band voxels per block

// counters[] slots: the static map's (K15a writes RAYS and SKIPPED; TRIPPED is the tripwire), then the mesh's
enum : int { MS_CTR_WALKED = SM_CTR_COUNT, MS_CTR_OBSERVED, MS_CTR_FACES, MS_CTR_COUNT };

// K21a: every ray's band walk marked in the rank index over the widened box (zero beforehand); a walk voxel outside the
// box (never, by the header's bound) raises counters[TRIPPED] instead of a store.
void ms_mark_launch(const SmEntry* table, int n_entries, unsigned tiles, const MsConst& c, const SmBox& box, RankWord* index,
                    unsigned long long* counters, cudaStream_t stream);
// K21b: every ray's band walk again: sum[rank] += s (two's complement), weight[rank] += 1 (both zero beforehand);
// counters[WALKED] += the voxels walked. A voxel without a rank below n_band raises counters[TRIPPED] instead.
void ms_fuse_launch(const SmEntry* table, int n_entries, unsigned tiles, const MsConst& c, const SmBox& box, const RankWord* index,
                    unsigned n_band, unsigned long long* sum, uint32_t* weight, unsigned long long* counters, cudaStream_t stream);
// K21c: active[r] = whether the cell whose lowest corner is band voxel r (ijk[3 r ..]) is ACTIVE; counts[tile] = the tile's
// ACTIVE cells; counters[OBSERVED] += the observed band voxels.
void ms_active_launch(const int* ijk, const unsigned long long* sum, const uint32_t* weight, const RankWord* index, const SmBox& box,
                      unsigned n_band, unsigned min_weight, unsigned char* active, unsigned* counts, unsigned long long* counters,
                      cudaStream_t stream);
// K21d: vid[r] = the vertex id of band voxel r's cell (tile_offsets[tile] + its rank among the tile's ACTIVE cells), or
// 0xffffffff when the cell is not ACTIVE; the vertex at xyz[3 vid ..] (an id at or beyond n_vertices raises
// counters[TRIPPED] instead); face_counts[tile] = the faces of the tile's voxels' three +a edges, counters[FACES] += them.
void ms_vertex_launch(const int* ijk, const unsigned long long* sum, const uint32_t* weight, const RankWord* index, const SmBox& box,
                      unsigned n_band, const MsConst& c, const unsigned char* active, const unsigned* tile_offsets, unsigned n_vertices,
                      uint32_t* vid, float* xyz, unsigned* face_counts, unsigned long long* counters, cudaStream_t stream);
// K21e: the faces, three vertex ids each, at face_offsets[tile] + their rank in the tile's order (rank of v, axis,
// triangle). A destination at or beyond n_faces (the count the host read back after K21d) raises counters[TRIPPED]
// instead of a store.
void ms_face_launch(const int* ijk, const unsigned long long* sum, const uint32_t* weight, const RankWord* index, const SmBox& box,
                    unsigned n_band, unsigned min_weight, const uint32_t* vid, const unsigned* face_offsets, unsigned n_faces,
                    uint32_t* faces, unsigned long long* counters, cudaStream_t stream);

}  // namespace b200
