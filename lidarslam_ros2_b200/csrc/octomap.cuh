// The OctoMap of the scan-matcher session (b200sm_build_octomap): the K22 kernels of octomap.cu. The arithmetic is
// csrc/octomap.hpp's; the rays, the occupied voxels' rank index and their dynamic flags come from the static map's
// K15a-K15e (static_map.cuh). These are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "octomap.hpp"
#include "static_map.cuh"

namespace b200 {

// The dense pyramid over the box's keys: level l (1..16) holds the cells key >> l of the box's keys, lo[l] .. lo[l] +
// dims[l] - 1 per axis, at first[l] .. first[l + 1] - 1 of the pyramid's arrays, in linear (z, y, x) order. Level 0 is the
// box itself (its keys; the voxel states live in the box's own array). Above the box the extents shrink to one cell per
// axis, a short chain up to the root, level 16's single cell.
struct OmPyramid {
  unsigned lo[OM_DEPTH + 1][3];
  unsigned dims[OM_DEPTH + 1][3];
  unsigned long long first[OM_DEPTH + 2];
};

// The pyramid over a box (host)
inline OmPyramid om_pyramid(const SmBox& box) {
  OmPyramid p{};
  for (int a = 0; a < 3; a++) {
    const unsigned k0 = (unsigned)(box.lo[a] + OM_KEY_OFFSET), k1 = k0 + box.dims[a] - 1u;
    for (int l = 0; l <= OM_DEPTH; l++) {
      p.lo[l][a] = k0 >> l;
      p.dims[l][a] = (k1 >> l) - (k0 >> l) + 1u;
    }
  }
  p.first[0] = p.first[1] = 0;
  for (int l = 1; l <= OM_DEPTH; l++)
    p.first[l + 1] = p.first[l] + (unsigned long long)p.dims[l][0] * p.dims[l][1] * p.dims[l][2];
  return p;
}

// counters[] slots: the static map's, then the OctoMap's
enum : int {
  OM_CTR_OCCUPIED_VOXELS = SM_CTR_COUNT,
  OM_CTR_FREE_VOXELS,
  OM_CTR_INNER,
  OM_CTR_OCCUPIED_LEAVES,
  OM_CTR_FREE_LEAVES,
  OM_CTR_COUNT
};

// K22a: the bit of every voxel (linear index in `box`) that some ray's freed walk crosses set in `freed` (zero
// beforehand), over the tiles of the whole map. A walk voxel outside the box (never, by construction) raises
// counters[TRIPPED] instead.
void om_free_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, uint32_t* freed,
                    unsigned long long* counters, cudaStream_t stream);
// K22b: one thread per level-1 cell: the states of its 8 voxels (om_state of the endpoint rank index over `ebox`, the
// dynamic flags of its n_voxels occupied voxels and `freed`) into states[] (the box's linear order; UNKNOWN included),
// and the cell's code and inner count (1 when inner) at its pyramid index; counters[OCCUPIED / FREE_VOXELS] += those
// voxels.
void om_leaf_launch(const OmPyramid& pyr, const SmBox& ebox, const RankWord* index, const unsigned char* dynamic,
                    unsigned n_voxels, const uint32_t* freed, unsigned char* states, unsigned char* codes, unsigned* counts,
                    unsigned long long* counters, cudaStream_t stream);
// K22c: level l (2..16) from level l - 1: each cell's code (om_parent) and its subtree's inner nodes.
void om_reduce_launch(const OmPyramid& pyr, int level, unsigned char* codes, unsigned* counts, cudaStream_t stream);
// K22d: level l (16..2) hands its inner cells' children (level l - 1) their pre-order byte offsets, in place of their
// inner counts (the root's offset is 0 and stays its count).
void om_offset_launch(const OmPyramid& pyr, int level, const unsigned char* codes, unsigned* counts, cudaStream_t stream);
// K22e: every inner cell of levels 1..16 writes its two bytes at its offset in out[0 .. n_bytes); counters[INNER /
// OCCUPIED_LEAVES / FREE_LEAVES] += the inner cells and their leaf children. A byte at or beyond n_bytes is not stored;
// counters[TRIPPED] is raised instead.
void om_write_launch(const OmPyramid& pyr, const unsigned char* states, const unsigned char* codes, const unsigned* counts,
                     unsigned char* out, unsigned long long n_bytes, unsigned long long* counters, cudaStream_t stream);

}  // namespace b200
