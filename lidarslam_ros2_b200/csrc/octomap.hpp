// The OctoMap of the session (b200sm_build_octomap): every voxel some submap's ray frees or ends in, labelled FREE or
// OCCUPIED, pruned into OctoMap's depth-16 key tree and written as the bytes of OctoMap's OcTree::writeBinary (a .bt file
// that octomap_server, MoveIt and rviz load). The kernels (octomap.cu) and a host compile (tests/hostmath/octomap_host.cpp,
// g++ -ffp-contract=off) both use the functions below and those of static_map.hpp. The octree is the output format only:
// the voxel states are the static map's per-submap counts, with no clamped log-odds.
//
// Definitions (this text is the contract; tests/octomapref.py replays it in Python integers):
//  * Rays, walks, parameters: exactly those of the static map (static_map.hpp): sm_ray, sm_walk, its skip rule and the
//    freed first ray_fraction of each ray, with b200sm_static_map_params.
//  * BOX: the bounding box of every ray's endpoint voxel and of the origin voxel og_cell(O) of every submap with at least
//    one ray. Every freed walk lies in it (its voxels lie between voxel(O) and voxel(E'), and E' between O and E). The
//    build is refused before anything is sized from the box when it has more than 2^31 - 1 voxels, when a box voxel index
//    lies outside [-32768, 32767] on some axis (OctoMap keys are 16 bits: key = index + 32768), and when
//    printf("%g", resolution) does not read back as the same double (a reader would put the voxels elsewhere).
//  * State of a box voxel: OCCUPIED when the static map counts it as an occupied voxel (an endpoint lies in it) and
//    sm_dynamic(hits, frees) is false, with the static map's hits and frees; FREE when it is not OCCUPIED and some ray's
//    freed walk crosses it or it is an endpoint voxel (so a dynamic voxel is FREE: what moved leaves free space behind);
//    UNKNOWN otherwise. The codes are OM_UNKNOWN 0, OM_FREE 1, OM_OCCUPIED 2.
//  * Tree: a node at level l (0 = voxel, 16 = root) covers the keys whose top 16 - l bits are its own; its children are
//    the level l - 1 nodes under it, child index bit (l - 1) of kx + 2 * that bit of ky + 4 * that bit of kz (bit
//    15 - depth, depth = 16 - l). A node exists iff some voxel under it is known. A node is a LEAF when all 8 children
//    exist, each is a leaf, and all have the same state; it takes that state. (A known voxel is a leaf.) This is the tree
//    OctoMap's toMaxLikelihood(); prune(); leaves, which writeBinary saves.
//  * Child code of a node as its parent's bytes hold it: 0 absent, 1 FREE leaf, 2 OCCUPIED leaf, 3 inner node (OM_INNER).
//    Level 0 codes are the voxel states, and om_parent gives a node's code from its children's.
//  * File bytes (octomap 1.9 OcTree::writeBinary): the header om_header(size, resolution), size = the nodes of the tree,
//    the root included; then, for every inner node in pre-order (children visited 0..7), two bytes: byte 0 holds children
//    0-3 and byte 1 children 4-7, child i at bits 2 (i mod 4) and 2 (i mod 4) + 1 (om_pack). An empty tree (no ray) is the
//    header with size 0 and no data.
//  * Pre-order offsets: the bytes of a subtree are 2 * its inner nodes, so an inner child's two bytes start at its
//    parent's offset + 2 + the subtree bytes of its earlier siblings; the root's are at 0.
// Every decision is integers and bit operations after the static map's one float transform and rounded multiply per
// coordinate, so the states and the bytes are bitwise deterministic.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <string>

#include "static_map.hpp"

namespace b200 {

enum : unsigned char { OM_UNKNOWN = 0, OM_FREE = 1, OM_OCCUPIED = 2, OM_INNER = 3 };
constexpr int OM_DEPTH = 16;
constexpr int OM_KEY_OFFSET = 32768;  // key = voxel index + 32768

// The state of a box voxel: endpoint (some ray ends in it), its dynamic flag (meaningful for an endpoint only) and whether
// some freed walk crosses it
OG_HD unsigned char om_state(bool endpoint, bool dynamic, bool freed) {
  if (endpoint && !dynamic) return OM_OCCUPIED;
  return (endpoint || freed) ? OM_FREE : OM_UNKNOWN;
}

// A node's code from its 8 children's codes: a leaf of their state when all are leaves of one state, absent when all
// are absent, else inner
OG_HD unsigned char om_parent(const unsigned char* child) {
  const unsigned char c0 = child[0];
  bool same = c0 == OM_FREE || c0 == OM_OCCUPIED, any = c0 != OM_UNKNOWN;
  for (int i = 1; i < 8; i++) {
    same = same && child[i] == c0;
    any = any || child[i] != OM_UNKNOWN;
  }
  return same ? c0 : (any ? (unsigned char)OM_INNER : (unsigned char)OM_UNKNOWN);
}

// Child index, under a node at level l, of the node holding keys (kx, ky, kz)
OG_HD int om_child(unsigned kx, unsigned ky, unsigned kz, int l) {
  const int b = l - 1;
  return (int)(((kx >> b) & 1u) | (((ky >> b) & 1u) << 1) | (((kz >> b) & 1u) << 2));
}

// An inner node's two bytes from its children's codes
OG_HD void om_pack(const unsigned char* child, unsigned char* b0, unsigned char* b1) {
  unsigned v0 = 0, v1 = 0;
  for (int i = 0; i < 4; i++) {
    v0 |= (unsigned)child[i] << (2 * i);
    v1 |= (unsigned)child[4 + i] << (2 * i);
  }
  *b0 = (unsigned char)v0;
  *b1 = (unsigned char)v1;
}

// ---- host side: the resolution, the box, the header ----

// false when printf("%g", resolution) does not read back as the same double
inline bool om_resolution_exact(double resolution) {
  char buf[64];
  std::snprintf(buf, sizeof(buf), "%g", resolution);
  return std::strtod(buf, nullptr) == resolution;
}

// The box's dimensions from its inclusive voxel bounds lo[3], hi[3]; nullptr when accepted, else the reason
inline const char* om_box(const int* lo, const int* hi, unsigned* dims, unsigned long long* cells) {
  if (!sm_box(lo, hi, dims, cells)) return "more than 2^31 - 1 voxels";
  for (int a = 0; a < 3; a++)
    if (lo[a] < -OM_KEY_OFFSET || hi[a] > OM_KEY_OFFSET - 1) return "a voxel index outside the 16-bit OctoMap key range [-32768, 32767]";
  return nullptr;
}

// The .bt header of a tree of `size` nodes
inline std::string om_header(unsigned long long size, double resolution) {
  char buf[256];
  std::snprintf(buf, sizeof(buf),
                "# Octomap OcTree binary file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
                "id OcTree\nsize %llu\nres %g\ndata\n",
                size, resolution);
  return buf;
}

}  // namespace b200
