// The changes between two recordings of the session's map (b200sm_build_map_changes): the voxels that APPEARED (free in
// the earlier recording, occupied in the later one) or VANISHED (the reverse), every point labelled by its voxel's change,
// and the map brought up to date (the assembled map without the points of what vanished). The rays, box, rank index and
// walks are the static map's (static_map.hpp) unchanged; only the counts are kept per epoch instead of pooled. The
// kernels (map_changes.cu, and static_map.cu's K15a-K15d) and a host compile (tests/hostmath/map_changes_host.cpp,
// g++ -ffp-contract=off) both use the functions below and those of static_map.hpp, so every decision is the same on
// either side.
//
// Definitions (this text is the contract; tests/changeref.py replays it in Python integers):
//  * Parameters: the static map's (SmParams, same defaults, same refusals through sm_prepare) and split_submap.
//  * Epochs. BEFORE is submaps [0, split), AFTER is [split, N), N the session's submaps. split_submap = -1 means the first
//    submap of the session's last segment (the recording b200sm_merge_session appended last); an explicit index also
//    covers one recording that revisits a place (lap 1 against lap 2). Refused (ch_split): -1 on a session of one segment,
//    0, any other negative value, and N or more.
//  * Rays, box, rank, walks: exactly the static map's (origins, sm_ray, sm_box over every ray's endpoint voxel of both
//    epochs, ranks in ascending linear index, sm_walk of the freed segment; a walk voxel outside the box or not occupied is
//    ignored).
//  * Counts. hits_e[v] and frees_e[v], e in {BEFORE, AFTER}: the static map's per-submap HIT and FREE booleans (a submap
//    that hits a voxel does not free it) counted over the submaps of epoch e only. Each is at most the epoch's submaps.
//  * Per voxel. free_e(v) = sm_dynamic(hits_e, frees_e, min_frees, dyn_value) (frees_e >= min_frees and og_value <=
//    rint(100 dynamic_thresh)); occ_e(v) = hits_e >= 1 && !free_e. The label is APPEARED when occ_AFTER && free_BEFORE,
//    VANISHED when occ_BEFORE && free_AFTER, otherwise UNCHANGED. occ_e excludes free_e, so the three are mutually
//    exclusive; a voxel one epoch never saw (no hit, fewer than min_frees frees) is neither occupied nor free in it.
//  * Per point (map order). A ray of an AFTER submap whose endpoint voxel is APPEARED is APPEARED; a ray of a BEFORE
//    submap whose endpoint voxel is VANISHED is VANISHED. Every other point is UNCHANGED: skipped and non-finite points, a
//    BEFORE point in an APPEARED voxel (the few rays of the earlier recording that ended in space the later one found
//    occupied), an AFTER point in a VANISHED voxel.
//  * Updated map: the assembled map in assembly order minus the VANISHED points. Nothing else is dropped: every AFTER
//    point is kept.
//  * Consequence. A voxel's counts in epoch e equal those of the static map of epoch e's submaps alone (the walks and
//    the per-submap booleans do not depend on the box, and that map's occupied voxels are a subset of this one's). So an
//    APPEARED or VANISHED point lies in a voxel that is occupied, hence not dynamic, in the static map of its own epoch:
//    that map would keep it. Something that only moves through one recording (a passing car) is dynamic or unseen in that
//    recording and is never reported as a change.
#pragma once
#include "static_map.hpp"

namespace b200 {

enum : unsigned char { CH_UNCHANGED = 0, CH_APPEARED = 1, CH_VANISHED = 2 };
enum : int { CH_BEFORE = 0, CH_AFTER = 1 };

// The change of a voxel from its counts in the two epochs
OG_HD unsigned char ch_voxel_label(unsigned hits_b, unsigned frees_b, unsigned hits_a, unsigned frees_a, unsigned min_frees,
                                   int dyn_value) {
  const bool free_b = sm_dynamic(hits_b, frees_b, min_frees, dyn_value), free_a = sm_dynamic(hits_a, frees_a, min_frees, dyn_value);
  const bool occ_b = hits_b >= 1 && !free_b, occ_a = hits_a >= 1 && !free_a;
  if (occ_a && free_b) return CH_APPEARED;
  if (occ_b && free_a) return CH_VANISHED;
  return CH_UNCHANGED;
}

// The label of a ray of epoch `epoch` whose endpoint voxel has label `voxel`
OG_HD unsigned char ch_point_label(unsigned char voxel, int epoch) {
  if (epoch == CH_AFTER && voxel == CH_APPEARED) return CH_APPEARED;
  if (epoch == CH_BEFORE && voxel == CH_VANISHED) return CH_VANISHED;
  return CH_UNCHANGED;
}

// nullptr when split_submap names a split of a session of n_sub submaps whose last segment starts at submap
// last_segment_first (0: one segment), and *split = the first AFTER submap; else the reason
inline const char* ch_split(long long split_submap, unsigned long long n_sub, unsigned long long last_segment_first,
                            unsigned long long* split) {
  if (split_submap == -1) {
    if (last_segment_first == 0) return "split_submap -1 needs a session of more than one segment";
    *split = last_segment_first;
    return nullptr;
  }
  if (split_submap < 0) return "split_submap must be -1 or in [1, n_submaps)";
  if (split_submap == 0) return "split_submap 0 leaves no submap before the split";
  if ((unsigned long long)split_submap >= n_sub) return "split_submap must be below the number of submaps";
  *split = (unsigned long long)split_submap;
  return nullptr;
}

}  // namespace b200
