"""An exact replay of the map changes of b200sm_build_map_changes (csrc/map_changes.hpp) in Python integers: the rays,
walks, box and rank are staticmapref's (its ray, walk and box_cells); the per-submap hit and free booleans are counted per
epoch; then the voxel labels, the point labels and the updated map.

MUTATIONS names subtly wrong variants, each of which tests/test_map_changes_cpu.py shows changes an outcome:
  split_late     the split one submap later than asked
  epoch_blind    the point rule ignores the epoch: every ray takes its voxel's label
  strict_dyn     free_e uses og_value < dyn_value instead of <=
  no_min_frees   free_e ignores min_frees
  pooled_before  the AFTER submaps' folds are added to the BEFORE counts too
"""
from __future__ import annotations

import numpy as np

import occupancyref as O
import staticmapref as SM

MUTATIONS = ("split_late", "epoch_blind", "strict_dyn", "no_min_frees", "pooled_before")
UNCHANGED, APPEARED, VANISHED = 0, 1, 2
BEFORE, AFTER = 0, 1
Refused = O.Refused
params = SM.params


def split_of(split_submap, n_sub, last_segment_first):
    """The first AFTER submap, or Refused(-5)."""
    if split_submap == -1:
        if last_segment_first == 0:
            raise Refused(-5, "split_submap -1 on one segment")
        return last_segment_first
    if split_submap <= 0 or split_submap >= n_sub:
        raise Refused(-5, "split_submap")
    return split_submap


def free(h, f, c, mut=()):
    """The static map's dynamic rule for one epoch's counts."""
    if "no_min_frees" not in mut and f < c["min_frees"]:
        return False
    v = O.value(h, f)  # -1 for a voxel the epoch never saw: only the no_min_frees mutation gets here with one
    return v < c["dyn"] if "strict_dyn" in mut else v <= c["dyn"]


def voxel_label(hb, fb, ha, fa, c, mut=()):
    free_b, free_a = free(hb, fb, c, mut), free(ha, fa, c, mut)
    occ_b, occ_a = hb >= 1 and not free_b, ha >= 1 and not free_a
    if occ_a and free_b:
        return APPEARED
    if occ_b and free_a:
        return VANISHED
    return UNCHANGED


def point_label(voxel, epoch, mut=()):
    if "epoch_blind" in mut:
        return voxel
    if epoch == AFTER and voxel == APPEARED:
        return APPEARED
    if epoch == BEFORE and voxel == VANISHED:
        return VANISHED
    return UNCHANGED


def build(submaps, split_submap, p=None, last_segment_first=0, mut=()):
    """submaps: list of (points (n, >= 3) float32, pose 4x4 float64). Returns a dict: lo, dims, split, n_rays, n_skipped,
    ijk ((V, 3) int32, rank order), hits_before, frees_before, hits_after, frees_after (uint32), label (uint8 per voxel),
    point_label (uint8 per point), offsets (n_sub + 1), n_voxels, n_appeared_voxels, n_vanished_voxels, n_points,
    n_appeared_points, n_vanished_points, n_updated_points, and the assembled points (M, 4) float32."""
    p = params(**(p or {}))
    c = SM.prepare(p)
    if not submaps:
        raise Refused(-4, "no submaps")
    split = split_of(split_submap, len(submaps), last_segment_first)
    if "split_late" in mut:
        split += 1
    Ts = [O.pose_f(P) for _, P in submaps]
    Os = [SM.origin(c, p, T) for T in Ts]
    rays, moved = [], []
    n_rays = n_skipped = 0
    for (pts, _), T, o in zip(submaps, Ts, Os):
        rs = []
        for row in np.asarray(pts, dtype=np.float32):
            e = O.transform(T, row[0], row[1], row[2])
            moved.append((e[0], e[1], e[2], np.float32(row[3]) if len(row) > 3 else np.float32(0)))
            r = SM.ray(c, o, e)
            rs.append(r)
            n_skipped += r is None
            n_rays += r is not None
        rays.append(rs)
    ends = [r[0] for rs in rays for r in rs if r is not None]
    if ends:
        lo = tuple(min(v[a] for v in ends) for a in range(3))
        hi = tuple(max(v[a] for v in ends) for a in range(3))
        if SM.box_cells(lo, hi) is None:
            raise Refused(-3, "box")
        dims = tuple(hi[a] - lo[a] + 1 for a in range(3))
    else:
        lo, dims = (0, 0, 0), (0, 0, 0)

    def lin(v):
        return ((v[2] - lo[2]) * dims[1] + (v[1] - lo[1])) * dims[0] + (v[0] - lo[0])

    occupied = sorted(set(ends), key=lin)
    rank = {v: r for r, v in enumerate(occupied)}
    hits = [np.zeros(len(occupied), dtype=np.uint32) for _ in range(2)]
    frees = [np.zeros(len(occupied), dtype=np.uint32) for _ in range(2)]
    for k, (rs, o) in enumerate(zip(rays, Os)):
        e = BEFORE if k < split else AFTER
        hit, crossed = set(), set()
        for r in rs:
            if r is None:
                continue
            hit.add(r[0])
            crossed |= {v for v in SM.walk(tuple(o), r[1]) if v in rank}
        into = (BEFORE, AFTER) if (e == AFTER and "pooled_before" in mut) else (e,)
        for t in into:
            for v in hit:
                hits[t][rank[v]] += 1
            for v in crossed - hit:
                frees[t][rank[v]] += 1
    label = np.array([voxel_label(int(hits[0][v]), int(frees[0][v]), int(hits[1][v]), int(frees[1][v]), c, mut)
                      for v in range(len(occupied))], dtype=np.uint8)
    plab, offsets, kept = [], [0], 0
    for k, rs in enumerate(rays):
        e = BEFORE if k < split else AFTER
        for r in rs:
            pl = UNCHANGED if r is None else point_label(int(label[rank[r[0]]]), e, mut)
            plab.append(pl)
            kept += pl != VANISHED
        offsets.append(kept)
    plab = np.array(plab, dtype=np.uint8)
    return dict(lo=lo, dims=dims, split=split, n_rays=n_rays, n_skipped=n_skipped,
                ijk=np.array(occupied, dtype=np.int32).reshape(-1, 3), hits_before=hits[0], frees_before=frees[0],
                hits_after=hits[1], frees_after=frees[1], label=label, point_label=plab,
                offsets=np.array(offsets, dtype=np.int64), n_voxels=len(occupied),
                n_appeared_voxels=int((label == APPEARED).sum()), n_vanished_voxels=int((label == VANISHED).sum()),
                n_points=len(plab), n_appeared_points=int((plab == APPEARED).sum()),
                n_vanished_points=int((plab == VANISHED).sum()), n_updated_points=kept,
                points=np.array(moved, dtype=np.float32).reshape(-1, 4), p=p, c=c)
