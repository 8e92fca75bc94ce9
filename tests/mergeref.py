"""A float64 numpy replay of the host part of b200sm_merge_session (csrc/session_merge.hpp and the segmented build_edges of
csrc/pose_graph.hpp): the per-row candidate selection and the global (D, b, a) order, the edge Z, the cycle error of two
accepted rows and its tolerance, the greedy consistent set, the rigid placement and the joint graph; plus the two-session
drive of the end-to-end GPU tests.

MUTATIONS names subtly wrong variants of the replay, each of which the CPU tests show changes an outcome:
  cycle_order      the cycle closed through B as P_{b_i}^-1 P_{b_j} instead of P_{b_j}^-1 P_{b_i}
  z_wrong_end      Z taken from the b end: (F P_b)^-1 P_a instead of P_a^-1 (F P_b)
  odometry_across  the odometry rule applied over the whole merged numbering, across the segment boundary
  tie_high         equal D (selection) or equal fitness (consistent set) broken by the higher index
  no_drift         the tolerance without its L term
"""
from __future__ import annotations

import math

import numpy as np

import posegraphref as PG
import scancontextref as SC
from lidarslam_ros2_b200 import synth

MUTATIONS = ("cycle_order", "z_wrong_end", "odometry_across", "tie_high", "no_drift")
TOL_FIELDS = ("consistency_translation", "consistency_rotation", "consistency_drift_translation", "consistency_drift_rotation")


def select_row(D, threshold, top_k, mut=()):
    """The a with D[a] < threshold ordered by (D, a), the first top_k."""
    rows = [a for a in range(len(D)) if D[a] < threshold]
    key = (lambda a: (D[a], -a)) if "tie_high" in mut else (lambda a: (D[a], a))
    return sorted(rows, key=key)[:top_k]


def order(D, threshold, top_k, max_verifications, mut=()):
    """All rows' selections of the (n_B, n_A) matrix D, as (D, b, a) ordered and cut to max_verifications."""
    c = [(float(D[b][a]), b, a) for b in range(len(D)) for a in select_row(D[b], threshold, top_k, mut)]
    return sorted(c)[:max_verifications]


def edge(Pa, F, Pb, mut=()):
    """Z, the edge from a to b."""
    Pa, F, Pb = (np.asarray(m, dtype=np.float64) for m in (Pa, F, Pb))
    if "z_wrong_end" in mut:
        return np.linalg.inv(F @ Pb) @ Pa
    return np.linalg.inv(Pa) @ (F @ Pb)


def cycle_error(i, j, mut=()):
    """(e_t, e_r) of rows i and j (dicts with Pa, Pb, Z)."""
    inv, c = PG.inverse, PG.compose  # Isometry3d's inverse (R^T, -R^T t), as the product's: Z is not exactly orthonormal
    if "cycle_order" in mut:
        E = c(c(c(inv(i["Z"]), c(inv(i["Pa"]), j["Pa"])), j["Z"]), c(inv(i["Pb"]), j["Pb"]))
    else:
        E = c(c(c(inv(i["Z"]), c(inv(i["Pa"]), j["Pa"])), j["Z"]), c(inv(j["Pb"]), i["Pb"]))
    e_t = float(np.linalg.norm(E[:3, 3]))
    e_r = math.acos(min(1.0, max(-1.0, (float(np.trace(E[:3, :3])) - 1.0) / 2.0)))
    return e_t, e_r


def cycle_length(i, j):
    return abs(i["da"] - j["da"]) + abs(i["db"] - j["db"])


def within(e_t, e_r, L, tol, mut=()):
    t0, r0, td, rd = (tol[k] for k in TOL_FIELDS)
    if "no_drift" in mut:
        L = 0.0
    return e_t <= t0 + td * L and e_r <= r0 + rd * L


def consistent(i, j, tol, mut=()):
    e_t, e_r = cycle_error(i, j, mut)
    return within(e_t, e_r, cycle_length(i, j), tol, mut)


def inliers(rows, tol, mut=()):
    """Indices of the greedy consistent set, in joining order: rows by (fitness, index), each kept iff consistent with every
    row kept before it."""
    key = (lambda r: (rows[r]["fitness"], -r)) if "tie_high" in mut else (lambda r: (rows[r]["fitness"], r))
    kept = []
    for r in sorted(range(len(rows)), key=key):
        if all(consistent(rows[q], rows[r], tol, mut) for q in kept):
            kept.append(r)
    return kept


def placement(T, Pb):
    return np.asarray(T, dtype=np.float64) @ np.asarray(Pb, dtype=np.float64)


def segment_edges(n, k, seg_first, mut=()):
    """The odometry edges (from, to) of the reference's rule applied inside each segment."""
    if "odometry_across" in mut:
        return PG.graph_edges(n, k)
    out = []
    bounds = list(seg_first) + [n]
    for s in range(len(seg_first)):
        f0 = bounds[s]
        out += [(f0 + f, f0 + t) for f, t in PG.graph_edges(bounds[s + 1] - f0, k)]
    return out


def joint_edges(poses, k, seg_first, loop_edges=(), mut=()):
    """(from, to, Z^-1) of the joint graph: per-segment odometry, then the loop edges (from, to, Z)."""
    inv, comp = PG.inverse, PG.compose
    E = [(f, t, inv(comp(inv(poses[f]), poses[t]))) for f, t in segment_edges(len(poses), k, seg_first, mut)]
    E += [(int(f), int(t), inv(np.asarray(Z, dtype=np.float64))) for f, t, Z in loop_edges]
    return E


def joint_adjust(poses, k, seg_first, loop_edges=(), max_iterations=10):
    return PG.optimize(poses, joint_edges(poses, k, seg_first, loop_edges), max_iterations)


# ---------------------------------------------------------------- the two-session drive of the end-to-end tests
A_IDX = list(range(SC.N_OUT))                       # the out-leg, drive indices 0..15
B_IDX = list(range(SC.N_OUT, 2 * SC.N_OUT - 1))     # the back-leg, 16..30
FOREIGN = synth.pose_matrix((50.0, -20.0, 0.0), (0.0, 0.0, math.radians(100.0)))  # W: B's poses are W^-1 P


def b_bias():
    """A fifth of scancontextref.odometry_bias() per STEP metres."""
    return synth.pose_matrix((0.1, 0.0, 0.0), (0.0, 0.0, 0.006))


def travelled(poses):
    d = [0.0]
    for k in range(1, len(poses)):
        d.append(d[-1] + float(np.linalg.norm(poses[k][:3, 3] - poses[k - 1][:3, 3])))
    return d


def sessions(poses):
    """(A poses, A distances, B poses in the foreign frame, B distances): A at the true poses of A_IDX, B integrated from
    the true relative motions of B_IDX with b_bias() per step, starting at W^-1 P_true."""
    A = [poses[k] for k in A_IDX]
    Bw = [poses[B_IDX[0]]]
    bias = b_bias()
    for a, b in zip(B_IDX[:-1], B_IDX[1:]):
        rel = np.linalg.inv(poses[a]) @ poses[b]
        Bw.append(Bw[-1] @ rel @ bias)
    Winv = np.linalg.inv(FOREIGN)
    B = [Winv @ P for P in Bw]
    return A, travelled(A), B, travelled(B)


def true_match(poses, b):
    """The A submap nearest to B submap b's true position."""
    p = poses[B_IDX[b]][:3, 3]
    return int(np.argmin([np.linalg.norm(poses[a][:3, 3] - p) for a in A_IDX]))


def unrelated_scene(stream=77):
    """A field of scattered boxes and posts with no facades and no pilasters: nothing in it repeats synth.make_scene()."""
    r = synth.Rng(stream)
    u = r.uniform(70 * 6).reshape(70, 6)
    boxes = []
    for k in range(70):
        lx, ly, lz = 2.0 + 9.0 * u[k, 0], 2.0 + 9.0 * u[k, 1], 1.0 + 7.0 * u[k, 2]
        cx, cy = -110.0 + 220.0 * u[k, 3], -45.0 + 90.0 * u[k, 4]
        if abs(cy) < 4.0:  # the road
            cy += 8.0 if cy >= 0 else -8.0
        boxes.append([cx - lx / 2, cy - ly / 2, 0.0, cx + lx / 2, cy + ly / 2, lz])
    u = r.uniform(40 * 4).reshape(40, 4)
    cyl = [[-110.0 + 220.0 * u[k, 0], (6.0 + 30.0 * u[k, 1]) * (1 if u[k, 2] < 0.5 else -1), 0.3, 2.0 + 8.0 * u[k, 3]]
           for k in range(40)]
    return synth.Scene(boxes=np.array(boxes), cylinders=np.array(cyl), facade_y=1.0e6, facade_h=0.0,
                       y_range=(-60.0, 60.0))
