"""A float64 numpy replay of the place search of b200sm_search_loop_place (csrc/scan_context.hpp): Scan Context bins by
atan2 / sqrt, the column norms, the distance at every shift, the best shift and the ranking; the guess of the verification;
and the ray-cast drive with odometry drift that the end-to-end tests close a loop on.

MUTATIONS names subtly wrong variants of the replay, each of which the CPU tests show changes an outcome:
  shift_reversed  newest column j compared with candidate column j - s instead of j + s
  any_nonzero     a column pair counts when either norm is non-zero (cos 0 for the other), not only when both are
  ring_exclusive  a point exactly on a ring bound t_k stays in the inner ring
  tie_high        among equal distances the highest shift wins
"""
from __future__ import annotations

import math

import numpy as np

from lidarslam_ros2_b200 import synth

MUTATIONS = ("shift_reversed", "any_nonzero", "ring_exclusive", "tie_high")
DEFAULTS = dict(num_rings=20, num_sectors=60, max_radius=80.0, lidar_height=2.0)


def bins(points, num_rings=20, num_sectors=60, max_radius=80.0, mut=()):
    """(ring, sector) of every row by r = sqrt(x^2 + y^2) and atan2; -1, -1 for a skipped row (non-finite, r > max_radius)."""
    p = np.asarray(points, dtype=np.float32)[:, :3].astype(np.float64)
    ok = np.isfinite(p).all(axis=1)
    x, y = np.where(ok, p[:, 0], 0.0), np.where(ok, p[:, 1], 0.0)
    r = np.sqrt(x * x + y * y)
    ok &= r <= max_radius
    width = max_radius / num_rings
    if "ring_exclusive" in mut:
        ring = np.ceil(r / width).astype(np.int64) - 1
    else:
        ring = np.floor(r / width).astype(np.int64)
    ring = np.clip(ring, 0, num_rings - 1)
    a = np.arctan2(y, x)
    a = np.where(a < 0, a + 2 * math.pi, a)
    sector = np.clip(np.floor(a / (2 * math.pi / num_sectors)).astype(np.int64), 0, num_sectors - 1)
    sector = np.where((x == 0) & (y == 0), 0, sector)
    return np.where(ok, ring, -1), np.where(ok, sector, -1)


def edge_distance(points, num_rings=20, num_sectors=60, max_radius=80.0):
    """Distance of every row (x, y) to the nearest ring bound or sector edge, in metres (inf for a skipped row)."""
    p = np.asarray(points, dtype=np.float32)[:, :3].astype(np.float64)
    r = np.hypot(p[:, 0], p[:, 1])
    width = max_radius / num_rings
    dr = np.abs(r - np.round(r / width) * width)
    a = np.arctan2(p[:, 1], p[:, 0])
    sw = 2 * math.pi / num_sectors
    da = np.abs(a - np.round(a / sw) * sw) * r
    d = np.minimum(dr, da)
    return np.where(np.isfinite(p).all(axis=1) & (r <= max_radius), d, np.inf)


def descriptor(points, num_rings=20, num_sectors=60, max_radius=80.0, lidar_height=2.0, mut=()):
    """(num_rings, num_sectors) float32: the largest z + (float)lidar_height (in float) of each bin, 0 for an empty bin."""
    p = np.asarray(points, dtype=np.float32)
    ring, sector = bins(p, num_rings, num_sectors, max_radius, mut)
    keep = ring >= 0
    v = (p[keep, 2] + np.float32(lidar_height)).astype(np.float32)
    D = np.full(num_rings * num_sectors, -np.inf, dtype=np.float32)
    np.maximum.at(D, ring[keep] * num_sectors + sector[keep], v)
    D[D == -np.inf] = 0.0
    # the device orders +0 above -0: a bin whose maximum is a zero holds +0 when any of its points gives +0
    zero = np.zeros(num_rings * num_sectors, dtype=bool)
    np.logical_or.at(zero, ring[keep] * num_sectors + sector[keep], (v == 0) & ~np.signbit(v))
    D[zero & (D == 0)] = 0.0
    return D.reshape(num_rings, num_sectors)


def norms(D):
    D = np.asarray(D, dtype=np.float64)
    return np.sqrt((D * D).sum(axis=0))


def distances(Q, C, mut=()):
    """d_s for every shift s (float64)."""
    Q, C = np.asarray(Q, dtype=np.float64), np.asarray(C, dtype=np.float64)
    S = Q.shape[1]
    nQ, nC = norms(Q), norms(C)
    out = np.empty(S)
    j = np.arange(S)
    for s in range(S):
        c = (j - s) % S if "shift_reversed" in mut else (j + s) % S
        dots = (Q * C[:, c]).sum(axis=0)
        den = nQ * nC[c]
        if "any_nonzero" in mut:
            use = (nQ > 0) | (nC[c] > 0)
            cos = np.where(den > 0, dots / np.where(den > 0, den, 1.0), 0.0)
        else:
            use = (nQ > 0) & (nC[c] > 0)
            cos = dots / np.where(use, den, 1.0)
        m = int(use.sum())
        out[s] = 1.0 - cos[use].sum() / m if m else 1.0
    return out


def distance(Q, C, mut=(), tol=0.0):
    """(D, s*): the minimum over shifts and the lowest shift within `tol` of it (the highest under tie_high)."""
    d = distances(Q, C, mut)
    best = d.min()
    ties = np.flatnonzero(d <= best + tol)
    return float(best), int(ties[-1] if "tie_high" in mut else ties[0])


def rank(D, ids, threshold):
    """Indices into D of the rows with D < threshold, by (D, id) ascending."""
    rows = [r for r in range(len(D)) if D[r] < threshold]
    return sorted(rows, key=lambda r: (D[r], ids[r]))


def matmul_seq(A, B):
    """4x4 product with every entry summed k = 0..3 from 0, as the session's host code does (no FMA)."""
    out = [[0.0] * 4 for _ in range(4)]
    for r in range(4):
        for c in range(4):
            a = 0.0
            for k in range(4):
                a += float(A[r][k]) * float(B[k][c])
            out[r][c] = a
    return out


def iso_inverse(P):
    P = [[float(v) for v in row] for row in P]
    inv = [[P[0][0], P[1][0], P[2][0], 0.0], [P[0][1], P[1][1], P[2][1], 0.0], [P[0][2], P[1][2], P[2][2], 0.0],
           [0.0, 0.0, 0.0, 1.0]]
    for r in range(3):
        inv[r][3] = -(inv[r][0] * P[0][3] + inv[r][1] * P[1][3] + inv[r][2] * P[2][3])
    return inv


def guess(P_cand, P_new, shift, num_sectors):
    """G = P_cand * Rz(2 pi shift / num_sectors) * P_new^-1 in double, cast to float32 (4x4)."""
    th = 2.0 * 3.141592653589793 * float(shift) / float(num_sectors)
    c, s = math.cos(th), math.sin(th)
    Rz = [[c, -s, 0.0, 0.0], [s, c, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]
    return np.array(matmul_seq(matmul_seq(P_cand, Rz), iso_inverse(P_new)), dtype=np.float64).astype(np.float32)


# ---------------------------------------------------------------- the ray-cast drive of the end-to-end tests
STEP = 4.0          # metres between submaps
N_OUT = 16          # submaps down the canyon (x = -30 .. 30)
X0 = -30.0
REVISIT_YAW = 37.0  # degrees: the extra turn of the last revisit, not a multiple of a 6-degree sector


def drive_poses():
    """Ground-truth sensor poses (world frame, z = sensor height) of the drive: N_OUT submaps down the canyon heading +x,
    then back up the canyon heading -x (180 degrees off) 0.4 m to the side, the last one over the first submap and turned
    a further REVISIT_YAW degrees. Returns (poses, index of a 180-degree revisit, its true match, index of the turned
    revisit, its true match)."""
    d = math.pi / 180.0
    poses = []
    for k in range(N_OUT):
        poses.append(synth.pose_matrix((X0 + STEP * k, 0.0, synth.SENSOR_HEIGHT), (0.0, 0.0, 0.02 * math.sin(k))))
    for k in range(N_OUT - 2, -1, -1):
        yaw = math.pi + 0.02 * math.cos(k) + (REVISIT_YAW * d if k == 0 else 0.0)
        poses.append(synth.pose_matrix((X0 + STEP * k + 0.3, 0.4, synth.SENSOR_HEIGHT), (0.0, 0.0, yaw)))
    return poses, len(poses) - 2, 1, len(poses) - 1, 0


def odometry_bias():
    """The error odometry adds per STEP metres driven: 0.5 m too far and 0.03 rad of yaw to the left."""
    return synth.pose_matrix((0.5, 0.0, 0.0), (0.0, 0.0, 0.03))


def drive(rings=16, azimuths=450):
    """The drive's scans (sensor frame) and true poses, plus the indices of drive_poses()."""
    scene = synth.make_scene()
    poses, back, back_match, rev, rev_match = drive_poses()
    scans = [synth.make_scan(scene, rings, azimuths, P, stream=9100 + k) for k, P in enumerate(poses)]
    return scans, poses, (back, back_match, rev, rev_match)


def session(poses, indices):
    """The submaps a backend would hold after driving through `indices` of the drive: poses integrated from the true
    relative motions, each followed by odometry_bias() once per STEP metres, and the travelled distance along them."""
    drifted = [poses[indices[0]]]
    B = odometry_bias()
    for a, b in zip(indices[:-1], indices[1:]):
        rel = np.linalg.inv(poses[a]) @ poses[b]
        step = rel @ np.linalg.matrix_power(B, max(1, int(round(np.linalg.norm(rel[:3, 3]) / STEP))))
        drifted.append(drifted[-1] @ step)
    dist = [0.0]
    for k in range(1, len(drifted)):
        dist.append(dist[-1] + float(np.linalg.norm(drifted[k][:3, 3] - drifted[k - 1][:3, 3])))
    return drifted, dist


def sessions(back, rev):
    """The two searches of the end-to-end tests, each the list of drive indices of its submaps: the drive up to the
    180-degree revisit, and the whole drive with the turned revisit newest."""
    return [list(range(back + 1)), list(range(rev + 1))]


def true_shift(P_cand, P_new, num_sectors):
    """The newest sensor's heading relative to the candidate's, in sectors (real-valued, in [0, num_sectors))."""
    R = P_cand[:3, :3].T @ P_new[:3, :3]
    th = math.atan2(R[1, 0], R[0, 0]) % (2 * math.pi)
    return th / (2 * math.pi / num_sectors)
