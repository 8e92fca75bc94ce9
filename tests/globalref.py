"""TEST INFRASTRUCTURE. A float64 replay of the hypothesis grid and the top-k choice of b200sm_localize_global
(csrc/global_grid.hpp; the contract is include/b200reg.h's). Python floats are IEEE doubles and every expression is
evaluated as written, un-fused; math.cos / math.sin are the C library's, as std::cos / std::sin are in the library, so
the tests compare the header with this replay bit for bit.

Every function takes `mut`, a set of mutation names (MUTATIONS): a replay of a subtly wrong grid or choice, used by
tests/test_global_grid_cpu.py to show that the fixtures tell it from the right one. Nothing here needs a GPU.
"""
from __future__ import annotations

import math

import numpy as np

import sessionref as S

F32 = np.float32
MAX_K, MAX_HYP, MAX_YAW, MAX_TOP = 4096, 1 << 24, 4096, 1024

MUTATIONS = (
    "yaw_outer",  # hypothesis k = m * positions + position_index: the yaw loop outside the position loop
    "disc_lt",    # `<` instead of `<=` on the disc
    "tie_high",   # the higher hypothesis index first among equal scores
)


def positions(radius, step, mut=()):
    """[(i, j)] of the kept positions, j outer and i inner, or None when a field is invalid or K > 4096."""
    radius, step = float(radius), float(step)
    if not (math.isfinite(radius) and math.isfinite(step) and radius >= 0 and step > 0):
        return None
    kd = math.floor(radius / step) if math.isfinite(radius / step) else math.inf
    if not kd <= MAX_K:
        return None
    K = int(kd)
    r2 = radius * radius
    out = []
    for j in range(-K - 1, K + 2):
        b = float(j) * step
        bb = b * b
        a = np.arange(-K - 1, K + 2, dtype=np.float64) * step
        d2 = a * a + bb
        keep = (d2 < r2) if "disc_lt" in mut else (d2 <= r2)
        out.extend((int(i), j) for i in np.flatnonzero(keep) - K - 1)
    return out


def count(radius, step, yaw_steps, top_k, mut=()) -> int:
    """hypotheses of a spec, -1 when it is invalid"""
    if not (1 <= yaw_steps <= MAX_YAW and 1 <= top_k <= MAX_TOP):
        return -1
    p = positions(radius, step, mut)
    if p is None or len(p) * yaw_steps > MAX_HYP:
        return -1
    return len(p) * yaw_steps


def grid(position, quat, radius, step, yaw_steps, mut=()) -> np.ndarray:
    """(H, 4, 4) float32 hypotheses around the pose (position, quaternion xyzw)."""
    M = S.pose_matrix(position, quat)
    P = positions(radius, step, mut)
    rots = []
    for m in range(yaw_steps):
        th = 2.0 * math.pi * m / yaw_steps
        c, s = math.cos(th), math.sin(th)
        Rz = ((c, -s, 0.0), (s, c, 0.0), (0.0, 0.0, 1.0))
        rots.append([[Rz[r][0] * M[0, col] + Rz[r][1] * M[1, col] + Rz[r][2] * M[2, col] for col in range(3)] for r in range(3)])
    out = np.zeros((len(P) * yaw_steps, 4, 4), dtype=F32)
    for q, (i, j) in enumerate(P):
        t = (M[0, 3] + float(i) * step, M[1, 3] + float(j) * step, M[2, 3])
        for m in range(yaw_steps):
            k = m * len(P) + q if "yaw_outer" in mut else q * yaw_steps + m
            out[k, :3, :3] = np.array(rots[m], dtype=np.float64).astype(F32)
            out[k, :3, 3] = np.array(t, dtype=np.float64).astype(F32)
            out[k, 3, 3] = 1.0
    return out


def select(scores, top_k, mut=()) -> list:
    """The top_k highest scores in descending order, the lower index first among equal scores."""
    s = np.asarray(scores, dtype=np.float64)
    idx = np.arange(len(s))
    order = np.lexsort((-idx if "tie_high" in mut else idx, -s))
    return [int(v) for v in order[:min(top_k, len(s))]]
