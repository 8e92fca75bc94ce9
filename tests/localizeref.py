"""TEST INFRASTRUCTURE. A float64 replay of the localising frontend (csrc/scanmatcher.cu: b200sm_set_prior_map*,
b200sm_localize_cloud, b200sm_localize_init; the contract is include/b200reg.h's, the reference has no such mode), driven by
what the device hands back: its `final` of every frame and the rows of its batch call. Python floats and numpy float64
elementwise arithmetic are IEEE and un-fused, so every expression is evaluated exactly as written and the tests compare
the device with this replay bit for bit.

  cut_mask          the rows of the prior map a cut keeps
  Localizer         per frame: when a cut is made, around what, when it becomes the engine's target, the pose, the
                    distance from the cut's centre and the re-cut decision
  choose_hypothesis b200sm_localize_init's choice among the rows of the batch call

Every function takes `mut`, a set of mutation names (MUTATIONS): a replay of a subtly wrong session, used by
tests/test_localizeref_cpu.py to show that the fixtures tell such a session from the right one. Nothing here needs a GPU.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

import sessionref as S

F32 = np.float32

MUTATIONS = (
    "radius_lt",        # `<` instead of `<=` on the crop radius
    "recut_gt",         # `>` instead of `>=` in the re-cut decision
    "fused",            # dx * dx + dy * dy with one rounding (an FMA) in the cut's predicate
    "adopt_same_frame",  # the re-cut becomes the target in the frame that made it instead of the next one
    "tie_last",         # the highest index wins a tie among the hypotheses
    "with_z",           # z included in the cut's distance (a sphere instead of a cylinder)
)


def cut_mask(cloud, cx, cy, r, mut=(), cz=0.0) -> np.ndarray:
    """keep = dx * dx + dy * dy <= r * r with dx = (double)x - cx, dy = (double)y - cy. NaN rows fail the comparison;
    z is not looked at. The device keeps exactly these rows, in this order."""
    c = np.asarray(cloud, dtype=F32).reshape(-1, 4)
    cx, cy, r = float(cx), float(cy), float(r)
    r2 = r * r
    with np.errstate(invalid="ignore", over="ignore"):
        dx = c[:, 0].astype(np.float64) - cx
        dy = c[:, 1].astype(np.float64) - cy
        d2 = dx * dx + dy * dy
        if "fused" in mut:  # fma(dx, dx, dy * dy): exact product, one rounding; only rows at the edge can differ
            yy = dy * dy
            near = np.flatnonzero(np.isfinite(d2) & (np.abs(d2 - r2) <= 1e-12 * r2))
            for i in near:
                d2[i] = float(Fraction(float(dx[i])) * Fraction(float(dx[i])) + Fraction(float(yy[i])))
        if "with_z" in mut:
            dz = c[:, 2].astype(np.float64) - float(cz)
            d2 = d2 + dz * dz
        return (d2 < r2) if "radius_lt" in mut else (d2 <= r2)


def horizontal_distance(position, centre) -> float:
    dx, dy = float(position[0]) - float(centre[0]), float(position[1]) - float(centre[1])
    return math.sqrt(dx * dx + dy * dy)


class Localizer:
    """The host state of a localising session. `frame(final)` replays b200sm_localize_cloud given the float 4x4 `final`
    the device's align() returned for that frame; it returns None instead when the frame fails with ERR_NO_TARGET (the
    cut it had to make keeps no row), in which case nothing has changed."""

    def __init__(self, prior_map, crop_radius, recrop_distance, position=(0.0, 0.0, 0.0), quat_xyzw=(0.0, 0.0, 0.0, 1.0)):
        self.map = np.asarray(prior_map, dtype=F32).reshape(-1, 4)
        self.crop_radius, self.recrop_distance = float(crop_radius), float(recrop_distance)
        self.position = [float(v) for v in position]
        self.quat = [float(v) for v in quat_xyzw]
        self.have_cut, self.stale, self.pending = False, True, False
        self.centre = (0.0, 0.0)         # of the current cut
        self.target_centre = None        # of the cut the engine registers against
        self.mask = None                 # of the current cut
        self.n_cuts = 0
        self.dist = 0.0
        self.adopted_at = []             # (frame, centre) every time a cut became the target
        self.k = 0

    def set_initial_pose(self, position, quat_xyzw):
        self.position = [float(v) for v in position]
        self.quat = [float(v) for v in quat_xyzw]
        self.stale = True

    def set_prior_map(self, prior_map):
        self.map = np.asarray(prior_map, dtype=F32).reshape(-1, 4)
        self.stale, self.pending, self.n_cuts = True, False, 0

    def sim_trans(self) -> np.ndarray:
        return S.pose_matrix(self.position, self.quat).astype(F32)

    def _cut(self, mut) -> bool:
        m = cut_mask(self.map, self.position[0], self.position[1], self.crop_radius, mut, cz=self.position[2])
        if not m.any():
            return False
        self.mask, self.centre = m, (self.position[0], self.position[1])
        self.n_cuts += 1
        self.have_cut, self.stale, self.pending = True, False, True
        return True

    def _adopt(self):
        if self.pending:
            self.pending = False
            self.target_centre = self.centre
            self.adopted_at.append((self.k, self.centre))

    def begin(self, mut=()) -> bool:
        """step 2: the cut a frame needs before it can register. False: ERR_NO_TARGET."""
        if (not self.have_cut or self.stale) and not self._cut(mut):
            return False
        self._adopt()
        return True

    def adopt_pose(self, final):
        final = np.asarray(final, dtype=F32)
        self.quat = S.quat_from_rot(final[:3, :3])
        self.position = [float(final[r, 3]) for r in range(3)]

    def frame(self, final, mut=()):
        if not self.begin(mut):
            return None
        self.adopt_pose(final)
        self.dist = horizontal_distance(self.position, self.centre)
        again = (self.dist > self.recrop_distance) if "recut_gt" in mut else (self.dist >= self.recrop_distance)
        recut = bool(again and self._cut(mut))
        if recut and "adopt_same_frame" in mut:
            self._adopt()
        out = dict(pose7=np.array(self.position + self.quat), dist=self.dist, recut=recut, n_cuts=self.n_cuts,
                   centre=self.centre, pending=self.pending, target_centre=self.target_centre)
        self.k += 1
        return out

    def cut(self) -> np.ndarray:
        return self.map[self.mask]


def choose_hypothesis(rows, mut=()) -> int:
    """rows: (converged, trans_probability, status) per guess. The converged row with the highest probability, the lowest
    index on a tie; -1 when none converged."""
    best = -1
    for k, (conv, tp, status) in enumerate(rows):
        if status != 0 or not conv:
            continue
        if best < 0 or (tp >= rows[best][1] if "tie_last" in mut else tp > rows[best][1]):
            best = k
    return best
