"""The recovery fixture of tests/test_gpu_localize_global.py checked on the CPU with the float64 NDT reference
(tests/ndtref.py): scored as the session scores it (the cut of the canyon map around the start, the range-filtered and
VoxelGrid-filtered scan, DIRECT7 at resolution 2), the hypothesis of the grid nearest the true pose outscores every other
yaw at its position, every other position at its yaw, and a random sample of the rest. So a session that adopts a pose far
from the truth on this fixture has a wrong score or a wrong choice, not an ambiguous scene. Needs no GPU."""
import math

import numpy as np

import globalref as GR
import gridref as R
import localizeref as L
import ndtref as N
import sessionref as S
import test_gpu_localize as TL
from test_gpu_localize_global import RECOVERY, _start

F32 = np.float32


def test_nearest_hypothesis_scores_highest():
    prior = TL.canyon_map()
    scan, T_true = TL.drive(6)[2]
    offset, dyaw, radius, step, yaw_steps = RECOVERY
    pos, quat = _start(T_true, offset, dyaw)
    cut = prior[L.cut_mask(prior, pos[0], pos[1], TL.CROP)][:, :3]
    kept = scan[S.range_keep(scan, TL.KW["scan_min_range"], TL.KW["scan_max_range"])]
    src = R.voxelgrid_ref(kept, TL.KW["vg_size_for_input"])[0][:, :3].astype(F32)
    res = TL.KW["ndt_resolution"]
    vox, geom = R.voxel_map_ref(cut, res), R.leaf_geometry(cut, res)
    grid = GR.grid(pos, quat, radius, step, yaw_steps)
    n_pos = len(grid) // yaw_steps
    # the hypothesis nearest the truth: the position nearest it and, there, the yaw nearest its heading
    d = np.hypot(grid[::yaw_steps, 0, 3] - T_true[0, 3], grid[::yaw_steps, 1, 3] - T_true[1, 3])
    q = int(np.argmin(d))
    yaw_true = math.atan2(T_true[1, 0], T_true[0, 0])
    yaws = np.arctan2(grid[q * yaw_steps:(q + 1) * yaw_steps, 1, 0], grid[q * yaw_steps:(q + 1) * yaw_steps, 0, 0])
    m = int(np.argmin(np.abs(np.angle(np.exp(1j * (yaws - yaw_true))))))
    near = q * yaw_steps + m
    assert d[q] < 0.5 * step and abs(np.angle(np.exp(1j * (yaws[m] - yaw_true)))) < math.pi / yaw_steps
    rng = np.random.default_rng(5)
    others = set(range(q * yaw_steps, (q + 1) * yaw_steps)) | set(range(m, len(grid), yaw_steps))
    others |= set(int(k) for k in rng.choice(len(grid), 200, replace=False))
    others.discard(near)

    def score(k):
        return N.derivatives(src, grid[k][:3], np.zeros(6), res, vox, geom, N.DIRECT7, compute_hessian=False)["score"]

    best = score(near)
    worst_gap = min(best - score(k) for k in sorted(others))
    print(f"\nnearest hypothesis {near} (position {q} of {n_pos}, {d[q]:.3f} m; yaw {m}): score {best:.1f}, "
          f"smallest lead over {len(others)} others {worst_gap:.1f}")
    assert worst_gap > 0
