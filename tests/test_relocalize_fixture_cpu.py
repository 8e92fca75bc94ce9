"""The canyon fixture of tests/test_gpu_relocalize.py checked on the CPU with the host compile of csrc/relocalize.hpp: the
scan filtered as the session filters it (range filter, VoxelGrid(vg_size_for_input)), the search started from the far
pose with the heading wrong, and the first ranked tile's best leaf within one cell and one heading step of the truth. So
a GPU run that adopts a pose far from the truth here has a wrong search or a wrong refinement, not an ambiguous scene.
Needs no GPU."""
import math

import numpy as np

import gridref as G
import relocref as R
import sessionref as S
import test_gpu_localize as TL
import test_relocalize_cpu as RC
from test_gpu_relocalize import FAR, _start

F32 = np.float32


def test_first_tile_holds_the_truth(tmp_path_factory):
    rl = RC.build_host_lib(tmp_path_factory.mktemp("rlf"))
    prior = TL.canyon_map()
    p = dict(R.DEFAULTS)
    host = RC.Host(rl, prior, p)
    assert not host.refused
    for f in (0, 2, 5):
        scan, T_true = TL.drive(6)[f]
        kept = scan[S.range_keep(scan, TL.KW["scan_min_range"], TL.KW["scan_max_range"])]
        src = G.voxelgrid_ref(kept, TL.KW["vg_size_for_input"])[0].astype(F32)
        pos, quat = _start(T_true, *FAR)
        assert host.set_scan(src, pos, quat) > 0
        res = host.search()
        idx = R.key_index(res["keys"][0])
        W, H = host.grid["W"], host.grid["H"]
        k, i, j = idx // (W * H), idx % W, (idx // W) % H
        ti = math.floor(T_true[0, 3] / p["resolution"]) - host.grid["i0"]
        tj = math.floor(T_true[1, 3] / p["resolution"]) - host.grid["j0"]
        yaw_k = math.atan2(*reversed(R.rotations(pos, quat, p["yaw_steps"])[0][k][:2, 0]))
        dyaw = abs(math.remainder(yaw_k - math.atan2(T_true[1, 0], T_true[0, 0]), 2 * math.pi))
        print(f"\nframe {f}: first tile's leaf ({k}, {i}, {j}) score {res['keys'][0] >> 40} of m {host.m}; truth cell ({ti}, {tj}), "
              f"heading off by {dyaw:.4f} rad; T0 {res['t0']} T {res['t']} nodes {res['nodes'][:6]}")
        assert abs(i - ti) <= 1 and abs(j - tj) <= 1 and dyaw <= 2 * math.pi / p["yaw_steps"], f
