"""GPU parity at BASELINE.json's full sizes for config 4 (loop-closure pairs: 32-ring scan ~56k pts vs 200k-pt local map,
NDT res 2.0, max_iter 100 as graph_based_slam_component.cpp:66) and config 5 (streaming frontend: 32 x 1875 rays per frame,
VoxelGrid 0.2 + NDT res 5.0 per frame, map update every 1.5 m with VoxelGrid 0.1 and the last 10 submaps, lidarslam.yaml) —
the CPU oracle runs a bounded sample of each (seconds), the GPU the same and more. Tolerance: 1e-3 m / 1e-3 rad."""
import os

import numpy as np
import pytest

import oracle
import oracle.scanmatcher as osm
from lidarslam_ros2_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    oracle.build()
    return m


def _threads():
    try:
        return len(os.sched_getaffinity(0))
    except Exception:
        return os.cpu_count() or 1


def test_c4_full_size_pairs(b200):
    """Four of the 64 loop-closure pairs at full size through the sweep entry point (b200reg_ndt_sweep) and, pair by pair,
    through the CPU path: pose, iteration count, convergence flag and fitness."""
    from concurrent.futures import ProcessPoolExecutor

    from lidarslam_ros2_b200 import batch

    idx = [0, 21, 42, 63]
    with ProcessPoolExecutor(max_workers=4) as ex:
        pairs = list(ex.map(_pair, idx))
    sw = batch.LoopSweep(b200, device=0, resolution=2.0, max_iterations=100)
    rows = batch.unpack_rows(sw.run([p[0] for p in pairs], [p[1] for p in pairs], idx))
    o = oracle.NDT(resolution=2.0, transformation_epsilon=0.01, max_iterations=100, search_method=oracle.DIRECT7, num_threads=_threads())
    for k, (src, tgt, T_rel) in enumerate(pairs):
        o.set_target(tgt)
        o.set_source(src)
        To = o.align()
        dt, dr = synth.pose_error(rows["pose"][k], To)
        assert dt < 1e-3 and dr < 1e-3, (idx[k], dt, dr)
        assert int(rows["iterations"][k]) == o.iterations and bool(rows["converged"][k]) == o.converged
        fo = o.fitness()
        assert abs(float(rows["fitness"][k]) - fo) <= 1e-3 * fo
        et, er = synth.pose_error(rows["pose"][k], T_rel)
        assert et < 0.2 and er < 1e-2  # it is a registration: close to the pose the scan was ray-cast from


def _pair(i):
    _, src, tgt, T_rel = next(iter(synth.loop_closure_pairs(64, first=i, count=1)))
    return src, tgt, T_rel


def test_c5_stream_full_frame_size(b200):
    """Config 5 at the BASELINE frame size: 40 frames of 32 x 1875 rays down the canyon through b200sm_receive_cloud with the
    node's parameters; the CPU restatement of the same callback follows the first 12 frames (several map updates) and must
    agree per frame; the remaining frames must keep tracking the ground truth."""
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    kw = dict(ndt_resolution=5.0, vg_size_for_input=0.2, vg_size_for_map=0.1, trans_for_mapupdate=1.5, num_targeted_cloud=10)
    frames = list(synth.drive_stream(40, rings=32, azimuths=1875, step=0.5, workers=min(32, _threads())))
    g = ScanMatcher(device=0, **kw)
    o = osm.ScanMatcher(num_threads=_threads(), **kw)
    n_upd = 0
    for k, (scan, T_gt) in enumerate(frames):
        pg, Tg, ug = g.receiveCloud(scan)
        n_upd += int(ug)
        if k < 12:
            po, To, uo = o.receive_cloud(scan)
            assert ug == uo, k
            dt, dr = synth.pose_error(Tg, To)
            assert dt < 1e-3 and dr < 1e-3, (k, dt, dr)
            assert np.abs(pg - po).max() < 1e-3
        et, er = synth.pose_error(Tg, T_gt)
        assert et < 0.25 and er < 1e-2, (k, et, er)
    assert n_upd >= 10 and g.numSubmaps() == n_upd + 1
