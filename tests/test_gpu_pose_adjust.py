"""Backend pose adjustment on the session (b200sm_pose_adjust, b200sm_assemble_map): doPoseAdjustment's solve against the
float64 restatement tests/posegraphref.py, and the map assembly kernel bitwise against pcl::transformPointCloud(Matrix4f)
restated in numpy (oracle/scanmatcher.py transform_f32)."""
import ctypes as C

import numpy as np
import pytest

import oracle.scanmatcher as osm
import posegraphref as R
from lidarslam_ros2_b200 import _capi, synth
from lidarslam_ros2_b200.registration import B200RegError
from test_posegraph_cpu import LOOP_ARGS, drift
from test_scanmatcher import _out_and_back

pytestmark = pytest.mark.gpu
KW = dict(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _expected_map(sm, poses=None):
    parts, sizes = [], []
    for i in range(sm.numSubmaps()):
        cloud, M, _ = sm.submap(i)
        P = M if poses is None else poses[i]
        parts.append(osm.transform_f32(cloud, P.astype(np.float32)))
        sizes.append(len(cloud))
    return np.concatenate(parts, axis=0), np.concatenate([[0], np.cumsum(sizes)])


def _drifted_session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher(**KW)
    truth = []
    for k, (scan, T) in enumerate(_out_and_back()):
        Td = drift(k) @ T
        g.setScan(scan)
        g.updateMap(Td.astype(np.float32), Td[:3, 3], osm.quat_from_matrix(Td[:3, :3]), adopt_now=False)
        truth.append(T)
    return g, truth


def test_assemble_map_with_the_session_poses_is_bitwise_pcl():
    g, _ = _drifted_session()
    want, want_off = _expected_map(g)
    got, off = g.assembleMap()
    assert got.dtype == np.float32 and got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert off.tolist() == want_off.tolist()
    part, _ = g.assembleMap(capacity=1000)  # a smaller capacity copies exactly that many points, the total is still reported
    assert len(part) == 1000 and np.array_equal(part.view(np.uint32), want[:1000].view(np.uint32))
    L = _capi.lib()
    n = C.c_size_t(0)
    buf = np.zeros((10, 4), dtype=np.float32)
    assert L.b200sm_assemble_map(g._h, None, buf.ctypes.data, 10, C.byref(n), None) == 0
    assert n.value == len(want) and np.array_equal(buf.view(np.uint32), want[:10].view(np.uint32))


def test_drifted_drive_loop_closure_and_adjustment():
    from lidarslam_ros2_b200.scanmatcher import backend_registration

    g, truth = _drifted_session()
    ref, _ = _drifted_session()  # the same drive, never adjusted
    reg = backend_registration("NDT", ndt_resolution=2.0)
    r = g.searchLoop(reg, **LOOP_ARGS)
    assert r["accepted"] and r["id_min"] == 0, r
    n = g.numSubmaps()
    loops = [(r["id_min"], n - 1, r["relative_pose"])]
    session_poses = [g.submap(i)[1] for i in range(n)]
    poses, res = g.poseAdjust(loops)
    Xo, ro, _ = R.pose_adjust(session_poses, 5, loops, 10)
    for a, b in zip(poses, Xo):
        dt, dr = synth.pose_error(a, b)
        assert dt < 1e-9 and dr < 1e-9, (dt, dr)
    assert res["n_vertices"] == n and res["n_edges"] == len(R.build_edges(session_poses, 5, loops))
    assert abs(res["chi2_initial"] - ro["chi2_initial"]) <= 1e-12 * ro["chi2_initial"]
    assert res["chi2_final"] < res["chi2_initial"] and 1 <= res["iterations"] <= 10 and res["trials"] >= res["iterations"]
    np.testing.assert_array_equal(poses[0], session_poses[0])  # vertex 0 is fixed
    before, after = synth.pose_error(session_poses[-1], truth[-1]), synth.pose_error(poses[-1], truth[-1])
    assert after[0] < 0.5 * before[0] and after[1] < 0.5 * before[1], (before, after)

    got, off = g.assembleMap(poses)
    want, want_off = _expected_map(g, poses)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)) and off.tolist() == want_off.tolist()

    # the session keeps the frontend's poses: submaps and the next loop search are those of the session never adjusted
    for i in range(n):
        a, b = g.submap(i), ref.submap(i)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0], b[0])
    ra, rb = g.searchLoop(reg, **LOOP_ARGS), ref.searchLoop(reg, **LOOP_ARGS)
    assert np.array_equal(ra["final"], rb["final"]) and ra["fitness"] == rb["fitness"]
    assert np.array_equal(ra["relative_pose"], rb["relative_pose"])


def test_pose_adjust_without_loops_and_argument_errors():
    g, _ = _drifted_session()
    n = g.numSubmaps()
    session_poses = np.array([g.submap(i)[1] for i in range(n)])
    poses, res = g.poseAdjust([])
    assert np.array_equal(poses, session_poses) and res["chi2_initial"] == 0.0 and res["chi2_final"] == 0.0
    for bad in ([(0, n, np.eye(4))], [(-1, 3, np.eye(4))], [(2, 2, np.eye(4))], [(0, n - 1, np.full((4, 4), np.nan))]):
        with pytest.raises(B200RegError) as e:
            g.poseAdjust(bad)
        assert e.value.code == _capi.ERR_ARG
    for kwargs in (dict(num_adjacent_pose_cnstraints=0), dict(max_iterations=-1)):
        with pytest.raises(B200RegError) as e:
            g.poseAdjust([], **kwargs)
        assert e.value.code == _capi.ERR_ARG
    poses0, res0 = g.poseAdjust([(0, n - 1, np.eye(4))], max_iterations=0)
    assert np.array_equal(poses0, session_poses) and res0["iterations"] == 0


def test_assemble_twenty_million_points_in_one_launch():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    rng = np.random.default_rng(5)
    g = ScanMatcher(**KW)
    n_sub, n_pts = 1000, 20_000
    clouds, poses = [], []
    for i in range(n_sub):
        c = np.concatenate([rng.uniform(-50, 50, size=(n_pts, 3)), rng.uniform(0, 255, size=(n_pts, 1))], axis=1).astype(np.float32)
        M = synth.pose_matrix(rng.normal(size=3) * 100.0, rng.uniform(-np.pi, np.pi, size=3))
        g.importSubmap(c, M, float(i))
        clouds.append(c)
        poses.append(M)
    adjusted = [synth.pose_matrix(rng.normal(size=3) * 100.0, rng.uniform(-np.pi, np.pi, size=3)) for _ in range(n_sub)]
    before = g.stats()["kernel_launches"]
    got, off = g.assembleMap(adjusted)
    assert g.stats()["kernel_launches"] - before == 1
    assert len(got) == n_sub * n_pts and off.tolist() == list(range(0, n_sub * n_pts + 1, n_pts))
    for i in range(n_sub):
        want = osm.transform_f32(clouds[i], adjusted[i].astype(np.float32))
        assert np.array_equal(got[off[i]:off[i + 1]].view(np.uint32), want.view(np.uint32)), i
