"""GPU parity of the IMU de-skew (SURVEY.md §8f row 4): b200sm_imu_* against the literal sequential restatement of
LidarUndistortion::getImu / adjustDistortion (oracle/deskew.py; lidar_undistortion.hpp:52-226).

Tolerances: ring state and corrected coordinates to float rounding (the kernels evaluate atan2 / sin / cos in double and
round, glibc / numpy evaluate them in float: <= 1-2 ulp apart) — 2e-4 m on 5..25 m ranges; the carried ring pointers
(imu_ptr_front_, imu_ptr_last_iter_) and the set of untouched points exactly."""
import numpy as np
import pytest

from oracle import deskew
from test_deskew_oracle import _spinning_scan

pytestmark = pytest.mark.gpu


def _feed(objs, t0, n, dt=0.01, seed=0):
    rng = np.random.default_rng(seed)
    yaw = 0.0
    for k in range(n):
        yaw += 0.4 * dt
        q = np.array([0.01 * np.sin(0.1 * k), 0.02 * np.cos(0.07 * k), np.sin(yaw / 2), np.cos(yaw / 2)])
        q /= np.linalg.norm(q)
        w = np.array([0.02, -0.01, 0.4]) + 0.01 * rng.normal(size=3)
        a = np.array([0.5, 0.1, 9.8]) + 0.05 * rng.normal(size=3)
        for o in objs:
            (o.get_imu if hasattr(o, "get_imu") else o.getImu)(w, a, q, t0 + k * dt)


@pytest.fixture(scope="module")
def sm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


def test_imu_ring_state_matches_oracle(sm):
    g, o = sm.LidarUndistortion(scan_period=0.1), deskew.LidarUndistortion(scan_period=0.1)
    _feed([g, o], t0=50.0, n=260)  # wraps the 200-entry ring
    assert g.pointers() == (o.ptr_front, o.ptr_last, o.ptr_last_iter)
    for k in range(deskew.QUE):
        t, rpy, sh, ve = g.sample(k)
        assert t == o.time[k]
        np.testing.assert_allclose(rpy, [o.roll[k], o.pitch[k], o.yaw[k]], rtol=0, atol=3e-7)
        np.testing.assert_allclose(sh, o.shift[k], rtol=2e-6, atol=1e-7)
        np.testing.assert_allclose(ve, o.velo[k], rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("scan_time_offset", [0.20, 0.95, -0.03, 1.5])  # mid coverage, off the end, before the start, outside
def test_adjust_distortion_parity(sm, scan_time_offset):
    g, o = sm.LidarUndistortion(scan_period=0.1), deskew.LidarUndistortion(scan_period=0.1)
    _feed([g, o], t0=100.0, n=100)
    cloud = _spinning_scan(n=24000, rings=16)
    for rep in range(2):  # the second scan continues from the carried pointer
        st = 100.0 + scan_time_offset + 0.1 * rep
        a = o.adjust_distortion(cloud, st)
        b = g.adjustDistortion(cloud, st)
        assert g.pointers() == (o.ptr_front, o.ptr_last, o.ptr_last_iter), (rep, scan_time_offset)
        np.testing.assert_array_equal(b[:, 3], cloud[:, 3])
        untouched_o = np.all(a[:, :3] == cloud[:, :3], axis=1)
        untouched_g = np.all(b[:, :3] == cloud[:, :3], axis=1)
        assert np.mean(untouched_o != untouched_g) < 1e-3  # a point the correction moves by < 1 ulp may read as untouched
        assert np.abs(a[:, :3] - b[:, :3]).max() < 2e-4
    if scan_time_offset == 0.20:
        assert np.linalg.norm(b[-50:, :3] - cloud[-50:, :3], axis=1).mean() > 0.01  # the sweep's tail really moved


def test_no_imu_means_no_change(sm):
    g = sm.LidarUndistortion()
    cloud = _spinning_scan(400)
    np.testing.assert_array_equal(g.adjustDistortion(cloud, 1.0), cloud)
    o = deskew.LidarUndistortion()
    o.adjust_distortion(cloud, 1.0)
    assert g.pointers() == (o.ptr_front, o.ptr_last, o.ptr_last_iter)


def test_deskew_inside_the_frontend_frame(sm):
    """b200sm_deskew_next_scan: the next uploaded frame is de-skewed on the device before the filters (sm.cpp:205-219).
    The 3 cm input VoxelGrid over a ~50 m scan also takes the sparse two-level rank index (29 M dense words > budget)."""
    import oracle as oracle_pkg

    oracle_pkg.build()
    s = sm.ScanMatcher(device=0, ndt_resolution=2.0, vg_size_for_input=0.03, vg_size_for_map=0.1)
    imu = sm.LidarUndistortion(session=s._h)
    o = deskew.LidarUndistortion(scan_period=0.1)
    _feed([imu, o], t0=10.0, n=100)
    cloud = _spinning_scan(n=8000, rings=8)
    want = oracle_pkg.voxelgrid(o.adjust_distortion(cloud, 10.3), 0.03)
    plain = oracle_pkg.voxelgrid(cloud, 0.03)
    s.deskewNextScan(10.3)
    n_f = s.setScan(cloud)
    got = s.filteredScan()
    assert n_f == len(got) and abs(len(got) - len(want)) <= 2
    if len(got) == len(want):
        assert np.abs(got[:, :3] - want[:, :3]).max() < 5e-4
        assert len(plain) != len(want) or np.abs(got[:, :3] - plain[:, :3]).max() > 1e-2  # it really was de-skewed
    assert imu.pointers() == (o.ptr_front, o.ptr_last, o.ptr_last_iter)
    # the following frame is NOT de-skewed unless armed again
    s.setScan(cloud)
    got2 = s.filteredScan()
    assert len(got2) == len(plain) and np.abs(got2[:, :3] - plain[:, :3]).max() < 5e-5
