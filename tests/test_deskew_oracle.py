"""oracle/deskew.py: the sequential restatement of LidarUndistortion::adjustDistortion (lidar_undistortion.hpp:110-226) and
its data-parallel reformulation (first-index reduction for the half-turn switch, prefix-max for the carried IMU pointer) must
agree exactly — the groundwork for the GPU kernel of SURVEY.md §8f row 4."""
import copy

import numpy as np
import pytest

from oracle import deskew


def _imu_stream(u, t0, n, dt=0.01, seed=0):
    rng = np.random.default_rng(seed)
    yaw = 0.0
    for k in range(n):
        yaw += 0.4 * dt
        q = np.array([0.01 * np.sin(0.1 * k), 0.02 * np.cos(0.07 * k), np.sin(yaw / 2), np.cos(yaw / 2)])
        q /= np.linalg.norm(q)
        u.get_imu(np.array([0.02, -0.01, 0.4]) + 0.01 * rng.normal(size=3), np.array([0.5, 0.1, 9.8]) + 0.05 * rng.normal(size=3),
                  q, t0 + k * dt)


def _spinning_scan(n=2400, rings=4, seed=1):
    """Points in firing order of a clockwise-spinning multi-beam LiDAR: azimuth sweeps one full turn."""
    rng = np.random.default_rng(seed)
    per = n // rings
    az = -np.linspace(0.05, 2 * np.pi - 0.05, per)  # clockwise
    pts = []
    for j in range(per):
        for r in range(rings):
            d = 5.0 + 20.0 * rng.random()
            el = np.deg2rad(-10 + 5 * r)
            pts.append([d * np.cos(el) * np.cos(az[j]), d * np.cos(el) * np.sin(az[j]), d * np.sin(el), rng.random()])
    return np.array(pts, dtype=np.float32)


@pytest.mark.parametrize("scan_time_offset", [0.20, 0.95, -0.03, 1.5])  # mid coverage, running off the end, before the start, outside
def test_parallel_form_equals_sequential(scan_time_offset):
    u = deskew.LidarUndistortion(scan_period=0.1)
    _imu_stream(u, t0=100.0, n=100)
    v = copy.deepcopy(u)
    cloud = _spinning_scan()
    a = u.adjust_distortion(cloud, 100.0 + scan_time_offset)
    b = v.adjust_distortion_parallel(cloud, 100.0 + scan_time_offset)
    np.testing.assert_array_equal(a, b)
    assert (u.ptr_front, u.ptr_last_iter) == (v.ptr_front, v.ptr_last_iter)
    # a second scan continues from the carried pointer
    a2 = u.adjust_distortion(cloud, 100.0 + scan_time_offset + 0.1)
    b2 = v.adjust_distortion_parallel(cloud, 100.0 + scan_time_offset + 0.1)
    np.testing.assert_array_equal(a2, b2)
    assert (u.ptr_front, u.ptr_last_iter) == (v.ptr_front, v.ptr_last_iter)


def test_deskew_moves_points_by_the_sensor_motion():
    """With IMU coverage the late points of the sweep are rotated back by the yaw the sensor gained since the first point."""
    u = deskew.LidarUndistortion(scan_period=0.1)
    _imu_stream(u, t0=10.0, n=100)
    cloud = _spinning_scan()
    out = u.adjust_distortion(cloud, 10.3)
    moved = np.linalg.norm(out[:, :3] - cloud[:, :3], axis=1)
    assert moved[0] == 0.0 and np.array_equal(out[:, 3], cloud[:, 3])
    assert moved[-100:].mean() > 5 * moved[4:104].mean() > 0  # grows along the sweep
    # yaw rate 0.4 rad/s over ~0.1 s of sweep on 5..25 m ranges: centimetres to a metre, not more
    assert 0.02 < moved[-100:].mean() < 1.5


def test_no_imu_means_no_change():
    u = deskew.LidarUndistortion()
    cloud = _spinning_scan(400)
    np.testing.assert_array_equal(u.adjust_distortion(cloud, 1.0), cloud)
    np.testing.assert_array_equal(u.adjust_distortion_parallel(cloud, 1.0), cloud)


@pytest.mark.parametrize("scan_time_offset", [0.20, 0.95])  # mid coverage, running off the end
def test_parallel_form_equals_sequential_with_nan_ray(scan_time_offset):
    """A NaN ray (fromROSMsg of an organised cloud keeps them): the walk runs to the newest sample for it and carries
    that pointer; the parallel form's lower bound (searchsorted sorts NaN last) does the same."""
    u = deskew.LidarUndistortion(scan_period=0.1)
    _imu_stream(u, t0=100.0, n=100)
    v = copy.deepcopy(u)
    cloud = _spinning_scan()
    cloud[700, :3] = np.nan
    for rep in range(2):
        a = u.adjust_distortion(cloud, 100.0 + scan_time_offset + 0.1 * rep)
        b = v.adjust_distortion_parallel(cloud, 100.0 + scan_time_offset + 0.1 * rep)
        np.testing.assert_array_equal(a, b)
        assert (u.ptr_front, u.ptr_last_iter) == (v.ptr_front, v.ptr_last_iter)
