"""The cloud callback's frame arithmetic on the CPU: the product's host header csrc/sensor_frame.hpp (the sensor-to-robot
matrix of tf2::doTransform, the point transform, the use_odom guess and its 4x4 inverse), compiled with g++, against the
float32 restatement tests/frontendref.py bit for bit; and the restated frontend with a mounted sensor and drifting
odometry tracking a drive."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import frontendref as fr
import oracle.scanmatcher as osm
from lidarslam_ros2_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))

# mapping_car.launch.py:27-28 mounts the LiDAR 1.2 m forward and 2.0 m up; a rotation is added so that every matrix entry
# takes part
MOUNT_POS = (1.2, 0.0, 2.0)
MOUNT_QUAT = osm.quat_from_matrix(synth.rpy_matrix(0.02, -0.04, 0.35))


@pytest.fixture(scope="module")
def sf():
    src = os.path.join(HERE, "hostmath", "sensor_frame_host.cpp")
    lib = os.path.join(HERE, "hostmath", "libsensor_frame_host.so")
    deps = [src] + [os.path.join(HERE, "..", "lidarslam_ros2_b200", "csrc", h) for h in ("sensor_frame.hpp", "pose_graph.hpp")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    return C.CDLL(lib)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _random_transforms(rng, n):
    t = rng.normal(size=(n, 3)) * rng.choice([0.01, 1.0, 100.0], size=(n, 1))
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[: n // 3] *= rng.uniform(0.5, 1.5, size=(n // 3, 1))  # non-unit quaternions: used as given, not normalised
    q[n // 3: n // 3 + 5] = [[0, 0, 0, 1], [1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, -1]]
    return np.ascontiguousarray(t), np.ascontiguousarray(q)


def test_sensor_matrix_and_point_transform_bitwise(sf):
    rng = np.random.default_rng(31)
    n = 400
    t, q = _random_transforms(rng, n)
    T = np.zeros((n, 12), dtype=np.float32)
    sf.sf_sensor_matrix(n, _p(t), _p(q), _p(T))
    pts = (rng.normal(size=(257, 3)) * 40).astype(np.float32)
    out = np.zeros_like(pts)
    for i in range(n):
        M = fr.sensor_matrix(t[i], q[i])
        assert np.array_equal(_bits(T[i].reshape(3, 4)), _bits(M[:3])), i
        sf.sf_transform_points(len(pts), _p(T[i]), _p(pts), _p(out))
        assert np.array_equal(_bits(out), _bits(fr.transform_cloud(pts, M))), i
    # a unit quaternion gives a rotation, and the transform is the float64 one to float rounding
    Md = osm.pose_matrix(t[-1], q[-1])
    np.testing.assert_allclose(fr.sensor_matrix(t[-1], q[-1]), Md, rtol=0, atol=1e-6 * max(1.0, np.abs(t[-1]).max()))
    # a non-unit quaternion is not normalised: |q|^2 scales the rotation part
    M2 = fr.sensor_matrix((0, 0, 0), 2.0 * np.asarray(q[-1]))
    assert abs(np.linalg.det(M2[:3, :3].astype(np.float64))) > 10.0


def test_inverse_bitwise_and_close_to_linalg(sf):
    rng = np.random.default_rng(32)
    t, q = _random_transforms(rng, 300)
    for i in range(300):
        M = fr.odom_matrix(t[i], q[i] / np.linalg.norm(q[i]))
        if i % 3 == 0:  # general (non-rigid) matrices too
            M = (M + 0.3 * rng.normal(size=(4, 4))).astype(np.float32)
        got = np.zeros(16, dtype=np.float32)
        sf.sf_inverse(_p(np.ascontiguousarray(M)), _p(got))
        ref = fr.mat4_inverse(M)
        assert np.array_equal(_bits(got.reshape(4, 4)), _bits(ref)), i
        Md = M.astype(np.float64)
        np.testing.assert_allclose(ref, np.linalg.inv(Md), rtol=0, atol=2e-5 * np.linalg.cond(Md) * max(1.0, np.abs(Md).max()))


def test_odometry_guess_bitwise(sf):
    """A stream of odometry steps through both: the guess, the stored previous odometry, and no delta while the previous
    odometry is exactly Identity (the first frame, and any odometry that is exactly Identity again)."""
    rng = np.random.default_rng(33)
    t, q = _random_transforms(rng, 300)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    prev_c = np.eye(4, dtype=np.float32).reshape(16).copy()
    prev_r = np.eye(4, dtype=np.float32)
    n_identity = n_applied = 0
    for i in range(300):
        sim = fr.odom_matrix(rng.normal(size=3) * 20, osm.quat_from_matrix(synth.rpy_matrix(*rng.uniform(-0.5, 0.5, 3))))
        if i % 50 == 7:
            ot, oq = np.zeros(3), np.array([0.0, 0.0, 0.0, 1.0])  # odometry exactly at the odom origin
        else:
            ot, oq = t[i], q[i]
        odom = np.zeros(16, dtype=np.float32)
        sf.sf_odom_matrix(_p(np.ascontiguousarray(ot, dtype=np.float64)), _p(np.ascontiguousarray(oq, dtype=np.float64)), _p(odom))
        assert np.array_equal(_bits(odom.reshape(4, 4)), _bits(fr.odom_matrix(ot, oq)))
        prev_before = prev_r
        sim_c = np.ascontiguousarray(sim).reshape(16).copy()
        sf.sf_odom_guess(_p(sim_c), _p(prev_c), _p(odom))
        sim_r, prev_r = fr.odom_guess(sim, prev_r, odom.reshape(4, 4))
        assert np.array_equal(_bits(sim_c.reshape(4, 4)), _bits(sim_r)), i
        assert np.array_equal(_bits(prev_c.reshape(4, 4)), _bits(prev_r)), i
        if np.array_equal(prev_before, np.eye(4, dtype=np.float32)):
            n_identity += 1
            assert np.array_equal(_bits(sim_r), _bits(sim)), i  # no delta applied
        else:
            n_applied += 1
            # the float guess is the float64 product to float rounding
            want = sim.astype(np.float64) @ np.linalg.inv(prev_before.astype(np.float64)) @ odom.reshape(4, 4).astype(np.float64)
            assert np.abs(sim_r - want).max() < 1e-4 * max(1.0, np.abs(want).max()), i
    assert n_identity == 7 and n_applied == 293  # frame 0 and the frame after each of the six exact-Identity odometries


def test_oracle_frontend_tracks_the_drive_with_mounted_sensor_and_odometry():
    """The restated callback with the LiDAR mounted 1.2 m forward, 2.0 m up and rotated, and odometry = ground truth times
    a drift growing by 2 cm and 1 mrad per frame: the robot-frame poses E T_k E^-1 are tracked within the bounds of
    test_oracle_frontend_tracks_the_drive."""
    sm = fr.ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=4, num_threads=8)
    sm.set_sensor_transform(MOUNT_POS, MOUNT_QUAT)
    E = osm.pose_matrix(MOUNT_POS, MOUNT_QUAT)
    Einv = np.linalg.inv(E)
    n_upd = 0
    for k, (scan, T_gt) in enumerate(synth.drive_stream(8, rings=16, azimuths=300, step=0.6)):
        R_gt = E @ T_gt @ Einv
        odom = R_gt @ synth.pose_matrix((0.02 * k, -0.01 * k, 0.0), (0.0, 0.0, 0.001 * k))
        pose, final, upd = sm.receive_cloud(scan, odom=(odom[:3, 3], osm.quat_from_matrix(odom[:3, :3])))
        n_upd += int(upd)
        dt, dr = synth.pose_error(final, R_gt)
        assert dt < 0.5 and dr < 0.02, (k, dt, dr)
    assert n_upd >= 2 and len(sm.submaps) == 1 + n_upd
    assert np.array_equal(sm.previous_odom, fr.odom_matrix(odom[:3, 3], osm.quat_from_matrix(odom[:3, :3])))
