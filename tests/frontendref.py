"""TEST INFRASTRUCTURE. float32 numpy restatement of the two cloud-callback steps the frontend session performs on top of
oracle/scanmatcher.py: tf2::doTransform of the incoming cloud into robot_frame_id_ (scanmatcher_component.cpp:188-199)
and the use_odom initial guess of receiveCloud (:333-348). numpy float32 scalar and elementwise arithmetic is IEEE and
un-fused, so each expression below is evaluated exactly as written; csrc/sensor_frame.hpp writes the same expressions in
C++ and tests/test_sensor_frame_cpu.py compares the two bit for bit.

`ScanMatcher` extends the oracle frontend with set_sensor_transform() and receive_cloud(points, odom=None); both are off
by default, so it computes what oracle.scanmatcher.ScanMatcher computes unless they are used.
"""
from __future__ import annotations

import numpy as np

import oracle
import oracle.scanmatcher as osm

F = np.float32


def sensor_matrix(position, quat_xyzw) -> np.ndarray:
    """Translation3f(t) * Quaternionf(w, x, y, z) with the doubles cast to float, toRotationMatrix in float (the quaternion
    is not normalised, as in tf2_sensor_msgs). Returns the 4x4 float32 matrix."""
    x, y, z, w = (F(v) for v in quat_xyzw)
    tx, ty, tz = F(2) * x, F(2) * y, F(2) * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    M = np.eye(4, dtype=np.float32)
    M[0, :3] = [F(1) - (tyy + tzz), txy - twz, txz + twy]
    M[1, :3] = [txy + twz, F(1) - (txx + tzz), tyz - twx]
    M[2, :3] = [txz - twy, tyz + twx, F(1) - (txx + tyy)]
    M[:3, 3] = [F(v) for v in position]
    return M


def transform_cloud(cloud, T) -> np.ndarray:
    """doTransform of the points: ((r0 x + r1 y) + r2 z) + t in float32, the other columns copied."""
    return osm.transform_f32(cloud, np.asarray(T, dtype=np.float32))


def odom_matrix(position, quat_xyzw) -> np.ndarray:
    """tf2::transformToEigen(odom).matrix().cast<float>()."""
    return osm.pose_matrix(position, quat_xyzw).astype(np.float32)


def mat4_mul(A, B) -> np.ndarray:
    """4x4 float32 product, each entry ((a0 b0 + a1 b1) + a2 b2) + a3 b3."""
    C = np.zeros((4, 4), dtype=np.float32)
    for r in range(4):
        for c in range(4):
            C[r, c] = ((A[r, 0] * B[0, c] + A[r, 1] * B[1, c]) + A[r, 2] * B[2, c]) + A[r, 3] * B[3, c]
    return C


def mat4_inverse(m) -> np.ndarray:
    """Laplace expansion in 2x2 minors, the formula and association of csrc/sensor_frame.hpp::mat4_inverse_f."""
    m = np.asarray(m, dtype=np.float32)
    a00, a01, a02, a03 = m[0]
    a10, a11, a12, a13 = m[1]
    a20, a21, a22, a23 = m[2]
    a30, a31, a32, a33 = m[3]
    s0, s1, s2 = a00 * a11 - a10 * a01, a00 * a12 - a10 * a02, a00 * a13 - a10 * a03
    s3, s4, s5 = a01 * a12 - a11 * a02, a01 * a13 - a11 * a03, a02 * a13 - a12 * a03
    c5, c4, c3 = a22 * a33 - a32 * a23, a21 * a33 - a31 * a23, a21 * a32 - a31 * a22
    c2, c1, c0 = a20 * a33 - a30 * a23, a20 * a32 - a30 * a22, a20 * a31 - a30 * a21
    det = ((((s0 * c5 - s1 * c4) + s2 * c3) + s3 * c2) - s4 * c1) + s5 * c0
    inv = F(1) / det
    o = [
        (a11 * c5 - a12 * c4 + a13 * c3) * inv, (-a01 * c5 + a02 * c4 - a03 * c3) * inv,
        (a31 * s5 - a32 * s4 + a33 * s3) * inv, (-a21 * s5 + a22 * s4 - a23 * s3) * inv,
        (-a10 * c5 + a12 * c2 - a13 * c1) * inv, (a00 * c5 - a02 * c2 + a03 * c1) * inv,
        (-a30 * s5 + a32 * s2 - a33 * s1) * inv, (a20 * s5 - a22 * s2 + a23 * s1) * inv,
        (a10 * c4 - a11 * c2 + a13 * c0) * inv, (-a00 * c4 + a01 * c2 - a03 * c0) * inv,
        (a30 * s4 - a31 * s2 + a33 * s0) * inv, (-a20 * s4 + a21 * s2 - a23 * s0) * inv,
        (-a10 * c3 + a11 * c1 - a12 * c0) * inv, (a00 * c3 - a01 * c1 + a02 * c0) * inv,
        (-a30 * s3 + a31 * s1 - a32 * s0) * inv, (a20 * s3 - a21 * s1 + a22 * s0) * inv,
    ]
    return np.array(o, dtype=np.float32).reshape(4, 4)


def odom_guess(sim, previous_odom, odom):
    """sm.cpp:342-347: (sim * previous^-1) * odom unless previous is exactly Identity. Returns (guess, new previous)."""
    sim = np.asarray(sim, dtype=np.float32)
    previous_odom = np.asarray(previous_odom, dtype=np.float32)
    if not np.array_equal(previous_odom, np.eye(4, dtype=np.float32)):
        sim = mat4_mul(mat4_mul(sim, mat4_inverse(previous_odom)), odom)
    return sim, np.asarray(odom, dtype=np.float32).copy()


class ScanMatcher(osm.ScanMatcher):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.sensor_T = None
        self.previous_odom = np.eye(4, dtype=np.float32)  # scanmatcher_component.h:170

    def set_sensor_transform(self, position, quat_xyzw):
        """lookupTransform(robot_frame_id_, frame_id) for every later frame; (None, None) turns it off."""
        self.sensor_T = None if position is None and quat_xyzw is None else sensor_matrix(position, quat_xyzw)

    def receive_cloud(self, points, odom=None):
        """cloud_callback + receiveCloud + publishMapAndPose, as oracle.scanmatcher.ScanMatcher.receive_cloud, with the
        doTransform first when a sensor transform is set and the use_odom guess when odom = (position, quat_xyzw)."""
        cloud = np.ascontiguousarray(points, dtype=np.float32)
        if cloud.shape[1] < 4:
            cloud = np.concatenate([cloud[:, :3], np.zeros((len(cloud), 1), dtype=np.float32)], axis=1)
        if self.sensor_T is not None:
            cloud = transform_cloud(cloud, self.sensor_T)
        cloud = self._range_filter(cloud)
        if not self.initial:
            self.initial = True
            sim = osm.pose_matrix(self.position, self.quat).astype(np.float32)
            self.update_map(cloud, sim, self.position, self.quat)
            self._adopt(False)
        self._adopt(self.method == "GICP")
        self.filtered = oracle.voxelgrid(cloud, self.vg_in)
        self.reg.set_source(self.filtered[:, :3])
        sim = osm.pose_matrix(self.position, self.quat).astype(np.float32)
        if odom is not None:
            sim, self.previous_odom = odom_guess(sim, self.previous_odom, odom_matrix(*odom))
        final = np.asarray(self.reg.align(sim), dtype=np.float32)
        pos = final[:3, 3].astype(np.float64)
        self.quat = osm.quat_from_matrix(final[:3, :3].astype(np.float64))
        self.position = pos
        self.trans = float(np.sqrt(np.sum((pos - self.previous_position) ** 2)))
        updated = False
        if self.trans >= self.trans_for_mapupdate:
            self.previous_position = pos.copy()
            self.latest_distance += self.trans
            self.update_map(cloud, final, self.position, self.quat)
            updated = True
        return np.concatenate([self.position, self.quat]), final, updated
