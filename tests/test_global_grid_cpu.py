"""The hypothesis grid and the top-k choice of b200sm_localize_global on the CPU: the product's header
csrc/global_grid.hpp compiled with g++ -ffp-contract=off (tests/hostmath/global_grid_host.cpp) against the float64 replay
tests/globalref.py bit for bit — at the disc's edge, at radii one ulp either side of a multiple of the step, at radius 0,
with one yaw step and at the caps — and the replay told apart from subtly wrong ones (globalref.MUTATIONS)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import globalref as R

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "global_grid_host.cpp")
HDRS = [os.path.join(HERE, "..", "lidarslam_ros2_b200", "csrc", h) for h in ("global_grid.hpp", "pose_graph.hpp")]
F32 = np.float32
POSE = ((3.25, -1.5, 0.75), (0.0123, -0.0456, 0.3826834, 0.9226))  # a tilted, rotated pose (quaternion x y z w)


def _unit(q):
    n = math.sqrt(sum(v * v for v in q))
    return tuple(v / n for v in q)


@pytest.fixture(scope="module")
def gg(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("gg"), "libglobal_grid_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    lib = C.CDLL(lib)
    lib.gg_count.restype = C.c_longlong
    lib.gg_count.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int]
    lib.gg_build.restype = C.c_longlong
    lib.gg_build.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_longlong]
    lib.gg_select.restype = C.c_int
    lib.gg_select.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    return lib


def _build(gg, position, quat, radius, step, yaw_steps):
    p = np.ascontiguousarray(position, dtype=np.float64)
    q = np.ascontiguousarray(quat, dtype=np.float64)
    n = gg.gg_count(radius, step, yaw_steps, 1)
    assert n >= 0
    out = np.zeros((max(n, 1), 16), dtype=F32)
    assert gg.gg_build(p.ctypes.data, q.ctypes.data, radius, step, yaw_steps, out.ctypes.data, n) == n
    return out[:n].reshape(n, 4, 4).transpose(0, 2, 1)


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


CASES = [  # (radius, step, yaw_steps)
    (5.0, 1.0, 3),                                 # the disc edge: (3, 4) has a * a + b * b == r * r
    (3.0, 1.0, 8), (math.nextafter(3.0, 0.0), 1.0, 8), (math.nextafter(3.0, 9.0), 1.0, 8),  # around a multiple of the step
    (2.1, 0.7, 5), (math.nextafter(2.1, 0.0), 0.7, 5), (math.nextafter(2.1, 9.0), 0.7, 5),
    (0.0, 1.0, 4), (0.0, 0.25, 1),                 # radius 0: the centre only
    (4.0, 1.0, 1),                                 # one yaw step
    (10.0, 1.0, 72),                               # the recovery search of the GPU test
]


@pytest.mark.parametrize("radius,step,yaw", CASES)
def test_grid_equals_replay(gg, radius, step, yaw):
    quat = _unit(POSE[1])
    got = _build(gg, POSE[0], quat, radius, step, yaw)
    want = R.grid(POSE[0], quat, radius, step, yaw)
    assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want))
    assert gg.gg_count(radius, step, yaw, 1) == R.count(radius, step, yaw, 1) == len(want)


def test_disc_edge_and_radius_zero():
    P = R.positions(5.0, 1.0)
    assert (3, 4) in P and (4, 3) in P and (-3, -4) in P and (5, 0) in P and (4, 4) not in P
    assert len(R.positions(5.0, 1.0, mut={"disc_lt"})) < len(P)
    assert R.positions(0.0, 1.0) == [(0, 0)]
    # a radius one ulp below a multiple of the step drops the axis points at that multiple
    assert (3, 0) in R.positions(3.0, 1.0) and (3, 0) not in R.positions(math.nextafter(3.0, 0.0), 1.0)


def test_identity_pose_yaw_zero_is_the_centre():
    g = R.grid((1.0, 2.0, 3.0), (0.0, 0.0, 0.0, 1.0), 0.0, 1.0, 4)
    assert np.array_equal(g[0], np.array([[1, 0, 0, 1], [0, 1, 0, 2], [0, 0, 1, 3], [0, 0, 0, 1]], dtype=F32))
    assert np.allclose(g[1][:2, :2], [[0, -1], [1, 0]], atol=1e-7)  # +90 degrees


@pytest.mark.parametrize("spec", [
    (math.nan, 1.0, 1, 1), (math.inf, 1.0, 1, 1), (-1.0, 1.0, 1, 1), (1.0, 0.0, 1, 1), (1.0, -1.0, 1, 1), (1.0, math.nan, 1, 1),
    (1.0, math.inf, 1, 1), (1.0, 1.0, 0, 1), (1.0, 1.0, 4097, 1), (1.0, 1.0, 1, 0), (1.0, 1.0, 1, 1025),
    (4097.0, 1.0, 1, 1), (1e300, 1e-300, 1, 1), (1e308, 1e-10, 1, 1)])
def test_invalid_specs(gg, spec):
    assert gg.gg_count(*spec) == -1 and R.count(*spec) == -1


def test_caps(gg):
    assert gg.gg_count(1.0, 1.0, 4096, 1024) == R.count(1.0, 1.0, 4096, 1024) == 5 * 4096
    # the hypothesis cap: 2^24 = 4096 positions x 4096 yaws; the radius where the disc passes 4096 positions
    seen = set()
    for r in np.arange(35.0, 37.01, 0.25):
        n_pos = len(R.positions(float(r), 1.0))
        want = n_pos * 4096 if n_pos * 4096 <= (1 << 24) else -1
        assert gg.gg_count(float(r), 1.0, 4096, 1) == R.count(float(r), 1.0, 4096, 1) == want, r
        seen.add(want == -1)
    assert seen == {True, False}
    # K = 4096 passes the half-width cap but not the hypothesis cap; K = 4097 fails the half-width cap
    assert gg.gg_count(4096.5, 1.0, 1, 1) == -1 and gg.gg_count(math.nextafter(4097.0, 0.0), 1.0, 1, 1) == -1
    assert gg.gg_count(2310.0, 1.0, 1, 1) == R.count(2310.0, 1.0, 1, 1) > 0  # the largest disc under 2^24 at step 1 fits


def _scores(seed, n, ties):
    rng = np.random.default_rng(seed)
    s = rng.normal(size=n)
    if ties:
        s = np.round(s, 1)  # many equal scores
    return s


@pytest.mark.parametrize("n,top_k,ties", [(1, 1, False), (1, 8, False), (7, 3, True), (100, 100, True), (1000, 8, True),
                                          (5000, 1024, True), (5000, 17, False)])
def test_selection_equals_replay(gg, n, top_k, ties):
    s = np.ascontiguousarray(_scores(n + top_k, n, ties))
    out = np.zeros(max(min(n, top_k), 1), dtype=np.int32)
    k = gg.gg_select(s.ctypes.data, n, top_k, out.ctypes.data)
    assert k == min(n, top_k)
    assert out[:k].tolist() == R.select(s, top_k)


def test_mutations_are_told_apart(gg):
    quat = _unit(POSE[1])
    good = R.grid(POSE[0], quat, 5.0, 1.0, 3)
    assert not np.array_equal(_bits(good), _bits(R.grid(POSE[0], quat, 5.0, 1.0, 3, mut={"yaw_outer"})))
    assert len(R.grid(POSE[0], quat, 5.0, 1.0, 3, mut={"disc_lt"})) != len(good)
    s = np.array([1.0, 3.0, 3.0, 2.0, 3.0])
    assert R.select(s, 3) == [1, 2, 4] and R.select(s, 3, mut={"tie_high"}) == [4, 2, 1]
    out = np.zeros(3, dtype=np.int32)
    gg.gg_select(np.ascontiguousarray(s).ctypes.data, 5, 3, out.ctypes.data)
    assert out.tolist() == [1, 2, 4]
