"""The place search's arithmetic on the CPU: the product's header csrc/scan_context.hpp compiled with g++ -ffp-contract=off
(tests/hostmath/scan_context_host.cpp) against the float64 replay tests/scancontextref.py. Bins agree for every point away
from a ring or sector edge, and the edges themselves are decided as the header defines them; distances agree to 1e-12,
ties go to the lowest shift and the lowest id; the replay is told apart from its named mutations; and on the ray-cast drive
of the end-to-end GPU test the true revisit is the best place with the right heading."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import scancontextref as R

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "scan_context_host.cpp")
F32 = np.float32


@pytest.fixture(scope="module")
def sc(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("sc"), "libscan_context_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    lib = C.CDLL(lib)
    vp, d, i, lg = C.c_void_p, C.c_double, C.c_int, C.c_long
    lib.sch_valid.argtypes = [i, i, d, d]
    lib.sch_bins.argtypes = [vp, lg, i, i, i, d, vp]
    lib.sch_descriptor.argtypes = [vp, lg, i, i, i, d, d, vp, vp]
    lib.sch_distance_at.argtypes = [vp, vp, vp, vp, i, i, i]
    lib.sch_distance_at.restype = d
    lib.sch_distance.argtypes = [vp, vp, vp, vp, i, i, C.POINTER(i)]
    lib.sch_distance.restype = d
    lib.sch_rank.argtypes = [vp, vp, lg, d, vp]
    lib.sch_guess.argtypes = [vp, vp, i, i, vp]
    return lib


def host_bins(sc, pts, R_=20, S=60, r=80.0):
    p = np.ascontiguousarray(pts, dtype=F32)
    out = np.zeros(len(p), dtype=np.int32)
    sc.sch_bins(p.ctypes.data, len(p), p.shape[1], R_, S, r, out.ctypes.data)
    return out


def host_descriptor(sc, pts, R_=20, S=60, r=80.0, h=2.0):
    p = np.zeros((len(pts), 4), dtype=F32)
    if len(pts):
        p[:, :3] = np.asarray(pts, dtype=F32)[:, :3]
    D = np.zeros((R_, S), dtype=F32)
    n = np.zeros(S, dtype=np.float64)
    sc.sch_descriptor(p.ctypes.data, len(p), 4, R_, S, r, h, D.ctypes.data, n.ctypes.data)
    return D, n


def host_distance(sc, Q, nQ, Cd, nC):
    Rr, S = Q.shape
    s = C.c_int(-1)
    args = [np.ascontiguousarray(a) for a in (Q, nQ, Cd, nC)]
    D = sc.sch_distance(*(a.ctypes.data for a in args), Rr, S, C.byref(s))
    return D, s.value


def random_cloud(seed, n, reach=90.0):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), dtype=F32)
    p[:, 0:2] = rng.uniform(-reach, reach, size=(n, 2))
    p[:, 2] = rng.uniform(-3.0, 12.0, size=n)
    p[:, 3] = rng.uniform(0, 255, size=n)
    return p


def edge_rows(R_=20, S=60, r=80.0, h=2.0):
    """Rows on the +-x / +-y axes, exactly on ring bounds t_k (as floats), at max_radius and one ulp beyond, the origin,
    non-finite rows and z = -lidar_height."""
    rows = []
    for k in range(1, R_ + 1):
        t = F32((k * r) / R_)
        for x, y in ((t, 0), (0, t), (-t, 0), (0, -t)):
            rows.append((x, y, 1.0))
    rm = F32(r)
    up = np.nextafter(rm, F32(np.inf))
    rows += [(rm, 0, 1.0), (up, 0, 1.0), (0, -up, 1.0), (-rm, 0, 0.5)]
    rows += [(0, 0, 3.0), (-0.0, 0.0, 4.0), (0.0, -0.0, 4.5), (np.nan, 1, 1), (1, np.inf, 1), (1, 1, -np.inf), (1, 2, np.nan)]
    rows += [(5.0, 5.0, -h), (-7.0, 0.0, -h), (3.0, -0.0, 1.0), (-3.0, -0.0, 1.0), (-3.0, 0.0, 1.0)]
    out = np.zeros((len(rows), 4), dtype=F32)
    out[:, :3] = np.array(rows, dtype=np.float64)
    return out


@pytest.mark.parametrize("R_,S,r", [(20, 60, 80.0), (1, 1, 80.0), (11, 720, 50.0), (128, 64, 100.0), (7, 13, 33.3)])
def test_bins_equal_replay_away_from_edges(sc, R_, S, r):
    p = random_cloud(R_ * 1000 + S, 20000, reach=1.15 * r)
    hb = host_bins(sc, p, R_, S, r)
    ring, sector = R.bins(p, R_, S, r)
    want = np.where(ring >= 0, ring * S + sector, -1)
    far = R.edge_distance(p, R_, S, r) > 1e-9
    assert far.mean() > 0.99
    assert np.array_equal(hb[far], want[far])


def test_edge_rows_are_decided_as_defined(sc):
    p = edge_rows()
    b = host_bins(sc, p)
    # on +x: sector 0; +y: sector 15; -x: sector 30; -y: sector 45 (each axis is a sector edge and lands in the sector above)
    for k in range(1, 21):
        ring = min(k, 19)  # t_k itself: B_k <= q, so ring k (the outer bound t_20 stays in ring 19)
        assert b[4 * (k - 1):4 * k].tolist() == [ring * 60 + 0, ring * 60 + 15, ring * 60 + 30, ring * 60 + 45], k
    n_axes = 80
    assert b[n_axes] == 19 * 60 and b[n_axes + 1] == -1 and b[n_axes + 2] == -1 and b[n_axes + 3] == 19 * 60 + 30
    assert b[n_axes + 4:n_axes + 7].tolist() == [0, 0, 0]  # the origin, with either zero sign
    assert (b[n_axes + 7:n_axes + 11] == -1).all()  # non-finite rows are skipped
    # y = -0 is the upper half-plane: (3, -0) is sector 0 and (-3, -0) sector 30 like (-3, +0)
    assert b[-3] == 0 and b[-2] == 30 and b[-1] == 30
    D, _ = host_descriptor(sc, p)
    Dr = R.descriptor(p)
    assert np.array_equal(D.view(np.uint32), Dr.view(np.uint32))
    # z = -lidar_height gives a +0 bin; the bin of (5, 5) holds exactly 0 with a positive sign
    b55 = host_bins(sc, np.array([[5.0, 5.0, 0.0, 0.0]], dtype=F32))[0]
    assert D.reshape(-1)[b55] == 0 and not np.signbit(D.reshape(-1)[b55])


def test_signed_zero_order(sc):
    # one bin with a -0 value only, one with -0 and +0: a value is -0 only for z = -0 with lidar_height = -0
    p = np.array([[1.0, 0.1, -0.0, 0], [1.0, -5.0, -0.0, 0], [1.0, -5.0, 0.0, 0]], dtype=F32)
    D, _ = host_descriptor(sc, p, h=-0.0)
    flat = D.reshape(-1)
    b = host_bins(sc, p)
    assert flat[b[0]] == 0 and np.signbit(flat[b[0]])
    assert flat[b[1]] == 0 and not np.signbit(flat[b[1]])
    assert np.array_equal(D.view(np.uint32), R.descriptor(p, lidar_height=-0.0).view(np.uint32))


@pytest.mark.parametrize("seed,R_,S", [(1, 20, 60), (2, 1, 1), (3, 11, 720), (4, 128, 64), (5, 5, 7)])
def test_descriptors_and_distances_equal_replay(sc, seed, R_, S):
    a, b = random_cloud(seed, 3000), random_cloud(seed + 100, 2500)
    keep = R.edge_distance(a, R_, S, 80.0) > 1e-9
    a = a[keep]
    b = b[R.edge_distance(b, R_, S, 80.0) > 1e-9]
    Qa, nQ = host_descriptor(sc, a, R_, S)
    Cb, nC = host_descriptor(sc, b, R_, S)
    assert np.array_equal(Qa, R.descriptor(a, R_, S)) and np.array_equal(Cb, R.descriptor(b, R_, S))
    assert np.allclose(nQ, R.norms(Qa), rtol=1e-15, atol=0)
    D, s = host_distance(sc, Qa, nQ, Cb, nC)
    d_all = R.distances(Qa, Cb)
    Dr, sr = R.distance(Qa, Cb, tol=1e-12)
    assert abs(D - Dr) <= 1e-12
    assert abs(d_all[s] - Dr) <= 1e-12  # the host's shift attains the minimum (to rounding)
    if sr == R.distance(Qa, Cb, tol=1e-9)[1]:
        assert s == sr


def test_ties_go_to_the_lowest_shift(sc):
    # a query with all columns equal: every shift gives the same distance -> shift 0
    Q = np.tile(np.arange(1, 6, dtype=F32)[:, None], (1, 12))
    Cd = np.tile(np.array([2, 1, 0, 1, 3], dtype=F32)[:, None], (1, 12))
    D, s = host_distance(sc, Q, R.norms(Q), Cd, R.norms(Cd))
    assert s == 0 and R.distance(Q, Cd)[1] == 0 and R.distance(Q, Cd, mut={"tie_high"})[1] == 11
    # a pattern of period 4 in 12 sectors: shifts s, s + 4, s + 8 tie; the lowest wins
    rng = np.random.default_rng(9)
    base = rng.uniform(0.5, 5, size=(6, 4)).astype(F32)
    Q = np.tile(base, (1, 3))
    Cd = np.roll(Q, 2, axis=1)  # C[:, (j + 2) % 12] == Q[:, j]
    D, s = host_distance(sc, Q, R.norms(Q), Cd, R.norms(Cd))
    assert s == 2 and abs(D) < 1e-12
    assert R.distance(Q, Cd, tol=1e-12) [1] == 2 and R.distance(Q, Cd, mut={"tie_high"}, tol=1e-12)[1] == 10


def test_no_effective_column_gives_one(sc):
    Q = np.zeros((4, 6), dtype=F32)
    Q[:, 0] = 1
    Cd = np.zeros((4, 6), dtype=F32)  # empty candidate
    D, s = host_distance(sc, Q, R.norms(Q), Cd, R.norms(Cd))
    assert D == 1.0 and s == 0 and R.distance(Q, Cd) == (1.0, 0)
    Z = np.zeros((4, 6), dtype=F32)
    assert host_distance(sc, Z, R.norms(Z), Z, R.norms(Z)) == (1.0, 0)


def test_ranking_ties_go_to_the_lowest_id(sc):
    D = np.array([0.3, 0.1, 0.3, 0.05, 0.1, 0.9, 0.3], dtype=np.float64)
    ids = np.array([10, 7, 3, 12, 2, 1, 5], dtype=np.int32)
    out = np.zeros(len(D), dtype=np.int32)
    k = sc.sch_rank(D.ctypes.data, ids.ctypes.data, len(D), 0.5, out.ctypes.data)
    assert out[:k].tolist() == R.rank(D, ids, 0.5) == [3, 4, 1, 2, 6, 0]
    assert sc.sch_rank(D.ctypes.data, ids.ctypes.data, len(D), 0.05, out.ctypes.data) == 0  # strict <


def test_guess_equals_replay(sc):
    from lidarslam_ros2_b200 import synth

    Pc = synth.pose_matrix((3.5, -2.25, 0.4), (0.01, -0.02, 0.7))
    Pn = synth.pose_matrix((40.1, 17.3, -0.2), (-0.015, 0.005, 2.9))
    for shift, S in ((0, 60), (17, 60), (30, 60), (359, 720), (0, 1)):
        G = np.zeros(16, dtype=F32)
        sc.sch_guess(np.ascontiguousarray(Pc).ctypes.data, np.ascontiguousarray(Pn).ctypes.data, shift, S, G.ctypes.data)
        want = R.guess(Pc, Pn, shift, S)
        assert np.array_equal(G.reshape(4, 4).T.view(np.uint32), want.view(np.uint32)), (shift, S)


@pytest.mark.parametrize("spec,ok", [((20, 60, 80.0, 2.0), 1), ((1, 1, 1e-300, -5.0), 1), ((128, 64, 80.0, 0.0), 1),
                                     ((11, 720, 80.0, 0.0), 1), ((0, 60, 80.0, 2.0), 0), ((129, 60, 80.0, 2.0), 0),
                                     ((20, 0, 80.0, 2.0), 0), ((20, 721, 80.0, 2.0), 0), ((12, 720, 80.0, 2.0), 0),
                                     ((20, 60, 0.0, 2.0), 0), ((20, 60, -1.0, 2.0), 0), ((20, 60, math.inf, 2.0), 0),
                                     ((20, 60, math.nan, 2.0), 0), ((20, 60, 80.0, math.nan), 0), ((20, 60, 80.0, math.inf), 0)])
def test_parameter_bounds(sc, spec, ok):
    assert sc.sch_valid(*spec) == ok


def test_mutations_change_an_outcome():
    rng = np.random.default_rng(4)
    Q = rng.uniform(0, 5, size=(8, 24)).astype(F32)
    Q[:, 3] = 0  # an empty column in the query
    Cd = np.roll(Q, 5, axis=1) + rng.uniform(0, 0.05, size=Q.shape).astype(F32)
    Cd[:, 20] = 0
    good = R.distance(Q, Cd)
    assert good[1] == 5
    assert R.distance(Q, Cd, mut={"shift_reversed"})[1] == 24 - 5
    assert R.distance(Q, Cd, mut={"any_nonzero"})[0] != good[0]
    p = edge_rows()
    assert not np.array_equal(R.bins(p)[0], R.bins(p, mut={"ring_exclusive"})[0])
    Qt = np.tile(np.arange(1, 6, dtype=F32)[:, None], (1, 12))
    assert R.distance(Qt, Qt)[1] == 0 and R.distance(Qt, Qt, mut={"tie_high"})[1] == 11


def test_replay_matches_header_on_the_ray_cast_drive(sc):
    """The premise of the end-to-end GPU test: on the drive with drifted poses, the true revisit's D is below every
    other eligible submap's by at least 0.02, its s* is within one sector of the true heading, and the host compile's D and
    s* agree with the replay's."""
    scans, poses, (back, back_match, rev, rev_match) = R.drive()
    for idx, match in zip(R.sessions(back, rev), (back_match, rev_match)):
        drifted, dist = R.session(poses, idx)
        newest = len(idx) - 1
        eligible = [i for i in range(newest) if dist[-1] - dist[i] > 40.0]
        # the reference's position gate at 20 m passes none of the submaps its distance gate passes
        assert all(np.linalg.norm(drifted[-1][:3, 3] - drifted[i][:3, 3]) > 20.0 for i in eligible)
        assert idx.index(match) in eligible
        Q = R.descriptor(scans[idx[-1]])
        Qh, nQ = host_descriptor(sc, scans[idx[-1]])
        assert np.array_equal(Q, Qh) or (R.edge_distance(scans[idx[-1]]) <= 1e-9).any()
        scores = {}
        for i in eligible:
            Cd, nC = host_descriptor(sc, scans[idx[i]])
            D, s = host_distance(sc, Qh, nQ, Cd, nC)
            Dr, _ = R.distance(R.descriptor(scans[idx[-1]]), R.descriptor(scans[idx[i]]))
            assert abs(D - Dr) < 1e-6  # the replay bins by atan2: a point within rounding of an edge may move
            scores[i] = (D, s)
        m = idx.index(match)
        others = [scores[i][0] for i in eligible if i != m]
        assert scores[m][0] + 0.02 < min(others), (scores[m], min(others))
        t = R.true_shift(poses[match], poses[idx[-1]], 60)
        assert abs(scores[m][1] - t) <= 1.0 or abs(scores[m][1] - t) >= 59.0, (scores[m][1], t)
