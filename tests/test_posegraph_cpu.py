"""The backend's pose adjustment (doPoseAdjustment, gbs.cpp:262-319) on the CPU: the float64 restatement
tests/posegraphref.py checked on its own (Jacobians against central differences, the graph of the reference's loop,
g2o's LM against scipy's least_squares), then the product's host optimiser csrc/pose_graph.hpp, compiled with g++, against
it trial by trial, and its envelope Cholesky against dense solves."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import posegraphref as R
from lidarslam_ros2_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def pg():
    src = os.path.join(HERE, "hostmath", "posegraph_host.cpp")
    lib = os.path.join(HERE, "hostmath", "libposegraph_host.so")
    deps = [src, os.path.join(HERE, "..", "lidarslam_ros2_b200", "csrc", "pose_graph.hpp")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    return C.CDLL(lib)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def product_adjust(pg, poses, k, loops, max_iterations=10):
    """csrc/pose_graph.hpp through the harness: (poses, [chi2_initial, chi2_final, iterations, trials], trials, n_edges)."""
    n = len(poses)
    P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(n, 16))
    ids = np.array([[f, t] for f, t, _ in loops], dtype=np.int32).reshape(-1)
    rel = np.ascontiguousarray(np.array([np.asarray(Z, dtype=np.float64) for _, _, Z in loops]).reshape(-1))
    out, res, tr, nt = np.zeros((n, 16)), np.zeros(4), np.zeros(4 * 1000), C.c_int(0)
    ne = pg.pg_adjust(n, _p(P), k, len(loops), _p(ids), _p(rel), max_iterations, _p(out), _p(res), 1000, _p(tr), C.byref(nt))
    return out.reshape(n, 4, 4), res, tr[:4 * nt.value].reshape(-1, 4), ne


def _random_pose(rng, angle):
    axis = rng.normal(size=3)
    M = np.eye(4)
    M[:3, :3] = Rotation.from_rotvec(axis / np.linalg.norm(axis) * angle).as_matrix()
    M[:3, 3] = rng.normal(size=3) * 5.0
    return M


def drifted_square(side=10, yaw_bias=0.01, lateral_bias=0.02):
    """A 4 x `side` m square driven in 1 m steps back to its start: ground truth, and odometry that turns 0.01 rad too far
    and slips 2 cm sideways every step."""
    gt, dr = [np.eye(4)], [np.eye(4)]
    for leg in range(4):
        for s in range(side):
            turn = np.pi / 2 if s == side - 1 else 0.0
            gt.append(gt[-1] @ synth.pose_matrix((1.0, 0, 0), (0, 0, turn)))
            dr.append(dr[-1] @ synth.pose_matrix((1.0, lateral_bias, 0), (0, 0, turn + yaw_bias)))
    return np.array(gt), np.array(dr)


def long_drive(n=300):
    """A 300-vertex winding drive with drift in every degree of freedom and five ground-truth loop edges, one of them to
    vertex 0."""
    gt, dr = [np.eye(4)], [np.eye(4)]
    for i in range(n - 1):
        M = synth.pose_matrix((1.0, 0, 0), (0, 0, 0.2 * np.sin(i / 15)))
        gt.append(gt[-1] @ M)
        dr.append(dr[-1] @ M @ synth.pose_matrix((0.01, 0.02, 0.005), (0.001, -0.002, 0.004)))
    gt, dr = np.array(gt), np.array(dr)
    pairs = [(0, n - 1), (10, 120), (50, 200), (130, 260), (200, 290)]
    return gt, dr, [(a, b, np.linalg.inv(gt[a]) @ gt[b]) for a, b in pairs]


# ---------------------------------------------------------------- the float64 restatement on its own
@pytest.mark.parametrize("angle", [0.0, 1e-6, 1e-3, 0.3, 1.5, 2.5, np.deg2rad(170.0)])
def test_edge_jacobians_match_central_differences(angle):
    rng = np.random.default_rng(int(angle * 1e6) + 1)
    h = 1e-6
    for _ in range(6):
        Xf, Xt, Z = _random_pose(rng, angle), _random_pose(rng, angle), _random_pose(rng, angle)
        Zinv = R.inverse(Z)
        _, E = R.edge_error(Xf, Xt, Zinv)
        J = R.edge_jacobians(E, Zinv)
        for which in (0, 1):
            Jn = np.zeros((6, 6))
            for c in range(6):
                d = np.zeros(6)
                d[c] = h
                plus, minus = [Xf, Xt], [Xf, Xt]
                plus[which] = R.compose(plus[which], R.from_vector_mqt(d))
                minus[which] = R.compose(minus[which], R.from_vector_mqt(-d))
                Jn[:, c] = (R.edge_error(*plus, Zinv)[0] - R.edge_error(*minus, Zinv)[0]) / (2 * h)
            np.testing.assert_allclose(J[which], Jn, rtol=0, atol=1e-7)


@pytest.mark.parametrize("k", [1, 5])
@pytest.mark.parametrize("n_of_k", [lambda k: 1, lambda k: k, lambda k: k + 1, lambda k: k + 2, lambda k: 40])
def test_graph_has_the_reference_edges(k, n_of_k):
    """gbs.cpp:276-305: `if (i > k) for (j = 0; j < k; j++) edge(i - k + j, i)`. Vertex 0 is never an odometry end, and a
    graph of k + 1 vertices or fewer has no odometry edge."""
    n = n_of_k(k)
    want = []
    for i in range(n):
        if i > k:
            for j in range(k):
                want.append((i - k + j, i))
    assert R.graph_edges(n, k) == want
    assert all(f >= 1 for f, _ in want)
    assert (len(want) == 0) == (n <= k + 1)
    rng = np.random.default_rng(n + 10 * k)
    poses = [_random_pose(rng, 0.5) for _ in range(n)]
    edges = R.build_edges(poses, k, [(0, n - 1, np.eye(4))] if n > 1 else [])
    assert [(f, t) for f, t, _ in edges] == want + ([(0, n - 1)] if n > 1 else [])
    for f, t, Zinv in edges[:len(want)]:  # measurement = pose_from^-1 * pose_to
        np.testing.assert_allclose(R.inverse(Zinv), np.linalg.inv(poses[f]) @ poses[t], atol=1e-12)


def test_without_loop_edges_the_poses_come_back_bitwise():
    _, dr = drifted_square()
    X, res, trials = R.pose_adjust(dr, 5, [], 10)
    assert res["chi2_initial"] == 0.0 and res["chi2_final"] == 0.0
    assert all(np.array_equal(a, b) for a, b in zip(X, dr))
    assert trials == [(0, 0, trials[0][2], 0.0)] and res["iterations"] == 1  # rho == 0 ends the run


def test_square_loop_converges_to_the_least_squares_minimum():
    """The loop edge closes the cycle 1 .. N-1 against the drifted odometry, so the minimum is not zero. chi2 never grows,
    the newest pose moves towards the truth, and 50 iterations reach scipy's minimum of the same residual."""
    gt, dr = drifted_square()
    n = len(dr)
    loops = [(1, n - 1, np.linalg.inv(gt[1]) @ gt[-1])]
    X, res, trials = R.pose_adjust(dr, 5, loops, 10)
    chis = [res["chi2_initial"]] + [c for _, acc, _, c in trials if acc]
    assert all(b <= a for a, b in zip(chis, chis[1:])) and res["chi2_final"] < 0.02 * res["chi2_initial"]
    before, after = synth.pose_error(dr[-1], gt[-1]), synth.pose_error(X[-1], gt[-1])
    assert after[0] < 0.7 * before[0] and after[1] < 0.7 * before[1], (before, after)

    _, res50, _ = R.pose_adjust(dr, 5, loops, 50)
    edges = R.build_edges(dr, 5, loops)
    free = sorted({v for f, t, _ in edges for v in (f, t)} - {0})

    def residual(x):
        Y = list(dr)
        for j, v in enumerate(free):
            Y[v] = R.compose(dr[v], R.from_vector_mqt(x[6 * j:6 * j + 6]))
        return np.concatenate([R.edge_error(Y[f], Y[t], Zinv)[0] for f, t, Zinv in edges])

    ls = least_squares(residual, np.zeros(6 * len(free)), method="trf", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    chi_ls = float(np.sum(ls.fun ** 2))
    assert chi_ls > 0.01
    assert abs(res50["chi2_final"] - chi_ls) <= 1e-8 * chi_ls, (res50["chi2_final"], chi_ls)


def test_oracle_pose_adjustment_corrects_a_drifted_drive(oracle_mod):
    """The out-and-back drive of test_scanmatcher.py, its submaps stored at drifted poses: the CPU searchLoop accepts the
    revisit of submap 0, and the adjustment moves the newest submap towards its ground truth."""
    import oracle.scanmatcher as osm
    from test_scanmatcher import _out_and_back

    o = osm.ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3, num_threads=8)
    truth = []
    for k, (scan, T) in enumerate(_out_and_back()):
        Td = drift(k) @ T
        o.update_map_external(scan, Td.astype(np.float32), Td[:3, 3], osm.quat_from_matrix(Td[:3, :3]))
        truth.append(T)
    reg = oracle_mod.NDT(resolution=2.0, transformation_epsilon=0.01, max_iterations=100, search_method=oracle_mod.DIRECT7,
                         num_threads=8)
    r = o.search_loop(reg, **LOOP_ARGS)
    assert r["accepted"] and r["id_min"] == 0, r
    poses = [M for _, M, _ in o.submaps]
    X, res, _ = R.pose_adjust(poses, 5, [(0, len(poses) - 1, r["relative_pose"])], 10)
    before, after = synth.pose_error(poses[-1], truth[-1]), synth.pose_error(X[-1], truth[-1])
    assert after[0] < 0.5 * before[0] and after[1] < 0.5 * before[1], (before, after)
    assert res["chi2_final"] < res["chi2_initial"]


def drift(k):
    """Odometry drift of the k-th submap of the out-and-back drive: 3 cm / 2 cm per submap and 0.004 rad of yaw."""
    return synth.pose_matrix((0.03 * k, 0.02 * k, 0.0), (0.0, 0.0, 0.004 * k))


LOOP_ARGS = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, range_of_searching_loop_closure=2.0, search_submap_num=1)


# ---------------------------------------------------------------- the product's host optimiser against the restatement
def _decisive_prefix(trials, chi2_initial):
    """Trials before the first one whose chi2 is within 1e-12 (relative) of the chi2 it is compared with: there rounding,
    not the algorithm, decides between accept and reject."""
    cur = chi2_initial
    for j, (_, acc, _, chi) in enumerate(trials):
        if abs(chi - cur) <= 1e-12 * cur:
            return j
        if acc:
            cur = chi
    return len(trials)


def _check_against_restatement(pg, poses, k, loops, min_prefix):
    Xo, ro, to = R.pose_adjust(poses, k, loops, 10)
    Xp, rp, tp, ne = product_adjust(pg, poses, k, loops, 10)
    to = np.array(to, dtype=np.float64)
    assert ne == len(R.build_edges(poses, k, loops))
    j = _decisive_prefix(to, ro["chi2_initial"])
    assert j >= min_prefix, j
    np.testing.assert_array_equal(tp[:j, :2], to[:j, :2])  # iteration and accept / reject of every trial
    np.testing.assert_allclose(tp[:j, 2:], to[:j, 2:], rtol=1e-9, atol=0)  # lambda and chi2
    if j == len(to):
        assert len(tp) == len(to) and rp[2] == ro["iterations"] and rp[3] == ro["trials"]
    assert abs(rp[0] - ro["chi2_initial"]) <= 1e-12 * ro["chi2_initial"]
    assert abs(rp[1] - ro["chi2_final"]) <= 1e-9 * ro["chi2_initial"]
    for a, b in zip(Xp, Xo):
        dt, dr = synth.pose_error(a, b)
        assert dt < 1e-9 and dr < 1e-9, (dt, dr)
    return Xp, rp


def test_product_lm_matches_on_the_drifted_square(pg):
    gt, dr = drifted_square()
    n = len(dr)
    Xp, rp = _check_against_restatement(pg, dr, 5, [(0, n - 1, np.linalg.inv(gt[0]) @ gt[-1])], min_prefix=8)
    assert synth.pose_error(Xp[-1], gt[-1])[0] < 0.01 * synth.pose_error(dr[-1], gt[-1])[0]


def test_product_lm_matches_on_the_drifted_out_and_back_drive(pg):
    from test_scanmatcher import _out_and_back

    truth = [T for _, T in _out_and_back(rings=4, azimuths=8)]
    poses = [drift(k) @ T for k, T in enumerate(truth)]
    loop = np.linalg.inv(truth[0]) @ truth[-1] @ synth.pose_matrix((0.01, -0.02, 0.0), (0.0, 0.0, 0.002))
    Xp, _ = _check_against_restatement(pg, poses, 5, [(0, len(poses) - 1, loop)], min_prefix=3)
    assert synth.pose_error(Xp[-1], truth[-1])[0] < 0.5 * synth.pose_error(poses[-1], truth[-1])[0]


def test_product_lm_matches_on_a_300_vertex_graph_with_loops(pg):
    gt, dr, loops = long_drive()
    _check_against_restatement(pg, dr, 5, loops, min_prefix=10)


def test_product_returns_the_poses_bitwise_without_loop_edges(pg):
    _, dr = drifted_square()
    for k in (1, 5):
        Xp, rp, tp, _ = product_adjust(pg, dr, k, [], 10)
        assert np.array_equal(Xp, dr) and rp[0] == 0.0 and rp[1] == 0.0 and rp[2] == 1 and rp[3] == 1
    Xp, rp, _, ne = product_adjust(pg, dr[:4], 5, [], 10)  # no edge at all: nothing to optimise
    assert ne == 0 and np.array_equal(Xp, dr[:4]) and rp[2] == 0


def test_envelope_cholesky_solves_band_plus_loop_systems(pg):
    rng = np.random.default_rng(17)
    for n, k, loops in [(1, 1, []), (12, 1, [(0, 11)]), (40, 5, [(2, 39), (10, 30), (0, 25)]), (120, 5, [(3, 100), (50, 119), (60, 90)])]:
        pairs = [(i - k + j, i) for i in range(1, n) for j in range(k) if i - k + j >= 0] + loops
        H = 1e-3 * np.eye(6 * n)
        for a, b in pairs + [(i, i) for i in range(n)]:
            B = np.zeros((6, 6 * n))
            B[:, 6 * a:6 * a + 6] += rng.normal(size=(6, 6))
            B[:, 6 * b:6 * b + 6] += rng.normal(size=(6, 6))
            H += B.T @ B
        x_true = rng.normal(size=6 * n)
        b = H @ x_true
        P = np.array(pairs, dtype=np.int32).reshape(-1)
        x = np.zeros(6 * n)
        assert pg.pg_envelope_solve(n, len(pairs), _p(P), _p(np.ascontiguousarray(H)), _p(b), _p(x)) == 1
        assert np.linalg.norm(H @ x - b) <= 1e-10 * np.linalg.norm(b)
        first = np.zeros(n, dtype=np.int32)
        pg.pg_envelope_first(n, len(pairs), _p(P), _p(first))
        want = [min([i] + [min(a, b) for a, b in pairs if max(a, b) == i]) for i in range(n)]
        assert first.tolist() == want
    H = -np.eye(12)  # not positive definite: the factorisation refuses it
    x = np.zeros(12)
    assert pg.pg_envelope_solve(2, 0, _p(np.zeros(2, dtype=np.int32)), _p(H), _p(np.ones(12)), _p(x)) == 0
