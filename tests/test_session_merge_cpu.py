"""The host part of b200sm_merge_session on the CPU: csrc/session_merge.hpp and the segmented build_edges of
csrc/pose_graph.hpp compiled with g++ -ffp-contract=off (tests/hostmath/session_merge_host.cpp) against the float64 replay
tests/mergeref.py. Candidate selection and ordering with ties and thresholds at equality; the cycle error and its
tolerance at equality and one ulp either side, with and without the drift term; the greedy consistent set; the edge and the
placement; the segmented odometry edges (bitwise today's with one segment); the joint LM against tests/posegraphref.py;
the replay told apart from its named mutations; and the consistency defaults on the two-session drive's poses."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import mergeref as M
import posegraphref as PG
from lidarslam_ros2_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "session_merge_host.cpp")
DEFAULT_TOL = dict(consistency_translation=1.5, consistency_rotation=0.1, consistency_drift_translation=0.02,
                   consistency_drift_rotation=0.003)


@pytest.fixture(scope="module")
def smh(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("smh"), "libsession_merge_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    lib = C.CDLL(lib)
    vp, d, i = C.c_void_p, C.c_double, C.c_int
    lib.smh_select_row.argtypes = [vp, i, d, i, vp]
    lib.smh_order.argtypes = [i, vp, vp, vp, i, vp, vp]
    lib.smh_edge.argtypes = [vp, vp, vp, vp]
    lib.smh_place.argtypes = [vp, vp, vp]
    lib.smh_cycle_error.argtypes = [vp, vp, vp, vp, vp, vp, C.POINTER(d), C.POINTER(d)]
    lib.smh_within.argtypes = [d, d, d, vp]
    lib.smh_inliers.argtypes = [i, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.smh_build_edges.argtypes = [i, vp, i, i, vp, i, vp, vp, vp, vp]
    lib.smh_adjust.argtypes = [i, vp, i, i, vp, i, vp, vp, i, vp, vp]
    return lib


def _p(a):
    return a.ctypes.data


def _tol4(tol):
    return np.array([tol[k] for k in M.TOL_FIELDS], dtype=np.float64)


def _rm(P):
    return np.ascontiguousarray(P, dtype=np.float64).reshape(16)


def host_select(smh, D, thr, top_k):
    D = np.ascontiguousarray(D, dtype=np.float64)
    out = np.zeros(max(1, top_k), dtype=np.int32)
    n = smh.smh_select_row(_p(D), len(D), thr, top_k, _p(out))
    return out[:n].tolist()


def host_order(smh, cands, maxv):
    D = np.array([c[0] for c in cands], dtype=np.float64)
    b = np.array([c[1] for c in cands], dtype=np.int32)
    a = np.array([c[2] for c in cands], dtype=np.int32)
    ob, oa = np.zeros(len(cands) + 1, dtype=np.int32), np.zeros(len(cands) + 1, dtype=np.int32)
    n = smh.smh_order(len(cands), _p(D), _p(b), _p(a), maxv, _p(ob), _p(oa))
    return list(zip(ob[:n].tolist(), oa[:n].tolist()))


def host_cycle(smh, i, j):
    args = [_rm(m) for m in (i["Pa"], i["Pb"], i["Z"], j["Pa"], j["Pb"], j["Z"])]
    et, er = C.c_double(), C.c_double()
    smh.smh_cycle_error(*(_p(a) for a in args), C.byref(et), C.byref(er))
    return et.value, er.value


def host_within(smh, et, er, L, tol):
    t = _tol4(tol)
    return bool(smh.smh_within(et, er, L, _p(t)))


def host_inliers(smh, rows, tol):
    n = len(rows)
    Pa = np.array([_rm(r["Pa"]) for r in rows])
    Pb = np.array([_rm(r["Pb"]) for r in rows])
    Z = np.array([_rm(r["Z"]) for r in rows])
    da, db, fit = (np.array([r[k] for r in rows], dtype=np.float64) for k in ("da", "db", "fitness"))
    out = np.zeros(n + 1, dtype=np.int32)
    t = _tol4(tol)
    k = smh.smh_inliers(n, _p(Pa), _p(Pb), _p(Z), _p(da), _p(db), _p(fit), _p(t), _p(out))
    return out[:k].tolist()


def host_edges(smh, poses, k, seg_first=None, loops=()):
    n = len(poses)
    P = np.ascontiguousarray(np.array(poses, dtype=np.float64).reshape(n, 16))
    segs = np.array(seg_first if seg_first is not None else [0], dtype=np.int32)
    lp = np.array([(f, t) for f, t, _ in loops] or [(0, 0)], dtype=np.int32)
    rel = np.array([_rm(Z) for _, _, Z in loops] or [np.eye(4).reshape(16)], dtype=np.float64)
    cap = n * k + len(loops) + 1
    ft = np.zeros(2 * cap, dtype=np.int32)
    zi = np.zeros(16 * cap, dtype=np.float64)
    m = smh.smh_build_edges(n, _p(P), k, 0 if seg_first is None else len(segs), _p(segs), len(loops), _p(lp), _p(rel), _p(ft), _p(zi))
    return ft[:2 * m].reshape(m, 2), zi[:16 * m].reshape(m, 4, 4)


def host_adjust(smh, poses, k, seg_first, loops, max_iterations=10):
    n = len(poses)
    P = np.ascontiguousarray(np.array(poses, dtype=np.float64).reshape(n, 16))
    segs = np.array(seg_first, dtype=np.int32)
    lp = np.array([(f, t) for f, t, _ in loops] or [(0, 0)], dtype=np.int32)
    rel = np.array([_rm(Z) for _, _, Z in loops] or [np.eye(4).reshape(16)], dtype=np.float64)
    out = np.zeros((n, 16), dtype=np.float64)
    res = np.zeros(4)
    smh.smh_adjust(n, _p(P), k, len(segs), _p(segs), len(loops), _p(lp), _p(rel), max_iterations, _p(out), _p(res))
    return out.reshape(n, 4, 4), res


def _rand_pose(rng, t=5.0, ang=0.4):
    return synth.pose_matrix(rng.uniform(-t, t, 3), rng.uniform(-ang, ang, 3))


def _row(rng, F, a=0, b=0, fitness=0.1, da=None, db=None):
    """An accepted row whose registration gave F (4x4 float32) for random end poses."""
    Pa, Pb = _rand_pose(rng, 30.0), _rand_pose(rng, 30.0)
    F = np.asarray(F, dtype=np.float32)
    return dict(a=a, b=b, Pa=Pa, Pb=Pb, Z=M.edge(Pa, F.astype(np.float64), Pb), fitness=fitness,
                da=float(rng.uniform(0, 100)) if da is None else da, db=float(rng.uniform(0, 100)) if db is None else db, F=F)


# ---------------------------------------------------------------- candidate selection and ordering
def test_row_selection_ties_and_threshold_at_equality(smh):
    D = np.array([0.3, 0.2, 0.3, 0.1, 0.2, 0.25, 0.3, 0.5])
    for thr, k in ((0.3, 8), (math.nextafter(0.3, 1.0), 8), (0.3, 3), (0.2, 2), (0.1, 5), (math.nextafter(0.3, 1.0), 4), (1.0, 1)):
        want = M.select_row(D, thr, k)
        assert host_select(smh, D, thr, k) == want, (thr, k)
    assert host_select(smh, D, 0.3, 8) == [3, 1, 4, 5]                          # D < thr: the 0.3s are out
    assert host_select(smh, D, math.nextafter(0.3, 1.0), 8) == [3, 1, 4, 5, 0, 2, 6]  # one ulp above: in, by index
    assert host_select(smh, D, math.nextafter(0.3, 1.0), 6) == [3, 1, 4, 5, 0, 2]
    assert M.select_row(D, 1.0, 8, mut=("tie_high",)) != M.select_row(D, 1.0, 8)


def test_global_order_and_verification_cut(smh):
    rng = np.random.default_rng(3)
    D = np.round(rng.uniform(0, 1, size=(9, 14)), 1)  # many ties in D
    for thr, k, maxv in ((0.5, 3, 1000), (0.5, 3, 7), (0.3, 32, 4), (math.nextafter(0.3, 1.0), 2, 11), (0.0, 3, 5)):
        want = M.order(D, thr, k, maxv)
        cands = [(float(D[b][a]), b, a) for b in range(len(D)) for a in host_select(smh, D[b], thr, k)]
        rng.shuffle(cands)
        got = host_order(smh, cands, maxv)
        assert got == [(b, a) for _, b, a in want], (thr, k, maxv)
        assert len(got) == min(maxv, sum(min(k, int((D[b] < thr).sum())) for b in range(len(D))))
    # a tie in D goes to the lower b, then the lower a
    assert host_order(smh, [(0.2, 3, 1), (0.2, 1, 5), (0.2, 1, 2), (0.1, 7, 7)], 3) == [(7, 7), (1, 2), (1, 5)]


# ---------------------------------------------------------------- edge, placement, cycle error and tolerance
def test_edge_and_placement(smh):
    rng = np.random.default_rng(5)
    for _ in range(20):
        Pa, Pb = _rand_pose(rng, 50.0), _rand_pose(rng, 50.0)
        F = _rand_pose(rng, 80.0, 3.0).astype(np.float32)
        Z = np.zeros(16)
        Fc = np.ascontiguousarray(F.T).reshape(16)
        smh.smh_edge(_p(_rm(Pa)), _p(Fc), _p(_rm(Pb)), _p(Z))
        np.testing.assert_allclose(Z.reshape(4, 4), M.edge(Pa, F.astype(np.float64), Pb), rtol=0, atol=1e-9)
        X = np.zeros(16)
        smh.smh_place(_p(_rm(F.astype(np.float64))), _p(_rm(Pb)), _p(X))
        np.testing.assert_allclose(X.reshape(4, 4), M.placement(F, Pb), rtol=0, atol=1e-12)
        # the edge from a to b: P_a Z is the placement of b
        np.testing.assert_allclose(Pa @ Z.reshape(4, 4), X.reshape(4, 4), rtol=0, atol=1e-9)
    # Z from the wrong end is not the edge
    assert not np.allclose(M.edge(Pa, F.astype(np.float64), Pb, mut=("z_wrong_end",)), Z.reshape(4, 4), atol=1e-3)


def test_cycle_error_matches_the_replay(smh):
    rng = np.random.default_rng(7)
    F = _rand_pose(rng, 40.0, 3.0)
    for _ in range(50):
        dF = synth.pose_matrix(rng.uniform(-0.5, 0.5, 3), rng.uniform(-0.05, 0.05, 3))
        i, j = _row(rng, F), _row(rng, dF @ F)
        et, er = host_cycle(smh, i, j)
        rt, rr = M.cycle_error(i, j)
        assert abs(et - rt) <= 1e-9 and abs(er - rr) <= 1e-7, (et, rt, er, rr)
    i, j = _row(rng, F), _row(rng, F)  # the same F: no cycle error
    et, er = host_cycle(smh, i, j)
    assert et < 1e-4 and er < 1e-3


def test_tolerance_at_equality_and_one_ulp_either_side(smh):
    tol = dict(DEFAULT_TOL)
    for L in (0.0, 37.25):
        bt = tol["consistency_translation"] + tol["consistency_drift_translation"] * L
        br = tol["consistency_rotation"] + tol["consistency_drift_rotation"] * L
        for et, er, want in ((bt, br, True), (math.nextafter(bt, 0), br, True), (math.nextafter(bt, 99), br, False),
                             (bt, math.nextafter(br, 0), True), (bt, math.nextafter(br, 99), False)):
            assert host_within(smh, et, er, L, tol) == want == M.within(et, er, L, tol), (L, et, er)
    # the L term: an error only the drift allowance admits
    L = 50.0
    et = tol["consistency_translation"] + 0.5 * tol["consistency_drift_translation"] * L
    assert host_within(smh, et, 0.0, L, tol) and M.within(et, 0.0, L, tol)
    assert not M.within(et, 0.0, L, tol, mut=("no_drift",))
    assert not host_within(smh, et, 0.0, 0.0, tol)


def test_greedy_consistent_set(smh):
    rng = np.random.default_rng(11)
    F = _rand_pose(rng, 40.0, 3.0)
    off = synth.pose_matrix((7.0, 0.0, 0.0), (0.0, 0.0, 0.0)) @ F  # one pilaster along
    tol = dict(DEFAULT_TOL)
    # fitness ties: rows 0 (right) and 1 (wrong) tie; the lower index joins first and keeps the wrong one out, while
    # tie_high lets the wrong one lead and keeps the right ones out
    rows = [_row(rng, F, fitness=0.2, da=10.0, db=10.0), _row(rng, off, fitness=0.2, da=12.0, db=11.0),
            _row(rng, F, fitness=0.3, da=20.0, db=30.0)]
    assert host_inliers(smh, rows, tol) == M.inliers(rows, tol) == [0, 2]
    assert M.inliers(rows, tol, mut=("tie_high",)) == [1]
    # the best fitness leads even when it is wrong: then the right ones cannot join it
    rows += [_row(rng, F, fitness=0.1, da=40.0, db=5.0), _row(rng, off, fitness=0.05, da=60.0, db=60.0)]
    assert host_inliers(smh, rows, tol) == M.inliers(rows, tol) == [4, 1]
    rows[4]["fitness"] = 0.5
    assert host_inliers(smh, rows, tol) == M.inliers(rows, tol) == [3, 0, 2]


# ---------------------------------------------------------------- the joint graph
def _two_chains(rng, nA=12, nB=9):
    truth = [synth.pose_matrix((2.0 * k, 0.3 * math.sin(k), 0.0), (0.0, 0.0, 0.05 * k)) for k in range(nA + nB)]
    drift = [synth.pose_matrix((0.02 * k, 0.03 * k, 0.0), (0.0, 0.0, 0.003 * k)) for k in range(nB)]
    poses = truth[:nA] + [truth[nA] @ drift[k] @ np.linalg.inv(truth[nA]) @ truth[nA + k] for k in range(nB)]
    loops = [(3, nA + 2, np.linalg.inv(truth[3]) @ truth[nA + 2]), (9, nA + 7, np.linalg.inv(truth[9]) @ truth[nA + 7])]
    return truth, poses, loops


def test_segmented_edges_equal_the_replay(smh):
    rng = np.random.default_rng(13)
    truth, poses, loops = _two_chains(rng)
    for k, segs in ((5, [0, 12]), (1, [0, 12]), (3, [0, 4, 12, 15]), (5, [0, 3, 12])):
        ft, zi = host_edges(smh, poses, k, segs, loops)
        want = M.joint_edges(poses, k, segs, loops)
        assert [tuple(e) for e in ft.tolist()] == [(f, t) for f, t, _ in want], (k, segs)
        for a, (_, _, b) in zip(zi, want):
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-9)
        assert all(not (f < s <= t) for f, t in ft[:len(ft) - len(loops)].tolist() for s in segs[1:])
    assert M.segment_edges(len(poses), 5, [0, 12], mut=("odometry_across",)) != M.segment_edges(len(poses), 5, [0, 12])


def test_one_segment_is_todays_build_edges_bitwise(smh):
    rng = np.random.default_rng(17)
    truth, poses, loops = _two_chains(rng)
    for k in (1, 3, 5):
        ft0, zi0 = host_edges(smh, poses, k, None, loops)
        ft1, zi1 = host_edges(smh, poses, k, [0], loops)
        assert np.array_equal(ft0, ft1) and np.array_equal(zi0.view(np.uint64), zi1.view(np.uint64))
        assert [tuple(e) for e in ft0.tolist()][:len(ft0) - len(loops)] == PG.graph_edges(len(poses), k)


def test_joint_lm_matches_the_restatement(smh):
    rng = np.random.default_rng(19)
    truth, poses, loops = _two_chains(rng)
    segs = [0, 12]
    Xp, rp = host_adjust(smh, poses, 5, segs, loops, 10)
    Xo, ro, _ = M.joint_adjust(poses, 5, segs, loops, 10)
    assert abs(rp[0] - ro["chi2_initial"]) <= 1e-12 * max(ro["chi2_initial"], 1e-300)
    assert abs(rp[1] - ro["chi2_final"]) <= 1e-9 * ro["chi2_initial"]
    for a, b in zip(Xp, Xo):
        dt, dr = synth.pose_error(a, b)
        assert dt < 1e-9 and dr < 1e-9, (dt, dr)
    assert synth.pose_error(Xp[-1], truth[-1])[0] < synth.pose_error(poses[-1], truth[-1])[0]


# ---------------------------------------------------------------- mutations
def test_each_mutation_changes_an_outcome():
    rng = np.random.default_rng(23)
    tol = dict(DEFAULT_TOL)
    caught = set()
    F = _rand_pose(rng, 40.0, 3.0)
    i, j = _row(rng, F, da=0.0, db=0.0), _row(rng, F, da=60.0, db=60.0)
    if M.cycle_error(i, j, ("cycle_order",))[0] > 1.0 and M.cycle_error(i, j)[0] < 1e-6:
        caught.add("cycle_order")
    Pa, Pb = i["Pa"], i["Pb"]
    if not np.allclose(M.edge(Pa, F, Pb, ("z_wrong_end",)), M.edge(Pa, F, Pb), atol=1e-3):
        caught.add("z_wrong_end")
    if M.segment_edges(20, 5, [0, 10], ("odometry_across",)) != M.segment_edges(20, 5, [0, 10]):
        caught.add("odometry_across")
    if M.select_row([0.1, 0.1, 0.2], 1.0, 1, ("tie_high",)) != M.select_row([0.1, 0.1, 0.2], 1.0, 1):
        caught.add("tie_high")
    drifted = synth.pose_matrix((2.0, 0.0, 0.0), (0.0, 0.0, 0.0)) @ F
    j2 = _row(rng, drifted, da=60.0, db=60.0)
    if M.consistent(i, j2, tol) and not M.consistent(i, j2, tol, ("no_drift",)):
        caught.add("no_drift")
    assert caught == set(M.MUTATIONS), set(M.MUTATIONS) - caught


# ---------------------------------------------------------------- the defaults on the two-session drive
def test_consistency_defaults_on_the_drive():
    """With the true registration of every B submap onto its nearest A submap, every pair of rows is consistent; with one
    of them off by a pilaster (7 m along the canyon) none is, even at the drive's largest L."""
    import scancontextref as SC
    from lidarslam_ros2_b200 import _capi

    tol = {k: _capi.MERGE_DEFAULTS[k] for k in M.TOL_FIELDS}
    assert tol == DEFAULT_TOL
    poses = SC.drive_poses()[0]
    A, dA, B, dB = M.sessions(poses)
    rows = []
    for b in range(len(B)):
        a = M.true_match(poses, b)
        F = poses[M.B_IDX[b]] @ np.linalg.inv(B[b])
        rows.append(dict(a=a, b=b, Pa=A[a], Pb=B[b], Z=M.edge(A[a], F, B[b]), da=dA[a], db=dB[b], fitness=0.1, F=F))
    L_max = max(M.cycle_length(i, j) for i in rows for j in rows)
    assert L_max > 100.0
    for i in rows:
        for j in rows:
            if i is j:
                continue
            assert M.consistent(i, j, tol), (i["b"], j["b"])
            for dx in (7.0, -7.0):
                F7 = synth.pose_matrix((dx, 0.0, 0.0), (0.0, 0.0, 0.0)) @ j["F"]
                jw = dict(j, Z=M.edge(j["Pa"], F7, j["Pb"]))
                assert not M.consistent(i, jw, tol), (i["b"], j["b"], dx)
    assert tol["consistency_translation"] + tol["consistency_drift_translation"] * L_max < 7.0


def test_joint_graph_on_the_drive_with_exact_inter_session_edges(smh):
    """What the joint adjustment can do on the two-session drive, with the true registration of every B submap onto its
    nearest A submap as the inter-session edges (no registration error at all) and the rigid placement by B's submap 13
    (the GPU runs' first inlier with NDT and GICP): the product's graph and LM equal the replay, and neither halves B's
    mean error against the rigid placement. The graph is the issue's: the reference's odometry rule per segment, identity
    information, vertex 0 fixed. Vertex 0 has no odometry edge under that rule, so A's chain is held only through the
    inter-session edges and moves with B: B's odometry (2.5 % too long per step) is split between both chains."""
    import scancontextref as SC

    poses = SC.drive_poses()[0]
    A, dA, B, dB = M.sessions(poses)
    nA, nB = len(A), len(B)
    loops = []
    for b in range(nB):
        a = M.true_match(poses, b)
        loops.append((a, nA + b, M.edge(A[a], poses[M.B_IDX[b]] @ np.linalg.inv(B[b]), B[b])))
    T = poses[M.B_IDX[13]] @ np.linalg.inv(B[13])
    X = A + [M.placement(T, P) for P in B]

    def mean_errors(Y, idx, truth):
        e = [synth.pose_error(Y[i], truth[j]) for i, j in idx]
        return np.mean([v[0] for v in e]), np.mean([v[1] for v in e])

    b_idx = [(nA + b, M.B_IDX[b]) for b in range(nB)]
    rigid = mean_errors(X, b_idx, poses)
    assert 0.9 < rigid[0] < 1.05 and 0.03 < rigid[1] < 0.045, rigid
    for iters in (10, 30):
        Xp, _ = host_adjust(smh, X, 5, [0, nA], loops, iters)
        Xo, _, _ = M.joint_adjust(X, 5, [0, nA], loops, iters)
        for a, b in zip(Xp, Xo):
            assert max(synth.pose_error(a, b)) < 1e-6  # a weakly held graph: rounding differences grow
        adj = mean_errors(Xp, b_idx, poses)
        a_moved = mean_errors(Xp, [(a, a) for a in range(nA)], poses)
        assert adj[0] > 0.5 * rigid[0] and adj[1] > 0.5 * rigid[1], (iters, rigid, adj)
        assert a_moved[0] > 0.5, a_moved  # A's chain, at its true poses before, moved with B
