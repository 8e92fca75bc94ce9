"""Merging a second mapping session into the session's map (b200sm_merge_session) on the GPU: K16's scores bitwise the host
compile of csrc/scan_context.hpp and K13b's, the device's selection equal to the host's ordering of the read-back matrix;
every verification row bitwise the plain registration calls; end to end on NDT and GICP, a second recording in a foreign
frame placed and adjusted onto the first; wrong matches kept out of the consistent set; an unrelated scene refused with
the session untouched; and the session rules and argument errors."""
import ctypes as C
import math

import numpy as np
import pytest

import mergeref as M
import scancontextref as R
from test_scan_context_cpu import host_descriptor, host_distance, random_cloud, sc  # noqa: F401 (fixture)

F32 = np.float32
pytestmark = pytest.mark.gpu


def _session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    return ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _registration(kind):
    from lidarslam_ros2_b200.scanmatcher import backend_registration

    return backend_registration(kind, ndt_resolution=2.0)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype in (F32, np.int32) else np.uint64)


def _pose(k):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix((1.5 * k, 0.25 * k, 0.0), (0.0, 0.0, 0.3 * k))


def _load(g, clouds, d0=0.0):
    for k, c in enumerate(clouds):
        g.importSubmap(c, _pose(k), d0 + 2.0 * k)


def _tile(R_, S):
    g, h = _session(), _session()
    g.setScanContextParams(R_, S, 80.0, 2.0)
    h.setScanContextParams(R_, S, 80.0, 2.0)
    g.importSubmap(random_cloud(1, 50), _pose(0), 0.0)
    h.importSubmap(random_cloud(2, 50), _pose(0), 0.0)
    _, _, res = g.mergeSession(h, _registration("NDT"), sc_threshold=-1.0)
    return res["query_tile"]


def _scores(R_, S, nA, nB, seed):
    """dst of nA and src of nB submaps (random clouds, a few empty ones and duplicates), merged with no candidate."""
    def clouds(n, s0):
        out = [random_cloud(s0 + k, 400 + 13 * (k % 7)) for k in range(n)]
        if n > 3:
            out[1] = out[0].copy()                     # equal D for two candidates
            out[2] = np.zeros((0, 4), dtype=F32)       # an all-zero descriptor
        return out
    A, B = clouds(nA, seed), clouds(nB, seed + 5000)
    g, h = _session(), _session()
    for s in (g, h):
        s.setScanContextParams(R_, S, 80.0, 2.0)
    _load(g, A)
    _load(h, B)
    rows, poses, res = g.mergeSession(h, _registration("NDT"), sc_threshold=-1.0)
    assert rows == [] and poses is None and not res["merged"] and res["candidates"] == 0
    assert res["pairs_scored"] == nA * nB
    D, Sh = g.mergeScores()
    assert D.shape == (nB, nA) and Sh.shape == (nB, nA)
    return g, h, A, B, D, Sh


@pytest.mark.parametrize("R_,S", [(20, 60), (1, 1), (128, 64)])
def test_k16_scores_bitwise_host(sc, R_, S):  # noqa: F811
    t = _tile(R_, S)
    assert 1 <= t <= 32
    sizes = [(1, 1), (t - 1 or 1, t + 1), (t, t), (t + 1, t - 1 or 1), (300, t + 1)]
    if (R_, S) == (20, 60):
        sizes += [(t + 1, 300), (300, 300)]
    for nA, nB in sizes:
        _, _, A, B, D, Sh = _scores(R_, S, nA, nB, 100 * nA + nB)
        hd = [host_descriptor(sc, c, R_, S) for c in A]
        for b in range(nB):
            Q, nQ = host_descriptor(sc, B[b], R_, S)
            for a in range(nA):
                d, s = host_distance(sc, Q, nQ, *hd[a])
                assert _bits(np.float64(D[b, a])) == _bits(np.float64(d)) and Sh[b, a] == s, (nA, nB, b, a)
            if nA > 3:
                assert D[b, 2] == 1.0 and D[b, 0] == D[b, 1]  # all-zero descriptor; duplicated candidate


def test_k16_scores_bitwise_k13b(sc):  # noqa: F811
    g, h, A, B, D, Sh = _scores(20, 60, 40, 5, 9)
    for b in (0, 4):
        p = _session()
        _load(p, A + [B[b]])
        p.searchLoopPlace(_registration("NDT"), voxel_leaf_size=0.5, distance_loop_closure=-1e9, sc_threshold=-1.0, top_k=1)
        Dp, Sp = p.placeScores()
        assert np.array_equal(_bits(Dp[:40]), _bits(D[b])) and np.array_equal(Sp[:40], Sh[b])


def test_selection_equals_host_ordering():
    g, h, A, B, D, Sh = _scores(20, 60, 45, 12, 31)
    for thr, top_k, maxv in ((float(np.median(D)), 3, 8), (float(D.min()), 2, 5), (float(np.quantile(D, 0.3)), 32, 40)):
        rows, _, res = g.mergeSession(h, _registration("NDT"), sc_threshold=thr, top_k=top_k, max_verifications=maxv,
                                      threshold_loop_closure_score=-1.0)
        want = M.order(D, thr, top_k, maxv)
        assert res["candidates"] == sum(len(M.select_row(D[b], thr, top_k)) for b in range(len(D)))
        assert [(r["sc_distance"], r["src_id"], r["id_min"]) for r in rows] == want, thr
        assert all(r["shift"] == Sh[r["src_id"], r["id_min"]] for r in rows)
        assert not res["merged"] and res["accepted"] == 0


# ---------------------------------------------------------------- the two-session drive
@pytest.fixture(scope="module")
def drive():
    scans, poses, _ = R.drive()
    return scans, poses, M.sessions(poses)


def _sessions(drive):
    scans, poses, (A, dA, B, dB) = drive
    g, h = _session(), _session()
    for j, k in enumerate(M.A_IDX):
        g.importSubmap(scans[k], A[j], dA[j])
    for j, k in enumerate(M.B_IDX):
        h.importSubmap(scans[k], B[j], dB[j])
    return g, h


def _state(s):
    cloud, off = s.assembleMap()
    subs = [s.submap(k) for k in range(s.numSubmaps())]
    return cloud, off, subs, [s.scanContext(k) for k in range(s.numSubmaps())], s.segments()


def _same_state(x, y):
    assert np.array_equal(_bits(x[0]), _bits(y[0])) and np.array_equal(x[1], y[1]) and x[4] == y[4]
    for a, b in zip(x[2], y[2]):
        assert np.array_equal(_bits(a[0]), _bits(b[0])) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    assert len(x[3]) == len(y[3]) and all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(x[3], y[3]))


@pytest.mark.parametrize("kind", ["NDT", "GICP"])
def test_rows_are_the_plain_calls(drive, kind):
    import lidarslam_ros2_b200 as m

    scans, poses, (A, dA, B, dB) = drive
    g, h = _sessions(drive)
    cloud, off = g.assembleMap()
    src, soff = h.assembleMap()
    rows, _, res = g.mergeSession(h, _registration(kind), max_verifications=6)
    assert len(rows) == res["verified"] == min(6, res["candidates"]) and rows
    plain = _registration(kind)
    for r in rows:
        a, b = r["id_min"], r["src_id"]
        G = R.guess(A[a], B[b], r["shift"], 60)
        assert np.array_equal(_bits(r["guess"]), _bits(G))
        lo, hi = max(a - 1, 0), min(a + 1, len(A) - 1)
        window = m.voxel_grid_filter(cloud[off[lo]:off[hi + 1]], 0.3)
        plain.setInputTarget(window)
        plain.setInputSource(src[soff[b]:soff[b + 1]])
        fin = plain.align(G)
        fit = plain.getFitnessScore()
        assert r["n_target"] == len(window) and r["n_source"] == soff[b + 1] - soff[b]
        assert np.array_equal(_bits(r["final"]), _bits(fin)) and r["fitness"] == fit, (a, b)
        FP = fin.astype(np.float64) @ B[b]
        assert r["min_dist"] == pytest.approx(np.linalg.norm(A[a][:3, 3] - FP[:3, 3]), abs=1e-9)
        assert r["accepted"] == (fit < 1.0)
        if r["accepted"]:
            np.testing.assert_allclose(r["relative_pose"], M.edge(A[a], fin.astype(np.float64), B[b]), atol=1e-9)


@pytest.mark.parametrize("kind", ["NDT", "GICP"])
def test_end_to_end_two_sessions(drive, kind):
    from lidarslam_ros2_b200 import synth

    scans, poses, (A, dA, B, dB) = drive
    g, h = _sessions(drive)
    before_src = _state(h)
    nA, nB = len(A), len(B)
    rows, X, res = g.mergeSession(h, _registration(kind))
    assert res["merged"] and res["inliers"] >= 2 and res["first_submap"] == nA, res
    assert g.segments() == [0, nA] and g.numSubmaps() == nA + nB
    first = next(r for r in rows if r["inlier_rank"] == 0)
    b0 = first["src_id"]
    np.testing.assert_array_equal(res["T"], first["final"].astype(np.float64))
    dt, dr = synth.pose_error(res["T"] @ B[b0], poses[M.B_IDX[b0]])
    assert dt <= 0.3 and dr <= 0.02, (dt, dr)
    rigid = [synth.pose_error(res["T"] @ B[b], poses[M.B_IDX[b]]) for b in range(nB)]
    adj = [synth.pose_error(X[nA + b], poses[M.B_IDX[b]]) for b in range(nB)]
    r_t, r_r = np.mean([e[0] for e in rigid]), np.mean([e[1] for e in rigid])
    a_t, a_r = np.mean([e[0] for e in adj]), np.mean([e[1] for e in adj])
    # The joint adjustment turns B towards the truth but does not pull it in: with identity information, B's odometry
    # edges (2.5 % too long, 0.006 rad a step) outweigh one inter-session edge per submap, and the stretch is split between
    # both chains (DESIGN.md section 7b). Measured: heading 0.026 -> 0.021 rad (NDT), 0.037 -> 0.026 rad (GICP); position
    # 0.56 -> 0.58 m and 0.97 -> 0.68 m.
    assert a_r < r_r and a_t < 1.0 and res["adjust"]["chi2_final"] < res["adjust"]["chi2_initial"], (kind, r_t, r_r, a_t, a_r)
    assert all(synth.pose_error(r["final"].astype(np.float64) @ B[r["src_id"]], poses[M.B_IDX[r["src_id"]]])[0] < 2.0
               for r in rows if r["inlier"])
    # the appended submaps: src's clouds at the rigid placement, distance d_A,last + d_b
    for b in range(nB):
        c, P, d = g.submap(nA + b)
        c0, _, d0 = h.submap(b)
        assert np.array_equal(_bits(c), _bits(c0)) and d == dA[-1] + d0
        np.testing.assert_allclose(P, M.placement(res["T"], B[b]), rtol=0, atol=1e-9)
    # the merged map at poses_out: both sessions' submaps moved by their adjusted poses cast to float, bitwise what a
    # session holding the same submaps assembles, and the float transform on the host
    cloud, off = g.assembleMap(X)
    ref = _session()
    for i in range(nA + nB):
        c, P, d = g.submap(i)
        ref.importSubmap(c, P, d)
    cloud2, off2 = ref.assembleMap(X)
    assert np.array_equal(_bits(cloud), _bits(cloud2)) and np.array_equal(off, off2)
    for i in range(nA + nB):
        src_pts = g.submap(i)[0]
        assert np.array_equal(_bits(src_pts[:, :3]), _bits(scans[(M.A_IDX + M.B_IDX)[i]][:, :3]))
        T = X[i].astype(F32)
        np.testing.assert_allclose(cloud[off[i]:off[i + 1], :3], src_pts[:, :3] @ T[:3, :3].T + T[:3, 3], rtol=0, atol=2e-4)
    # poseAdjust with the returned edges reproduces the joint adjustment bit for bit
    Y, info = g.poseAdjust(res["edges"], num_adjacent_pose_cnstraints=5, max_iterations=10)
    assert np.array_equal(_bits(Y), _bits(X)) and info["n_edges"] == res["adjust"]["n_edges"]
    _same_state(before_src, _state(h))  # src is only read


def test_wrong_matches_stay_out_of_the_consistent_set(drive):
    scans, poses, (A, dA, B, dB) = drive
    g, h = _sessions(drive)
    rows, _, res = g.mergeSession(h, _registration("NDT"), threshold_loop_closure_score=50.0, sc_threshold=0.7, top_k=8,
                                  max_verifications=200)
    wrong = []
    for r in rows:
        if not r["accepted"]:
            continue
        b, a = r["src_id"], r["id_min"]
        place = r["final"].astype(np.float64) @ B[b]
        off = np.linalg.norm(place[:3, 3] - poses[M.B_IDX[b]][:3, 3])
        if abs(a - M.true_match(poses, b)) > 2 or off > 2.0:
            wrong.append(r)
    assert wrong, "no wrong row was accepted"
    assert not any(r["inlier"] for r in wrong), [(r["src_id"], r["id_min"]) for r in wrong if r["inlier"]]
    assert res["merged"] and res["inliers"] >= 2


def test_unrelated_scene_is_refused_and_dst_unchanged(drive):
    from lidarslam_ros2_b200 import synth

    scans, poses, (A, dA, B, dB) = drive
    g, _ = _sessions(drive)
    field = M.unrelated_scene()
    h = _session()
    for j in range(12):
        P = synth.pose_matrix((-40.0 + 4.0 * j, 0.0, synth.SENSOR_HEIGHT), (0.0, 0.0, 0.01 * j))
        h.importSubmap(synth.make_scan(field, 16, 450, P, stream=4400 + j), np.linalg.inv(M.FOREIGN) @ P, 4.0 * j)
    before = _state(g)
    rows, X, res = g.mergeSession(h, _registration("NDT"))
    assert not res["merged"] and X is None and res["first_submap"] == -1
    assert res["inliers"] < 2
    _same_state(before, _state(g))
    assert len(rows) == res["verified"]


def test_session_rules_and_argument_errors(drive):
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    scans, poses, (A, dA, B, dB) = drive
    g, h = _sessions(drive)
    reg = _registration("NDT")
    L = _capi.lib()
    n = C.c_size_t(0)
    res = _capi.SmMergeResult()
    rows = (_capi.SmMergeRow * 4)()
    before = _state(g)
    p0 = dict(_capi.MERGE_DEFAULTS)

    def call(dst, src, edges=(), rows_=rows, cap=4, **kw):
        p = _capi.SmMergeParams(**{**p0, **kw})
        arr = (_capi.SmLoopEdge * max(1, len(edges)))()
        for k, (f, t) in enumerate(edges):
            arr[k].from_, arr[k].to = f, t
            arr[k].relative_pose[:] = np.eye(4).reshape(16).tolist()
        return L.b200sm_merge_session(dst, src, reg._h, C.byref(p), arr, len(edges), rows_, cap, C.byref(n), None, C.byref(res))

    assert call(g._h, g._h) == _capi.ERR_ARG
    assert call(None, h._h) == _capi.ERR_ARG and call(g._h, None) == _capi.ERR_ARG
    for bad in (dict(top_k=0), dict(top_k=33), dict(max_verifications=0), dict(max_verifications=1025),
                dict(sc_threshold=math.nan), dict(voxel_leaf_size=0.0), dict(search_submap_num=-1), dict(min_inliers=0),
                dict(consistency_translation=-1.0), dict(consistency_drift_rotation=math.inf),
                dict(num_adjacent_pose_cnstraints=0), dict(max_iterations=-1), dict(threshold_loop_closure_score=math.nan)):
        assert call(g._h, h._h, **bad) == _capi.ERR_ARG, bad
    nA, nB = g.numSubmaps(), h.numSubmaps()
    for e in ((0, nA + nB), (-1, 3), (4, 4)):
        assert call(g._h, h._h, edges=[e]) == _capi.ERR_ARG, e
    assert call(g._h, h._h, rows_=None, cap=4) == _capi.ERR_ARG
    empty = _session()
    assert call(g._h, empty._h) == _capi.ERR_ARG and call(empty._h, h._h) == _capi.ERR_ARG
    other = _session()
    other.setScanContextParams(20, 72, 80.0, 2.0)
    other.importSubmap(scans[0], A[0], 0.0)
    assert call(g._h, other._h) == _capi.ERR_ARG
    _same_state(before, _state(g))
    # the pair cap: (2^14 + 1)^2 > 2^28 pairs are refused before anything is allocated
    big1, big2 = _session(), _session()
    one = np.zeros((1, 4), dtype=F32)
    for k in range((1 << 14) + 1):
        big1.importSubmap(one, np.eye(4), float(k))
        big2.importSubmap(one, np.eye(4), float(k))
    assert call(big1._h, big2._h) == _capi.ERR_ARG
    assert "2^28" in L.b200sm_last_error(big1._h).decode()
    # a merged session is a backend's map: the frontend's calls are refused and change nothing
    _, _, r = g.mergeSession(h, reg)
    assert r["merged"]
    merged = _state(g)
    st = g.stats()
    pts = scans[0]
    for f in (lambda: g.setScan(pts), lambda: g.receiveCloud(pts),
              lambda: g.updateMap(np.eye(4), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))):
        with pytest.raises(B200RegError) as e:
            f()
        assert e.value.code == _capi.ERR_ARG
    assert g.stats() == st
    _same_state(merged, _state(g))
    # import appends to the last segment
    g.importSubmap(pts, np.eye(4), 999.0)
    assert g.segments() == [0, nA] and g.numSubmaps() == nA + nB + 1


def test_a_merged_src_keeps_its_segments(drive):
    """Merging a session that is itself a merged map: its segments are appended, so no odometry edge joins its two
    recordings, in the merge's joint graph or in a later poseAdjust."""
    scans, poses, (A, dA, B, dB) = drive
    g, h = _sessions(drive)  # g: A; h: B
    other = _session()  # A's recording again, in a frame of its own: merged into h, h holds two segments
    W2 = np.linalg.inv(M.FOREIGN) @ np.linalg.inv(M.FOREIGN)
    for j, k in enumerate(M.A_IDX):
        other.importSubmap(scans[k], W2 @ A[j], dA[j])
    _, _, r1 = h.mergeSession(other, _registration("NDT"))
    assert r1["merged"] and h.segments() == [0, len(B)]
    nA, nH = g.numSubmaps(), h.numSubmaps()
    rows, X, res = g.mergeSession(h, _registration("NDT"))
    assert res["merged"] and g.segments() == [0, nA, nA + len(B)] and g.numSubmaps() == nA + nH
    k = 5
    odo = sum(max(0, n - k - 1) * k for n in (nA, len(B), len(A)))  # the reference's rule inside each segment
    assert res["adjust"]["n_edges"] == odo + res["inliers"]
    Y, info = g.poseAdjust(res["edges"], num_adjacent_pose_cnstraints=k, max_iterations=10)
    assert np.array_equal(_bits(Y), _bits(X)) and info["n_edges"] == res["adjust"]["n_edges"]


def test_empty_submaps_give_rows_that_are_not_accepted():
    """A selected src submap without points, and a dst window without points, are rows that are not accepted: the merge
    still reports every row and leaves dst as it was."""
    def clouds(n, s0):
        out = [random_cloud(s0 + k, 600) for k in range(n)]
        out[2] = np.zeros((0, 4), dtype=F32)
        return out
    g, h = _session(), _session()
    _load(g, clouds(6, 70))
    _load(h, clouds(4, 90))
    before = _state(g)
    rows, X, res = g.mergeSession(h, _registration("NDT"), sc_threshold=2.5, top_k=32, max_verifications=100,
                                  search_submap_num=0)
    assert len(rows) == res["verified"] == res["candidates"] == 24
    is_empty = [r["src_id"] == 2 or r["id_min"] == 2 for r in rows]
    empty = [r for r, e in zip(rows, is_empty) if e]
    assert len(empty) == 9 and all(not r["accepted"] and r["fitness"] == math.inf and not r["inlier"] for r in empty)
    assert all(r["n_source"] > 0 and r["n_target"] > 0 for r, e in zip(rows, is_empty) if not e)
    if not res["merged"]:
        _same_state(before, _state(g))
