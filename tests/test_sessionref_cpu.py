"""The frontend-session replay of tests/sessionref.py, checked on the CPU before any GPU comparison: driven by what
oracle/scanmatcher.py computes (its own NDT drives, and drives whose registration is scripted so that they reach the
edges) it must reproduce the oracle's decisions, poses, distances and targeted clouds exactly, and its loop search's
candidate, window and counts exactly; the fixture generators must reach the edges they are named for; and replays of a
subtly wrong session (sessionref.MUTATIONS) must disagree with at least one fixture."""
import math

import numpy as np
import pytest

import gridref as R
import sessionref as S

F32 = np.float32
U = 2.0**-53


class ScriptedReg:
    """A registration whose align() returns the next scripted transform and whose fitness() a scripted score: drives
    the oracle's bookkeeping and loop search through poses chosen to sit on their edges."""

    def __init__(self, finals, fitness=0.5):
        self.finals, self.k, self.score = [np.asarray(f, dtype=F32) for f in finals], 0, fitness

    def set_source(self, c):
        self.n_source = len(c)

    def set_target(self, c):
        self.n_target = len(c)

    def align(self, guess=None):
        f = self.finals[self.k]
        self.k += 1
        return f

    def fitness(self):
        return self.score


def _rot_final(R3, t):
    F = np.eye(4, dtype=F32)
    F[:3, :3] = np.asarray(R3, dtype=F32)
    F[:3, 3] = np.asarray(t, dtype=F32)
    return F


def _bookkeeping_finals():
    """trans_for_mapupdate 5.0 from the origin: a step of exactly 5 (3-4-5), a step of 0, 180-degree turns about x, y
    and z (trace -1: every largest-diagonal branch of Eigen's quaternion), a generic rotation, a step one ulp short."""
    c, s = math.cos(0.4), math.sin(0.4)
    gen = [[c, -s, 0.0], [s * 0.96, c * 0.96, 0.28], [-s * 0.28, -c * 0.28, 0.96]]
    return [_rot_final(np.eye(3), (3, 4, 0)), _rot_final(np.eye(3), (3, 4, 0)),
            _rot_final(np.diag([1, -1, -1]), (3, 4, 12)), _rot_final(np.diag([-1, 1, -1]), (3, 4, 12)),
            _rot_final(np.diag([-1, -1, 1]), (6, 8, 12)), _rot_final(gen, (6.0, 8.0, 7.0)),
            _rot_final(gen, (6.0, 8.0, np.nextafter(F32(12.0), F32(0))))]


def _scripted_drive(finals, thr, nt=3, filt=None):
    """oracle.scanmatcher.ScanMatcher through the scripted finals; returns (oracle, [(pose7, final, updated, trans,
    latest_distance, targeted copy)])."""
    import oracle.scanmatcher as osm

    kw = dict(filt) if filt else {}
    o = osm.ScanMatcher(trans_for_mapupdate=thr, vg_size_for_input=0.5, vg_size_for_map=0.3, num_targeted_cloud=nt, **kw)
    o.reg = ScriptedReg(finals)
    rng = np.random.default_rng(len(finals))
    rows = []
    for k in range(len(finals)):
        cloud = rng.uniform(-20, 20, (300, 4)).astype(F32)
        pose7, final, upd = o.receive_cloud(cloud)
        rows.append((pose7, final, upd, o.trans, o.latest_distance, o.targeted.copy()))
    return o, rows


def _replay_drive(o, rows, thr, nt, mut=()):
    """The replay driven by the oracle's finals and submap clouds: returns the list of mismatches."""
    bk = S.Bookkeeping(trans_for_mapupdate=thr)
    bad = []
    sim = bk.initialize()
    n_seen = 0
    for k, (pose7, final, upd, trans, dist, tgt) in enumerate(rows):
        r = bk.frame(final, mut)
        if not np.array_equal(r["pose7"], pose7):
            bad.append((k, "pose7"))
        if r["updated"] != upd or r["trans"] != trans or r["latest_distance"] != dist:
            bad.append((k, "decision", r["updated"], upd, r["trans"], trans))
        if len(bk.poses) > n_seen:  # this frame updated the map: the targeted cloud of the newest submap
            n_seen = len(bk.poses)
            m = n_seen - 1
            if m >= len(o.submaps):
                bad.append((k, "submap missing"))
                continue
            prev = [(o.submaps[i][0], bk.poses[i]) for i in range(m)]
            t = S.targeted(o.submaps[m][0], sim if m == 0 else final, prev, nt, mut)
            if not (t.shape == tgt.shape and np.array_equal(t, tgt)):
                bad.append((k, "targeted"))
    if len(bk.poses) != len(o.submaps):
        bad.append(("n_submaps", len(bk.poses), len(o.submaps)))
    for i, (_, M, d) in enumerate(o.submaps[:len(bk.poses)]):
        if not (np.array_equal(bk.poses[i], M) and bk.distances[i] == d):
            bad.append(("submap", i))
    return bad


# ---- the oracle's own drives --------------------------------------------------------------------------------------
_drives = {}


def _oracle_drive(use_filter):
    import oracle
    import oracle.scanmatcher as osm
    from lidarslam_ros2_b200 import synth

    if use_filter not in _drives:
        kw = dict(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3,
                  use_min_max_filter=use_filter, scan_min_range=2.0, scan_max_range=60.0)
        o = osm.ScanMatcher(num_threads=oracle.max_threads(), **kw)
        rows = []
        for scan, _ in synth.drive_stream(8, rings=16, azimuths=300, step=0.6):
            pose7, final, upd = o.receive_cloud(scan)
            rows.append((pose7, final, upd, o.trans, o.latest_distance, o.targeted.copy()))
        _drives[use_filter] = (o, rows)
    return _drives[use_filter]


@pytest.mark.parametrize("use_filter", [False, True])
def test_replay_reproduces_the_oracle_drive(oracle_mod, use_filter):
    o, rows = _oracle_drive(use_filter)
    assert sum(r[2] for r in rows) >= 2
    assert _replay_drive(o, rows, 1.5, 3) == []


def test_replay_reproduces_scripted_drives(oracle_mod):
    finals = _bookkeeping_finals()
    for thr, nt in ((5.0, 3), (5.0, 1), (5.0, 50), (0.0, 2)):
        o, rows = _scripted_drive(finals, thr, nt)
        assert _replay_drive(o, rows, thr, nt) == [], (thr, nt)


def test_range_filter_matches_the_oracle(oracle_mod):
    import oracle.scanmatcher as osm

    for cloud, rmin, rmax in _range_fixtures():
        o = osm.ScanMatcher(use_min_max_filter=True, scan_min_range=rmin, scan_max_range=rmax)
        with np.errstate(invalid="ignore", over="ignore"):
            want = o._range_filter(cloud)
        got = cloud[S.range_keep(cloud, rmin, rmax)]
        assert np.array_equal(got, want, equal_nan=True)


# ---- loop search --------------------------------------------------------------------------------------------------
gate_fixture = S.gate_fixture


def _oracle_search(poses, dists, clouds, final, fitness, **args):
    import oracle.scanmatcher as osm

    o = osm.ScanMatcher()
    o.submaps = [(c, M, d) for c, M, d in zip(clouds, poses, dists)]
    return o.search_loop(ScriptedReg([final], fitness), **args)


def _loop_replay(poses, dists, clouds, final, fitness, mut=(), voxel_leaf_size=0.2, threshold_loop_closure_score=1.0,
                 distance_loop_closure=20.0, range_of_searching_loop_closure=20.0, search_submap_num=3):
    cands = S.loop_candidates(poses, dists, distance_loop_closure, range_of_searching_loop_closure, mut)
    best = S.closest(cands, mut)
    if best is None:
        return {"is_candidate": False, "id_min": -1, "accepted": False, "cands": cands}
    idxs = S.window(best[0], search_submap_num, len(poses), mut)
    out = {"is_candidate": True, "id_min": best[0], "min_dist": best[1], "cands": cands, "window": idxs,
           "n_source": len(clouds[-1]), "accepted": S.accepted(fitness, threshold_loop_closure_score)}
    try:
        out["n_target"] = len(R.voxelgrid_ref(S.loop_target_parts(clouds, poses, idxs), voxel_leaf_size)[0])
    except IndexError:  # a window index past the newest submap
        out["n_target"] = None
    if out["accepted"]:
        out["relative_pose"] = S.relative_pose(final, poses[-1], poses[best[0]], mut)
    return out


def _loop_fixtures():
    """(poses, distances, clouds, final, fitness, args): the gate edges, the window past both ends, a negative
    distance_loop_closure, and the oracle's out-and-back drive."""
    rng = np.random.default_rng(7)
    fin = np.eye(4, dtype=F32)
    fin[:3, :3] = S.pose_matrix((0, 0, 0), np.array([0.01, -0.02, 0.03, 1.0]) / np.linalg.norm([0.01, -0.02, 0.03, 1.0]))[:3, :3]
    fin[:3, 3] = (0.05, -0.02, 0.01)
    out = []
    for rotated in (False, True):
        poses, dists = gate_fixture(rotated)
        clouds = [S.lattice_cloud(seed=i) for i in range(len(poses))]
        gate = dict(distance_loop_closure=20.0, range_of_searching_loop_closure=13.0)
        for ssn in (0, 1, 3, 10):
            out.append((poses, dists, clouds, fin, 0.25, dict(gate, search_submap_num=ssn)))
        out.append((poses, dists, clouds, fin, 1.0, dict(gate, search_submap_num=1)))  # fitness == threshold
        # the tied pair exactly at the range: no candidate at all
        out.append((poses, dists, clouds, fin, 0.25, dict(gate, range_of_searching_loop_closure=10.0, search_submap_num=1)))
        out.append((poses, dists, clouds, fin, 0.25, dict(distance_loop_closure=-1.0, range_of_searching_loop_closure=0.5,
                                                            search_submap_num=2)))
    poses, dists = gate_fixture(True)
    clouds = [rng.uniform(-3, 3, (200, 4)).astype(F32) for _ in poses]
    clouds[1] = np.zeros((0, 4), F32)  # an empty submap inside the window
    out.append((poses, dists, clouds, fin, 0.5, dict(distance_loop_closure=20.0, range_of_searching_loop_closure=13.0,
                                                     search_submap_num=1)))
    return out


def _loop_disagreements(fx, mut=()):
    poses, dists, clouds, final, fitness, args = fx
    o = _oracle_search(poses, dists, clouds, final, fitness, voxel_leaf_size=0.2, **args)
    r = _loop_replay(poses, dists, clouds, final, fitness, mut, voxel_leaf_size=0.2, **args)
    bad = [k for k in ("is_candidate", "id_min", "accepted") if r[k] != o[k]]
    if o["is_candidate"]:
        bad += [k for k in ("min_dist", "n_source", "n_target") if r.get(k) != o[k]]
    if o.get("accepted") and r.get("accepted"):
        # the oracle multiplies with BLAS: its edge is within the float64 rounding of a 4x4 product chain
        ref = o["relative_pose"]
        if not np.all(np.abs(r["relative_pose"] - ref) <= 64 * U * (1.0 + np.abs(ref).max())):
            bad.append("relative_pose")
    return bad


def test_loop_replay_reproduces_the_oracle(oracle_mod):
    for k, fx in enumerate(_loop_fixtures()):
        assert _loop_disagreements(fx) == [], k


def test_loop_replay_on_the_oracle_out_and_back(oracle_mod):
    import oracle
    import oracle.scanmatcher as osm

    o = osm.ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3, num_threads=8)
    bk = S.Bookkeeping()
    for scan, T in S.out_and_back():
        q = osm.quat_from_matrix(T[:3, :3])
        o.update_map_external(scan, T.astype(F32), T[:3, 3], q)
        bk.update_map_external(T[:3, 3], q)
        assert bk.trans == o.trans and bk.latest_distance == o.latest_distance
    assert all(np.array_equal(a, M) and d == e for a, d, (_, M, e) in zip(bk.poses, bk.distances, o.submaps))
    reg = oracle.NDT(resolution=2.0, transformation_epsilon=0.01, max_iterations=100, search_method=oracle.DIRECT7, num_threads=8)
    args = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, range_of_searching_loop_closure=1.0, search_submap_num=1)
    ro = o.search_loop(reg, **args)
    clouds = [c for c, _, _ in o.submaps]
    r = _loop_replay(bk.poses, bk.distances, clouds, ro["final"], ro["fitness"], **args)
    assert ro["accepted"] and r["accepted"] and r["id_min"] == ro["id_min"] == 0 and r["min_dist"] == ro["min_dist"]
    assert r["n_source"] == ro["n_source"] and r["n_target"] == ro["n_target"]
    assert np.all(np.abs(r["relative_pose"] - ro["relative_pose"]) <= 64 * U * (1.0 + np.abs(ro["relative_pose"]).max()))


def test_shards_reassemble_the_candidate_list():
    poses, dists = gate_fixture()
    cands = S.loop_candidates(poses, dists, -1.0, 100.0)
    assert len(cands) == 6
    for world in (1, 2, 3, 7):
        parts = [S.shard(cands, r, world) for r in range(world)]
        assert sorted(c for p in parts for c in p) == cands
        assert all(p == cands[r::world] for r, p in enumerate(parts))


# ---- the fixtures reach their edges ---------------------------------------------------------------------------------
def _range_fixtures():
    cloud, rmin, rmax = S.range_edge_cloud()
    out = [(cloud, rmin, rmax)]
    h = S.hypot_disagreements(16)
    hd, xd, yd = np.hypot(h[:, 0].astype(float), h[:, 1].astype(float)), h[:, 0].astype(float), h[:, 1].astype(float)
    a = np.sqrt(xd * xd + yd * yd)
    lo = a[hd > a].min()  # rmin at a point whose hypot is larger: the explicit sum drops it, hypot keeps it
    hi = a[(hd < a) & (a > lo)].max()
    hc = np.c_[h, np.arange(len(h), dtype=F32) * F32(0.5), np.ones(len(h), F32)].astype(F32)
    out.append((hc, float(lo), float(hi)))
    return out


def test_generators_reach_their_edges(oracle_mod):
    # the range filter: points exactly at both bounds, one ulp either side, NaN / inf rows, a hypot disagreement
    cloud, rmin, rmax = S.range_edge_cloud()
    x, y = cloud[:, 0].astype(float), cloud[:, 1].astype(float)
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.sqrt(x * x + y * y)
    assert (r == rmin).sum() >= 3 and (r == rmax).sum() >= 3
    assert ((r > rmin) & (r < rmin * (1 + 1e-6))).any() and ((r < rmin) & (r > rmin * (1 - 1e-6))).any()
    assert ((r > rmax) & (r < rmax * (1 + 1e-6))).any() and ((r < rmax) & (r > rmax * (1 - 1e-6))).any()
    assert np.isnan(cloud[:, :3]).any() and np.isinf(cloud[:, :3]).any() and (np.abs(cloud[:, 2]) > 1e4).any()
    hc, lo, hi = _range_fixtures()[1]
    assert not np.array_equal(S.range_keep(hc, lo, hi), S.range_keep(hc, lo, hi, ("hypot",)))
    # the bookkeeping: an update at trans == trans_for_mapupdate, and every quaternion branch
    o, rows = _scripted_drive(_bookkeeping_finals(), 5.0)
    assert rows[0][3] == 5.0 and rows[0][2]
    branches = set()
    for F in _bookkeeping_finals():
        m = F[:3, :3].astype(float)
        tr = (m[0, 0] + m[1, 1]) + m[2, 2]
        branches.add("trace" if tr > 0 else int(np.argmax(np.diag(m))))
    assert branches == {"trace", 0, 1, 2}
    # the loop gates: a candidate exactly at the range, a travelled distance exactly at distance_loop_closure, a tie
    poses, dists = gate_fixture()
    d = [S.distance3(poses[-1][:3, 3], p[:3, 3]) for p in poses]
    assert d[0] == 13.0 and dists[-1] - dists[1] == 20.0 and d[2] == d[3] == 10.0
    assert S.loop_candidates(poses, dists, 20.0, 13.0) == [(2, 10.0), (3, 10.0)]
    assert S.closest(S.loop_candidates(poses, dists, 20.0, 13.0)) == (2, 10.0)
    assert S.loop_candidates(poses, dists, -1.0, 0.5) == [(5, 0.0)]  # the newest is its own candidate
    # windows past both ends
    assert S.window(2, 3, 6) == [0, 1, 2, 3, 4, 5] and S.window(2, 10, 6) == list(range(6)) and S.window(0, 1, 6) == [0, 1]
    assert S.window(5, 2, 6) == [3, 4, 5]
    # the cancelling submap: the double sums' order shows in the float cast
    c, M = S.cancelling_submap()
    assert not np.array_equal(S.transform_f64(c, M), S.transform_f64(c, M, ("f64_reassoc",)))
    # lattice clouds: one point per leaf, exactly the input back
    lat = S.transform_f32(S.lattice_cloud(), S.pose_matrix((3.0, -2.5, 1.0), (0, 0, 0, 1)).astype(F32))
    cen, _ = R.voxelgrid_ref(lat, 0.2)
    assert len(cen) == len(lat) and np.array_equal(cen.astype(F32), lat[np.lexsort((lat[:, 0], lat[:, 1], lat[:, 2]))])


# ---- power --------------------------------------------------------------------------------------------------------
def _power_fixtures():
    """Each fixture returns the disagreements of a (possibly mutated) replay with it."""
    import oracle.scanmatcher as osm

    fx = {}
    finals = _bookkeeping_finals()
    for thr, nt in ((5.0, 3), (5.0, 50)):
        o, rows = _scripted_drive(finals, thr, nt)
        fx[f"scripted/{thr}/{nt}"] = lambda mut, o=o, rows=rows, thr=thr, nt=nt: _replay_drive(o, rows, thr, nt, mut)
    for use_filter in (False, True):
        o, rows = _oracle_drive(use_filter)
        fx[f"drive/{use_filter}"] = lambda mut, o=o, rows=rows: _replay_drive(o, rows, 1.5, 3, mut)
    for k, lf in enumerate(_loop_fixtures()):
        fx[f"loop/{k}"] = lambda mut, lf=lf: _loop_disagreements(lf, mut)
    c, M = S.cancelling_submap()
    fx["cancelling"] = lambda mut: [] if np.array_equal(S.transform_f64(c, M, mut), osm.transform_f64(c, M)) else ["f64"]
    for j, (cloud, rmin, rmax) in enumerate(_range_fixtures()):
        o = osm.ScanMatcher(use_min_max_filter=True, scan_min_range=rmin, scan_max_range=rmax)
        with np.errstate(invalid="ignore", over="ignore"):
            want = o._range_filter(cloud)
        fx[f"range/{j}"] = lambda mut, cloud=cloud, rmin=rmin, rmax=rmax, want=want: (
            [] if np.array_equal(cloud[S.range_keep(cloud, rmin, rmax, mut)], want, equal_nan=True) else ["range"])
    # relative_pose: the oracle's BLAS product is not bitwise, so the mutant is held against the unmutated replay, which
    # the GPU tests hold against the device bit for bit
    for k, (poses, dists, clouds, fin, fit, args) in enumerate(_loop_fixtures()):
        best = S.closest(S.loop_candidates(poses, dists, args["distance_loop_closure"], args["range_of_searching_loop_closure"]))
        if best is not None:
            ref = S.relative_pose(fin, poses[-1], poses[best[0]])
            fx[f"relative/{k}"] = lambda mut, fin=fin, P=poses[-1], Q=poses[best[0]], ref=ref: (
                [] if np.array_equal(S.relative_pose(fin, P, Q, mut), ref) else ["relative_pose"])
    return fx


_power = {}


@pytest.mark.parametrize("mut", S.MUTATIONS)
def test_power_of_the_replay(oracle_mod, mut):
    """A replay of a subtly wrong session disagrees with at least one fixture; the right one with none."""
    if not _power:
        _power.update(_power_fixtures())
        for label, f in _power.items():
            assert f(()) == [], label
    failed = [label for label, f in _power.items() if f((mut,))]
    print(f"\n{mut}: disagrees with {len(failed)} of {len(_power)} fixtures")
    assert failed, mut
