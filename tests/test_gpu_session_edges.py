"""The frontend session (csrc/scanmatcher.cu, b200sm_*) against the float64 replay of tests/sessionref.py, bit for bit:
given the device's own align() output and its own VoxelGrid output (read back as submaps), every pose, decision,
distance, targeted cloud, loop window and loop edge the session produces is deterministic arithmetic the replay
reproduces exactly. Covered: NDT and GICP drives frame by frame, the update threshold at equality, GICP's filtered
target and in-place source, the loop search's scratch shared with the GICP target, the range filter at its bounds and
warp edges, the submap arena's chunk boundary and the targeted-cloud window, and the loop gates at equality.
Run on an H100 with -m gpu."""
import numpy as np
import pytest

import gridref as R
import sessionref as S

pytestmark = pytest.mark.gpu

F32 = np.float32
KW = dict(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3, scan_min_range=2.0,
          scan_max_range=60.0)
LOOP = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, range_of_searching_loop_closure=1.0, search_submap_num=1)


@pytest.fixture(scope="module")
def smm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


def _sorted_rows(c):
    c = np.asarray(c)
    return c[np.lexsort(tuple(c[:, k] for k in range(c.shape[1] - 1, -1, -1)))]


def _check_voxelgrid(out, pts, leaf, what):
    """VoxelGrid output against gridref.voxelgrid_ref: the same leaves in the same order, each value within one float
    ulp of the float64 centroid plus the bound on the kernel's f64 summation order."""
    ref, err = R.voxelgrid_ref(pts, leaf)
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    tol = np.spacing(np.abs(ref).astype(F32)).astype(np.float64) + err
    bad = ~(np.abs(out - ref) <= tol)
    assert not bad.any(), (what, int(bad.sum()))


def _frames(n, azimuths=400):
    from lidarslam_ros2_b200 import synth

    return [scan for scan, _ in synth.drive_stream(n, rings=16, azimuths=azimuths, step=0.6)]


def _check_target(reg, cloud, filtered_leaf, what):
    """The registration's target is `cloud` (filtered_leaf None) or VoxelGrid(filtered_leaf) of it: the same count, and
    every reference point finds its own target point, within the VoxelGrid bound."""
    if filtered_leaf is None:
        ref, tol = np.asarray(cloud, dtype=np.float64), np.zeros((len(cloud), 4))
    else:
        ref, err = R.voxelgrid_ref(cloud, filtered_leaf)
        tol = np.spacing(np.abs(ref).astype(F32)).astype(np.float64) + err
    assert reg.stats()["n_target"] == len(ref), what
    idx, d2 = reg.nearest(ref.astype(F32))
    assert np.array_equal(np.sort(idx), np.arange(len(ref))), what  # one to one
    bound = ((2.0 * tol[:, :3]) ** 2).sum(axis=1) * (1 + 1e-6)
    assert np.all(d2.astype(np.float64) <= bound), what


def _reference_target(cloud, filtered_leaf):
    """The registration target as the tests know it: `cloud` itself (exact, e = 0), or the float64 VoxelGrid centroids
    cast to float, each within e (a distance) of the device's centroid."""
    if filtered_leaf is None:
        return np.asarray(cloud, dtype=F32), 0.0
    ref, err = R.voxelgrid_ref(cloud, filtered_leaf)
    tol = np.spacing(np.abs(ref).astype(F32)).astype(np.float64) + err
    return ref.astype(F32), float(2.0 * np.sqrt((tol[:, :3] ** 2).sum(axis=1)).max())


def _aligned(reg, n):
    """getAligned() of a source the session handed over in place (the Python object never saw its size)."""
    from lidarslam_ros2_b200.registration import _ptr

    out = np.zeros((n, 4), dtype=F32)
    reg._check(reg._lib.b200reg_get_aligned(reg._h, _ptr(out), 16))
    return out[:, :3]


def _drive(smm, frames, method="NDT", between=None, **kw):
    """Runs the frames through a fresh session and checks every frame bitwise against the replay of the device's own
    final and read-back submaps. `between(g)` runs after every frame. Returns (session, per-frame records)."""
    kw = dict(KW, **kw)
    g = smm.ScanMatcher(registration_method=method, **kw)
    bk = S.Bookkeeping(trans_for_mapupdate=kw.get("trans_for_mapupdate", 1.5))
    sim = bk.initialize()  # initializeMap runs inside the first receiveCloud
    nt = kw["num_targeted_cloud"]
    recs, n_seen, pending, target = [], 0, None, None
    for k, scan in enumerate(frames):
        guess = bk.sim_trans()  # getTransformation of the pose before this frame
        pose7, final, upd = g.receiveCloud(scan)
        r = bk.frame(final)
        st = g.stats()
        assert np.array_equal(pose7, r["pose7"]), k
        assert upd == r["updated"], k
        assert st["trans"] == r["trans"] and st["latest_distance"] == r["latest_distance"], k
        assert g.numSubmaps() == len(bk.poses), k
        subs = None
        if len(bk.poses) > n_seen:  # this frame updated the map
            n_seen = len(bk.poses)
            subs = [g.submap(i) for i in range(n_seen)]
            for i, (_, M, d) in enumerate(subs):
                assert np.array_equal(M, bk.poses[i]) and d == bk.distances[i], (k, i)
            m = len(bk.poses) - 1
            want = S.targeted(subs[m][0], sim if m == 0 else final, [(subs[i][0], bk.poses[i]) for i in range(m)], nt)
            got = g.targetedCloud()
            assert got.shape == want.shape and np.array_equal(got, want), k
        tgt = g.targetedCloud()
        if method == "GICP":
            reg = g.registration
            if k == 0:  # initializeMap hands the transformed first scan over unfiltered
                first = subs[0][0] if subs else g.submap(0)[0]
                target = (S.transform_f32(first, sim), None)
                _check_target(reg, *target, k)
            elif pending is not None:  # adopted at the start of this frame: VoxelGrid(vg_size_for_input) of the targeted cloud
                target = (pending, kw["vg_size_for_input"])
                _check_target(reg, *target, k)
            # the source is the session's filtered scan, read in place: still the one align() used
            fs = g.filteredScan()
            aligned = S.transform_f32(fs, final)
            assert np.array_equal(_aligned(reg, len(fs)), aligned[:, :3]), k
            # getFitnessScore of that source against the reference target, nearest neighbours by brute force
            pts, e = _reference_target(*target)
            _, d2 = R.nn1_ref(pts, aligned)
            d2 = d2.astype(np.float64)
            want_fit = d2.sum() / len(d2)
            # e = 0: the same target points, so the same float32 distances and only the sum's order differs. Else each
            # target point may be off by e: a distance moves by at most e, its float32 square by its own rounding too.
            bound = 1e-12 * want_fit if e == 0 else np.mean(2 * np.sqrt(d2) * e + e * e + 2.0**-20 * d2) + 1e-12 * want_fit
            assert abs(reg.getFitnessScore() - want_fit) <= bound, (k, reg.getFitnessScore(), want_fit, bound)
        pending = tgt if upd else None
        recs.append(dict(pose7=pose7, final=final, updated=upd, trans=st["trans"], targeted=tgt, guess=guess,
                         source=g.filteredScan(), target=target))
        if between is not None:
            between(g)
    return g, recs


# ---- NDT drive ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_filter", [False, True])
def test_ndt_drive_frame_by_frame(smm, use_filter):
    _, recs = _drive(smm, _frames(10), use_min_max_filter=use_filter)
    assert sum(r["updated"] for r in recs) >= 2


def test_update_threshold_at_equality(smm):
    frames = _frames(10)
    _, recs = _drive(smm, frames)
    k = next(i for i, r in enumerate(recs) if r["updated"])
    t = recs[k]["trans"]
    assert all(r["trans"] < t for r in recs[:k])  # no earlier frame updates under either threshold below
    for thr, want in ((t, True), (float(np.nextafter(t, np.inf)), False)):
        _, again = _drive(smm, frames[:k + 1], trans_for_mapupdate=thr)
        assert np.array_equal(again[k]["final"], recs[k]["final"])  # the solver repeats itself bit for bit
        assert again[k]["trans"] == t and again[k]["updated"] is want, (thr, want)


# ---- GICP frontend --------------------------------------------------------------------------------------------------
def test_gicp_frontend(smm):
    import oracle
    import oracle.scanmatcher as osm
    from lidarslam_ros2_b200 import synth

    frames = _frames(6, azimuths=300)
    _, recs = _drive(smm, frames, method="GICP")
    assert sum(r["updated"] for r in recs) >= 1
    kw = {k: v for k, v in KW.items() if k not in ("scan_min_range", "scan_max_range")}
    o = osm.ScanMatcher(registration_method="GICP", num_threads=oracle.max_threads(), **kw)
    for k, scan in enumerate(frames):
        _, To, uo = o.receive_cloud(scan)
        assert recs[k]["updated"] == uo, k
        # each registration is compared on equal inputs (the device's target, in-place source and guess): in the two
        # drives every frame starts from its own side's previous pose, so they are compared decision by decision only
        cloud, leaf = recs[k]["target"]
        ref = oracle.GICP(max_correspondence_distance=5.0, transformation_epsilon=1e-8)
        # the device's VoxelGrid centroid is its float64 mean cast to float: voxelgrid_ref's, up to summation order
        ref.set_target((cloud if leaf is None else R.voxelgrid_ref(cloud, leaf)[0].astype(F32))[:, :3])
        ref.set_source(recs[k]["source"][:, :3])
        Tr = np.asarray(ref.align(recs[k]["guess"]), dtype=F32)
        dt, dr = synth.pose_error(recs[k]["final"], Tr)
        assert dt < 1e-3 and dr < 1e-3, (k, dt, dr)


def _out_and_back_session(smm, **kw):
    """The out-and-back drive through the caller-driven updateMap, checked against the replay after every call."""
    g = smm.ScanMatcher(**dict(KW, **kw))
    bk = S.Bookkeeping()
    for scan, T in S.out_and_back():
        q = S.quat_from_rot(T[:3, :3])
        g.setScan(scan)
        g.updateMap(T.astype(F32), T[:3, 3], q, adopt_now=False)
        n = len(bk.poses)
        bk.update_map_external(T[:3, 3], q)
        subs = [g.submap(i) for i in range(n + 1)]
        assert g.stats()["latest_distance"] == bk.latest_distance
        assert all(np.array_equal(M, bk.poses[i]) and d == bk.distances[i] for i, (_, M, d) in enumerate(subs))
        want = S.targeted(subs[n][0], T.astype(F32), [(subs[i][0], bk.poses[i]) for i in range(n)], KW["num_targeted_cloud"])
        assert np.array_equal(g.targetedCloud(), want)
    clouds = [g.submap(i)[0] for i in range(g.numSubmaps())]
    return g, bk, clouds


def _check_loop_result(r, clouds, poses, dists, args, threshold=1.0, exact_target=False):
    """One evaluated candidate against the replay: id, distance, counts and loop edge bitwise, the acceptance rule on
    the device's own fitness; with exact_target the fitness against a float64 sum of nn1_ref distances."""
    idxs = S.window(r["id_min"], args["search_submap_num"], len(poses))
    dist = S.distance3(poses[-1][:3, 3], poses[r["id_min"]][:3, 3])
    assert r["min_dist"] == dist, r["id_min"]
    src = S.loop_source(clouds[-1], poses[-1])
    parts = S.loop_target_parts(clouds, poses, idxs)
    tgt, _ = R.voxelgrid_ref(parts, args["voxel_leaf_size"])
    assert r["n_source"] == len(src) and r["n_target"] == len(tgt), r["id_min"]
    assert r["accepted"] == S.accepted(r["fitness"], threshold)
    if r["accepted"]:
        rel = S.relative_pose(r["final"], poses[-1], poses[r["id_min"]])
        assert np.array_equal(r["relative_pose"], rel), r["id_min"]
    if exact_target:
        assert len(tgt) == len(parts)  # one point per leaf: the target is the window's points themselves
        _, d2 = R.nn1_ref(tgt.astype(F32), S.transform_f32(src, r["final"]))
        want = d2.astype(np.float64).sum() / len(d2)
        assert abs(r["fitness"] - want) <= 1e-12 * want, (r["fitness"], want)


def test_gicp_loop_search_finds_the_ndt_candidate(smm):
    g, bk, clouds = _out_and_back_session(smm)
    rn = g.searchLoop(smm.backend_registration("NDT", ndt_resolution=2.0), **LOOP)
    rg = g.searchLoop(smm.backend_registration("GICP"), **LOOP)
    cands = S.loop_candidates(bk.poses, bk.distances, LOOP["distance_loop_closure"], LOOP["range_of_searching_loop_closure"])
    assert rn["id_min"] == rg["id_min"] == S.closest(cands)[0] == 0
    for r in (rn, rg):
        assert r["accepted"]
        _check_loop_result(r, clouds, bk.poses, bk.distances, LOOP)


# ---- scratch shared by the loop search and GICP's target adoption ------------------------------------------------------
@pytest.mark.parametrize("method", ["NDT", "GICP"])
def test_loop_search_between_frames_changes_nothing(smm, method):
    frames = _frames(6, azimuths=300)
    _, plain = _drive(smm, frames, method=method)
    reg = smm.backend_registration(method, ndt_resolution=2.0)
    args = dict(voxel_leaf_size=0.3, distance_loop_closure=0.5, range_of_searching_loop_closure=100.0, search_submap_num=1)
    found = []

    def between(g):
        found.append(g.searchLoop(reg, **args)["is_candidate"])
        g.searchLoopAll(reg, **args)

    _, mixed = _drive(smm, frames, method=method, between=between)
    assert any(found)  # the loop search really ran between some frames
    for a, b in zip(plain, mixed):
        assert np.array_equal(a["pose7"], b["pose7"]) and np.array_equal(a["final"], b["final"])
        assert a["updated"] == b["updated"] and np.array_equal(a["targeted"], b["targeted"])


# ---- range filter ---------------------------------------------------------------------------------------------------
def _check_range(smm, cloud, rmin, rmax, leaf, what, exact_leaves=True):
    g = smm.ScanMatcher(use_min_max_filter=True, scan_min_range=rmin, scan_max_range=rmax, vg_size_for_input=leaf)
    keep = S.range_keep(cloud, rmin, rmax)
    g.setScan(cloud)
    assert g.stats()["n_scan"] == keep.sum(), what
    fs = g.filteredScan()
    if exact_leaves:  # every kept point is alone in its leaf, or the grid overflowed and VoxelGrid returned the scan
        # unchanged (a non-finite z passes the range filter): either way the filtered scan is the kept set
        assert np.array_equal(_sorted_rows(fs), _sorted_rows(cloud[keep]), equal_nan=True), what
    else:
        _check_voxelgrid(fs, cloud[keep], leaf, what)


def test_range_filter_bounds(smm):
    cloud, rmin, rmax = S.range_edge_cloud()
    _check_range(smm, cloud, rmin, rmax, 0.05, "edges")
    h = S.hypot_disagreements(16)
    x, y = h[:, 0].astype(float), h[:, 1].astype(float)
    a, hy = np.sqrt(x * x + y * y), np.hypot(x, y)
    lo = a[hy > a].min()
    hi = a[(hy < a) & (a > lo)].max()
    hc = np.c_[h, np.arange(len(h)) * 0.5, np.ones(len(h))].astype(F32)
    _check_range(smm, hc, float(lo), float(hi), 0.05, "hypot")


def _separated(n, seed):
    """n points on distinct cells of a 0.35 m (x, y) lattice over [-70, 70]^2, some inside 2 < r < 60, some not."""
    rng = np.random.default_rng(seed)
    cells = rng.choice(400 * 400, n, replace=False)
    x, y = (cells % 400) * 0.35 - 70.0 + 0.11, (cells // 400) * 0.35 - 70.0 + 0.13
    return np.c_[x, y, rng.uniform(-2, 2, n), rng.uniform(0, 100, n)].astype(F32)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 257])
def test_range_filter_warp_edges(smm, n):
    cloud = _separated(n, n)
    if n == 1:
        cloud[0, :2] = (3.0, 4.0)
    _check_range(smm, cloud, 2.0, 60.0, 0.05, n)
    # the filtered scan is VoxelGrid's leaf order of the kept set
    g = smm.ScanMatcher(use_min_max_filter=True, scan_min_range=2.0, scan_max_range=60.0, vg_size_for_input=0.05)
    g.setScan(cloud)
    ref, _ = R.voxelgrid_ref(cloud[S.range_keep(cloud, 2.0, 60.0)], 0.05)
    assert np.array_equal(g.filteredScan(), ref.astype(F32))


def test_range_filter_million_points(smm):
    rng = np.random.default_rng(5)
    n = 1 << 20
    r, th = rng.uniform(0.0, 80.0, n), rng.uniform(0, 2 * np.pi, n)
    cloud = np.c_[r * np.cos(th), r * np.sin(th), rng.uniform(-3, 3, n), rng.uniform(0, 100, n)].astype(F32)
    cloud[:7] = [(3, 4, 0, 1), (-4, 3, 1, 1), (36, 48, 0, 1), (-48, 36, 1, 1), (np.nan, 1, 1, 1), (np.inf, 0, 0, 1), (1, 1, 1e4, 1)]
    _check_range(smm, cloud, 5.0, 60.0, 0.2, "1M", exact_leaves=False)


# ---- submap arena and the targeted-cloud window, on imported submaps ------------------------------------------------------
ARENA_SIZES = [0, 1, 15, 16, 17, 2_000_000, 2_500_000, (4 << 20) + 1000, 17]  # 2.5 M crosses the 4 Mi chunk; then one larger


def _set_num_targeted_cloud(g, kw, nt):
    """num_targeted_cloud of a live session; every other parameter stays what the session was built with (`kw`, with
    ScanMatcher's defaults). b200sm_set_params(s, vg_size_for_input, vg_size_for_map, num_targeted_cloud,
    trans_for_mapupdate, use_min_max_filter, scan_min_range, scan_max_range), include/b200reg.h."""
    import inspect

    p = {k: v.default for k, v in inspect.signature(type(g).__init__).parameters.items() if v.default is not inspect.Parameter.empty}
    p.update(kw, num_targeted_cloud=nt)
    g._check(g._lib.b200sm_set_params(g._h, float(p["vg_size_for_input"]), float(p["vg_size_for_map"]), int(p["num_targeted_cloud"]),
                                      float(p["trans_for_mapupdate"]), int(bool(p["use_min_max_filter"])),
                                      float(p["scan_min_range"]), float(p["scan_max_range"])))


def test_arena_and_targeted_window(smm):
    rng = np.random.default_rng(17)
    g = smm.ScanMatcher(**KW)
    bk = S.Bookkeeping()
    clouds = []
    for i, n in enumerate(ARENA_SIZES):
        c = np.c_[rng.uniform(-50, 50, (n, 3)), rng.uniform(0, 100, n)].astype(F32)
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        M = S.pose_matrix(rng.uniform(-20, 20, 3), q)
        g.importSubmap(c, M, 3.0 * i)
        bk.import_submap(M, 3.0 * i)
        clouds.append(c)
    for i, c in enumerate(clouds):  # every submap reads back as it went in, across the chunk boundaries
        got, M, d = g.submap(i)
        assert got.shape == c.shape and np.array_equal(got, c) and np.array_equal(M, bk.poses[i]) and d == bk.distances[i], i
    scans = _frames(3, azimuths=300)
    for j, nt in enumerate((1, 3, 20)):
        _set_num_targeted_cloud(g, KW, nt)
        q = S.quat_from_rot(np.eye(3))
        pos = (1.0 + j, -0.5 * j, 0.25)
        final = S.pose_matrix(pos, q).astype(F32)
        g.setScan(scans[j])
        n = len(bk.poses)
        g.updateMap(final, pos, q, adopt_now=False)
        bk.update_map_external(pos, q)
        new, M, d = g.submap(n)
        assert np.array_equal(M, bk.poses[n]) and d == bk.distances[n] and g.stats()["latest_distance"] == bk.latest_distance
        _check_voxelgrid(new, np.c_[scans[j], np.zeros(len(scans[j]))], KW["vg_size_for_map"], nt)
        want = S.targeted(new, final, list(zip(clouds, bk.poses[:n])), nt)
        got = g.targetedCloud()
        assert got.shape == want.shape and np.array_equal(got, want), nt
        clouds.append(new)
    mp, off = g.assembleMap()
    assert off[-1] == sum(len(c) for c in clouds)
    for i, c in enumerate(clouds):
        assert np.array_equal(mp[off[i]:off[i + 1]], S.transform_f32(c, bk.poses[i].astype(F32))), i


def test_targeted_cloud_summation_order(smm):
    """Submaps whose double transform sums two large terms that cancel (sessionref.cancelling_submap): on these points
    the float cast shows the order and rounding of transform_f64's sum, so the targeted cloud tells the left-to-right
    un-fused sum from a re-associated or fused one."""
    g = smm.ScanMatcher(**dict(KW, num_targeted_cloud=3))
    bk = S.Bookkeeping()
    clouds = []
    for i in range(2):
        c, M = S.cancelling_submap(seed=i)
        g.importSubmap(c, M, 1.0 + i)
        bk.import_submap(M, 1.0 + i)
        clouds.append(c)
    scan = _frames(1, azimuths=300)[0]
    q = S.quat_from_rot(np.eye(3))
    final = S.pose_matrix((0.5, 0.25, 0.0), q).astype(F32)
    g.setScan(scan)
    g.updateMap(final, (0.5, 0.25, 0.0), q, adopt_now=False)
    new = g.submap(2)[0]
    prev = list(zip(clouds, bk.poses))
    want = S.targeted(new, final, prev, 3)
    for mut in ("f64_reassoc", "f64_fused"):  # the fixture has the power: either change shows in the float cast
        assert not np.array_equal(S.targeted(new, final, prev, 3, (mut,)), want), mut
    got = g.targetedCloud()
    assert got.shape == want.shape and np.array_equal(got, want)


# ---- the loop gates at equality, on imported submaps -------------------------------------------------------------------
def _gate_session(smm, empty=None, rotated=False):
    poses, dists = S.gate_fixture(rotated)
    clouds = [S.lattice_cloud(seed=i) for i in range(len(poses))]
    if empty is not None:
        clouds[empty] = np.zeros((0, 4), F32)
    g = smm.ScanMatcher(**KW)
    for c, M, d in zip(clouds, poses, dists):
        g.importSubmap(c, M, d)
    return g, clouds, poses, dists


def test_loop_gates_at_equality(smm):
    g, clouds, poses, dists = _gate_session(smm)
    reg = smm.backend_registration("NDT", ndt_resolution=2.0)
    thr = 1.0e9  # every registration is accepted: its loop edge is compared too
    for ssn in (0, 1, 3, 10):  # 10: the window runs past both ends
        args = dict(voxel_leaf_size=0.2, distance_loop_closure=20.0, range_of_searching_loop_closure=13.0, search_submap_num=ssn)
        one = g.searchLoop(reg, threshold_loop_closure_score=thr, **args)
        assert one["id_min"] == 2, ssn  # 0 is exactly at the range, 1 exactly at the travelled distance; 2 and 3 tie
        _check_loop_result(one, clouds, poses, dists, args, thr, exact_target=True)
        every = g.searchLoopAll(reg, threshold_loop_closure_score=thr, **args)
        assert [r["id_min"] for r in every] == [2, 3] and every[0]["n_candidates_total"] == 2
        for r in every:
            _check_loop_result(r, clouds, poses, dists, args, thr, exact_target=True)
        assert np.array_equal(every[0]["final"], one["final"]) and np.array_equal(every[0]["relative_pose"], one["relative_pose"])
    # the tied pair exactly at the range: nothing
    none = dict(voxel_leaf_size=0.2, distance_loop_closure=20.0, range_of_searching_loop_closure=10.0, search_submap_num=1)
    assert not g.searchLoop(reg, **none)["is_candidate"] and g.searchLoopAll(reg, **none) == []
    # a negative distance_loop_closure: the newest submap is its own candidate, at distance 0
    args = dict(voxel_leaf_size=0.2, distance_loop_closure=-1.0, range_of_searching_loop_closure=0.5, search_submap_num=2)
    own = g.searchLoop(reg, threshold_loop_closure_score=thr, **args)
    assert own["id_min"] == 5 and own["min_dist"] == 0.0
    _check_loop_result(own, clouds, poses, dists, args, thr, exact_target=True)
    # every submap a candidate, dealt over 2 and 3 shards: the shards reassemble the full list
    wide = dict(voxel_leaf_size=0.2, distance_loop_closure=-1.0, range_of_searching_loop_closure=100.0, search_submap_num=1)
    full = g.searchLoopAll(reg, threshold_loop_closure_score=thr, **wide)
    assert [r["id_min"] for r in full] == list(range(6))
    for r in full:
        _check_loop_result(r, clouds, poses, dists, wide, thr, exact_target=True)
    for world in (2, 3):
        parts = [g.searchLoopAll(reg, threshold_loop_closure_score=thr, shard_rank=k, shard_world=world, **wide)
                 for k in range(world)]
        for k, p in enumerate(parts):
            assert [r["id_min"] for r in p] == [c[0] for c in S.shard(S.loop_candidates(poses, dists, -1.0, 100.0), k, world)]
        merged = sorted((r for p in parts for r in p), key=lambda r: r["id_min"])
        for a, b in zip(merged, full):
            assert a["id_min"] == b["id_min"] and a["n_target"] == b["n_target"]
            assert np.array_equal(a["final"], b["final"]) and np.array_equal(a["relative_pose"], b["relative_pose"])


def test_loop_window_with_an_empty_submap(smm):
    g, clouds, poses, dists = _gate_session(smm, empty=1)
    reg = smm.backend_registration("NDT", ndt_resolution=2.0)
    args = dict(voxel_leaf_size=0.2, distance_loop_closure=20.0, range_of_searching_loop_closure=13.0, search_submap_num=1)
    r = g.searchLoop(reg, threshold_loop_closure_score=1.0e9, **args)
    assert r["id_min"] == 2 and S.window(2, 1, 6) == [1, 2, 3]
    _check_loop_result(r, clouds, poses, dists, args, 1.0e9, exact_target=True)
    assert g.submap(1)[0].shape == (0, 4)


def test_loop_edge_with_rotated_poses(smm):
    """Candidates whose pose has a generic rotation: Isometry's R^T, -R^T t inverse and a general 4x4 inverse round
    differently there, so the loop edges tell them apart (checked below on the device's own results)."""
    g, clouds, poses, dists = _gate_session(smm, rotated=True)
    reg = smm.backend_registration("NDT", ndt_resolution=2.0)
    thr = 1.0e9
    args = dict(voxel_leaf_size=0.2, distance_loop_closure=20.0, range_of_searching_loop_closure=13.0, search_submap_num=1)
    one = g.searchLoop(reg, threshold_loop_closure_score=thr, **args)
    assert one["id_min"] == 2
    _check_loop_result(one, clouds, poses, dists, args, thr)
    wide = dict(voxel_leaf_size=0.2, distance_loop_closure=-1.0, range_of_searching_loop_closure=100.0, search_submap_num=1)
    full = g.searchLoopAll(reg, threshold_loop_closure_score=thr, **wide)
    assert [r["id_min"] for r in full] == list(range(6))
    differs = 0
    for r in full:
        _check_loop_result(r, clouds, poses, dists, wide, thr)
        general = S.relative_pose(r["final"], poses[-1], poses[r["id_min"]], ("rel_full_inverse",))
        differs += not np.array_equal(general, r["relative_pose"])
    assert differs > 0  # the fixture has the power
