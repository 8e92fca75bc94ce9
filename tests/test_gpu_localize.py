"""Localisation in a prior map (csrc/scanmatcher.cu: b200sm_set_prior_map*, b200sm_localize_cloud, b200sm_localize_init)
against the float64 replay of tests/localizeref.py: the cut is bitwise map[mask] in map order; given the device's own
`final` of every frame, every pose, distance, re-cut decision and adoption is arithmetic the replay reproduces exactly;
and each frame's registration is bitwise that of the plain calls on the read-back cut and filtered scan. The cases run from
a 1-point map upwards. The fixtures (edge maps, the canyon map and drive) are defined here and shared with the CPU tests
tests/test_localizeref_cpu.py and tests/test_localize_host.py. Run on an H100 with -m gpu."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import frontendref as fr
import localizeref as L
import oracle.scanmatcher as osm
from lidarslam_ros2_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
TILE = 2048  # CUT_TILE of csrc/map_cut.hpp (tests/test_localize_host.py checks it)
EDGE_SIZES = (1, 31, 32, 33, TILE - 1, TILE, TILE + 1, 3 * TILE + 17)
PATTERNS = ("all", "none", "alternate", "last", "mixed")
CENTRE, RADIUS = (3.0, -2.0), 5.0

# the drive: the canyon map in the frame of synth.sample_map, the sensor starting 60 m up the street
X_START, STEP, N_FRAMES = -60.0, 1.5, 14
KW = dict(ndt_resolution=2.0, vg_size_for_input=0.4, use_min_max_filter=True, scan_min_range=2.0, scan_max_range=30.0)
CROP, RECROP = 45.0, 6.0
MOUNT_POS = (1.2, 0.0, 2.0)
MOUNT_QUAT = osm.quat_from_matrix(synth.rpy_matrix(0.02, -0.04, 0.35))


# ---- fixtures (plain functions: the CPU tests import them) --------------------------------------------------------------
def edge_map(n, pattern, centre=CENTRE, radius=RADIUS) -> np.ndarray:
    """n rows around `centre`: inside rows at 0.9 r, outside rows at 1.8 r; intensity = row index, z spread over +-30 m.
    'mixed' also has NaN / inf rows, rows at distance exactly r (3-4-5 triangles), one float32 step either side of them,
    and the origin (the row fused_case() is about)."""
    u = synth.Rng(9300 + n % 977 + 7 * PATTERNS.index(pattern)).uniform(2 * n).reshape(n, 2)
    i = np.arange(n)
    inside = {"all": np.ones(n, bool), "none": np.zeros(n, bool), "alternate": i % 2 == 0, "last": i == n - 1,
              "mixed": u[:, 1] < 0.5}[pattern]
    rad = np.where(inside, 0.9 * radius, 1.8 * radius)
    a = 2.0 * math.pi * u[:, 0]
    m = np.stack([centre[0] + rad * np.cos(a), centre[1] + rad * np.sin(a), 60.0 * (u[:, 1] - 0.5), i.astype(np.float64)],
                 axis=1).astype(F32)
    if pattern == "mixed" and n >= 31:
        s = radius / 5.0
        m[3, :2] = (centre[0] + 3 * s, centre[1] + 4 * s)           # exactly r (for the default centre and radius)
        m[5, :2] = (centre[0] - 4 * s, centre[1] + 3 * s)
        m[7, :2] = (np.nextafter(m[3, 0], F32(np.inf)), m[3, 1])   # one float32 step outside
        m[9, :2] = (np.nextafter(m[3, 0], F32(-np.inf)), m[3, 1])  # ... and inside
        m[11, 0], m[13, 1], m[17, 0], m[19, 1] = np.nan, np.nan, np.inf, -np.inf
        m[15, :3] = (centre[0] + 1.0, centre[1] + 1.0, np.nan)     # z is not looked at: rows 15 and 21 are kept
        m[21, :3] = (centre[0] - 1.0, centre[1] + 1.0, np.inf)
        m[23, :3] = (0.0, 0.0, 0.0)
        m[n - 1, :2] = (centre[0], centre[1])                       # the last row kept
    return m


def fused_case():
    """(cx, cy, r) for which the origin row is kept by dx * dx + dy * dy <= r * r evaluated un-fused and dropped by
    fma(dx, dx, dy * dy): the two sums differ by one ulp and r * r is exactly the smaller one."""
    u = synth.Rng(9400).uniform(4000).reshape(-1, 2)
    for a, b in u:
        dx, dy = 1.0 + 3.0 * a, 1.0 + 3.0 * b
        plain = dx * dx + dy * dy
        fused = float(Fraction(dx) * Fraction(dx) + Fraction(dy * dy))
        if fused <= plain:
            continue
        r0 = math.sqrt(plain)
        for r in (r0, math.nextafter(r0, 0.0), math.nextafter(r0, 10.0)):
            if r * r == plain:
                return -dx, -dy, r  # the origin row: (double)0.0f - cx = dx exactly
    raise AssertionError("no fused / un-fused case found")


def canyon_map(n=150_000) -> np.ndarray:
    pts = synth.sample_map(synth.make_scene(), n, stream=9101)
    inten = (255.0 * synth.Rng(9102).uniform(n)).astype(F32)
    return np.concatenate([pts, inten[:, None]], axis=1)


def drive(n_frames=N_FRAMES):
    """[(scan with an intensity column, pose of the sensor in the map frame)] down the canyon."""
    M0 = synth.pose_matrix((X_START, 0.0, 0.0), (0.0, 0.0, 0.0))
    out = []
    for k, (scan, T_rel) in enumerate(synth.drive_stream(n_frames, rings=16, azimuths=400, step=STEP, x_start=X_START)):
        inten = (255.0 * synth.Rng(9200 + k).uniform(len(scan))).astype(F32)
        out.append((np.concatenate([scan, inten[:, None]], axis=1), M0 @ T_rel))
    return out


def hypotheses(T_true):
    """3 yaw x 3 lateral offsets around the true pose, (9, 4, 4) float32; index 4 is the true pose."""
    out = []
    for yaw in (-0.03, 0.0, 0.03):
        for lat in (-0.6, 0.0, 0.6):
            out.append((T_true @ synth.pose_matrix((0.0, lat, 0.0), (0.0, 0.0, yaw))).astype(F32))
    return np.stack(out)


# ---- helpers ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


@pytest.fixture(scope="module")
def world():
    return canyon_map(), drive()


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _session(sm, prior, method="NDT", crop=CROP, recrop=RECROP, **kw):
    g = sm.ScanMatcher(registration_method=method, **dict(KW, **kw))
    if prior is not None:
        assert g.setPriorMap(prior) == len(prior)
    g.setLocalizationParams(crop, recrop)
    g.setInitialPose((X_START, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    return g


def _cut_of(sm, prior, centre, radius, scan):
    """The cut a session makes of `prior` around `centre` on its first frame (None when the frame is ERR_NO_TARGET)."""
    from lidarslam_ros2_b200.registration import B200RegError

    g = sm.ScanMatcher(**KW)
    g.setPriorMap(prior)
    g.setLocalizationParams(radius, 1e9)
    g.setInitialPose((centre[0], centre[1], 0.0), (0.0, 0.0, 0.0, 1.0))
    try:
        g.localizeCloud(scan)
    except B200RegError as e:
        assert e.code == sm._capi.ERR_NO_TARGET, e
        assert g.localizeStats()["n_cuts"] == 0
        return None
    st = g.localizeStats()
    assert st["n_cuts"] == 1 and st["cut_centre"] == (centre[0], centre[1]) and st["n_map"] == len(prior)
    return g.cutCloud()


def _check_cut(sm, prior, centre, radius, scan):
    want = prior[L.cut_mask(prior, centre[0], centre[1], radius)]
    got = _cut_of(sm, prior, centre, radius, scan)
    if len(want) == 0:
        assert got is None
    else:
        assert got is not None and got.shape == want.shape and np.array_equal(_bits(got), _bits(want))


# ---- the cut, smallest first ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", EDGE_SIZES)
def test_cut_is_map_mask_in_map_order(sm, world, n):
    scan = world[1][0][0]
    for pattern in PATTERNS:
        _check_cut(sm, edge_map(n, pattern), CENTRE, RADIUS, scan)


def test_cut_at_the_radius(sm, world):
    """Rows at distance exactly r are kept, at r shortened by one double ulp dropped; the un-fused sum decides."""
    scan = world[1][0][0]
    prior = edge_map(TILE + 1, "mixed")
    exact = [3, 5]
    for r in (RADIUS, math.nextafter(RADIUS, 0.0), math.nextafter(RADIUS, 10.0)):
        mask = L.cut_mask(prior, *CENTRE, r)
        assert all(mask[i] == (r >= RADIUS) for i in exact) and not mask[7] and mask[9]
        _check_cut(sm, prior, CENTRE, r, scan)
    cx, cy, r = fused_case()
    assert L.cut_mask(prior, cx, cy, r)[23] and not L.cut_mask(prior, cx, cy, r, mut={"fused"})[23]
    _check_cut(sm, prior, (cx, cy), r, scan)


def test_cut_of_a_large_map(sm, world):
    scan = world[1][0][0]
    _check_cut(sm, edge_map((1 << 22) + 5, "mixed"), CENTRE, RADIUS, scan)


def test_cut_of_a_saved_map(sm, world, tmp_path):
    """A map saved by saveMapPCDASCII and loaded by setPriorMapPCD cuts to the rows the same points cut to from host memory."""
    prior, frames = world
    build = sm.ScanMatcher(**dict(KW, vg_size_for_map=0.3, trans_for_mapupdate=1.0))
    for scan, _ in frames[:4]:
        build.receiveCloud(scan)
    path = os.path.join(tmp_path, "map.pcd")
    n_saved, _ = build.saveMapPCDASCII(path)
    import lidarslam_ros2_b200 as m

    pts = m.read_pcd(path)
    assert len(pts) == n_saved
    a, b = (_session(sm, None, crop=12.0) for _ in range(2))
    assert a.setPriorMapPCD(path) == n_saved
    b.setPriorMap(pts)
    for g in (a, b):
        g.setInitialPose((1.0, 0.5, 0.0), (0.0, 0.0, 0.0, 1.0))
        g.localizeCloud(frames[1][0])
    want = pts[L.cut_mask(pts, 1.0, 0.5, 12.0)]
    assert 0 < len(want) < len(pts)
    assert np.array_equal(_bits(a.cutCloud()), _bits(want)) and np.array_equal(_bits(b.cutCloud()), _bits(want))


# ---- the drive -------------------------------------------------------------------------------------------------------------
def _plain(sm, method):
    """A registration object with the session's parameters, driven by the plain calls."""
    return sm.ScanMatcher(registration_method=method, **KW).registration


def _drive(sm, world, method, recrop=RECROP, n_frames=N_FRAMES, check_plain=True):
    import lidarslam_ros2_b200 as m

    prior, frames = world
    g = _session(sm, prior, method, recrop=recrop)
    loc = L.Localizer(prior, CROP, recrop, position=(X_START, 0.0, 0.0))
    plain = _plain(sm, method)
    recs = []
    for k, (scan, T_gt) in enumerate(frames[:n_frames]):
        guess = loc.sim_trans()
        pose7, final, recut = g.localizeCloud(scan)
        n_adopted = len(loc.adopted_at)
        r = loc.frame(final)
        st = g.localizeStats()
        assert np.array_equal(pose7, r["pose7"]), k
        assert recut == r["recut"] and st["dist_from_centre"] == r["dist"], (k, st, r)
        assert st["n_cuts"] == r["n_cuts"] and st["cut_centre"] == r["centre"] and bool(st["cut_pending"]) == r["pending"], k
        assert np.array_equal(_bits(g.cutCloud()), _bits(loc.cut())), k
        adopted = len(loc.adopted_at) > n_adopted
        target = prior[L.cut_mask(prior, *r["target_centre"], CROP)]
        if check_plain:
            # the session adds nothing of its own to the registration: the plain calls on the same target, source and guess
            # give the same bits (the solvers repeat themselves bit for bit, tests/test_gpu_session_edges.py)
            if adopted:
                plain.setInputTarget(m.voxel_grid_filter(target, KW["vg_size_for_input"]) if method == "GICP" else target)
                assert st["n_target"] == plain.stats()["n_target"], k
            assert g.registration.stats()["n_target"] == plain.stats()["n_target"], k
            plain.setInputSource(g.filteredScan())
            want = plain.align(guess)
            assert np.array_equal(_bits(final), _bits(want)), (k, synth.pose_error(final, want))
        dt, dr = synth.pose_error(final, T_gt)
        assert dt < 0.3 and dr < 0.02, (k, dt, dr)
        assert g.numSubmaps() == 0 and g.stats()["latest_distance"] == 0.0
        recs.append(dict(r, final=final, guess=guess, adopted=adopted, target=target, source=g.filteredScan()))
    return g, loc, recs


@pytest.mark.parametrize("method", ["NDT", "GICP"])
def test_drive_frame_by_frame(sm, world, method, oracle_mod):
    _, loc, recs = _drive(sm, world, method)
    assert loc.n_cuts >= 3 and sum(r["recut"] for r in recs) == loc.n_cuts - 1
    # a cut made in frame k is the target from frame k + 1 on
    assert [k for k, _ in loc.adopted_at] == [0] + [k + 1 for k, r in enumerate(recs[:-1]) if r["recut"]]
    if method == "NDT":  # the oracle registered on the same cut, scan and guess
        for k in (0, len(recs) - 1):
            o = oracle_mod.NDT(resolution=2.0, transformation_epsilon=0.01)
            o.set_target(recs[k]["target"][:, :3])
            o.set_source(recs[k]["source"][:, :3])
            dt, dr = synth.pose_error(recs[k]["final"], o.align(recs[k]["guess"]))
            assert dt < 1e-3 and dr < 1e-3, (k, dt, dr)


def test_recut_at_equality(sm, world):
    """recrop_distance equal to a frame's dist_from_centre re-cuts in that frame; one ulp above it does not."""
    _, _, recs = _drive(sm, world, "NDT", recrop=1e9, n_frames=4, check_plain=False)
    d = recs[2]["dist"]
    assert recs[1]["dist"] < d and not any(r["recut"] for r in recs)
    _, _, at = _drive(sm, world, "NDT", recrop=d, n_frames=4, check_plain=False)
    assert [r["recut"] for r in at[:3]] == [False, False, True]
    _, _, above = _drive(sm, world, "NDT", recrop=math.nextafter(d, 1e9), n_frames=3, check_plain=False)
    assert [r["recut"] for r in above] == [False, False, False]


def test_frame_preparation_on_device_equals_host(sm, world):
    """Sensor transform, armed de-skew, range filter and the use_odom guess of a localising frame: records in the LiDAR frame
    + setSensorTransform give bitwise the result of records moved on the host by the float32 restatement."""
    from test_gpu_deskew import _feed

    prior, frames = world
    a, b = _session(sm, prior), _session(sm, prior)
    a.setSensorTransform(MOUNT_POS, MOUNT_QUAT)
    E = fr.sensor_matrix(MOUNT_POS, MOUNT_QUAT)
    Einv = np.linalg.inv(osm.pose_matrix(MOUNT_POS, MOUNT_QUAT))
    imus = [sm.LidarUndistortion(session=a._h), sm.LidarUndistortion(session=b._h)]
    _feed(imus, t0=100.0, n=80)
    plain = _session(sm, prior)
    differs = False
    for k, (scan, T_gt) in enumerate(frames[:6]):
        lidar = fr.transform_cloud(scan, Einv.astype(F32))  # what the mounted LiDAR would have measured
        for g in (a, b):
            g.deskewNextScan(100.0 + 0.1 * k)
            M = T_gt @ synth.pose_matrix((0.02 * k, -0.01 * k, 0.0), (0.0, 0.0, 0.001 * k))
            g.odomNextScan(M[:3, 3], osm.quat_from_matrix(M[:3, :3]))
        pa, Ta, ra = a.localizeCloud(lidar)
        pb, Tb, rb = b.localizeCloud(fr.transform_cloud(lidar, E))
        assert ra == rb and np.array_equal(pa, pb) and np.array_equal(_bits(Ta), _bits(Tb)), k
        sa, sb = a.filteredScan(), b.filteredScan()
        assert np.array_equal(_bits(sa[np.lexsort(sa.T[::-1])]), _bits(sb[np.lexsort(sb.T[::-1])])), k
        _, Tp, _ = plain.localizeCloud(fr.transform_cloud(lidar, E))
        differs = differs or not np.array_equal(_bits(Tp), _bits(Tb))
    assert differs  # the de-skew and the odometry guess did take part
    assert imus[0].pointers() == imus[1].pointers() and imus[0].pointers()[1] > 0


# ---- error paths -----------------------------------------------------------------------------------------------------
def test_error_paths(sm, world, tmp_path):
    from lidarslam_ros2_b200.registration import B200RegError

    prior, frames = world
    scan = frames[0][0]
    E = sm._capi
    g = _session(sm, None)
    with pytest.raises(B200RegError) as e:
        g.localizeCloud(scan)
    assert e.value.code == E.ERR_NO_TARGET
    for bad in ((0.0, 1.0), (-1.0, 1.0), (math.nan, 1.0), (math.inf, 1.0), (10.0, -1.0), (10.0, math.nan)):
        with pytest.raises(B200RegError) as e:
            g.setLocalizationParams(*bad)
        assert e.value.code == E.ERR_ARG
    # the first cut empty: the pose is 1 km from the map
    g.setPriorMap(prior)
    g.setInitialPose((1000.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    with pytest.raises(B200RegError) as e:
        g.localizeCloud(scan)
    assert e.value.code == E.ERR_NO_TARGET and "1000.000" in str(e.value)
    st = g.localizeStats()
    assert st["n_cuts"] == 0 and st["n_cut"] == 0 and len(g.cutCloud()) == 0
    assert g.registration.stats()["n_target"] == 0
    # back inside the map the same session localises
    g.setInitialPose((X_START, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    g.localizeCloud(scan)
    cut0, n_target = g.cutCloud(), g.registration.stats()["n_target"]
    assert n_target == len(cut0) > 0
    # a missing / malformed PCD leaves the prior map and the cut in place
    bad = os.path.join(tmp_path, "bad.pcd")
    with open(bad, "w") as f:
        f.write("# .PCD v0.7\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\nWIDTH 2\nHEIGHT 1\nPOINTS 2\n"
                "DATA ascii\n1 2 3\n1 2\n")
    for path, code in ((os.path.join(tmp_path, "missing.pcd"), E.ERR_IO), (bad, E.ERR_FORMAT)):
        with pytest.raises(B200RegError) as e:
            g.setPriorMapPCD(path)
        assert e.value.code == code
        assert g.localizeStats()["n_map"] == len(prior) and np.array_equal(_bits(g.cutCloud()), _bits(cut0))
    _, _, recut = g.localizeCloud(frames[1][0])
    assert not recut and g.localizeStats()["n_cuts"] == 1 and g.registration.stats()["n_target"] == n_target


def test_empty_recut_keeps_the_old_target(sm, world):
    """The pose leaves the map: the re-cut keeps no row. The frame is still OK, registered against the old target; the old
    cut and target stay and the next frame tries the re-cut again. The map here ends 2 m ahead of the start and the
    odometry guess carries the pose 19.5 m down the street, further than the solver's steps could bring it back."""
    prior, frames = world
    behind = np.ascontiguousarray(prior[prior[:, 0] <= F32(X_START + 2.0)])
    crop, recrop = 6.0, 3.0
    g = _session(sm, behind, crop=crop, recrop=recrop)
    loc = L.Localizer(behind, crop, recrop, position=(X_START, 0.0, 0.0))
    n_target = cut0 = None
    for k, j in enumerate((0, 13, 13)):
        scan, T_gt = frames[j]
        if k < 2:
            g.odomNextScan(T_gt[:3, 3], osm.quat_from_matrix(T_gt[:3, :3]))
        pose7, final, recut = g.localizeCloud(scan)
        before = loc.n_cuts
        r = loc.frame(final)
        st = g.localizeStats()
        assert np.array_equal(pose7, r["pose7"]) and recut == r["recut"] and st["n_cuts"] == r["n_cuts"], k
        assert bool(st["cut_pending"]) == r["pending"] and st["dist_from_centre"] == r["dist"], k
        if k == 0:
            n_target, cut0 = g.registration.stats()["n_target"], g.cutCloud()
            continue
        # the frame asked for a re-cut and the re-cut was empty
        assert r["dist"] >= recrop and not recut and r["n_cuts"] == before and not r["pending"], (k, r)
        assert not L.cut_mask(behind, pose7[0], pose7[1], crop).any(), k
        assert g.registration.stats()["n_target"] == n_target and np.array_equal(_bits(g.cutCloud()), _bits(cut0)), k


def test_new_prior_map_recuts_on_the_next_frame(sm, world):
    prior, frames = world
    g = _session(sm, prior, recrop=1e9)
    for scan, _ in frames[:3]:
        g.localizeCloud(scan)
    assert g.localizeStats()["n_cuts"] == 1
    half = np.ascontiguousarray(prior[::2])
    g.setPriorMap(half)
    assert g.localizeStats()["n_cuts"] == 0 and g.localizeStats()["n_map"] == len(half)
    pose = g.localizeCloud(frames[3][0])[0]
    st = g.localizeStats()
    assert st["n_cuts"] == 1 and st["cut_pending"] == 0
    # the cut was made around the pose BEFORE that frame: recompute it from the previous frame's pose
    assert np.array_equal(_bits(g.cutCloud()), _bits(half[L.cut_mask(half, *st["cut_centre"], CROP)]))
    assert g.registration.stats()["n_target"] == len(g.cutCloud()) and np.all(np.isfinite(pose))
    # mixing in a mapping frame uses the session's other buffers and leaves the cut alone
    cut = g.cutCloud()
    g.receiveCloud(frames[4][0])
    assert np.array_equal(_bits(g.cutCloud()), _bits(cut)) and g.numSubmaps() >= 1  # initializeMap, and an update if it moved
    assert g.localizeStats()["n_cuts"] == 1 and g.stats()["n_targeted"] > 0


# ---- the initial pose from several hypotheses -------------------------------------------------------------------------------
def test_localize_init(sm, world):
    from lidarslam_ros2_b200.registration import B200RegError

    prior, frames = world
    scan, T_true = frames[2]
    G = hypotheses(T_true)
    g = _session(sm, prior)
    g.setInitialPose(T_true[:3, 3] + np.array([0.5, -0.4, 0.0]), (0.0, 0.0, 0.0, 1.0))  # a rough pose: where the cut is made
    best, rows = g.localizeInit(scan, G)
    assert len(rows) == 9 and all(r["status"] == 0 for r in rows)
    plain = _plain(sm, "NDT")
    plain.setInputTarget(g.cutCloud())
    plain.setInputSource(g.filteredScan())
    for k, r in enumerate(rows):
        want = plain.align(G[k])
        assert np.array_equal(_bits(r["final"]), _bits(want)), k
        assert r["converged"] == plain.hasConverged() and r["trans_probability"] == plain.getTransformationProbability(), k
    want_best = L.choose_hypothesis([(r["converged"], r["trans_probability"], r["status"]) for r in rows])
    assert best == want_best and best >= 0
    dt, dr = synth.pose_error(rows[best]["final"], T_true)
    assert dt < 0.3 and dr < 0.02, (dt, dr)
    # the adopted pose is that row's: the next frame's replay starts from it
    g2 = _session(sm, prior)
    g2.setInitialPose(T_true[:3, 3], (0.0, 0.0, 0.0, 1.0))
    b2, rows2 = g2.localizeInit(scan, G)
    loc2 = L.Localizer(prior, CROP, 1e9, position=[float(v) for v in T_true[:3, 3]])
    assert loc2.begin()
    loc2.adopt_pose(rows2[b2]["final"])
    guess = loc2.sim_trans()
    g2.setLocalizationParams(CROP, 1e9)
    pose7, final, _ = g2.localizeCloud(frames[3][0])
    plain.setInputTarget(g2.cutCloud())
    plain.setInputSource(g2.filteredScan())
    assert np.array_equal(_bits(final), _bits(plain.align(guess)))
    # equal hypotheses: the lowest index wins the tie
    same = np.stack([G[4]] * 3)
    g3 = _session(sm, prior)
    g3.setInitialPose(T_true[:3, 3], (0.0, 0.0, 0.0, 1.0))
    b3, rows3 = g3.localizeInit(scan, same)
    assert all(np.array_equal(_bits(r["final"]), _bits(rows3[0]["final"])) for r in rows3)
    assert b3 == (0 if rows3[0]["converged"] else -1)
    # hypotheses far off, one iteration allowed: whatever the rows say, the choice is the replay's, and the pose the next
    # frame starts from is the chosen row's (the initial pose when none converged)
    g4 = _session(sm, prior, recrop=1e9)
    g4.setInitialPose(T_true[:3, 3], (0.0, 0.0, 0.0, 1.0))
    g4.registration.setMaximumIterations(1)
    far = np.stack([(T_true @ synth.pose_matrix((3.0, 2.0, 0.0), (0.0, 0.0, 0.3))).astype(F32)] * 2)
    b4, rows4 = g4.localizeInit(scan, far)
    assert b4 == L.choose_hypothesis([(r["converged"], r["trans_probability"], r["status"]) for r in rows4])
    loc4 = L.Localizer(prior, CROP, 1e9, position=[float(v) for v in T_true[:3, 3]])
    if b4 >= 0:
        loc4.adopt_pose(rows4[b4]["final"])
    _, final4, _ = g4.localizeCloud(scan)
    plain.setMaximumIterations(1)
    plain.setInputTarget(g4.cutCloud())
    plain.setInputSource(g4.filteredScan())
    assert np.array_equal(_bits(final4), _bits(plain.align(loc4.sim_trans())))
    # a GICP handle
    gi = _session(sm, prior, "GICP")
    with pytest.raises(B200RegError) as e:
        gi.localizeInit(scan, G)
    assert e.value.code == sm._capi.ERR_ARG
