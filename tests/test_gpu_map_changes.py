"""The map changes of the scan-matcher session (b200sm_build_map_changes: the static map's K15a-K15d per epoch, then K20 in
csrc/map_changes.cu) on the GPU: every count, label, info field, the updated map, its offsets and the saved file bitwise the
serial host compile of csrc/map_changes.hpp (tests/hostmath/map_changes_host.cpp) on the hand-built rays, random submaps,
the two-day drive, caller poses, several walk batches on each side of the split, shuffled points, a saved-and-loaded
session and two recordings merged by mergeSession; each epoch's counts equal to buildStaticMap on that epoch's submaps
alone; refused calls change nothing; and a change build and the static map, occupancy grid, elevation map and consistency
builds leave each other's read-backs as they were."""
import numpy as np
import pytest

import changeref as R
from test_gpu_session_merge import _registration, _sessions, drive  # noqa: F401 (fixture)
from test_map_changes_cpu import COUNTS, cases, host  # noqa: F401 (fixture)
from test_pcd_format_cpu import build_pcd_host, reference_pcd_bytes

F32 = np.float32
pytestmark = pytest.mark.gpu
INFO = (("split_submap", "split"), ("n_rays", "n_rays"), ("n_skipped", "n_skipped"), ("n_voxels", "n_voxels"),
        ("n_appeared_voxels", "n_appeared_voxels"), ("n_vanished_voxels", "n_vanished_voxels"), ("n_points", "n_points"),
        ("n_appeared_points", "n_appeared_points"), ("n_vanished_points", "n_vanished_points"),
        ("n_updated_points", "n_updated_points"))


@pytest.fixture(scope="module")
def ph(tmp_path_factory):
    return build_pcd_host(str(tmp_path_factory.mktemp("pcd_host")))


def _session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    return ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _import(g, submaps):
    for k, (pts, P) in enumerate(submaps):
        q = np.zeros((len(pts), 4), dtype=F32)
        if len(pts):
            q[:, :np.asarray(pts).shape[1]] = np.asarray(pts, dtype=F32)[:, :4]
        g.importSubmap(q, P, float(k))


def _build(g, p, split, poses=None):
    q = R.params(**p)
    return g.buildMapChanges(poses=poses, split_submap=split, resolution=q["resolution"], max_range=q["max_range"],
                             sensor_origin=q["sensor_origin"], ray_fraction=q["ray_fraction"], min_frees=q["min_frees"],
                             dynamic_thresh=q["dynamic_thresh"])


def _same_points(a, b):
    """Bit for bit, except that a NaN coordinate only has to be a NaN (the device returns the canonical NaN)."""
    a, b = np.asarray(a, dtype=F32), np.asarray(b, dtype=F32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb])


def _outputs(g):
    return g.changeVoxels(), g.mapChanges(), g.updatedMap()


def _check(g, host, submaps, split, p, info, poses=None, last=0):  # noqa: F811
    """The session's last build against the host compile of the same submaps, and its updated map against assembleMap."""
    want = host.build(submaps, split, p, last)
    assert isinstance(want, dict), want
    assert info["box_origin"] == want["lo"] and info["box_dims"] == want["dims"]
    for k, w in INFO:
        assert info[k] == want[w], k
    vox, labels, (cloud, offsets) = _outputs(g)
    assert np.array_equal(vox["ijk"], want["ijk"]) and np.array_equal(vox["label"], want["label"])
    for k in COUNTS:
        assert np.array_equal(vox[k], want[k]), k
    assert np.array_equal(labels, want["point_label"])
    assert np.array_equal(offsets, want["offsets"])
    assert _same_points(cloud, want["updated"])
    full, _ = g.assembleMap(poses)
    assert np.array_equal(cloud.view(np.uint32), full[want["point_label"] != R.VANISHED].view(np.uint32))
    return want


@pytest.mark.parametrize("name,subs,split,p,last", cases(), ids=[c[0] for c in cases()])
def test_hand_built_bitwise_host(host, name, subs, split, p, last):  # noqa: F811
    if last:
        pytest.skip("split_submap -1 needs a merged session: test_merged_sessions_bitwise_host")
    g = _session()
    _import(g, subs)
    info = _build(g, p, split)
    _check(g, host, subs, split, p, info)
    assert info["n_batches"] <= 2  # one per epoch with points


def _random_submap(seed, n, reach=60.0):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), dtype=F32)
    p[:, 0:2] = rng.uniform(-reach, reach, size=(n, 2))
    p[:, 2] = rng.uniform(-3.0, 5.0, size=n)
    p[:, 3] = rng.uniform(0, 255, size=n)
    if n > 10:
        p[3::97, 0] = np.nan
        p[5::89, 2] = np.inf
        p[7::11, :3] *= 0.3  # points in front of others: voxels that other rays cross
    return p


def test_random_submaps_bitwise_host(host):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sizes = [0, 1, 31, 1000, 4097, 1 << 20, 3000, 0]
    subs = [(_random_submap(20 + k, n), synth.pose_matrix((3.0 * k - 7.3, -2.1 * k, 1.0 + 0.1 * k), (0.01 * k, -0.02, 0.9 * k)))
            for k, n in enumerate(sizes)]
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.5, max_range=70.0, sensor_origin=(0.2, -0.1, 0.3), min_frees=1, dynamic_thresh=0.5)
    changed = 0
    for split in (3, 5, 1, 7):
        info = _build(g, p, split)
        _check(g, host, subs, split, p, info)
        changed += info["n_appeared_points"] + info["n_vanished_points"]
    assert changed > 0


@pytest.fixture(scope="module")
def two_days():
    import changescene

    d1, d2 = changescene.day(1), changescene.day(2)
    return list(zip(d1[0], d1[1])) + list(zip(d2[0], d2[1])), np.concatenate(d1[2]), np.concatenate(d2[2])


def test_two_day_drive_bitwise_host(host, ph, tmp_path, two_days):  # noqa: F811
    import changescene as S

    subs, l1, l2 = two_days
    g = _session()
    _import(g, subs)
    info = _build(g, {}, S.N_SUB)
    want = _check(g, host, subs, S.N_SUB, {}, info)
    lab = want["point_label"]
    assert (lab[:len(l1)][l1 == S.VANISHED_CAR] == R.VANISHED).mean() >= 0.75
    assert (lab[len(l1):][l2 == S.CONTAINER] == R.APPEARED).mean() >= 0.75
    # the saved file: PCL's writer restated on the updated map
    cloud, _ = g.updatedMap()
    points, size = g.saveUpdatedMapPcd(tmp_path / "updated.pcd")
    ref = reference_pcd_bytes(ph, cloud)
    assert points == len(cloud) and size == len(ref) and (tmp_path / "updated.pcd").read_bytes() == ref
    # two builds in a row: the same bits
    before = _outputs(g)
    assert _build(g, {}, S.N_SUB) == info
    after = _outputs(g)
    assert all(np.array_equal(before[0][k], after[0][k]) for k in before[0])
    assert np.array_equal(before[1], after[1]) and np.array_equal(before[2][0].view(np.uint32), after[2][0].view(np.uint32))


def test_caller_poses_equal_imported_poses(host, two_days):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    subs = two_days[0][20:40]
    moved = [P @ synth.pose_matrix((0.03 * k, -0.02, 0.01), (0.0, 0.001, 0.002 * k)) for k, (_, P) in enumerate(subs)]
    a = _session()
    _import(a, subs)
    ia = _build(a, {}, 10, poses=np.array(moved))
    b = _session()
    _import(b, [(s, P) for (s, _), P in zip(subs, moved)])
    ib = _build(b, {}, 10)
    assert ia == ib
    ca, oa = a.updatedMap()
    cb, ob = b.updatedMap()
    assert np.array_equal(ca.view(np.uint32), cb.view(np.uint32)) and np.array_equal(oa, ob)
    _check(a, host, [(s, P) for (s, _), P in zip(subs, moved)], 10, {}, ia, poses=np.array(moved))


def test_several_batches_each_side_bitwise_host(host):  # noqa: F811
    """One submap of 400 000 scattered points at 0.05 m makes some 400 000 occupied voxels: two bitmaps of about 12 500
    words per submap, so the 64 MiB budget holds about 670 submaps per batch. With 1 400 more submaps and the split at 701
    each epoch takes two batches, and a batch ends at the split."""
    from lidarslam_ros2_b200 import synth

    rng = np.random.default_rng(78)
    big = rng.uniform(-40, 40, size=(400000, 3)).astype(F32)
    big[:, 2] = rng.uniform(-2, 2, size=400000)
    subs = [(big, synth.pose_matrix((0.0, 0.0, 1.0), (0.0, 0.0, 0.0)))]
    for k in range(1400):
        q = rng.uniform(-30, 30, size=(8, 3)).astype(F32)
        q[:, 2] = rng.uniform(-2, 1, size=8)
        subs.append((q, synth.pose_matrix((rng.uniform(-5, 5), rng.uniform(-5, 5), 1.0), (0.0, 0.0, rng.uniform(0, 6.28)))))
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.05, max_range=100.0, min_frees=1, dynamic_thresh=0.5)
    info = _build(g, p, 701)
    assert info["n_batches"] >= 4, info
    _check(g, host, subs, 701, p, info)


def test_shuffled_points_permute_the_labels(two_days):
    """Shuffling the points of every submap permutes the labels and changes no voxel, count or info field."""
    import changescene as S

    subs = two_days[0][20:40]
    rng = np.random.default_rng(3)
    perms = [rng.permutation(len(s)) for s, _ in subs]
    a, b = _session(), _session()
    _import(a, subs)
    _import(b, [(s[q], P) for (s, P), q in zip(subs, perms)])
    ia, ib = _build(a, {}, S.N_SUB - 20), _build(b, {}, S.N_SUB - 20)
    assert ia == ib
    va, la, (ca, oa) = _outputs(a)
    vb, lb, (cb, ob) = _outputs(b)
    assert all(np.array_equal(va[k], vb[k]) for k in va) and np.array_equal(oa, ob)
    at = 0
    for (s, _), q in zip(subs, perms):
        assert np.array_equal(la[at:at + len(s)][q], lb[at:at + len(s)])
        at += len(s)
    key = lambda c: np.sort(c.view(np.uint32).view(np.dtype((np.void, 16))).ravel())  # noqa: E731
    assert np.array_equal(key(ca), key(cb))


def _submaps(s):
    out = []
    for k in range(s.numSubmaps()):
        cloud, pose, _ = s.submap(k)
        out.append((cloud, pose))
    return out


def test_loaded_session_bitwise_host(host, tmp_path, two_days):  # noqa: F811
    subs = two_days[0][::3]
    g = _session()
    _import(g, subs)
    g.saveSession(str(tmp_path / "sess"))
    loaded = _session()
    loaded.loadSession(str(tmp_path / "sess"))
    info = _build(loaded, {}, 10)
    _check(loaded, host, _submaps(loaded), 10, {}, info)
    assert info == _build(g, {}, 10)


def test_merged_sessions_bitwise_host(host, drive):  # noqa: F811
    """The real path: two recordings in sessions of their own, merged by mergeSession, then split_submap -1 against the host
    compile of the merged submaps and the poses read back."""
    from lidarslam_ros2_b200.registration import B200RegError

    a, b = _sessions(drive)
    n_a = a.numSubmaps()
    with pytest.raises(B200RegError):
        a.buildMapChanges()  # one segment: -1 is refused
    rows, X, res = a.mergeSession(b, _registration("NDT"))
    assert res["merged"] and a.segments() == [0, n_a]
    for poses in (None, X):
        info = _build(a, {}, -1, poses=poses)
        assert info["split_submap"] == n_a
        subs = _submaps(a)
        if poses is not None:
            subs = [(pts, P) for (pts, _), P in zip(subs, poses)]
        _check(a, host, subs, -1, {}, info, poses=poses, last=n_a)


def test_epoch_counts_equal_static_map(two_days):
    """On a session holding only one epoch's submaps, buildStaticMap's mapVoxels are that epoch's counts voxel for voxel."""
    import changescene as S

    subs = two_days[0]
    g = _session()
    _import(g, subs)
    _build(g, {}, S.N_SUB)
    vox = g.changeVoxels()
    idx = {tuple(v): r for r, v in enumerate(vox["ijk"].tolist())}
    for e, part in ((0, subs[:S.N_SUB]), (1, subs[S.N_SUB:])):
        h = _session()
        _import(h, part)
        h.buildStaticMap()
        sv = h.mapVoxels()
        rows = np.array([idx[tuple(v)] for v in sv["ijk"].tolist()], dtype=np.int64)
        assert np.array_equal(vox[COUNTS[2 * e]][rows], sv["hits"]) and np.array_equal(vox[COUNTS[2 * e + 1]][rows], sv["frees"])


def test_refused_calls_change_nothing(tmp_path, two_days):
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    with pytest.raises(B200RegError) as e:
        g.buildMapChanges(split_submap=1)
    assert e.value.code == -1  # no submaps
    subs = two_days[0][25:35]
    _import(g, subs)
    for call in (lambda: g.mapChanges(), lambda: g.changeVoxels(), lambda: g.updatedMap(),
                 lambda: g.saveUpdatedMapPcd(tmp_path / "x.pcd")):
        with pytest.raises(B200RegError) as e:
            call()
        assert e.value.code == -1
    assert not (tmp_path / "x.pcd").exists()
    info = _build(g, {}, 5)
    before = _outputs(g)
    g.saveUpdatedMapPcd(tmp_path / "a.pcd")
    bad = [dict(resolution=0.0), dict(max_range=float("inf")), dict(ray_fraction=1.5), dict(min_frees=0), dict(dynamic_thresh=-0.1)]
    for p in bad:
        with pytest.raises(B200RegError) as e:
            _build(g, p, 5)
        assert e.value.code == -1, p
    for split in (-1, 0, -2, 10, 11):
        with pytest.raises(B200RegError) as e:
            _build(g, {}, split)
        assert e.value.code == -1 and "split_submap" in str(e.value), split
    with pytest.raises(B200RegError) as e:
        g.buildMapChanges(poses=np.full((10, 4, 4), np.nan), split_submap=5)
    assert e.value.code == -1
    far = [P.copy() for _, P in subs]  # a box beyond 2^31 - 1 voxels
    far[7][:3, 3] += (20000.0, 20000.0, 20000.0)
    with pytest.raises(B200RegError) as e:
        _build(g, dict(resolution=0.02, max_range=100.0), 5, poses=np.array(far))
    assert e.value.code == -1 and "2^31" in str(e.value)
    after = _outputs(g)
    assert all(np.array_equal(before[0][k], after[0][k]) for k in before[0]) and np.array_equal(before[1], after[1])
    assert np.array_equal(before[2][0].view(np.uint32), after[2][0].view(np.uint32)) and np.array_equal(before[2][1], after[2][1])
    g.saveUpdatedMapPcd(tmp_path / "b.pcd")
    assert (tmp_path / "a.pcd").read_bytes() == (tmp_path / "b.pcd").read_bytes()
    assert info["n_points"] == sum(len(s) for s, _ in subs)


def test_isolation_from_the_other_builds(two_days):
    """A change build leaves the static map, occupancy grid, elevation map and consistency read-backs bitwise as they were,
    and those builds leave the change build's read-backs."""
    subs = two_days[0][25:35]
    g = _session()
    _import(g, subs)

    def bits(a):
        a = np.ascontiguousarray(a)
        return a.view(np.uint8)

    def others():
        sm, off = g.staticMap()
        mv = g.mapVoxels()
        og = g.occupancyGrid()
        el = g.elevationMap()
        mc = g.mapConsistency()
        return [sm, off] + [mv[k] for k in sorted(mv)] + [og[k] for k in ("data", "hits", "frees")] + \
            [np.asarray(el[k]) for k in ("n", "h", "lo", "step", "value")] + [mc[k] for k in ("n", "h", "plane_var")]

    g.buildStaticMap(resolution=0.25)
    g.buildOccupancyGrid(resolution=0.1, z_min=0.3, z_max=2.5, max_range=100.0)
    g.buildElevationMap()
    g.buildMapConsistency()
    a = others()
    _build(g, {}, 5)
    ch = _outputs(g)
    b = others()
    assert len(a) == len(b) and all(np.array_equal(bits(x), bits(y)) for x, y in zip(a, b))
    g.buildStaticMap()
    g.buildMapConsistency(radius=0.3)
    ch2 = _outputs(g)
    assert all(np.array_equal(ch[0][k], ch2[0][k]) for k in ch[0]) and np.array_equal(ch[1], ch2[1])
    assert np.array_equal(ch[2][0].view(np.uint32), ch2[2][0].view(np.uint32)) and np.array_equal(ch[2][1], ch2[2][1])
