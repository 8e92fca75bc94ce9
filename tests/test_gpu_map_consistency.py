"""The map consistency of the scan-matcher session (b200sm_build_map_consistency, K19 in csrc/consistency.cu) on the GPU:
every per-point layer, every per-submap row, every count, MME and MPV bitwise the serial host compile of
csrc/map_consistency.hpp (tests/hostmath/consistency_host.cpp) on the hand-built cases, random submaps of 0 to 2^20
points, a cell dense enough to be split across blocks, the place-recognition drive at true, drifted and adjusted poses, a
loaded session and a merged one (the merge tests' drive); the saved PCD byte-equal to the host writer's text; a second
build replaces the first, refused calls change nothing readable, and a build leaves the other map products as they were."""
import numpy as np
import pytest

import consistencyref as R
from test_gpu_session_merge import drive  # noqa: F401 (fixture)
from test_map_consistency_cpu import INFO_KEYS, ROW_KEYS, T, bits, compile_host, drive_maps, hand_cases

F32 = np.float32
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return compile_host(str(tmp_path_factory.mktemp("mc")))


@pytest.fixture(scope="module")
def pcd_host(tmp_path_factory):
    from test_pcd_format_cpu import build_pcd_host

    return build_pcd_host(str(tmp_path_factory.mktemp("pcd_host")))


def _session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    return ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _import(g, submaps):
    for k, (pts, P) in enumerate(submaps):
        pts = np.asarray(pts, dtype=F32).reshape(len(pts), -1) if len(pts) else np.zeros((0, 3), F32)
        g.importSubmap(pts[:, :3], P, float(k))


def _build(g, p, poses=None):
    return g.buildMapConsistency(poses=poses, **R.params(**p))


def _same_as_host(g, host, submaps, p, info):
    want = host.build(submaps, p)
    assert isinstance(want, dict), want
    got = g.mapConsistency()
    for k in ("n", "h", "plane_var"):
        assert np.array_equal(bits(got[k]), bits(want[k])), k
    rows = g.submapConsistency()
    for k in ROW_KEYS:
        assert np.array_equal(rows[k].astype(np.int64), want["rows"][k].astype(np.int64)), k
    for k in ("mme", "mpv"):
        assert np.array_equal(bits(rows[k]), bits(want["rows"][k])), k
        assert bits(np.float64(info[k])) == bits(np.float64(want["info"][k])), k
    for k in INFO_KEYS:
        assert (tuple(info[k]) if k.startswith("box") else info[k]) == want["info"][k], k
    return got


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_built_bitwise_host(host, name):
    subs, p = hand_cases()[name]
    g = _session()
    _import(g, subs)
    _same_as_host(g, host, subs, p, _build(g, p))


def test_random_submaps_bitwise_host(host):
    rng = np.random.default_rng(17)
    for n_total, n_sub, p in [(0, 2, dict(radius=0.5)), (1, 1, dict(radius=0.5, min_neighbors=4)),
                              (30000, 5, dict(radius=0.3, query_stride=3)), (1 << 20, 9, dict(radius=0.5, min_neighbors=6))]:
        cuts = np.sort(rng.integers(0, n_total + 1, size=n_sub - 1))
        sizes = np.diff(np.concatenate([[0], cuts, [n_total]]))
        subs = []
        for m in sizes:
            pts = np.column_stack([rng.uniform(-30, 30, size=(m, 2)), rng.uniform(-5, 5, size=m)]).astype(F32)
            pts[rng.random(m) < 0.001, 1] = np.nan
            subs.append((pts, T(*rng.uniform(-2, 2, 3), yaw=rng.uniform(-3, 3))))
        g = _session()
        _import(g, subs)
        _same_as_host(g, host, subs, p, _build(g, p))


def test_dense_cell_split_across_blocks(host):
    rng = np.random.default_rng(3)
    dense = rng.uniform(0.01, 0.29, size=(12000, 3)).astype(F32)  # one 0.3 m cell: 47 blocks of queries
    spread = np.column_stack([rng.uniform(-2, 2, size=(5000, 2)), 0.02 * rng.standard_normal(5000)]).astype(F32)
    subs = [(dense, np.eye(4)), (spread, np.eye(4))]
    g = _session()
    _import(g, subs)
    info = _build(g, {})
    _same_as_host(g, host, subs, {}, info)
    assert info["n_neighbors"] > 12000 * 12000 // 2


@pytest.fixture(scope="module")
def pr_drive():
    return drive_maps()


def test_drive_true_drifted_adjusted_bitwise_host_and_rebuilds(host, pr_drive):
    from test_map_consistency_cpu import adjust

    import ctypes as C
    import os
    import subprocess
    import tempfile

    scans, gt, drifted, (rev, match) = pr_drive
    d = tempfile.mkdtemp()
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostmath", "posegraph_host.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o",
                           os.path.join(d, "pg.so")])
    pg = C.CDLL(os.path.join(d, "pg.so"))
    adjusted = adjust(pg, drifted, (match, rev, np.linalg.inv(gt[match]) @ gt[rev]))
    g = _session()
    _import(g, list(zip(scans, drifted)))
    mme = {}
    for tag, poses in (("drifted", None), ("true", np.array(gt)), ("adjusted", np.array(adjusted))):
        info = _build(g, {}, poses=poses)  # every build replaces the last
        _same_as_host(g, host, list(zip(scans, list(poses) if poses is not None else drifted)), {}, info)
        mme[tag] = info["mme"]
    # the true map is the crispest; the adjusted one is not below the drifted one on this drive (DESIGN.md section 7b)
    assert mme["true"] < mme["drifted"] and mme["true"] < mme["adjusted"]


def test_saved_pcd_is_the_host_writers_text(host, pcd_host, tmp_path):
    from test_pcd_format_cpu import reference_pcd_bytes

    rng = np.random.default_rng(8)
    subs = [(np.column_stack([rng.uniform(-2, 2, size=(3000, 2)), 0.01 * rng.standard_normal(3000)]).astype(F32), T(1, 0, 0, 0.2)),
            (rng.normal(0, 0.5, size=(2000, 3)).astype(F32), T(0, 1, 0.5))]
    g = _session()
    _import(g, subs)
    poses = np.array([T(1.05, 0, 0, 0.21), T(0, 1.02, 0.5)])
    _build(g, {}, poses=poses)
    n, size = g.saveMapConsistencyPcd(tmp_path / "h.pcd")
    cloud, _ = g.assembleMap(poses)
    cloud = cloud.copy()
    cloud[:, 3] = g.mapConsistency()["h"].astype(np.float32)
    ref = reference_pcd_bytes(pcd_host, cloud)
    assert n == len(cloud) and size == len(ref) and (tmp_path / "h.pcd").read_bytes() == ref


def test_refusals_change_nothing(host, tmp_path):
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    for call in (lambda: g.mapConsistency(), lambda: g.submapConsistency(), lambda: g.saveMapConsistencyPcd(tmp_path / "a.pcd"),
                 lambda: _build(g, {})):
        with pytest.raises(B200RegError):
            call()
    rng = np.random.default_rng(4)
    subs = [(rng.normal(0, 0.5, size=(3000, 3)).astype(F32), np.eye(4)), (rng.normal(0, 0.5, size=(2000, 3)).astype(F32), T(0.5))]
    _import(g, subs)
    info = _build(g, {})
    before = (g.mapConsistency(), g.submapConsistency())
    for bad in (dict(radius=0.001), dict(radius=101.0), dict(min_neighbors=3), dict(query_stride=0)):
        with pytest.raises(B200RegError):
            _build(g, bad)
    with pytest.raises(B200RegError):
        _build(g, {}, poses=np.full((2, 4, 4), np.nan))
    with pytest.raises(B200RegError):
        _build(g, {}, poses=np.array([np.eye(4), T(float(2 ** 30) * 0.5 * 1.01)]))  # |X| >= 2^46 at 0.5 m
    with pytest.raises(B200RegError):
        _build(g, dict(radius=100.0), poses=np.array([np.eye(4), T(2.0 ** 16 * 100, 2.0 ** 15 * 100)]))  # 2^31 cells
    with pytest.raises(B200RegError):
        g.saveMapConsistencyPcd(tmp_path / "no_such_dir" / "a.pcd")
    after = (g.mapConsistency(), g.submapConsistency())
    for k in ("n", "h", "plane_var"):
        assert np.array_equal(bits(before[0][k]), bits(after[0][k])), k
    for k in before[1]:
        assert np.array_equal(bits(before[1][k]), bits(after[1][k])), k
    _same_as_host(g, host, subs, {}, info)
    # submaps added since the build: the save is refused rather than pairing the wrong points with the values
    g.importSubmap(subs[0][0], np.eye(4), 9.0)
    with pytest.raises(B200RegError):
        g.saveMapConsistencyPcd(tmp_path / "b.pcd")


def test_build_leaves_the_other_products(pr_drive):
    scans, gt, drifted, _ = pr_drive
    g = _session()
    _import(g, list(zip(scans[:6], drifted[:6])))
    m0 = g.assembleMap()
    og0 = (g.buildOccupancyGrid(), g.occupancyGrid())
    sm0 = (g.buildStaticMap(), g.staticMap())
    el0 = (g.buildElevationMap(), g.elevationMap())
    subs0 = [g.submap(k) for k in range(g.numSubmaps())]
    _build(g, {})
    assert all(np.array_equal(a, b) for a, b in zip(g.assembleMap(), m0))
    og = g.occupancyGrid()
    assert all(np.array_equal(og[k], og0[1][k]) for k in ("data", "hits", "frees"))
    assert all(np.array_equal(a, b) for a, b in zip(g.staticMap(), sm0[1]))
    el = g.elevationMap()
    assert all(np.array_equal(bits(np.asarray(el[k])), bits(np.asarray(el0[1][k]))) for k in ("n", "h", "value"))
    for k, (c0, p0, _) in enumerate(subs0):
        c1, p1, _ = g.submap(k)
        assert np.array_equal(c0, c1) and np.array_equal(p0, p1)


def _submaps(s):
    out = []
    for k in range(s.numSubmaps()):
        cloud, pose, _ = s.submap(k)
        out.append((cloud[:, :3], pose))
    return out


def test_loaded_session_bitwise_host(host, tmp_path, pr_drive):
    scans, gt, drifted, _ = pr_drive
    g = _session()
    _import(g, list(zip(scans[::3], drifted[::3])))
    g.saveSession(str(tmp_path / "sess"))
    loaded = _session()
    loaded.loadSession(str(tmp_path / "sess"))
    info = _build(loaded, {})
    _same_as_host(loaded, host, _submaps(loaded), {}, info)
    assert info == _build(g, {})


def test_merged_session_bitwise_host(host, drive):  # noqa: F811
    from test_gpu_session_merge import _registration, _sessions

    a, b = _sessions(drive)
    rows, X, res = a.mergeSession(b, _registration("NDT"))
    assert res["merged"]
    p = dict(radius=0.5, query_stride=2)
    for poses in (None, X):
        info = _build(a, p, poses=poses)
        subs = _submaps(a)
        if poses is not None:
            subs = [(pts, P) for (pts, _), P in zip(subs, poses)]
        _same_as_host(a, host, subs, p, info)
