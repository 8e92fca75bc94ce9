"""The elevation / traversability map of the scan-matcher session (b200sm_build_elevation_map, K18 in csrc/elevation.cu) on
the GPU: every layer, every count and both map_server files bitwise / byte-equal to the serial host compile of
csrc/elevation_map.hpp (tests/hostmath/elevation_host.cpp) on the hand-built cases, random submaps of 0 to 2^20 points, the
terrain drive, caller poses, a loaded session and a merged one (the merge tests' drive); a second build replaces the
first, refused calls change nothing readable, a build leaves the other map products as they were, and shuffled points give the same bits."""
import numpy as np
import pytest

import elevationref as R
import terrainscene as TS
from test_elevation_cpu import CASES, LAYERS, bits, host  # noqa: F401 (fixture)
from test_gpu_session_merge import drive  # noqa: F401 (fixture)

F32 = np.float32
pytestmark = pytest.mark.gpu


def _session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    return ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _import(g, submaps):
    for k, (pts, P) in enumerate(submaps):
        pts = np.asarray(pts, dtype=F32).reshape(len(pts), -1) if len(pts) else np.zeros((0, 3), F32)
        g.importSubmap(pts, P, float(k))


def _build(g, p, poses=None):
    return g.buildElevationMap(poses=poses, **R.params(**p))


def _check(g, host, submaps, p, tmp_path, info):  # noqa: F811
    """The session's last map and files against the host compile of the same submaps."""
    want = host.build(submaps, p)
    assert isinstance(want, dict), want
    got = g.elevationMap()
    assert (info["width"], info["height"]) == (want["width"], want["height"])
    assert info["origin"] == want["origin"] and info["resolution"] == R.params(**p)["resolution"]
    for k in ("n_points", "n_skipped", "n_overhang", "n_observed", "n_lethal", "n_traversable", "n_unknown"):
        assert info[k] == want[k], k
    for k in LAYERS:
        assert np.array_equal(bits(got[k]), bits(want[k])), k
    g.saveTraversabilityMap(tmp_path / "gpu.pgm", tmp_path / "gpu.yaml")
    assert host.save(str(tmp_path / "gpu.pgm.host"), str(tmp_path / "host.yaml")) == 0
    assert (tmp_path / "gpu.pgm").read_bytes() == (tmp_path / "gpu.pgm.host").read_bytes()
    assert (tmp_path / "gpu.yaml").read_text() == (tmp_path / "host.yaml").read_text().replace("gpu.pgm.host", "gpu.pgm")
    return got


def _layers_equal(a, b):
    return all(np.array_equal(bits(a[k]), bits(b[k])) for k in LAYERS)


@pytest.mark.parametrize("name,subs,p", CASES, ids=[c[0] for c in CASES])
def test_hand_built_bitwise_host(host, tmp_path, name, subs, p):  # noqa: F811
    g = _session()
    _import(g, subs)
    _check(g, host, subs, p, tmp_path, _build(g, p))


def _random_submap(seed, n, reach=60.0):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), dtype=F32)
    p[:, 0:2] = rng.uniform(-reach, reach, size=(n, 2))
    p[:, 2] = 0.02 * p[:, 0] + rng.normal(0.0, 0.03, size=n) + np.where(rng.random(n) < 0.05, 3.0, 0.0)
    if n > 10:
        p[3::97, 0] = np.nan
        p[5::89, 2] = np.inf
    return p


def test_random_submaps_bitwise_host(host, tmp_path):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sizes = [0, 1, 31, 1000, 4097, 1 << 20]
    subs = [(_random_submap(10 + k, n), synth.pose_matrix((3.0 * k - 7.3, -2.1 * k, 1.0 + 0.1 * k), (0.01 * k, -0.02, 0.9 * k)))
            for k, n in enumerate(sizes)]
    g = _session()
    _import(g, subs)
    for p in (dict(resolution=0.2, max_range=50.0, sensor_origin=(0.2, -0.1, 0.3)), dict(resolution=0.1, window_cells=8, min_cells=20)):
        info = _build(g, p)
        _check(g, host, subs, p, tmp_path, info)
        assert info["n_skipped"] > 0 and info["n_points"] > (1 << 19) and info["n_overhang"] > 0
    # the points of every submap shuffled: the same bits
    first = g.elevationMap()
    rng = np.random.default_rng(7)
    g2 = _session()
    _import(g2, [(pts[rng.permutation(len(pts))], P) for pts, P in subs])
    _build(g2, p)
    assert _layers_equal(first, g2.elevationMap())


@pytest.fixture(scope="module")
def terrain():
    return TS.drive()[0]


def test_terrain_drive_bitwise_host_and_rebuilds(host, tmp_path, terrain):  # noqa: F811
    g = _session()
    _import(g, terrain)
    info = _build(g, {})
    _check(g, host, terrain, {}, tmp_path, info)
    first = g.elevationMap()
    # other parameters replace the map; the first parameters give the first map back
    other = dict(resolution=0.2, window_cells=2, min_cells=5, max_slope=15.0)
    info2 = _build(g, other)
    _check(g, host, terrain, other, tmp_path, info2)
    assert info2["width"] != info["width"]
    assert _build(g, {}) == info
    assert _layers_equal(first, g.elevationMap())


def test_caller_poses_bitwise_host(host, tmp_path, terrain):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    subs = terrain[::5]
    moved = [P @ synth.pose_matrix((0.05 * k, -0.03 * k, 0.01), (0.0, 0.002 * k, 0.01 * k)) for k, (_, P) in enumerate(subs)]
    g = _session()
    _import(g, subs)
    info = _build(g, {}, poses=np.array(moved))
    _check(g, host, [(pts, P) for (pts, _), P in zip(subs, moved)], {}, tmp_path, info)


def test_refusals_change_nothing(host, tmp_path, terrain):  # noqa: F811
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    with pytest.raises(B200RegError):
        g.elevationMap()
    with pytest.raises(B200RegError):
        g.saveTraversabilityMap(tmp_path / "a.pgm", tmp_path / "a.yaml")
    with pytest.raises(B200RegError):
        _build(g, {})  # no submaps
    subs = terrain[:3]
    _import(g, subs)
    info = _build(g, {})
    before = g.elevationMap()
    for bad in (dict(window_cells=9), dict(max_slope=90.0), dict(min_cells=2), dict(max_step=0.0)):
        with pytest.raises(B200RegError):
            _build(g, bad)
    with pytest.raises(B200RegError):
        _build(g, {}, poses=np.full((3, 4, 4), np.nan))
    with pytest.raises(B200RegError):
        g.saveTraversabilityMap(tmp_path / "no_such_dir" / "a.pgm", tmp_path / "a.yaml")
    assert _layers_equal(before, g.elevationMap())
    _check(g, host, subs, {}, tmp_path, info)
    # the height-extent refusal comes after the statistics pass: the last map still stays
    h = _session()
    _import(h, [(np.array([(0.5, 0.5, 0.0), (1.5, 0.5, 1.0)], F32), np.eye(4))])
    base = _build(h, dict(resolution=1.0, min_points=1, min_cells=3, window_cells=1))
    kept = h.elevationMap()
    h.importSubmap(np.array([(0.5, 0.5, 16777216.0)], F32), np.eye(4), 1.0)
    with pytest.raises(B200RegError):
        _build(h, dict(resolution=1.0, min_points=1, min_cells=3, window_cells=1))
    again = h.elevationMap()
    assert _layers_equal(kept, again) and again["width"] == base["width"]


def test_build_leaves_the_other_products(tmp_path, terrain):
    g = _session()
    _import(g, terrain[:6])
    m0 = g.assembleMap()
    og0 = (g.buildOccupancyGrid(), g.occupancyGrid())
    sm0 = (g.buildStaticMap(), g.staticMap())
    _build(g, {})
    assert all(np.array_equal(a, b) for a, b in zip(g.assembleMap(), m0))
    og = g.occupancyGrid()
    assert all(np.array_equal(og[k], og0[1][k]) for k in ("data", "hits", "frees"))
    sm = g.staticMap()
    assert all(np.array_equal(a, b) for a, b in zip(sm, sm0[1]))
    assert g.numSubmaps() == 6


def _submaps(s):
    out = []
    for k in range(s.numSubmaps()):
        cloud, pose, _ = s.submap(k)
        out.append((cloud[:, :3], pose))
    return out


def test_loaded_session_bitwise_host(host, tmp_path, terrain):  # noqa: F811
    g = _session()
    _import(g, terrain[::4])
    g.saveSession(str(tmp_path / "sess"))
    loaded = _session()
    loaded.loadSession(str(tmp_path / "sess"))
    info = _build(loaded, {})
    _check(loaded, host, _submaps(loaded), {}, tmp_path, info)
    assert info == _build(g, {})


def test_merged_session_bitwise_host(host, tmp_path, drive):  # noqa: F811
    from test_gpu_session_merge import _registration, _sessions

    a, b = _sessions(drive)
    rows, X, res = a.mergeSession(b, _registration("NDT"))
    assert res["merged"]
    p = dict(resolution=0.2, window_cells=2, min_cells=5)
    for poses in (None, X):
        info = _build(a, p, poses=poses)
        subs = _submaps(a)
        if poses is not None:
            subs = [(pts, P) for (pts, _), P in zip(subs, poses)]
        _check(a, host, subs, p, tmp_path, info)
