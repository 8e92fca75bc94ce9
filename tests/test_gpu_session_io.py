"""A mapping session saved to disk and loaded back (b200sm_save_session / b200sm_load_session) on the GPU: a driven session
with its loop edges and adjusted poses comes back bitwise in every product (submaps, segments, descriptors, the graph, the
pose adjustment, the assembled and saved maps, the occupancy grid, the static map, the loop searches); a merge into a map
loaded from disk is bitwise the merge in memory, on NDT and GICP; the files are PCL's binary PCD and the restated g2o text;
and a failed save or load leaves nothing behind."""
import os

import numpy as np
import pytest

import sessionioref as R
from test_gpu_session_edges import KW, LOOP, _out_and_back_session, smm  # noqa: F401 (fixture)
from test_gpu_session_merge import _registration, _session, _sessions, drive  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
F32 = np.float32


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]) if a.dtype.kind == "f" else a


def _same(x, y, what="value"):
    """bitwise equality of nested dicts / lists / tuples / arrays / floats"""
    if isinstance(x, dict):
        assert set(x) == set(y), what
        for k in x:
            _same(x[k], y[k], f"{what}.{k}")
    elif isinstance(x, (list, tuple)):
        assert len(x) == len(y), what
        for k, (a, b) in enumerate(zip(x, y)):
            _same(a, b, f"{what}[{k}]")
    elif isinstance(x, np.ndarray) or isinstance(y, np.ndarray):
        assert np.asarray(x).shape == np.asarray(y).shape and np.array_equal(_bits(np.asarray(x)), _bits(np.asarray(y))), what
    elif isinstance(x, float):
        assert np.array_equal(_bits(np.float64(x)), _bits(np.float64(y))), (what, x, y)
    else:
        assert x == y, (what, x, y)


def _submaps(s):
    return [s.submap(i) for i in range(s.numSubmaps())]


# ---------------------------------------------------------------- 1. a driven session
def test_round_trip_of_a_driven_session(smm, tmp_path):  # noqa: F811
    g, _, _ = _out_and_back_session(smm)
    reg = smm.backend_registration("NDT", ndt_resolution=2.0)
    n = g.numSubmaps()
    rows = g.searchLoopAll(reg, **LOOP)
    edges = [(r["id_min"], n - 1, r["relative_pose"]) for r in rows if r["accepted"]]
    assert edges, rows
    X, adj = g.poseAdjust(edges, num_adjacent_pose_cnstraints=3)
    d = str(tmp_path / "drive")
    info = g.saveSession(d, edges, 3, X)
    h = smm.ScanMatcher(**KW)
    e2, X2, k2, info2 = h.loadSession(d)
    g2o_bytes = os.path.getsize(os.path.join(d, "pose_graph.g2o"))  # written, never read back
    assert {k: v for k, v in info2.items() if k != "n_bytes"} == {k: v for k, v in info.items() if k != "n_bytes"}
    assert info2["n_bytes"] == info["n_bytes"] - g2o_bytes
    assert info["n_submaps"] == n and info["n_loop_edges"] == len(edges) and info["adjusted"] == 1
    _same(_submaps(h), _submaps(g), "submaps")
    assert h.segments() == g.segments() == [0]
    _same([h.scanContext(i) for i in range(n)], [g.scanContext(i) for i in range(n)], "descriptors")
    assert k2 == 3
    _same(e2, [(f, t, np.asarray(Z)) for f, t, Z in edges], "graph edges")
    _same(X2, X, "graph poses")
    _same(h.poseAdjust(e2, num_adjacent_pose_cnstraints=k2), (X, adj), "poseAdjust")
    for P in (None, X):
        _same(h.assembleMap(P), g.assembleMap(P), "assembleMap")
        for s, name in ((g, "a.pcd"), (h, "b.pcd")):
            s.saveMapPCDASCII(str(tmp_path / name), P)
        assert (tmp_path / "a.pcd").read_bytes() == (tmp_path / "b.pcd").read_bytes()
    _same(h.buildOccupancyGrid(), g.buildOccupancyGrid(), "occupancy info")
    _same(h.occupancyGrid(), g.occupancyGrid(), "occupancy grid")
    _same(h.buildStaticMap(), g.buildStaticMap(), "static map info")
    _same(h.staticMap(), g.staticMap(), "static map")
    _same(h.searchLoopAll(reg, **LOOP), rows, "searchLoopAll")
    place = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, search_submap_num=1)
    _same(h.searchLoopPlace(reg, **place), g.searchLoopPlace(reg, **place), "searchLoopPlace")


# ---------------------------------------------------------------- 2. merge across days
@pytest.mark.parametrize("kind", ["NDT", "GICP"])
def test_merge_into_a_map_loaded_from_disk(drive, kind, tmp_path):  # noqa: F811
    g, h = _sessions(drive)
    nA = g.numSubmaps()
    g.saveSession(str(tmp_path / "A"))
    del g
    a2 = _session()
    assert a2.loadSession(str(tmp_path / "A"))[:3] == ([], None, 5)
    got = a2.mergeSession(h, _registration(kind))
    g0, h0 = _sessions(drive)
    want = g0.mergeSession(h0, _registration(kind))
    assert want[2]["merged"]
    _same(got, want, "merge")
    _same(_submaps(a2), _submaps(g0), "merged submaps")
    rows, X, res = got
    a2.saveSession(str(tmp_path / "M"), res["edges"], 5, X)
    m = _session()
    e, P, k, info = m.loadSession(str(tmp_path / "M"))
    assert m.segments() == [0, nA] and info["n_segments"] == 2 and k == 5
    _same(e, res["edges"], "merged edges")
    _same(P, X, "merged poses")
    _same(m.poseAdjust(e, num_adjacent_pose_cnstraints=k)[0], X, "poseAdjust of the merged map")


# ---------------------------------------------------------------- 3. files
def _random_cloud(rng, n):
    c = rng.uniform(-50, 50, (n, 4)).astype(F32)
    c[:, 3] = rng.integers(0, 256, n).astype(F32) + F32(0.5)
    return c


def _pose(rng):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix(rng.uniform(-20, 20, 3), rng.uniform(-3, 3, 3))


def test_files_are_pcl_binary_and_the_restated_graph(tmp_path):
    from lidarslam_ros2_b200 import read_pcd

    rng = np.random.default_rng(5)
    sizes = list(range(18)) + [3_000_000, 2_000_000]  # the last one does not fit the 4 Mi-point arena chunk the first opened
    clouds = [_random_cloud(rng, n) for n in sizes]
    poses = [_pose(rng) for _ in sizes]
    dists = np.cumsum(rng.uniform(0, 3, len(sizes))).tolist()
    g = _session()
    g.setScanContextParams(12, 30, 40.0, 1.5)
    for c, P, dd in zip(clouds, poses, dists):
        g.importSubmap(c, P, dd)
    loops = [(3, 15, _pose(rng)), (19, 0, _pose(rng))]
    adj = [_pose(rng) for _ in sizes]
    d = tmp_path / "files"
    info = g.saveSession(str(d), loops, 2, adj)
    total = 0
    for i, c in enumerate(clouds):
        f = d / "submaps" / ("%06d.pcd" % i)
        body = f.read_bytes()
        assert body == R.submap_file(c), i
        total += len(body)
        assert np.array_equal(_bits(read_pcd(str(f))), _bits(c)), i
    manifest = R.write_manifest((12, 30, 40.0, 1.5), [0], sizes, dists, poses, 2, loops, adj)
    assert (d / "session.txt").read_text() == manifest
    g2o = R.write_g2o(poses, 2, [0], loops, adj)
    assert (d / "pose_graph.g2o").read_text() == g2o
    assert info["n_bytes"] == total + len(manifest) + len(g2o) and info["n_points"] == sum(sizes)
    assert not (d / "session.txt.tmp").exists()
    h = _session()
    h.loadSession(str(d))
    _same(_submaps(h), _submaps(g), "submaps")
    _same([h.scanContext(i) for i in range(len(sizes))], [g.scanContext(i) for i in range(len(sizes))], "descriptors")
    g2o_own = R.write_g2o(poses, 2, [0], loops)
    g.saveSession(str(d), loops, 2)  # over the earlier save, without adjusted poses
    assert (d / "pose_graph.g2o").read_text() == g2o_own


# ---------------------------------------------------------------- 4. failures
def _small_session():
    rng = np.random.default_rng(11)
    g = _session()
    g.setScanContextParams(10, 24, 30.0, 1.0)
    for k in range(6):
        g.importSubmap(_random_cloud(rng, 200 + 10 * k), _pose(rng), 1.0 * k)
    return g


def _descriptor_with_params(rng_seed=2):
    """a cloud, and the descriptor a fresh session with Scan Context parameters (7, 18, 25, 0.5) gives it"""
    c = _random_cloud(np.random.default_rng(rng_seed), 300)
    ref = _session()
    ref.setScanContextParams(7, 18, 25.0, 0.5)
    ref.importSubmap(c, np.eye(4), 0.0)
    return c, ref.scanContext(0)


def test_failures_leave_nothing_behind(tmp_path):
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    g = _small_session()
    bad = tmp_path / "refused"
    for args in (dict(num_adjacent_pose_cnstraints=0), dict(loop_edges=[(0, 6, np.eye(4))]), dict(loop_edges=[(2, 2, np.eye(4))]),
                 dict(loop_edges=[(0, 1, np.full((4, 4), np.nan))]), dict(poses=[np.full((4, 4), np.inf)] * 6)):
        with pytest.raises(B200RegError) as e:
            g.saveSession(str(bad), **args)
        assert e.value.code == _capi.ERR_ARG and not bad.exists(), args
    with pytest.raises(B200RegError) as e:
        _session().saveSession(str(bad))
    assert e.value.code == _capi.ERR_ARG and not bad.exists()
    good = tmp_path / "good"
    g.saveSession(str(good), [(0, 5, np.eye(4))], 2)
    text = (good / "session.txt").read_text()
    lines = text.split("\n")[:-1]
    sub0 = good / "submaps" / "000000.pcd"
    body0 = sub0.read_bytes()

    s = _session()
    s.setScanContextParams(7, 18, 25.0, 0.5)

    def refused(code):
        with pytest.raises(B200RegError) as e:
            s.loadSession(str(good))
        assert e.value.code == code, str(e.value)
        assert s.numSubmaps() == 0 and s.segments() == []
        return str(e.value)

    sub0.write_bytes(body0[:-5])  # a truncated body
    assert "POINTS 200" in refused(_capi.ERR_FORMAT)
    sub0.write_bytes(body0.replace(b"WIDTH 200", b"WIDTH 199").replace(b"POINTS 200", b"POINTS 199"))  # POINTS against the manifest
    assert "the manifest says 200" in refused(_capi.ERR_FORMAT)
    sub0.unlink()  # a missing file
    refused(_capi.ERR_IO)
    sub0.write_bytes(body0)
    for k, (line, new) in enumerate([(0, "b200sm_session 2"), (3, "segments 1 1"), (4, lines[4] + " 0"), (10, "odometry 0"),
                                     (12, "loop 0 6" + lines[12][8:]), (13, "adjusted 3")]):
        (good / "session.txt").write_text("\n".join(lines[:line] + [new] + lines[line + 1:]) + "\n")
        assert f"line {line + 1}:" in refused(_capi.ERR_FORMAT), k
    (good / "session.txt").write_text(text + "pose 0\n")
    assert "line 15:" in refused(_capi.ERR_FORMAT)
    (good / "session.txt").unlink()
    refused(_capi.ERR_IO)
    # the parameters survived every refusal: a descriptor is the one (7, 18, 25, 0.5) gives
    c, want = _descriptor_with_params()
    s.importSubmap(c, np.eye(4), 0.0)
    assert s.scanContext(0).shape == want.shape and np.array_equal(_bits(s.scanContext(0)), _bits(want))
    with pytest.raises(B200RegError) as e:  # not empty any more
        (good / "session.txt").write_text(text)
        s.loadSession(str(good))
    assert e.value.code == _capi.ERR_ARG and s.numSubmaps() == 1
    t = _session()
    t.setScanContextParams(7, 18, 25.0, 0.5)
    e2, P, k, info = t.loadSession(str(good))  # the next good load succeeds, with the saved parameters
    assert info["n_submaps"] == 6 and k == 2 and P is None and len(e2) == 1
    _same(_submaps(t), _submaps(g), "submaps")
    _same([t.scanContext(i) for i in range(6)], [g.scanContext(i) for i in range(6)], "descriptors")


def test_session_rules_on_a_loaded_map(drive, tmp_path):  # noqa: F811
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    g, h = _sessions(drive)
    nA = g.numSubmaps()
    rows, X, res = g.mergeSession(h, _registration("NDT"))
    assert res["merged"]
    g.saveSession(str(tmp_path / "M"), res["edges"], 5, X)
    m = _session()
    m.loadSession(str(tmp_path / "M"))
    scan = drive[0][0]
    T = np.eye(4, dtype=F32)
    for call in (lambda: m.setScan(scan), lambda: m.receiveCloud(scan), lambda: m.updateMap(T, [0, 0, 0], [0, 0, 0, 1])):
        with pytest.raises(B200RegError) as e:
            call()
        assert e.value.code == _capi.ERR_ARG
    n = m.numSubmaps()
    before = _submaps(m)
    m.importSubmap(scan, np.eye(4), 99.0)
    assert m.numSubmaps() == n + 1 and m.segments() == [0, nA]
    _same(_submaps(m)[:n], before, "submaps")
    one = _session()  # a single-segment map loaded from disk refuses the frontend too
    g1, _ = _sessions(drive)
    g1.saveSession(str(tmp_path / "A"))
    one.loadSession(str(tmp_path / "A"))
    with pytest.raises(B200RegError) as e:
        one.setScan(scan)
    assert e.value.code == _capi.ERR_ARG and "loaded" in str(e.value)
    one.importSubmap(scan, np.eye(4), 99.0)
    assert one.segments() == [0] and one.numSubmaps() == g1.numSubmaps() + 1
