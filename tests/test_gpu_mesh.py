"""The surface mesh of the scan-matcher session (b200sm_build_mesh: the static map's K15a bounds, then K21 in csrc/mesh.cu)
on the GPU: every info field, band voxel, sum, weight, vertex (as bits) and face bitwise the serial host compile of
csrc/mesh.hpp (tests/hostmath/mesh_host.cpp) on the hand-built rays, random submaps of up to 2^20 points, the drive, caller
poses from poseAdjust, a saved-and-loaded session and repeated builds; shuffled points change nothing; the PLY byte-equal
to a struct writer of the host's arrays; refused calls change nothing; and a mesh build and the static map, map changes,
occupancy grid, elevation map and consistency builds leave each other's read-backs as they were."""
import numpy as np
import pytest

import meshref as R
from test_mesh_cpu import cases, host  # noqa: F401 (fixture)

F32 = np.float32
pytestmark = pytest.mark.gpu
INFO = ("n_points", "n_rays", "n_skipped", "n_walked", "n_band_voxels", "n_observed_voxels", "n_vertices", "n_faces")


def _session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    return ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _import(g, submaps):
    for k, (pts, P) in enumerate(submaps):
        q = np.zeros((len(pts), 4), dtype=F32)
        if len(pts):
            q[:, :np.asarray(pts).shape[1]] = np.asarray(pts, dtype=F32)[:, :4]
        g.importSubmap(q, P, float(k))


def _build(g, p, poses=None):
    q = R.params(**p)
    return g.buildMesh(poses=poses, resolution=q["resolution"], truncation=q["truncation"], max_range=q["max_range"],
                       sensor_origin=q["sensor_origin"], min_weight=q["min_weight"])


def _outputs(g):
    v, f = g.mesh()
    return g.meshVoxels(), v, f


def _same_outputs(a, b):
    return all(np.array_equal(a[0][k], b[0][k]) for k in a[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and \
        np.array_equal(a[2], b[2])


def _check(g, host, submaps, p, info):  # noqa: F811
    want = host.build(submaps, p)
    assert isinstance(want, dict), want
    if want["n_rays"]:
        assert info["box_origin"] == want["lo"] and info["box_dims"] == want["dims"]
    for k in INFO:
        assert info[k] == want[k], k
    vox, v, f = _outputs(g)
    assert np.array_equal(vox["ijk"], want["ijk"]) and np.array_equal(vox["sdf_sum"], want["sum"])
    assert np.array_equal(vox["weight"], want["weight"])
    assert np.array_equal(v.view(np.uint32), want["vertices"].view(np.uint32)) and np.array_equal(f, want["faces"])
    return want


@pytest.mark.parametrize("name,subs,p", cases(), ids=[c[0] for c in cases()])
def test_hand_built_bitwise_host(host, name, subs, p):  # noqa: F811
    g = _session()
    _import(g, subs)
    _check(g, host, subs, p, _build(g, p))


def _random_submap(seed, n, reach=30.0):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), dtype=F32)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p[:, :3] = d * rng.choice([6.0, 11.0, reach], size=(n, 1)) + rng.normal(scale=0.02, size=(n, 3))
    p[:, 3] = rng.uniform(0, 255, size=n)
    if n > 10:
        p[3::97, 0] = np.nan
        p[5::89, 2] = np.inf
    return p


def test_random_submaps_bitwise_host(host):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sizes = [0, 1, 31, 1000, 4097, 1 << 20, 3000, 0]
    subs = [(_random_submap(40 + k, n), synth.pose_matrix((0.3 * k - 0.7, -0.2 * k, 1.0 + 0.1 * k), (0.01 * k, -0.02, 0.9 * k)))
            for k, n in enumerate(sizes)]
    g = _session()
    _import(g, subs)
    for p in (dict(resolution=0.25, truncation=0.75, max_range=40.0, sensor_origin=(0.2, -0.1, 0.3), min_weight=2),
              dict(resolution=0.5, truncation=0.5, max_range=20.0, min_weight=1)):
        info = _build(g, p)
        _check(g, host, subs, p, info)
        assert info["n_faces"] > 0


@pytest.fixture(scope="module")
def drive():
    import staticscene

    scans, poses, _ = staticscene.drive()
    return list(zip(scans, poses))


def test_drive_bitwise_host_ply_and_repeat(host, drive, tmp_path):  # noqa: F811
    g = _session()
    _import(g, drive)
    info = _build(g, {})
    want = _check(g, host, drive, {}, info)
    size = g.saveMeshPly(tmp_path / "mesh.ply")
    ref = R.ply_bytes(want["vertices"], want["faces"])
    assert size == len(ref) and (tmp_path / "mesh.ply").read_bytes() == ref
    before = _outputs(g)
    assert _build(g, {}) == info
    assert _same_outputs(before, _outputs(g))


def test_caller_poses_from_pose_adjust(host, drive):  # noqa: F811
    """Poses from poseAdjust (one loop edge, the true relative pose) against the host compile at those poses."""
    subs = drive[::2]
    g = _session()
    _import(g, subs)
    P0, P1 = subs[0][1], subs[-1][1]
    rel = np.linalg.inv(P0) @ P1 @ np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.03], [0, 0, 1, 0], [0, 0, 0, 1]])  # a loop edge a little off
    X, _ = g.poseAdjust([(0, len(subs) - 1, rel)])
    X = np.asarray(X, dtype=np.float64).reshape(len(subs), 4, 4)
    assert not np.array_equal(X, np.array([P for _, P in subs]))
    info = _build(g, {}, poses=X)
    _check(g, host, [(s, P) for (s, _), P in zip(subs, X)], {}, info)


def test_shuffled_points_change_nothing(drive):
    subs = drive[10:20]
    rng = np.random.default_rng(4)
    a, b = _session(), _session()
    _import(a, subs)
    _import(b, [(s[rng.permutation(len(s))], P) for s, P in subs])
    assert _build(a, {}) == _build(b, {})
    assert _same_outputs(_outputs(a), _outputs(b))


def test_loaded_session_bitwise_host(host, drive, tmp_path):  # noqa: F811
    g = _session()
    _import(g, drive[::3])
    g.saveSession(str(tmp_path / "sess"))
    loaded = _session()
    loaded.loadSession(str(tmp_path / "sess"))
    info = _build(loaded, {})
    subs = []
    for k in range(loaded.numSubmaps()):
        cloud, pose, _ = loaded.submap(k)
        subs.append((cloud, pose))
    _check(loaded, host, subs, {}, info)
    assert info == _build(g, {})


def test_refused_calls_change_nothing(tmp_path, drive):
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    with pytest.raises(B200RegError) as e:
        g.buildMesh()
    assert e.value.code == -1  # no submaps
    subs = drive[12:18]
    _import(g, subs)
    for call in (lambda: g.mesh(), lambda: g.meshVoxels(), lambda: g.saveMeshPly(tmp_path / "x.ply")):
        with pytest.raises(B200RegError) as e:
            call()
        assert e.value.code == -1
    assert not (tmp_path / "x.ply").exists()
    info = _build(g, {})
    before = _outputs(g)
    g.saveMeshPly(tmp_path / "a.ply")
    for p in (dict(resolution=0.0), dict(truncation=0.19), dict(truncation=3.3), dict(max_range=float("inf")), dict(min_weight=0),
              dict(max_range=0.2 * 16385)):
        with pytest.raises(B200RegError) as e:
            _build(g, p)
        assert e.value.code == -1, p
    with pytest.raises(B200RegError) as e:
        g.buildMesh(poses=np.full((len(subs), 4, 4), np.nan))
    assert e.value.code == -1
    far = [P.copy() for _, P in subs]
    far[3][:3, 3] += (20000.0, 20000.0, 20000.0)
    with pytest.raises(B200RegError) as e:
        _build(g, dict(resolution=0.02, truncation=0.04), poses=np.array(far))
    assert e.value.code == -1 and "2^31" in str(e.value)
    with pytest.raises(B200RegError) as e:
        g.saveMeshPly(tmp_path / "no_such_dir" / "m.ply")
    assert e.value.code == -7
    assert _same_outputs(before, _outputs(g))
    g.saveMeshPly(tmp_path / "b.ply")
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()
    # an empty mesh (one submap, min_weight above any weight): no file, and the build still replaces the last one
    _build(g, dict(min_weight=1 << 30))
    with pytest.raises(B200RegError) as e:
        g.saveMeshPly(tmp_path / "empty.ply")
    assert e.value.code == -1 and not (tmp_path / "empty.ply").exists()
    assert info["n_faces"] > 0


def test_isolation_from_the_other_builds(drive):
    subs = drive[12:20]
    g = _session()
    _import(g, subs)

    def bits(a):
        return np.ascontiguousarray(a).view(np.uint8)

    def others():
        sm, off = g.staticMap()
        mv = g.mapVoxels()
        og = g.occupancyGrid()
        el = g.elevationMap()
        mc = g.mapConsistency()
        ch = g.changeVoxels()
        return [sm, off] + [mv[k] for k in sorted(mv)] + [og[k] for k in ("data", "hits", "frees")] + \
            [np.asarray(el[k]) for k in ("n", "h", "lo", "step", "value")] + [mc[k] for k in ("n", "h", "plane_var")] + \
            [ch[k] for k in sorted(ch)] + [g.mapChanges()]

    g.buildStaticMap(resolution=0.25)
    g.buildOccupancyGrid(resolution=0.1, z_min=0.3, z_max=2.5, max_range=100.0)
    g.buildElevationMap()
    g.buildMapConsistency()
    g.buildMapChanges(split_submap=4)
    a = others()
    _build(g, {})
    ms = _outputs(g)
    b = others()
    assert len(a) == len(b) and all(np.array_equal(bits(x), bits(y)) for x, y in zip(a, b))
    g.buildStaticMap()
    g.buildOccupancyGrid()
    g.buildElevationMap()
    g.buildMapConsistency(radius=0.3)
    g.buildMapChanges(split_submap=3)
    assert _same_outputs(ms, _outputs(g))
