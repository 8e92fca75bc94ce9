"""The static map of the scan-matcher session (b200sm_build_static_map, K15 in csrc/static_map.cu) on the GPU: the voxel
list, hits, frees, flags, info and the static map bitwise the serial host compile of csrc/static_map.hpp
(tests/hostmath/static_map_host.cpp) on the hand-built rays, random submaps of 0 to 2^20 points, the moving-object drive, a
build that takes several walk batches, caller poses and repeated builds; the static map equal to assembleMap's points at
the same poses masked by the host's keep set, offsets included; the saved file byte-equal to PCL's writer restated;
refused calls change nothing; and the map assembly, the PCD save, the occupancy grid and the loop search give what they
gave before a build."""
import numpy as np
import pytest

import staticmapref as R
from test_pcd_format_cpu import build_pcd_host, reference_pcd_bytes
from test_static_map_cpu import cases, host  # noqa: F401 (fixture)

F32 = np.float32
pytestmark = pytest.mark.gpu


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


def _build(g, p, poses=None):
    q = R.params(**p)
    return g.buildStaticMap(poses=poses, resolution=q["resolution"], max_range=q["max_range"], sensor_origin=q["sensor_origin"],
                            ray_fraction=q["ray_fraction"], min_frees=q["min_frees"], dynamic_thresh=q["dynamic_thresh"])


def _same_points(a, b):
    """Bit for bit, except that a NaN coordinate only has to be a NaN: the device's float arithmetic returns the canonical
    NaN, the host's propagates the input's payload."""
    a, b = np.asarray(a, dtype=F32), np.asarray(b, dtype=F32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb])


def _check(g, host, submaps, p, info, poses=None):  # noqa: F811
    """The session's last build against the host compile of the same submaps, and its static map against assembleMap."""
    want = host.build(submaps, p)
    assert isinstance(want, dict), want
    assert info["box_origin"] == want["lo"] and info["box_dims"] == want["dims"]
    for k, w in (("n_rays", "n_rays"), ("n_skipped", "n_skipped"), ("n_voxels", "n_voxels"), ("n_dynamic_voxels", "n_dynamic"),
                 ("n_points", "n_points"), ("n_static_points", "n_static")):
        assert info[k] == want[w], k
    vox = g.mapVoxels()
    assert np.array_equal(vox["ijk"], want["ijk"]) and np.array_equal(vox["hits"], want["hits"])
    assert np.array_equal(vox["frees"], want["frees"]) and np.array_equal(vox["dynamic"], want["dynamic"].astype(bool))
    cloud, offsets = g.staticMap()
    assert np.array_equal(offsets, want["offsets"])
    assert _same_points(cloud, want["static"])
    full, _ = g.assembleMap(poses)
    assert np.array_equal(cloud.view(np.uint32), full[want["keep"]].view(np.uint32))
    return want


@pytest.mark.parametrize("name,subs,p", cases(), ids=[c[0] for c in cases()])
def test_hand_built_bitwise_host(host, name, subs, p):  # noqa: F811
    g = _session()
    _import(g, subs)
    info = _build(g, p)
    _check(g, host, subs, p, info)
    assert info["n_batches"] == 1


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

    sizes = [0, 1, 31, 1000, 4097, 1 << 20]
    subs = [(_random_submap(10 + k, n), synth.pose_matrix((3.0 * k - 7.3, -2.1 * k, 1.0 + 0.1 * k), (0.01 * k, -0.02, 0.9 * k)))
            for k, n in enumerate(sizes)]
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.5, max_range=70.0, sensor_origin=(0.2, -0.1, 0.3), min_frees=1, dynamic_thresh=0.5)
    info = _build(g, p)
    _check(g, host, subs, p, info)
    assert info["n_skipped"] > 0 and info["n_rays"] > (1 << 19) and info["n_dynamic_voxels"] > 0


@pytest.fixture(scope="module")
def moving():
    import staticscene

    scans, poses, labels = staticscene.drive()
    return list(zip(scans, poses)), np.concatenate(labels)


def test_moving_drive_bitwise_host(host, ph, tmp_path, moving):  # noqa: F811
    subs, labels = moving
    g = _session()
    _import(g, subs)
    info = _build(g, {})
    want = _check(g, host, subs, {}, info)
    import staticscene as S

    gone = ~want["keep"]
    assert gone[labels == S.CAR].mean() >= 0.80 and gone[labels != S.CAR].mean() <= 0.01
    # the saved file: PCL's writer restated on the static map
    cloud, _ = g.staticMap()
    points, size = g.saveStaticMapPcd(tmp_path / "static.pcd")
    ref = reference_pcd_bytes(ph, cloud)
    assert points == len(cloud) and size == len(ref) and (tmp_path / "static.pcd").read_bytes() == ref
    # two builds in a row: the same bits
    vox = g.mapVoxels()
    again = _build(g, {})
    assert again == info
    vox2 = g.mapVoxels()
    cloud2, _ = g.staticMap()
    for k in ("ijk", "hits", "frees", "dynamic"):
        assert np.array_equal(vox[k], vox2[k])
    assert np.array_equal(cloud.view(np.uint32), cloud2.view(np.uint32))


def test_several_batches_bitwise_host(host):  # noqa: F811
    """One submap of 200 000 scattered points at 0.05 m makes some 200 000 occupied voxels: two bitmaps of about 6 250 words
    per submap, so the 64 MiB budget holds about 1 340 submaps per batch, and 1 401 submaps take two batches; the first
    batch also takes the fold past its 1 023-submap chunk. The host compile folds every submap in one pass."""
    from lidarslam_ros2_b200 import synth

    rng = np.random.default_rng(77)
    subs = []
    big = rng.uniform(-40, 40, size=(200000, 3)).astype(F32)  # 200 000 scattered voxels at 0.05 m
    big[:, 2] = rng.uniform(-2, 2, size=200000)
    subs.append((big, synth.pose_matrix((0.0, 0.0, 1.0), (0.0, 0.0, 0.0))))
    for k in range(1400):
        pts = rng.uniform(-30, 30, size=(8, 3)).astype(F32)
        pts[:, 2] = rng.uniform(-2, 1, size=8)
        subs.append((pts, synth.pose_matrix((rng.uniform(-5, 5), rng.uniform(-5, 5), 1.0), (0.0, 0.0, rng.uniform(0, 6.28)))))
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.05, max_range=100.0, min_frees=1, dynamic_thresh=0.5)
    info = _build(g, p)
    assert info["n_batches"] > 1, info
    _check(g, host, subs, p, info)


def test_caller_poses_equal_imported_poses(host, moving):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sub = moving[0][:10]
    moved = [P @ synth.pose_matrix((0.3 * k, -0.2, 0.05), (0.0, 0.01, 0.02 * k)) for k, (_, P) in enumerate(sub)]
    a = _session()
    _import(a, sub)
    ia = _build(a, {}, poses=np.array(moved))
    b = _session()
    _import(b, [(s, P) for (s, _), P in zip(sub, moved)])
    ib = _build(b, {})
    assert ia == ib
    ca, oa = a.staticMap()
    cb, ob = b.staticMap()
    assert np.array_equal(ca.view(np.uint32), cb.view(np.uint32)) and np.array_equal(oa, ob)
    _check(a, host, [(s, P) for (s, _), P in zip(sub, moved)], {}, ia, poses=np.array(moved))


def test_refused_calls_change_nothing(tmp_path, moving):
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    with pytest.raises(B200RegError) as e:
        g.buildStaticMap()
    assert e.value.code == -1  # no submaps
    subs = moving[0][:4]
    _import(g, subs)
    for call in (lambda: g.staticMap(), lambda: g.mapVoxels(), lambda: g.saveStaticMapPcd(tmp_path / "x.pcd")):
        with pytest.raises(B200RegError) as e:
            call()
        assert e.value.code == -1
    assert not (tmp_path / "x.pcd").exists()
    info = _build(g, {})
    before, off = g.staticMap()
    vox = g.mapVoxels()
    g.saveStaticMapPcd(tmp_path / "a.pcd")
    bad = [dict(resolution=0.0), dict(resolution=-0.1), dict(max_range=0.0), dict(max_range=float("inf")),
           dict(resolution=0.001, max_range=20.0), dict(sensor_origin=(0.0, float("inf"), 0.0)), dict(ray_fraction=0.0),
           dict(ray_fraction=1.5), dict(min_frees=0), dict(dynamic_thresh=1.5), dict(dynamic_thresh=-0.1)]
    for p in bad:
        with pytest.raises(B200RegError) as e:
            _build(g, p)
        assert e.value.code == -1, p
    with pytest.raises(B200RegError) as e:
        g.buildStaticMap(poses=np.full((4, 4, 4), np.nan))
    assert e.value.code == -1
    far = [P.copy() for _, P in subs]  # a box beyond 2^31 - 1 voxels: a submap 20 km away in x, y and z at 0.02 m
    far[3][:3, 3] += (20000.0, 20000.0, 20000.0)
    with pytest.raises(B200RegError) as e:
        _build(g, dict(resolution=0.02, max_range=100.0), poses=np.array(far))
    assert e.value.code == -1 and "2^31" in str(e.value)
    high = [P.copy() for _, P in subs]  # a sensor origin beyond 2^30 voxels
    high[0][2, 3] = 3e8
    with pytest.raises(B200RegError) as e:
        _build(g, {}, poses=np.array(high))
    assert e.value.code == -1
    after, off2 = g.staticMap()
    vox2 = g.mapVoxels()
    assert np.array_equal(before.view(np.uint32), after.view(np.uint32)) and np.array_equal(off, off2)
    for k in ("ijk", "hits", "frees", "dynamic"):
        assert np.array_equal(vox[k], vox2[k])
    g.saveStaticMapPcd(tmp_path / "b.pcd")
    assert (tmp_path / "a.pcd").read_bytes() == (tmp_path / "b.pcd").read_bytes()
    with pytest.raises(B200RegError) as e:
        g.saveStaticMapPcd(tmp_path / "no" / "such" / "dir.pcd")
    assert e.value.code == -7
    assert info["n_points"] == sum(len(s) for s, _ in subs)


def test_other_outputs_unchanged_by_a_build(tmp_path, moving):
    from lidarslam_ros2_b200.scanmatcher import backend_registration

    subs = moving[0][:12]
    g = _session()
    _import(g, subs)
    reg = backend_registration("NDT", ndt_resolution=2.0)
    gate = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, range_of_searching_loop_closure=200.0, search_submap_num=1)
    occ = dict(resolution=0.1, z_min=0.3, z_max=2.5, max_range=100.0)

    def outputs(tag):
        cloud, offsets = g.assembleMap()
        g.saveMapPCDASCII(tmp_path / f"{tag}.pcd")
        g.buildOccupancyGrid(**occ)
        grid = g.occupancyGrid()
        return cloud, offsets, (tmp_path / f"{tag}.pcd").read_bytes(), grid, g.searchLoop(reg, **gate)

    a = outputs("a")
    _build(g, {})
    b = outputs("b")
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    for k in ("data", "hits", "frees"):
        assert np.array_equal(a[3][k], b[3][k])
    assert a[4]["id_min"] == b[4]["id_min"] and np.array_equal(a[4]["final"], b[4]["final"]) and a[4]["fitness"] == b[4]["fitness"]


def test_empty_and_all_skipped_maps(host):  # noqa: F811
    """Submaps whose every point is skipped: no box, no voxel, the static map is the whole map."""
    from lidarslam_ros2_b200 import synth

    subs = [(np.array([[np.nan, 0, 0], [500.0, 0, 0]], dtype=F32), synth.pose_matrix((0, 0, 0), (0, 0, 0))),
            (np.zeros((0, 3), dtype=F32), synth.pose_matrix((1, 0, 0), (0, 0, 0)))]
    g = _session()
    _import(g, subs)
    info = _build(g, {})
    assert info["n_voxels"] == 0 and info["n_static_points"] == 2 and info["n_batches"] == 0
    _check(g, host, subs, {}, info)
