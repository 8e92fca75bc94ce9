"""The OctoMap of the scan-matcher session (b200sm_build_octomap, K22 in csrc/octomap.cu) on the GPU: the info, the box's
voxel states and the .bt bytes bitwise the serial host compile of csrc/octomap.hpp (tests/hostmath/octomap_host.cpp) on
the hand-built rays, random submaps, caller poses, repeated builds, a build of several walk batches and the moving-object
drive (whose cars are FREE); the OCCUPIED voxels equal to the static map's non-dynamic voxels; the saved file decoded back
into the state grid leaf by leaf; refused calls change nothing; the other products are unchanged by a build; and the
build's kernel launches follow from its info."""
import numpy as np
import pytest

import octomapref as R
import staticmapref as SR
from test_octomap_cpu import CASES, host  # noqa: F401 (fixture)

F32 = np.float32
pytestmark = pytest.mark.gpu


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
    return g.buildOctoMap(poses=poses, **SR.params(**(p or {})))


def _check(g, host, submaps, p, info):  # noqa: F811
    want = host.build(submaps, p)
    assert isinstance(want, dict), want
    for k, w in (("n_rays", "n_rays"), ("n_skipped", "n_skipped"), ("n_occupied_voxels", "n_occupied"),
                 ("n_dynamic_voxels", "n_dynamic"), ("n_free_voxels", "n_free"), ("n_inner_nodes", "inner"),
                 ("n_occupied_leaves", "occupied_leaves"), ("n_free_leaves", "free_leaves"), ("tree_size", "size")):
        assert info[k] == want[w], k
    if want["n_rays"]:
        assert info["box_origin"] == want["lo"] and info["box_dims"] == want["dims"]
    st = g.octoMapStates()
    assert np.array_equal(st["states"], want["states"])
    data = g.octoMapBytes()
    assert data == want["bytes"] and info["n_bytes"] == len(data)
    return want


@pytest.mark.parametrize("name,subs,p", CASES, ids=[c[0] for c in CASES])
def test_hand_built_bitwise_host(host, name, subs, p):  # noqa: F811
    g = _session()
    _import(g, subs)
    _check(g, host, subs, p, _build(g, p))


def _random_submap(seed, n, reach=40.0):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), dtype=F32)
    p[:, 0:2] = rng.uniform(-reach, reach, size=(n, 2))
    p[:, 2] = rng.uniform(-3.0, 5.0, size=n)
    if n > 10:
        p[3::97, 0] = np.nan
        p[7::11, :3] *= 0.3
    return p


def test_random_submaps_repeated_builds_bitwise_host(host):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sizes = [0, 1, 31, 1000, 4097, 1 << 17]
    subs = [(_random_submap(10 + k, n), synth.pose_matrix((3.0 * k - 7.3, -2.1 * k, 1.0 + 0.1 * k), (0.01 * k, -0.02, 0.9 * k)))
            for k, n in enumerate(sizes)]
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.5, max_range=70.0, sensor_origin=(0.2, -0.1, 0.3), min_frees=1, dynamic_thresh=0.5)
    first = _build(g, p)
    want = _check(g, host, subs, p, first)
    assert first["n_dynamic_voxels"] > 0 and first["n_free_leaves"] > 0 and first["n_occupied_leaves"] > 0
    # another build at other parameters, then the first again: the same bytes
    _check(g, host, subs, dict(p, resolution=0.25), _build(g, dict(p, resolution=0.25)))
    assert _build(g, p) == first and g.octoMapBytes() == want["bytes"]
    # the OCCUPIED voxels are the static map's non-dynamic voxels
    g.buildStaticMap(**SR.params(**p))
    vox = g.mapVoxels()
    lo = np.array(first["box_origin"])
    ijk = np.argwhere(g.octoMapStates()["states"] == R.OCCUPIED)[:, ::-1] + lo
    keep = vox["ijk"][~vox["dynamic"]]
    assert np.array_equal(np.array(sorted(map(tuple, ijk))), np.array(sorted(map(tuple, keep))))


@pytest.fixture(scope="module")
def moving():
    import staticscene

    scans, poses, labels = staticscene.drive()
    return list(zip(scans, poses)), labels


def test_moving_drive_cars_are_free(host, moving, tmp_path):  # noqa: F811
    import staticscene

    subs, labels = moving
    g = _session()
    _import(g, subs)
    info = _build(g, {})
    _check(g, host, subs, {}, info)
    # the voxels of the points the static map removes (the cars') are FREE
    g.buildStaticMap()
    vox = g.mapVoxels()
    st = g.octoMapStates()
    dyn = vox["ijk"][vox["dynamic"]] - np.array(st["box_origin"])
    assert len(dyn) > 0 and (st["states"][dyn[:, 2], dyn[:, 1], dyn[:, 0]] == R.FREE).all()
    assert info["n_dynamic_voxels"] == len(dyn)
    # the saved file decodes back into the state grid, leaf by leaf
    n = g.saveOctoMapBt(tmp_path / "map.bt")
    data = (tmp_path / "map.bt").read_bytes()
    assert n == len(data) and data == g.octoMapBytes()
    res, size, leaves = R.decode(data)
    assert res == 0.2 and size == info["tree_size"]
    assert np.array_equal(R.expand(leaves, info["box_origin"], info["box_dims"]), st["states"])
    del staticscene


def test_caller_poses_equal_imported_poses(host, moving):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sub = moving[0][:10]
    moved = [P @ synth.pose_matrix((0.3 * k, -0.2, 0.05), (0.0, 0.01, 0.02 * k)) for k, (_, P) in enumerate(sub)]
    a = _session()
    _import(a, sub)
    ia = _build(a, {}, poses=np.array(moved))
    b = _session()
    _import(b, [(s, P) for (s, _), P in zip(sub, moved)])
    assert ia == _build(b, {})
    assert a.octoMapBytes() == b.octoMapBytes()
    _check(a, host, [(s, P) for (s, _), P in zip(sub, moved)], {}, ia)


def test_several_batches_bitwise_host(host):  # noqa: F811
    """As the static map's: 200 000 scattered occupied voxels at 0.05 m and 1 401 submaps take two walk batches."""
    from lidarslam_ros2_b200 import synth

    rng = np.random.default_rng(77)
    big = rng.uniform(-40, 40, size=(200000, 3)).astype(F32)
    big[:, 2] = rng.uniform(-2, 2, size=200000)
    subs = [(big, synth.pose_matrix((0.0, 0.0, 1.0), (0.0, 0.0, 0.0)))]
    for _ in range(1400):
        pts = rng.uniform(-30, 30, size=(8, 3)).astype(F32)
        pts[:, 2] = rng.uniform(-2, 1, size=8)
        subs.append((pts, synth.pose_matrix((rng.uniform(-5, 5), rng.uniform(-5, 5), 1.0), (0.0, 0.0, rng.uniform(0, 6.28)))))
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.05, max_range=100.0, min_frees=1, dynamic_thresh=0.5)
    before = g.stats()["kernel_launches"]
    info = _build(g, p)
    assert info["n_batches"] > 1, info
    # K15a, the rank pass, the walk batches, K15e, K22a, K22b, K22c x 15, K22d x 15, K22e
    assert g.stats()["kernel_launches"] - before == 1 + 3 + 2 * info["n_batches"] + 3 + 30 + 1
    _check(g, host, subs, p, info)


def test_launches_follow_from_the_info(moving):
    g = _session()
    with_rays = moving[0][:3]
    _import(g, with_rays + [(np.full((2, 3), np.nan, dtype=F32), with_rays[0][1])])
    before = g.stats()["kernel_launches"]
    info = _build(g, {})
    assert g.stats()["kernel_launches"] - before == 1 + 3 + 2 * info["n_batches"] + 3 + 30 + 1
    for call in (g.octoMapStates, g.octoMapBytes):
        before = g.stats()["kernel_launches"]
        call()
        assert g.stats()["kernel_launches"] == before
    skipped = _session()
    _import(skipped, [(np.full((3, 3), np.nan, dtype=F32), with_rays[0][1])])
    before = skipped.stats()["kernel_launches"]
    info = _build(skipped, {})
    assert skipped.stats()["kernel_launches"] - before == 1 and info["tree_size"] == 0 and info["n_batches"] == 0


def test_refused_calls_change_nothing(tmp_path, moving):
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    with pytest.raises(B200RegError) as e:
        g.buildOctoMap()
    assert e.value.code == -1
    subs = moving[0][:4]
    _import(g, subs)
    for call in (g.octoMapStates, g.octoMapBytes, lambda: g.saveOctoMapBt(tmp_path / "x.bt")):
        with pytest.raises(B200RegError) as e:
            call()
        assert e.value.code == -1
    assert not (tmp_path / "x.bt").exists()
    _build(g, {})
    states, data = g.octoMapStates()["states"], g.octoMapBytes()
    far = [P.copy() for _, P in subs]  # a box beyond 2^31 - 1 voxels
    far[3][:3, 3] += (20000.0, 20000.0, 20000.0)
    wide = [P.copy() for _, P in subs]  # a box within 2^31 - 1 voxels but beyond the 16-bit keys
    wide[3][0, 3] += 7000.0
    for p, poses, what in ((dict(resolution=0.1000001), None, "printf"), (dict(resolution=0.02), np.array(far), "2^31"),
                           (dict(resolution=0.2), np.array(wide), "key"), (dict(resolution=0.0), None, "resolution")):
        with pytest.raises(B200RegError) as e:
            _build(g, p, poses=poses)
        assert e.value.code == -1 and what in str(e.value), (p, str(e.value))
    assert np.array_equal(g.octoMapStates()["states"], states) and g.octoMapBytes() == data
    with pytest.raises(B200RegError) as e:
        g.saveOctoMapBt(tmp_path / "no" / "such" / "dir.bt")
    assert e.value.code == -7
    # an empty tree is kept, readable, and not saved
    empty = _session()
    _import(empty, [(np.full((2, 3), np.nan, dtype=F32), subs[0][1])])
    assert _build(empty, {})["tree_size"] == 0
    assert empty.octoMapBytes().endswith(b"size 0\nres 0.2\ndata\n")
    with pytest.raises(B200RegError) as e:
        empty.saveOctoMapBt(tmp_path / "empty.bt")
    assert e.value.code == -1 and not (tmp_path / "empty.bt").exists()


def test_other_outputs_unchanged_by_a_build(tmp_path, moving):
    from lidarslam_ros2_b200.scanmatcher import backend_registration

    subs = moving[0][:12]
    g = _session()
    _import(g, subs)
    reg = backend_registration("NDT", ndt_resolution=2.0)
    gate = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, range_of_searching_loop_closure=200.0, search_submap_num=1)
    g.buildStaticMap()
    g.buildMapChanges(split_submap=6)
    g.buildMesh()

    def outputs(tag):
        g.saveMapPCDASCII(tmp_path / f"{tag}.pcd")
        vox = g.mapVoxels()
        return (g.staticMap()[0], vox["hits"], vox["frees"], vox["dynamic"], g.updatedMap()[0], g.changeVoxels()["label"],
                g.mesh()[0], g.mesh()[1], (tmp_path / f"{tag}.pcd").read_bytes(), g.searchLoop(reg, **gate)["final"])

    a = outputs("a")
    _build(g, dict(resolution=0.25, min_frees=1))
    b = outputs("b")
    for x, y in zip(a, b):
        if isinstance(x, bytes):
            assert x == y
        else:
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
