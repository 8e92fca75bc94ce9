"""Kernel launches of the session's six map builds and of the read-backs that launch (mapVoxels, changeVoxels,
saveMapConsistencyPcd), counted by stats()["kernel_launches"]: each build's count follows from its info on small fixed
scenes, an empty and an all-skipped map among them, and on scenes whose walks take more than one batch. A change to a
build's host orchestration that adds, drops or repeats a launch shows here."""
import numpy as np
import pytest

F32 = np.float32
pytestmark = pytest.mark.gpu


def _session(submaps):
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)
    for k, (pts, P) in enumerate(submaps):
        q = np.zeros((len(pts), 4), dtype=F32)
        if len(pts):
            q[:, :3] = np.asarray(pts, dtype=F32)[:, :3]
        g.importSubmap(q, P, float(k))
    return g


def _pose(t, yaw):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix(t, (0.0, 0.0, yaw))


def _small():
    """Three submaps of points on a few walls and the ground, and an empty one."""
    rng = np.random.default_rng(5)
    subs = []
    for k, n in enumerate((1500, 0, 2500, 40)):
        p = np.zeros((n, 3), dtype=F32)
        p[:, 0] = rng.uniform(-6, 6, size=n)
        p[:, 1] = rng.choice([-4.0, 4.0], size=n) + rng.normal(0, 0.01, size=n)
        p[:, 2] = rng.uniform(-1.0, 1.5, size=n)
        p[: n // 3, 1] = rng.uniform(-4, 4, size=n // 3)
        p[: n // 3, 2] = -1.0
        subs.append((p, _pose((0.7 * k, 0.2 * k, 0.0), 0.1 * k)))
    return subs


def _skipped():
    """Every point non-finite, and an empty submap."""
    nan = np.array([[np.nan, 0, 0], [0, np.inf, 0]], dtype=F32)
    return [(nan, _pose((0, 0, 0), 0)), (np.zeros((0, 3), dtype=F32), _pose((1, 0, 0), 0))]


def _empty():
    return [(np.zeros((0, 3), dtype=F32), _pose((0, 0, 0), 0)), (np.zeros((0, 3), dtype=F32), _pose((2, 1, 0), 0))]


SCENES = dict(small=_small, skipped=_skipped, empty=_empty)


def _delta(g, call):
    before = g.stats()["kernel_launches"]
    out = call()
    return out, g.stats()["kernel_launches"] - before


def _entries(subs):
    return int(any(len(p) for p, _ in subs))


def _occupancy(g, subs, **kw):
    info, n = _delta(g, lambda: g.buildOccupancyGrid(**kw))
    assert n == _entries(subs) + 2 * info["n_batches"] + 1, info
    return info


def _static(g, subs, **kw):
    info, n = _delta(g, lambda: g.buildStaticMap(**kw))
    e = _entries(subs)
    assert n == (e + 3 * (info["n_rays"] > 0) + 2 * info["n_batches"] + (info["n_voxels"] > 0) + 3 * e
                 + (info["n_static_points"] > 0)), info
    _, n = _delta(g, g.mapVoxels)
    assert n == (info["n_voxels"] > 0)
    return info


def _changes(g, subs, split, **kw):
    info, n = _delta(g, lambda: g.buildMapChanges(split_submap=split, **kw))
    e = _entries(subs)
    assert n == (e + 3 * (info["n_rays"] > 0) + 2 * info["n_batches"] + (info["n_voxels"] > 0) + 3 * e
                 + (info["n_updated_points"] > 0)), info
    _, n = _delta(g, g.changeVoxels)
    assert n == (info["n_voxels"] > 0)
    return info


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_build_launches(scene, tmp_path):
    subs = SCENES[scene]()
    g = _session(subs)
    e = _entries(subs)
    _occupancy(g, subs, resolution=0.1)
    if scene == "small":
        info, n = _delta(g, lambda: g.buildElevationMap())
        assert n == 4, info
    _static(g, subs)
    _changes(g, subs, 1)
    info, n = _delta(g, lambda: g.buildMesh())
    assert n == e + 3 * (info["n_rays"] > 0) + 8 * (info["n_band_voxels"] > 0) + (info["n_faces"] > 0), info
    if scene == "small":
        assert info["n_faces"] > 0
    # consistency: K19a, K19b and its scan, the cell counts, chunks and voxel list, the scatter, K19c; as on the parent
    info, n = _delta(g, lambda: g.buildMapConsistency())
    assert n == dict(small=15, skipped=2, empty=0)[scene], info
    if info["n_points"]:
        # the map assembled at the build's poses, its intensity replaced, then the writer of saveMapPCDASCII
        _, n_map = _delta(g, lambda: g.saveMapPCDASCII(tmp_path / "map.pcd"))
        _, n = _delta(g, lambda: g.saveMapConsistencyPcd(tmp_path / "consistency.pcd"))
        assert n == n_map + 1


def test_several_walk_batches():
    """Occupancy: 40 submaps whose 70 m rays at 0.05 m give windows of some 2 800 cells square, about 0.5 Mi words of
    bitmaps each, so the 16 Mi-word scratch takes two batches. Static map and map changes: one submap of 2 Mi scattered
    points at 0.05 m makes some 2 Mi occupied voxels, so a batch holds about 130 submaps and 150 take two."""
    rng = np.random.default_rng(11)
    ring = np.array([[70.0, 0, 1.0], [-70.0, 0, 1.0], [0, 70.0, 1.0], [0, -70.0, 1.0]], dtype=F32)
    subs = [(ring + rng.normal(0, 0.5, size=ring.shape).astype(F32), _pose((rng.uniform(-3, 3), rng.uniform(-3, 3), 0.0), 0.0))
            for _ in range(40)]
    g = _session(subs)
    info = _occupancy(g, subs, resolution=0.05)
    assert info["n_batches"] > 1, info

    big = np.empty((2 << 20, 3), dtype=F32)
    big[:, :2] = rng.uniform(-20, 20, size=(len(big), 2))
    big[:, 2] = rng.uniform(-2, 2, size=len(big))
    subs = [(big, _pose((0.0, 0.0, 1.0), 0.0))]
    for _ in range(150):
        pts = rng.uniform(-15, 15, size=(8, 3)).astype(F32)
        pts[:, 2] = rng.uniform(-2, 1, size=8)
        subs.append((pts, _pose((rng.uniform(-5, 5), rng.uniform(-5, 5), 1.0), rng.uniform(0, 6.28))))
    g = _session(subs)
    p = dict(resolution=0.05, min_frees=1, dynamic_thresh=0.5)
    info = _static(g, subs, **p)
    assert info["n_batches"] > 1, info
    info = _changes(g, subs, 75, **p)
    assert info["n_batches"] > 1, info
