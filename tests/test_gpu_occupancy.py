"""The occupancy grid of the scan-matcher session (b200sm_build_occupancy_grid, K14 in csrc/occupancy.cu) on the GPU: hits,
frees, values and both map_server files bitwise / byte-equal to the serial host compile of csrc/occupancy_grid.hpp
(tests/hostmath/occupancy_host.cpp) on the hand-built rays, random submaps of 0 to 2^20 points, the ray-cast canyon drive,
a build that takes several walk batches, caller poses and repeated builds; refused calls change nothing; and the map
assembly, the PCD save and the loop search give what they gave before a build."""
import math

import numpy as np
import pytest

import occupancyref as R
from test_occupancy_cpu import cases, host  # noqa: F401 (fixture)

F32 = np.float32
pytestmark = pytest.mark.gpu
DRIVE = dict(resolution=0.1, z_min=0.3, z_max=2.5, max_range=100.0)


def _session():
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    return ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3)


def _import(g, submaps):
    for k, (pts, P) in enumerate(submaps):
        g.importSubmap(np.asarray(pts, dtype=F32), P, float(k))


def _build(g, p, poses=None):
    q = R.params(**p)
    return g.buildOccupancyGrid(poses=poses, resolution=q["resolution"], z_min=q["z_min"], z_max=q["z_max"],
                                max_range=q["max_range"], sensor_origin=q["sensor_origin"],
                                occupied_thresh=q["occupied_thresh"], free_thresh=q["free_thresh"])


def _check(g, host, submaps, p, tmp_path, info):  # noqa: F811
    """The session's last grid and files against the host compile of the same submaps."""
    want = host.build(submaps, p)
    assert isinstance(want, dict), want
    got = g.occupancyGrid()
    assert (info["width"], info["height"]) == (want["width"], want["height"])
    assert info["origin"] == want["origin"] and info["resolution"] == R.params(**p)["resolution"]
    for k in ("n_rays", "n_skipped", "n_occupied", "n_free", "n_unknown"):
        assert info[k] == want[k], k
    assert np.array_equal(got["hits"], want["hits"]) and np.array_equal(got["frees"], want["frees"])
    assert np.array_equal(got["data"], want["values"])
    g.saveOccupancyMap(tmp_path / "gpu.pgm", tmp_path / "gpu.yaml")
    assert host.save(str(tmp_path / "gpu.pgm.host"), str(tmp_path / "host.yaml")) == 0
    assert (tmp_path / "gpu.pgm").read_bytes() == (tmp_path / "gpu.pgm.host").read_bytes()
    assert (tmp_path / "gpu.yaml").read_text() == (tmp_path / "host.yaml").read_text().replace("gpu.pgm.host", "gpu.pgm")
    return got


@pytest.mark.parametrize("name,subs,p", cases(), ids=[c[0] for c in cases()])
def test_hand_built_bitwise_host(host, tmp_path, name, subs, p):  # noqa: F811
    g = _session()
    _import(g, subs)
    info = _build(g, p)
    _check(g, host, subs, p, tmp_path, info)
    assert info["n_batches"] == 1


def _random_submap(seed, n, reach=70.0):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 4), dtype=F32)
    p[:, 0:2] = rng.uniform(-reach, reach, size=(n, 2))
    p[:, 2] = rng.uniform(-3.0, 5.0, size=n)
    p[:, 3] = rng.uniform(0, 255, size=n)
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
    p = dict(resolution=0.1, z_min=0.0, z_max=2.0, max_range=60.0, sensor_origin=(0.2, -0.1, 0.3))
    info = _build(g, p)
    _check(g, host, subs, p, tmp_path, info)
    assert info["n_skipped"] > 0 and info["n_rays"] > (1 << 19)


@pytest.fixture(scope="module")
def drive():
    import scancontextref as SC

    scans, poses, _ = SC.drive()
    return [(s, P) for s, P in zip(scans, poses)]


def test_canyon_drive_bitwise_host(host, tmp_path, drive):  # noqa: F811
    g = _session()
    _import(g, drive)
    info = _build(g, DRIVE)
    _check(g, host, drive, DRIVE, tmp_path, info)
    # two builds in a row: the same bits
    first = g.occupancyGrid()
    again = _build(g, DRIVE)
    second = g.occupancyGrid()
    assert again == info
    for k in ("data", "hits", "frees"):
        assert np.array_equal(first[k], second[k])


def test_several_batches_bitwise_host(host, tmp_path):  # noqa: F811
    """24 submaps whose windows span 200 m at 0.05 m: 4 MB of bitmaps each, more than the 64 MiB batch budget holds, so the
    walks run in several batches; the grid is the host compile's, which folds all submaps in one pass."""
    from lidarslam_ros2_b200 import synth

    subs = []
    for k in range(24):
        rng = np.random.default_rng(500 + k)
        n = 3000
        a = rng.uniform(0, 2 * math.pi, size=n)
        r = np.where(np.arange(n) < 64, 99.5, rng.uniform(1.0, 99.0, size=n))
        pts = np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-2.0, 1.0, size=n)], axis=1).astype(F32)
        subs.append((pts, synth.pose_matrix((2.5 * k, 0.7 * k, 1.5), (0.0, 0.0, 0.3 * k))))
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.05, z_min=0.2, z_max=2.0, max_range=100.0)
    info = _build(g, p)
    assert info["n_batches"] > 1
    _check(g, host, subs, p, tmp_path, info)
    # the host compile folds every submap in one pass: the batched device build is its bitwise equal (checked above)


def test_many_submaps_on_a_small_grid_bitwise_host(host, tmp_path):  # noqa: F811
    """100 submaps inside one 60 m room at 0.05 m, on a fresh session: every window covers most of a 1.4 M-cell grid, so
    one batch holds the bitmaps of all of them (about 9 M words, six times two bits per grid cell). The scratch must be
    sized to that batch, not to the grid."""
    from lidarslam_ros2_b200 import synth

    subs = []
    for k in range(100):
        rng = np.random.default_rng(900 + k)
        c = np.array([rng.uniform(-20, 20), rng.uniform(-20, 20)])
        n = 2000
        wall = rng.integers(0, 4, size=n)
        t = rng.uniform(-30.0, 30.0, size=n)
        xy = np.stack([np.where(wall == 0, -30.0, np.where(wall == 1, 30.0, t)),
                       np.where(wall == 2, -30.0, np.where(wall == 3, 30.0, t))], axis=1)
        xy[:100] = rng.uniform(-29.0, 29.0, size=(100, 2))  # furniture inside the room
        z = rng.uniform(-1.0, 1.0, size=n)
        P = synth.pose_matrix((c[0], c[1], 1.2), (0.0, 0.0, 0.0))
        pts = np.concatenate([xy - c, z[:, None]], axis=1).astype(F32)
        subs.append((pts, P))
    g = _session()
    _import(g, subs)
    p = dict(resolution=0.05, z_min=0.2, z_max=2.0, max_range=100.0)
    info = _build(g, p)
    cells = info["width"] * info["height"]
    window_words = 2 * ((info["width"] + 31) // 32) * info["height"]
    assert cells < (8 << 20) and info["n_batches"] == 1 and 100 * window_words * 0.8 > 4 * cells  # > twice 2 words per cell
    _check(g, host, subs, p, tmp_path, info)


def test_caller_poses_equal_imported_poses(host, tmp_path, drive):  # noqa: F811
    from lidarslam_ros2_b200 import synth

    sub = drive[:8]
    moved = [P @ synth.pose_matrix((0.3 * k, -0.2, 0.05), (0.0, 0.01, 0.02 * k)) for k, (_, P) in enumerate(sub)]
    a = _session()
    _import(a, sub)
    ia = _build(a, DRIVE, poses=np.array(moved))
    b = _session()
    _import(b, [(s, P) for (s, _), P in zip(sub, moved)])
    ib = _build(b, DRIVE)
    assert ia == ib
    ga, gb = a.occupancyGrid(), b.occupancyGrid()
    for k in ("data", "hits", "frees"):
        assert np.array_equal(ga[k], gb[k])
    _check(a, host, [(s, P) for (s, _), P in zip(sub, moved)], DRIVE, tmp_path, ia)


def test_yaml_reads_back_bitwise(tmp_path, drive):
    import yaml

    g = _session()
    _import(g, drive[:4])
    info = _build(g, dict(DRIVE, resolution=0.07, occupied_thresh=0.7, free_thresh=0.196))
    g.saveOccupancyMap(tmp_path / "map.pgm", tmp_path / "map.yaml")
    y = yaml.safe_load((tmp_path / "map.yaml").read_text())
    assert y["image"] == "map.pgm" and y["mode"] == "trinary" and y["negate"] == 0
    assert np.float64(y["resolution"]).view(np.uint64) == np.float64(info["resolution"]).view(np.uint64)
    for k in (0, 1):
        assert np.float64(y["origin"][k]).view(np.uint64) == np.float64(info["origin"][k]).view(np.uint64)
    assert float(y["origin"][2]) == 0.0 and y["occupied_thresh"] == 0.7 and y["free_thresh"] == 0.196
    data = (tmp_path / "map.pgm").read_bytes()
    head = f"{info['width']} {info['height']}\n255\n".encode()
    assert data.startswith(b"P5\n# ") and data.index(head) + len(head) == len(data) - info["width"] * info["height"]


def test_refused_calls_change_nothing(tmp_path, drive):
    from lidarslam_ros2_b200.registration import B200RegError

    g = _session()
    with pytest.raises(B200RegError) as e:
        g.buildOccupancyGrid()
    assert e.value.code == -1  # no submaps
    _import(g, drive[:3])
    with pytest.raises(B200RegError) as e:
        g.saveOccupancyMap(tmp_path / "x.pgm", tmp_path / "x.yaml")
    assert e.value.code == -1 and not (tmp_path / "x.pgm").exists()  # no grid yet
    info = _build(g, DRIVE)
    before = g.occupancyGrid()
    g.saveOccupancyMap(tmp_path / "a.pgm", tmp_path / "a.yaml")
    bad = [dict(resolution=0.0), dict(resolution=-0.1), dict(z_min=3.0, z_max=3.0), dict(z_max=float("nan")),
           dict(max_range=0.0), dict(max_range=float("inf")), dict(resolution=0.01, max_range=200.0),
           dict(sensor_origin=(0.0, float("inf"), 0.0)), dict(occupied_thresh=0.2, free_thresh=0.2),
           dict(occupied_thresh=1.5), dict(free_thresh=-0.1)]
    for p in bad:
        with pytest.raises(B200RegError) as e:
            _build(g, dict(DRIVE, **p))
        assert e.value.code == -1, p
    with pytest.raises(B200RegError) as e:
        g.buildOccupancyGrid(poses=np.full((3, 4, 4), np.nan))
    assert e.value.code == -1
    # over the cell cap: a submap 30 km away at 0.05 m
    far = [P.copy() for _, P in drive[:3]]
    far[2][:3, 3] += (30000.0, 30000.0, 0.0)
    with pytest.raises(B200RegError) as e:
        _build(g, dict(DRIVE, resolution=0.05), poses=np.array(far))
    assert e.value.code == -1 and " x " in str(e.value) and "2^28" in str(e.value)
    # a sensor origin 10 km above the band
    high = [P.copy() for _, P in drive[:3]]
    high[0][2, 3] = 1e4
    with pytest.raises(B200RegError) as e:
        _build(g, dict(DRIVE, resolution=0.05), poses=np.array(high))
    assert e.value.code == -1
    after = g.occupancyGrid()
    for k in ("data", "hits", "frees"):
        assert np.array_equal(before[k], after[k])
    assert {k: after[k] for k in info} == info
    g.saveOccupancyMap(tmp_path / "b.pgm", tmp_path / "b.yaml")
    assert (tmp_path / "a.pgm").read_bytes() == (tmp_path / "b.pgm").read_bytes()
    assert (tmp_path / "a.yaml").read_text().replace("a.pgm", "b.pgm") == (tmp_path / "b.yaml").read_text()
    with pytest.raises(B200RegError) as e:
        g.saveOccupancyMap(tmp_path / "no" / "such" / "dir.pgm", tmp_path / "c.yaml")
    assert e.value.code == -7


def test_other_outputs_unchanged_by_a_build(tmp_path, drive):
    from lidarslam_ros2_b200.scanmatcher import backend_registration

    g = _session()
    _import(g, drive[:12])
    reg = backend_registration("NDT", ndt_resolution=2.0)
    gate = dict(voxel_leaf_size=0.3, distance_loop_closure=5.0, range_of_searching_loop_closure=200.0, search_submap_num=1)
    cloud, offsets = g.assembleMap()
    g.saveMapPCDASCII(tmp_path / "a.pcd")
    one = g.searchLoop(reg, **gate)
    _build(g, DRIVE)
    cloud2, offsets2 = g.assembleMap()
    g.saveMapPCDASCII(tmp_path / "b.pcd")
    one2 = g.searchLoop(reg, **gate)
    assert np.array_equal(cloud.view(np.uint32), cloud2.view(np.uint32)) and np.array_equal(offsets, offsets2)
    assert (tmp_path / "a.pcd").read_bytes() == (tmp_path / "b.pcd").read_bytes()
    assert one["id_min"] == one2["id_min"] and np.array_equal(one["final"], one2["final"]) and one["fitness"] == one2["fitness"]


def test_image_name_with_yaml_characters(host, tmp_path):  # noqa: F811
    """The session writes the image name as the host compile does: a double-quoted scalar that reads back as the name."""
    import yaml

    subs, p = cases()[0][1], cases()[0][2]
    g = _session()
    _import(g, subs)
    _build(g, p)
    host.build(subs, p)
    name = 'map: v2 #1 "a\\b".pgm'
    g.saveOccupancyMap(tmp_path / name, tmp_path / "gpu.yaml")
    assert host.save(str(tmp_path / name) + ".h", str(tmp_path / "host.yaml")) == 0
    gpu_text = (tmp_path / "gpu.yaml").read_text(encoding="utf-8")
    assert yaml.safe_load(gpu_text)["image"] == name
    assert gpu_text == R.yaml_text(R.build(subs, p), str(tmp_path / name))
    assert (tmp_path / name).read_bytes() == (tmp_path / (name + ".h")).read_bytes()
