"""Relocalisation anywhere in the prior map (b200sm_relocalize, K17 of csrc/relocalize.cu) on the H100: the pyramid, node
scores (out-of-grid ones included), per-level node counts, T and candidates bitwise the host compile of
csrc/relocalize.hpp (tests/test_relocalize_cpu.py) on hand-built and random maps and on the canyon; num_levels = 1 (the
exhaustive search, every cell its own tile) equal to the host's definition and giving the default's first candidate; every
refined row bitwise the plain calls and the adoption rule; the next frame that of a fresh session at the adopted pose; NDT
and GICP; recovery from a far start with the heading wrong on every fixture frame; and the error paths, the limits that
depend on yaw_steps included on a pyramid built for fewer headings. Run with -m gpu."""
import math

import numpy as np
import pytest

import globalref as GR
import localizeref as L
import relocref as R
import test_gpu_localize as TL
import test_relocalize_cpu as RC
from lidarslam_ros2_b200 import synth, voxel_grid_filter

pytestmark = pytest.mark.gpu

F32 = np.float32
FAR = ((-40.0, 3.0), math.radians(120.0))  # the start: metres down the canyon and the heading wrong


@pytest.fixture(scope="module")
def sm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


@pytest.fixture(scope="module")
def world():
    return TL.canyon_map(), TL.drive(6)


@pytest.fixture(scope="module")
def rl(tmp_path_factory):
    return RC.build_host_lib(tmp_path_factory.mktemp("rlg"))


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _start(T_true, offset, dyaw):
    yaw = math.atan2(float(T_true[1, 0]), float(T_true[0, 0])) + dyaw
    pos = [float(T_true[0, 3]) + offset[0], float(T_true[1, 3]) + offset[1], float(T_true[2, 3])]
    return pos, (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))


def _kw(p):
    return {k: p[k] for k in R.DEFAULTS}


def _against_host(rl, g, prior, pos, quat, p, best, rows, info):
    """the session's search against the host compile on the session's own filtered scan"""
    host = RC.Host(rl, prior, p)
    assert not host.refused
    scan = g.filteredScan()
    assert host.set_scan(scan, pos, quat) == info["m"]
    want = host.search()
    if host.grid is None:
        assert info["width"] == 0 and rows == []
        return host, want
    assert (info["width"], info["height"], info["origin_cell"]) == (host.grid["W"], host.grid["H"], (host.grid["i0"], host.grid["j0"]))
    for h in range(p["num_levels"]):
        assert np.array_equal(g.relocalizeGrid(h), host.level(h)), h
    if info["m"]:
        rng = np.random.default_rng(5)
        for h in range(p["num_levels"]):
            nodes = RC._probe_nodes(dict(W=host.grid["W"], H=host.grid["H"]), p["yaw_steps"], rng, 200)
            assert np.array_equal(g.relocalizeScoreNodes(h, nodes), host.scores(h, nodes)), h
    assert (info["t0"], info["t"], info["nodes"]) == (want["t0"], want["t"], want["nodes"])
    assert len(rows) == len(want["tiles"])
    W, H = host.grid["W"], host.grid["H"]
    for r, key in zip(rows, want["keys"]):
        idx = R.key_index(key)
        assert (r["yaw_index"], r["cell"], r["score"]) == (idx // (W * H), (idx % W, (idx // W) % H), key >> 40)
        assert np.array_equal(_bits(r["guess"]), _bits(host.guess(r["yaw_index"], *r["cell"])))
    return host, want


def _session(sm, prior, method="NDT", **kw):
    g = TL._session(sm, prior, method, **kw)
    return g


# ---- 1. hand cases and random maps against the host compile ------------------------------------------------------------
def test_hand_and_random_maps_equal_host(sm, rl):
    cases = [(c[1], c[2], c[3], RC._yaw_quat(c[4]), c[5]) for c in RC.HAND] + [RC._random_case(s) for s in range(0, 200, 4)]
    checked = 0
    for m, s, pos, quat, p in cases:
        g = _session(sm, m, use_min_max_filter=False, vg_size_for_input=0.01)
        g.setInitialPose(pos, quat)
        best, rows, info = g.relocalize(s, **_kw(p))
        _against_host(rl, g, m, pos, quat, p, best, rows, info)
        checked += info["m"] > 0 and info["width"] > 0
    assert checked > 40


# ---- 2. the canyon: the search, the exhaustive search, the refinement -----------------------------------------------------
@pytest.mark.parametrize("method", ["NDT", "GICP"])
def test_canyon_rows_are_the_plain_calls(sm, rl, world, method):
    prior, frames = world
    scan, T_true = frames[2]
    pos, quat = _start(T_true, *FAR)
    p = dict(R.DEFAULTS)
    g = _session(sm, prior, method)
    g.setInitialPose(pos, quat)
    best, rows, info = g.relocalize(scan)
    host, want = _against_host(rl, g, prior, pos, quat, p, best, rows, info)
    assert len(rows) == p["top_k"] and info["search_ms"] > 0
    print(f"\n{method}: grid {info['width']} x {info['height']}, m {info['m']}, T0 {info['t0']}, T {info['t']}, "
          f"nodes {info['nodes'][:p['num_levels']]}, search {info['search_ms']:.3f} ms, rows "
          f"{[(r['score'], round(r['fitness'], 4), r['converged']) for r in rows]}, best {best}")
    # every row: setInputTarget(cut around the row) / setInputSource(filtered) / align(guess) / getFitnessScore()
    filtered = g.filteredScan()
    plain = TL._plain(sm, method)
    for r in rows:
        cx = (info["origin_cell"][0] + r["cell"][0]) * p["resolution"]
        cy = (info["origin_cell"][1] + r["cell"][1]) * p["resolution"]
        cut = TL._cut_of(sm, prior, (cx, cy), TL.CROP, scan)
        plain.setInputTarget(voxel_grid_filter(cut, TL.KW["vg_size_for_input"]) if method == "GICP" else cut)
        plain.setInputSource(filtered)
        final = plain.align(r["guess"])
        assert np.array_equal(_bits(r["final"]), _bits(final))
        assert r["fitness"] == plain.getFitnessScore() and r["converged"] == plain.hasConverged() and r["status"] == 0
    ok = [k for k, r in enumerate(rows) if r["status"] == 0 and r["converged"] and r["fitness"] < p["accept_fitness"]]
    want_best = min(ok, key=lambda k: (rows[k]["fitness"], k)) if ok else -1
    assert best == want_best >= 0
    # the exhaustive search (num_levels = 1: every leaf scored, every cell its own tile) is the host's definition, and its
    # first row is the best leaf of the whole map, the default search's first row
    g1 = _session(sm, prior, method)
    g1.setInitialPose(pos, quat)
    b1, rows1, info1 = g1.relocalize(scan, num_levels=1)
    _against_host(rl, g1, prior, pos, quat, dict(p, num_levels=1), b1, rows1, info1)
    assert (rows1[0]["yaw_index"], rows1[0]["cell"], rows1[0]["score"]) == (rows[0]["yaw_index"], rows[0]["cell"], rows[0]["score"])
    assert info1["nodes"][0] == info1["leaves"] == 360 * info["width"] * info["height"]
    print(f"exhaustive: {info1['leaves']} leaves in {info1['search_ms']:.3f} ms")


def test_next_frame_equals_fresh_session_bitwise(sm, world):
    prior, frames = world
    scan, T_true = frames[2]
    pos, quat = _start(T_true, *FAR)
    g = _session(sm, prior)
    g.setInitialPose(pos, quat)
    best, rows, _ = g.relocalize(scan)
    assert best >= 0
    # the next frame: the cut around the adopted pose, registered from it (localizeref's pose bookkeeping)
    loc = L.Localizer(prior, TL.CROP, 1e9, position=pos, quat_xyzw=quat)
    assert loc.begin()
    loc.adopt_pose(rows[best]["final"])
    g.setLocalizationParams(TL.CROP, 1e9)
    _, final, _ = g.localizeCloud(frames[3][0])
    st = g.localizeStats()
    assert np.allclose(st["cut_centre"], loc.position[:2], rtol=0, atol=0)
    plain = TL._plain(sm, "NDT")
    plain.setInputTarget(g.cutCloud())
    plain.setInputSource(g.filteredScan())
    assert np.array_equal(_bits(final), _bits(plain.align(loc.sim_trans())))


# ---- 3. recovery from a far start on every fixture frame ---------------------------------------------------------------
def test_recovery_on_every_frame(sm, world):
    prior, frames = world
    for f, (scan, T_true) in enumerate(frames):
        pos, quat = _start(T_true, *FAR)
        g = _session(sm, prior)
        g.setInitialPose(pos, quat)
        best, rows, info = g.relocalize(scan)
        assert best >= 0, f
        dt, dr = synth.pose_error(rows[best]["final"], T_true)
        print(f"\nframe {f}: best {best}, dt {dt:.4f} m, dr {dr:.5f} rad, search {info['search_ms']:.3f} ms")
        assert dt < 0.3 and dr < 0.02, (f, dt, dr)


# ---- 4. errors, limits and the pyramid's lifetime -------------------------------------------------------------------------
def test_errors_limits_and_rebuilds(sm, world):
    from lidarslam_ros2_b200.registration import B200RegError

    prior, frames = world
    scan, T_true = frames[2]
    E = sm._capi
    pos, quat = _start(T_true, (0.5, -0.5), 0.0)
    g = _session(sm, None)
    g.setInitialPose(pos, quat)
    with pytest.raises(B200RegError) as e:
        g.relocalize(scan)
    assert e.value.code == E.ERR_NO_TARGET
    g.setPriorMap(prior)
    g.localizeCloud(scan)
    g.setInitialPose(pos, quat)
    g.localizeCloud(scan)
    g.setInitialPose(pos, quat)
    cut0, st0, n_t0 = g.cutCloud(), g.localizeStats(), g.registration.stats()["n_target"]

    def pose_is(p, q):  # through a radius-0 global search, whose only hypothesis is the pose (it adopts a pose)
        g.localizeGlobal(scan, 0.0, 1.0, 1, 1)
        return np.array_equal(_bits(g.globalSearch()[0]), _bits(GR.grid(p, q, 0.0, 1.0, 1)))

    for bad in (dict(resolution=0.0), dict(resolution=math.nan), dict(z_min=3.0, z_max=3.0), dict(yaw_steps=0),
                dict(yaw_steps=4097), dict(num_levels=0), dict(num_levels=17), dict(min_score=1.5), dict(top_k=0),
                dict(top_k=65), dict(accept_fitness=0.0),
                dict(resolution=0.001),                     # W * H over 2^28 cells
                dict(resolution=0.01, num_levels=16),       # the pyramid over 2^32 bytes
                dict(resolution=0.1, yaw_steps=4096, num_levels=1)):  # over 2^32 roots
        with pytest.raises(B200RegError) as e:
            g.relocalize(scan, **bad)
        assert e.value.code == E.ERR_ARG, bad
        assert np.array_equal(_bits(g.cutCloud()), _bits(cut0)) and g.localizeStats() == st0, bad
        assert g.registration.stats()["n_target"] == n_t0, bad
    assert pose_is(pos, quat)
    # the limits that depend on the headings are checked by every search, also on a pyramid built for fewer headings:
    # 0.1 m with one level is 8 x 1.1 M roots, fine; 4096 headings would be 4.5e9 roots
    _, _, ib = g.relocalize(scan, resolution=0.1, num_levels=1, yaw_steps=8)
    g.setInitialPose(pos, quat)
    cut1, st1, n_t1 = g.cutCloud(), g.localizeStats(), g.registration.stats()["n_target"]
    with pytest.raises(B200RegError) as e:
        g.relocalize(scan, resolution=0.1, num_levels=1, yaw_steps=4096)
    assert e.value.code == E.ERR_ARG and "roots" in str(e.value)
    assert np.array_equal(_bits(g.cutCloud()), _bits(cut1)) and g.localizeStats() == st1
    assert g.registration.stats()["n_target"] == n_t1 and pose_is(pos, quat)
    _, _, ic = g.relocalize(scan, resolution=0.1, num_levels=1, yaw_steps=8)
    assert ic["pyramid_builds"] == ib["pyramid_builds"]  # the refused call neither rebuilt nor dropped the pyramid
    g.setInitialPose(pos, quat)
    # the pyramid: built once, rebuilt after a parameter change or a new prior map
    _, _, i1 = g.relocalize(scan, yaw_steps=8)
    _, _, i2 = g.relocalize(scan, yaw_steps=16)
    assert i2["pyramid_builds"] == i1["pyramid_builds"]
    _, _, i3 = g.relocalize(scan, yaw_steps=8, resolution=0.5)
    assert i3["pyramid_builds"] == i2["pyramid_builds"] + 1
    g.setPriorMap(prior)
    _, _, i4 = g.relocalize(scan, yaw_steps=8, resolution=0.5)
    assert i4["pyramid_builds"] == i3["pyramid_builds"] + 1
    # no map row in the band: no rows, best -1, the pose unchanged
    g.setInitialPose(pos, quat)
    best, rows, info = g.relocalize(scan, z_min=500.0, z_max=501.0)
    assert best == -1 and rows == [] and info["width"] == 0 and pose_is(pos, quat)
