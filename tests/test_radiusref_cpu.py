"""The float64 reference of the NDT radius paths (tests/radiusref.py) and its bounds, checked on the CPU before any GPU
comparison: against the oracle's radius Hessian and calculateScore (FLANN-style radius search over every centroid) entry by
entry; on the escape fixtures, where the oracle finds a voxel two lookup cells from the query that a 27-cell rule cannot
see; on the equality fixtures; and under mutations of the reference, each of which some check here must catch."""
import numpy as np
import pytest

import gridref as R
import ndtref as N
import radiusref as RR

F32 = np.float32
POSES = (np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02]), np.array([-0.4, 0.3, -0.1, 2.9, 0.01, -0.3]))
ESCAPES = [(leaf, axis, d, inside) for leaf in (0.3, 0.6) for axis in range(3) for d in (1, -1) for inside in (True, False)]


def _oracle(oracle_mod, src, tgt, res):
    o = oracle_mod.NDT(resolution=res)
    o.set_target(tgt)
    o.set_source(src)
    return o


def _scenes(golden, pair_tiny, pair_small):
    return {"tiny": (pair_tiny[0], pair_tiny[1], 2.0), "small": (pair_small[0], pair_small[1], 2.0),
            "golden": (golden["source"], golden["target"], 1.0)}


def _hessian_vs_oracle(o, src, res, p, **kw):
    T = o_pose(p)
    ref = RR.hessian(src, T[:3], p, res, o.voxels(), serial=True, **kw)
    return RR.within_h(o.hessian_radius(T, p), ref)[0], ref


def o_pose(p):
    import oracle

    return oracle.pose_to_matrix(p)


def test_hessian_matches_oracle(oracle_mod, golden, pair_tiny, pair_small):
    worst = {}
    for name, (src, tgt, res) in _scenes(golden, pair_tiny, pair_small).items():
        o = _oracle(oracle_mod, src, tgt, res)
        for p in POSES + tuple(N.pitch_poses()):
            w, ref = _hessian_vs_oracle(o, src, res, p)
            assert ref["near_threshold"] == 0 and ref["hits"] > 0, (name, p)
            assert w <= 1.0, (name, p, w)
            worst[name] = max(worst.get(name, 0.0), w)
    print("\nmax |oracle - ref| / bound, radius Hessian: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_score_matches_oracle(oracle_mod, golden, pair_tiny, pair_small):
    for name, (src, tgt, res) in _scenes(golden, pair_tiny, pair_small).items():
        o = _oracle(oracle_mod, src, tgt, res)
        for p in POSES[:2]:
            T = o_pose(p)
            ref = RR.score(N.transform_points(T[:3], src), res, o.voxels(), serial=True)
            assert ref["near_threshold"] == 0 and ref["hits"] > 0
            assert RR.within_score(o.calculate_score(T), ref) <= 1.0, (name, p)


def test_bounds_are_tight():
    """The Hessian bound is near 1e-12 of each entry's own size, not 1e-9 of the largest entry."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("small", 2.0)
    v = R.voxel_map_ref(tgt, 2.0)
    p = POSES[1]
    ref = RR.hessian(src, o_pose(p)[:3], p, 2.0, v)
    rel = np.array([ref["tol"][i, j] / abs(ref["H"][i, j]) for i, j in RR.TRI if abs(ref["H"][i, j]) > 1e-3 * np.abs(ref["H"]).max()])
    assert np.median(rel) < 1e-11 and rel.max() < 1e-9, rel


@pytest.mark.parametrize("leaf,axis,direction,inside", ESCAPES)
def test_escape_fixture_needs_every_centroid(oracle_mod, leaf, axis, direction, inside):
    tgt, q, cen, w, qq = RR.escape_fixture(leaf, axis, direction, inside)
    k = int(R.build_ref(np.array([w]), leaf)[0])
    assert int(R.lookup_ref(np.array([qq]), leaf)[0]) == k - 2 * direction
    o = _oracle(oracle_mod, q, tgt, leaf)
    v, geom = o.voxels(), R.leaf_geometry(tgt, leaf)
    if not inside:  # the query is two cells outside the grid
        assert geom["div_b"][axis] == 1 and int(R.lookup_ref(np.array([qq]), leaf)[0]) - geom["min_b"][axis] in (-2, 2)
    full = RR.score(q, leaf, v, serial=True)
    block = RR.score(q, leaf, v, rule="block27", geom=geom, serial=True)
    assert full["hits"] == 1 and block["hits"] == 0 and full["near_threshold"] == 0
    so = o.calculate_score(np.eye(4))
    assert so != 0 and RR.within_score(so, full) <= 1.0
    assert RR.within_score(so, block) > 1.0
    # the same query through the radius Hessian at the identity pose
    Ho = o.hessian_radius(np.eye(4, dtype=F32), np.zeros(6))
    ref = RR.hessian(q, np.eye(4, dtype=F32)[:3], np.zeros(6), leaf, v, serial=True)
    assert ref["hits"] == 1 and RR.within_h(Ho, ref)[0] <= 1.0 and np.abs(Ho).max() > 0
    # and the derivative reference's KDTREE rule
    assert N.per_point_hits(q, np.eye(4, dtype=F32)[:3], leaf, v, geom, N.KDTREE)[0] == 1


EQUALITY_WALLS = {1.0: (2.0, 0.5, 0.25), 0.3: (0.75, 0.45, 0.15)}  # (wall x, centre y, z) per resolution


def equality_case(res):
    x, y, z = (F32(c) for c in EQUALITY_WALLS[res])
    return RR.wall(0, x, (y, z), res), np.array([x, y, z], dtype=F32)


def test_equality_fixtures(oracle_mod):
    for res in EQUALITY_WALLS:
        tgt, cen = equality_case(res)
        qs = RR.equality_queries(res, cen)
        r2 = RR.radius2(res)
        assert len(qs) >= 2 and qs[0][1] < r2 <= qs[-1][1]
        if res == 1.0:
            assert any(d2 == r2 for _, d2 in qs)
        for qv, d2 in qs:
            o = _oracle(oracle_mod, qv[None, :], tgt, res)
            ref = RR.score(qv[None, :], res, o.voxels(), serial=True)
            assert ref["hits"] == int(d2 < r2), (res, d2)
            assert (o.calculate_score(np.eye(4)) != 0) == (d2 < r2), (res, d2)


# ---- mutations: each must make some check above fail ----------------------------------------------------------------
def _caught_block27(oracle_mod):
    tgt, q, *_ = RR.escape_fixture(0.3, 0, 1)
    o = _oracle(oracle_mod, q, tgt, 0.3)
    ref = RR.score(q, 0.3, o.voxels(), rule="block27", geom=R.leaf_geometry(tgt, 0.3), serial=True)
    return RR.within_score(o.calculate_score(np.eye(4)), ref) > 1.0


def _caught_le(oracle_mod):
    tgt, cen = equality_case(1.0)
    qv =[q for q, d2 in RR.equality_queries(1.0, cen) if d2 == RR.radius2(1.0)][0]
    o = _oracle(oracle_mod, qv[None, :], tgt, 1.0)
    ref = RR.score(qv[None, :], 1.0, o.voxels(), strict=False, serial=True)
    return ref["hits"] != 0 and o.calculate_score(np.eye(4)) == 0


def _caught_no_eguard(oracle_mod, pair_tiny):
    """A voxel with a negative definite icov: e = d2 exp(+...) > 1, so the guarded Hessian equals the one without that
    voxel, and the unguarded one does not."""
    src, tgt, _ = pair_tiny
    v = R.voxel_map_ref(tgt, 2.0)
    T, p = o_pose(POSES[1]), POSES[1]
    _, vi, _ = RR.neighbours(N.transform_points(T[:3], src), 2.0, v)
    worst = int(np.bincount(vi).argmax())  # the voxel with the most pairs
    bad = dict(v, icov=v["icov"].copy())
    bad["icov"][worst] = -100 * np.eye(3)
    keep = np.arange(len(v["idx"])) != worst
    without = {k: (a[keep] if isinstance(a, np.ndarray) and len(a) == len(keep) else a) for k, a in v.items()}
    ref_without = RR.hessian(src, T[:3], p, 2.0, without)
    assert RR.within_h(RR.hessian(src, T[:3], p, 2.0, bad)["H"], ref_without)[0] <= 1.0
    return RR.within_h(RR.hessian(src, T[:3], p, 2.0, bad, e_guard=False)["H"], ref_without)[0] > 1.0


def _caught_global_average(oracle_mod, pair_small):
    src, tgt, _ = pair_small
    o = _oracle(oracle_mod, src, tgt, 2.0)
    ref = RR.score(src, 2.0, o.voxels(), average="global", serial=True)
    return RR.within_score(o.calculate_score(np.eye(4)), ref) > 1.0


def _caught_plus_sy(oracle_mod, pair_small):
    src, tgt, _ = pair_small
    o = _oracle(oracle_mod, src, tgt, 2.0)
    return any(_hessian_vs_oracle(o, src, 2.0, p, minus_sy=False)[0] > 1.0 for p in N.pitch_poses())


def _caught_icov_f32(oracle_mod, pair_small):
    src, tgt, _ = pair_small
    o = _oracle(oracle_mod, src, tgt, 2.0)
    return _hessian_vs_oracle(o, src, 2.0, POSES[1], icov_f32=True)[0] > 1.0


@pytest.mark.parametrize("mutation", ["block27", "le", "no_eguard", "global_average", "plus_sy", "icov_f32"])
def test_mutations_are_caught(oracle_mod, pair_tiny, pair_small, mutation):
    caught = {"block27": lambda: _caught_block27(oracle_mod), "le": lambda: _caught_le(oracle_mod),
              "no_eguard": lambda: _caught_no_eguard(oracle_mod, pair_tiny),
              "global_average": lambda: _caught_global_average(oracle_mod, pair_small),
              "plus_sy": lambda: _caught_plus_sy(oracle_mod, pair_small),
              "icov_f32": lambda: _caught_icov_f32(oracle_mod, pair_small)}[mutation]()
    assert caught, mutation


def test_nonfinite_and_huge_rows_have_no_neighbour(pair_tiny):
    src, tgt, _ = pair_tiny
    v = R.voxel_map_ref(tgt, 2.0)
    base = RR.score(src, 2.0, v)
    for cloud, ok in (R.with_nonfinite_rows(src), RR.huge_rows(src)):
        got = RR.score(cloud, 2.0, v)
        assert got["hits"] == base["hits"] and got["n"] == len(cloud) > base["n"] == ok.sum()
        assert abs(got["score"] * got["n"] - base["score"] * base["n"]) <= 1e-12 * abs(base["score"] * base["n"])
    assert np.isnan(RR.score(src[:0], 2.0, v)["score"])  # the reference's 0 / 0
