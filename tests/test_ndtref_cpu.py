"""The float64 derivative reference of tests/ndtref.py and its bound, checked on the CPU before any GPU comparison: against
the oracle's independent f32 restatement (oracle.NDT.derivatives), entry by entry, for every search method with and
without the Hessian; and each fixture generator against the edge it is named for."""
import numpy as np
import pytest

import gridref as R
import ndtref as N

F32 = np.float32
POSES = (np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02]), np.array([-0.4, 0.3, -0.1, 2.9, 0.01, -0.3]))
METHODS = [(2, "DIRECT7"), (3, "DIRECT1"), (1, "DIRECT26"), (0, "KDTREE")]


def _oracle_ndt(oracle_mod, src, tgt, res, method):
    o = oracle_mod.NDT(resolution=res, search_method=method)
    o.set_target(tgt)
    o.set_source(src)
    return o


def _check_against_oracle(oracle_mod, src, tgt, res, method, poses, what, offset=(0.0, 0.0, 0.0)):
    o = _oracle_ndt(oracle_mod, src, tgt, res, method)
    v, geom = o.voxels(), R.leaf_geometry(tgt, res)
    worst = 0.0
    for p in poses:
        p = np.array(p, dtype=np.float64)
        p[:3] += offset
        T = oracle_mod.pose_to_matrix(p)
        for hess in (True, False):
            ref = N.derivatives(src, T[:3], p, res, v, geom, method, compute_hessian=hess)
            assert ref["near_threshold"] == 0, (what, p)
            got = o.derivatives(T, p, hess)
            r = N.within(got, ref, scale=2.0)  # the oracle sums in another order: twice the bound
            assert r["max"] <= 1.0, (what, method, p, hess, r)
            if not hess:
                assert np.all(got[2] == 0)
            worst = max(worst, r["max"])
    return worst


@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_ndtref_matches_oracle_synthetic(oracle_mod, pair_tiny, pair_small, method):
    for name, (src, tgt, _) in (("tiny", pair_tiny), ("small", pair_small)):
        _check_against_oracle(oracle_mod, src, tgt, 2.0, method, POSES + tuple(N.pitch_poses()), name)


@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_ndtref_matches_oracle_edges(oracle_mod, golden, pair_small, method):
    _check_against_oracle(oracle_mod, golden["source"], golden["target"], 1.0, method, POSES[:2], "golden")
    src, tgt = N.illconditioned_pair()
    _check_against_oracle(oracle_mod, src, tgt, 2.0, method, POSES[:2], "illconditioned")
    src, tgt = N.shifted_pair(*pair_small[:2])
    _check_against_oracle(oracle_mod, src, tgt, 2.0, method, POSES[:2], "shifted", offset=N.SHIFT)
    src, tgt, _ = pair_small
    _check_against_oracle(oracle_mod, src, tgt, 2.0, method, [p for p, _, _ in N.snap_poses()[:6]], "snap")


def test_angle_tables_match_the_oracle_bitwise(oracle_mod):
    for p in list(POSES) + N.pitch_poses() + [p for p, _, _ in N.snap_poses()]:
        j, h = N.angle_tables(p)
        jo, ho = oracle_mod.angle_tables(p)
        np.testing.assert_array_equal(j, jo)
        np.testing.assert_array_equal(h, ho)
        assert h[6, 2] == F32(np.sin(p[4]) if abs(p[4]) >= 1e-4 else 0.0)  # the live table keeps +sy


def test_snap_poses_straddle_the_snap():
    seen = set()
    for p, axis, snapped in N.snap_poses():
        j_on, _ = N.angle_tables(p)
        q = p.copy()
        q[axis] = 0.0
        j_zero, _ = N.angle_tables(q)
        assert np.array_equal(j_on, j_zero) == snapped, (axis, p[axis])
        seen.add((axis, snapped))
    assert len(seen) == 6


def test_quirk_is_visible_at_large_pitch(oracle_mod, pair_small):
    """Flipping d1.z from +sy to -sy moves H(4,4) by ~2 sy z S0: at |pitch| >= 0.6 far beyond the bound (so a test that
    compares H(4,4) would notice the flip), at the moderate poses below it."""
    src, tgt, _ = pair_small
    o = _oracle_ndt(oracle_mod, src, tgt, 2.0, 2)
    v, geom = o.voxels(), R.leaf_geometry(tgt, 2.0)
    for p in N.pitch_poses():
        T = oracle_mod.pose_to_matrix(p)
        plus = N.derivatives(src, T[:3], p, 2.0, v, geom)
        minus = N.derivatives(src, T[:3], p, 2.0, v, geom, minus_sy=True)
        assert abs(plus["H"][4, 4] - minus["H"][4, 4]) > 10 * plus["tol_H"][4, 4], p
        assert np.array_equal(plus["g"], minus["g"])


def test_xprime_split_is_within_one_ulp_and_not_always_equal():
    """x' = (x_t - mean_hi) - mean_lo in f32 against f32(f64(x_t) - mean): at most one float32 ulp apart, and not always
    equal, near the origin and at km scale."""
    rng = np.random.default_rng(3)
    for centre, spread in ((0.0, 3.0), (60.0, 60.0), (3000.0, 60.0)):
        mean = centre + rng.uniform(-spread, spread, 400000)
        xt = (mean + rng.normal(0, 1.5, len(mean))).astype(F32)
        got = N.kernel_xprime(xt, mean)
        exact = (xt.astype(np.float64) - mean).astype(F32)
        ulp = np.spacing(np.abs(exact))
        assert np.all(np.abs(got.astype(np.float64) - exact) <= ulp), centre
        assert np.any(got != exact), centre


def test_illconditioned_pair_is_illconditioned(oracle_mod):
    src, tgt = N.illconditioned_pair()
    o = _oracle_ndt(oracle_mod, src, tgt, 2.0, 2)
    v = o.voxels()
    ev = np.linalg.eigvalsh(v["icov"])
    cond = ev[:, -1] / ev[:, 0]  # the eigenvalue floor of 0.01 ev_max caps it at 100; scan-like voxels sit near 2
    assert cond.max() > 20 and len(v["idx"]) >= 3 + 6
    assert sorted(v["npts"].tolist())[:6] == [6, 6, 6, 7, 7, 7]


def test_shifted_pair_is_at_km_scale(pair_small):
    src, tgt = N.shifted_pair(*pair_small[:2])
    assert np.abs(tgt.mean(axis=0) - np.array(N.SHIFT)).max() < 100 and np.abs(src).max() < 200


def test_ladder_sizes_hit_their_edges():
    for sms in (132, 114, 78):
        n_eval = sms - N.CTL_CTAS
        sizes = N.ladder_sizes(sms)
        assert len(set(sizes)) == len(sizes)
        per_thread = {n: N.points_per_thread(n, sms) for n in sizes}
        cap = 768 * n_eval
        assert per_thread[cap] == 1 and per_thread[cap + 1] == 2 and per_thread[cap + 33] == 2
        for n in sizes:
            rank, tid, rows = N.point_owner(n, sms)
            assert rows == max(1, min((n + 127) // 128, n_eval))
            assert np.bincount(rank * 768 + tid).max() == per_thread[n]
        assert N.point_owner(128 * n_eval, sms)[2] == n_eval and N.point_owner(128 * (n_eval - 1), sms)[2] == n_eval - 1
        assert 33 % 32 and (cap + 33) % 32  # ragged last units


def test_kdtree_reaches_a_voxel_two_lookup_cells_away(oracle_mod):
    """KDTREE is a radius search over every centroid: on an escape fixture (a wall on a build-cell face, the query two
    lookup cells below it, inside the radius) the reference and the oracle both score the wall voxel."""
    import radiusref as RR

    for axis in range(3):
        tgt, q, *_ = RR.escape_fixture(0.3, axis, 1)
        o = _oracle_ndt(oracle_mod, q, tgt, 0.3, N.KDTREE)
        v, geom = o.voxels(), R.leaf_geometry(tgt, 0.3)
        eye = np.eye(4, dtype=F32)
        ref = N.derivatives(q, eye[:3], np.zeros(6), 0.3, v, geom, N.KDTREE)
        assert ref["hits"] == 1 and ref["near_threshold"] == 0, axis
        assert N.within(o.derivatives(eye, np.zeros(6), True), ref, scale=2.0)["max"] <= 1.0, axis
        assert ref["score"] != 0
