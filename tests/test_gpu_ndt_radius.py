"""The NDT radius paths on the device (ndt_aux.cu: the K2 radius Hessian and calculateScore; ndt_solver.cu: K1's KDTREE
branch) against the float64 reference of tests/radiusref.py, entry by entry within its bound, with the handle's own
voxels. The fixtures sit where the radius rule goes wrong: voxels two lookup cells from the query (the builder's
floor(x * inv_leaf) and the lookup's floor(x / leaf) disagree near a face), squared distances at r^2 exactly and one ulp
either side, grid-stride sizes, 16- and 32-byte records, non-finite and huge rows, km-scale coordinates and leaf sizes that
are not powers of two. The reference uses the handle's own f32 centroids and the kernels' un-fused f32 distance, so
every radius decision is exact, at r^2 itself included. Run on an H100 with -m gpu; each test prints the largest |GPU - ref| / bound it saw."""
import numpy as np
import pytest

import gridref as R
import ndtref as N
import radiusref as RR

pytestmark = pytest.mark.gpu

F32 = np.float32
MODERATE = [np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02]), np.array([-0.4, 0.3, -0.1, 2.9, 0.01, -0.3])]
EYE = np.eye(4, dtype=F32)
ESCAPES = [(leaf, axis, d, inside) for leaf in (0.3, 0.6, 0.9) for axis in range(3) for d in (1, -1) for inside in (True, False)]
GRID_STRIDE = 1056 * 128  # the radius kernels' largest grid (H100_SMS * 8 blocks of 128 threads)


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


@pytest.fixture(scope="module")
def n_sms(b200):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _ndt(b200, tgt, src, res, method=2):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setNeighborhoodSearchMethod(method)
    g.setInputTarget(tgt)
    if src is not None:
        g.setInputSource(src)
    return g


def _pose(p):
    import oracle

    return oracle.pose_to_matrix(p)


def _scenes(golden):
    from lidarslam_ros2_b200 import synth

    small = synth.registration_pair("small", 2.0)[:2]
    return {"tiny": (synth.registration_pair("tiny", 2.0)[:2], 2.0, (0.0, 0.0, 0.0)), "small": (small, 2.0, (0.0, 0.0, 0.0)),
            "c1": (synth.registration_pair("c1", 2.0)[:2], 2.0, (0.0, 0.0, 0.0)),
            "golden": ((golden["source"], golden["target"]), 1.0, (0.0, 0.0, 0.0)),
            "illconditioned": (N.illconditioned_pair(), 2.0, (0.0, 0.0, 0.0)),
            "shifted": (N.shifted_pair(*small), 2.0, N.SHIFT),
            "shifted_far": (N.shifted_pair(*small, offset=R.SHIFTS[1]), 2.0, R.SHIFTS[1])}


def _check_k2(g, src, res, p, what, T=None):
    T = _pose(p) if T is None else T
    ref = RR.hessian(src, T[:3], p, res, g.voxels())
    w, _ = RR.within_h(g.hessian_radius(T, p), ref)
    assert w <= 1.0, (what, p, w)
    return w, ref


def test_k2_hessian_per_entry(b200, golden):
    worst = {}
    for name, ((src, tgt), res, off) in _scenes(golden).items():
        g = _ndt(b200, tgt, src, res)
        poses = MODERATE + N.pitch_poses() + ([p for p, _, _ in N.snap_poses()[:6]] if name == "small" else [])
        for p in poses:
            p = np.array(p, dtype=np.float64)
            p[:3] += off
            w, ref = _check_k2(g, src, res, p, name)
            assert ref["hits"] > 0, name
            worst[name] = max(worst.get(name, 0.0), w)
    print("\nmax |K2 - ref| / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def _big_cloud():
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("headline", 2.0)
    offs = np.array([(0.0, 0.0, 0.0), (0.013, -0.007, 0.005), (-0.011, 0.009, -0.004)], dtype=F32)
    return np.ascontiguousarray(np.concatenate([src + o for o in offs])[:300_000], dtype=F32), tgt


def test_calculate_score_sizes_and_records(b200):
    src_all, tgt = _big_cloud()
    g = _ndt(b200, tgt, None, 2.0)
    v = g.voxels()
    worst = 0.0
    T = _pose(MODERATE[1])
    moved = N.transform_points(T[:3], src_all)
    sizes = [1, 31, 32, 33, GRID_STRIDE - 1, GRID_STRIDE, GRID_STRIDE + 1, len(moved)]
    for n in sizes:
        cloud = np.ascontiguousarray(moved[:n])
        ref = RR.score(cloud, 2.0, v)
        assert ref["hits"] > 0, n
        rec16 = np.c_[cloud, np.full(n, 7.0, F32)]
        rec32 = np.zeros((n, 8), F32)
        rec32[:, :3], rec32[:, 3], rec32[:, 5] = cloud, 1.0, -3.0
        for what, c in (("12 B", cloud), ("16 B", rec16), ("32 B", rec32)):
            w = RR.within_score(g.calculateScore(c), ref)
            assert w <= 1.0, (n, what, w)
            worst = max(worst, w)
    # the reference computes 0 / 0 for an empty cloud; the C-ABI returns 0 (DESIGN.md section 3)
    assert np.isnan(RR.score(moved[:0], 2.0, v)["score"]) and g.calculateScore(moved[:0]) == 0.0
    # a target without a valid voxel: every point has no neighbour
    sparse = _ndt(b200, tgt[::5000], None, 2.0)
    assert len(sparse.voxels()["idx"]) == 0 and sparse.calculateScore(moved[:1000]) == 0.0
    print(f"\nmax |calculateScore - ref| / bound over sizes {sizes}: {worst:.3g}")


def _escape_case(leaf, axis, direction, inside):
    tgt, q, cen, w, qq = RR.escape_fixture(leaf, axis, direction, inside)
    return tgt, q


@pytest.mark.parametrize("leaf,axis,direction,inside", ESCAPES)
def test_escape_fixtures_through_every_radius_user(b200, n_sms, leaf, axis, direction, inside):
    """A voxel two lookup cells from the query, inside the radius: K2, calculateScore and K1's KDTREE branch must all see
    it (the 27-cell block around the lookup cell does not hold it)."""
    tgt, q = _escape_case(leaf, axis, direction, inside)
    g = _ndt(b200, tgt, q, leaf, method=0)
    v, geom = g.voxels(), R.leaf_geometry(tgt, leaf)
    ref_s = RR.score(q, leaf, v)
    assert ref_s["hits"] == 1 and RR.score(q, leaf, v, rule="block27", geom=geom)["hits"] == 0
    s = g.calculateScore(q)
    assert s != 0 and RR.within_score(s, ref_s) <= 1.0, (s, ref_s["score"])
    w, ref_h = _check_k2(g, q, leaf, np.zeros(6), "escape", T=EYE)
    assert ref_h["hits"] == 1 and np.abs(ref_h["H"]).max() > 0
    ref_d = N.derivatives(q, EYE[:3], np.zeros(6), leaf, v, geom, N.KDTREE, n_sms=n_sms)
    got = g.derivatives(EYE, np.zeros(6), True)
    assert ref_d["hits"] == 1 and g.stats()["hits"] == 1
    assert N.within(got, ref_d)["max"] <= 1.0
    print(f"\nescape leaf {leaf} axis {axis} dir {direction} inside {inside}: score {RR.within_score(s, ref_s):.3g}, "
          f"K2 {w:.3g} of the bound")


def test_equality_fixtures_through_every_radius_user(b200, n_sms):
    for res, (x, y, z) in {1.0: (2.0, 0.5, 0.25), 0.3: (0.75, 0.45, 0.15), 0.6: (1.5, 0.9, 0.3)}.items():
        cen = np.array([x, y, z], dtype=F32)
        tgt = RR.wall(0, cen[0], (cen[1], cen[2]), res)
        qs = RR.equality_queries(res, cen)
        r2 = RR.radius2(res)
        assert qs[0][1] < r2 <= qs[-1][1]
        src = np.array([q for q, _ in qs], dtype=F32)
        expect = sum(int(d2 < r2) for _, d2 in qs)
        g = _ndt(b200, tgt, src, res, method=0)
        v = g.voxels()
        ref_s = RR.score(src, res, v)
        assert ref_s["hits"] == expect
        assert RR.within_score(g.calculateScore(src), ref_s) <= 1.0, res
        ref_h = RR.hessian(src, EYE[:3], np.zeros(6), res, v)
        assert ref_h["hits"] == expect and RR.within_h(g.hessian_radius(EYE, np.zeros(6)), ref_h)[0] <= 1.0, res
        g.derivatives(EYE, np.zeros(6), True)
        assert g.stats()["hits"] == expect, res
        for qv, d2 in qs:  # one query at a time: only the ones strictly inside score
            assert (g.calculateScore(qv.reshape(1, 3).copy()) != 0) == (d2 < r2), (res, d2)


def test_nonfinite_and_huge_rows(b200, n_sms):
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("small", 2.0)
    p = MODERATE[1]
    T = _pose(p)
    clean = _ndt(b200, tgt, src, 2.0, method=0)
    v = clean.voxels()
    H0 = clean.hessian_radius(T, p)
    moved = N.transform_points(T[:3], src)
    s0 = clean.calculateScore(moved)
    d0 = clean.derivatives(T, p, True)
    hits0 = clean.stats()["hits"]
    worst = 0.0
    for what, (cloud, ok) in (("non-finite", R.with_nonfinite_rows(src)), ("huge", RR.huge_rows(src))):
        g = _ndt(b200, tgt, cloud, 2.0, method=0)
        ref = RR.hessian(cloud, T[:3], p, 2.0, v)
        assert ref["hits"] == RR.hessian(src, T[:3], p, 2.0, v)["hits"]
        H = g.hessian_radius(T, p)
        worst = max(worst, RR.within_h(H, ref)[0], RR.within_h(H0, ref)[0])
        assert RR.within_h(H, ref)[0] <= 1.0 and RR.within_h(H0, ref)[0] <= 1.0, what
        mc = N.transform_points(T[:3], cloud)
        mc[~ok] = cloud[~ok, :3]  # the non-finite / huge rows themselves as queries
        ref_s = RR.score(mc, 2.0, v)
        s = g.calculateScore(mc)
        assert RR.within_score(s, ref_s) <= 1.0, what
        assert abs(s * len(mc) - s0 * len(moved)) <= (ref_s["tol"] * len(mc) + RR.score(moved, 2.0, v)["tol"] * len(moved))
        d = g.derivatives(T, p, True)
        assert g.stats()["hits"] == hits0, what
        ref_d = N.derivatives(cloud, T[:3], p, 2.0, v, R.leaf_geometry(tgt, 2.0), N.KDTREE, n_sms=n_sms)
        assert N.within(d, ref_d)["max"] <= 1.0 and N.within(d0, ref_d, scale=2.0)["max"] <= 1.0, what
    print(f"\nmax |K2 - ref| / bound with non-finite and huge rows: {worst:.3g}")


def test_repeated_calls_agree_within_the_bound(b200):
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("c1", 2.0)
    g = _ndt(b200, tgt, src, 2.0)
    p = MODERATE[2]
    T = _pose(p)
    ref = RR.hessian(src, T[:3], p, 2.0, g.voxels())
    a, b = g.hessian_radius(T, p), g.hessian_radius(T, p)
    assert RR.within_h(a, dict(ref, H=b), scale=2.0)[0] <= 1.0
    moved = N.transform_points(T[:3], src)
    ref_s = RR.score(moved, 2.0, g.voxels())
    assert RR.within_score(g.calculateScore(moved), dict(ref_s, score=g.calculateScore(moved)), scale=2.0) <= 1.0
