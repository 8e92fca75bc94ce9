"""The CPU references and edge-cloud generators of tests/gridref.py, checked without a GPU: the references agree with
the oracle where the oracle covers the same operation, and every generator really produces the edge it is named for.
tests/test_gpu_grid_edges.py compares the CUDA kernels with these references."""
import numpy as np
import pytest

import gridref as R

F32 = np.float32


def _edge_clouds():
    rng = np.random.default_rng(5)
    scene = rng.uniform(-6, 6, size=(3000, 3)).astype(F32)
    scene[:, 2] *= 0.2
    pop, _ = R.population_leaves(1.0)
    bad, _ = R.with_nonfinite_rows(scene, seed=1)
    return {
        "scene": (scene, 1.0),
        "nonfinite": (bad, 1.0),
        "population": (pop, 1.0),
        "degenerate": (R.degenerate_leaves(2.0, n=1000), 2.0),
        "shift_km": (R.shifted(scene, R.SHIFTS[0]), 1.0),
        "shift_20km": (R.shifted(scene, R.SHIFTS[1]), 2.0),
    }


def _ulp(v):
    return np.spacing(np.abs(np.asarray(v, dtype=np.float64)).astype(F32)).astype(np.float64)


def test_leaf_geometry_matches_oracle(oracle_mod, golden):
    clouds = dict(_edge_clouds(), golden=(golden["target"], 1.0))
    for name, (pts, leaf) in clouds.items():
        g = R.leaf_geometry(pts, leaf)
        o = oracle_mod.NDT(resolution=leaf)
        o.set_target(np.ascontiguousarray(pts[:, :3]))
        mb, db = o.grid_geom()
        np.testing.assert_array_equal(g["min_b"], mb, err_msg=name)
        np.testing.assert_array_equal(g["div_b"], db, err_msg=name)


def test_voxelgrid_ref_matches_oracle(oracle_mod, golden):
    clouds = dict(_edge_clouds(), golden=(golden["raw"], 0.1), golden_coarse=(golden["raw"], 2.5))
    for name, (pts, leaf) in clouds.items():
        p = R._with_intensity(pts)
        p[:, 3] = np.linspace(0, 50, len(p), dtype=F32)
        ref, err = R.voxelgrid_ref(p, leaf)
        o = oracle_mod.voxelgrid(p, leaf)
        assert o.shape == ref.shape, name
        # the oracle sums in float like pcl::VoxelGrid: running-sum error <= n * 2^-24 * mean|value|, plus its final cast
        n_mean_abs = err / (2.0 * 2.0**-53)
        tol = n_mean_abs * 2.0**-24 + 2 * _ulp(ref)
        assert np.all(np.abs(o - ref) <= tol), (name, np.abs(o - ref).max())
        assert np.isfinite(ref).all()


def test_voxel_map_ref_matches_oracle(oracle_mod, golden):
    clouds = dict(_edge_clouds(), golden=(golden["target"], 1.0))
    for name, (pts, leaf) in clouds.items():
        ref = R.voxel_map_ref(pts, leaf)
        o = oracle_mod.NDT(resolution=leaf)
        o.set_target(np.ascontiguousarray(pts[:, :3]))
        ov = o.voxels()
        np.testing.assert_array_equal(ref["idx"], ov["idx"], err_msg=name)
        np.testing.assert_array_equal(ref["npts"], ov["npts"], err_msg=name)
        # same formula, same summation order: only the eigen-solvers differ (LAPACK here, Jacobi there)
        np.testing.assert_allclose(ref["mean"], ov["mean"], rtol=1e-15, atol=0, err_msg=name)
        scale = np.abs(ref["icov"]).max(axis=(1, 2))
        rel = np.abs(ref["icov"] - ov["icov"]).max(axis=(1, 2)) / scale
        assert np.all(rel <= 1e-9 * ref["lam_max"] / ref["lam_min"]), (name, rel.max())
    assert len(R.voxel_map_ref(*clouds["golden"])["idx"]) > 500


def test_leaf_edge_floats_hit_the_multiply_divide_disagreement():
    for leaf, expect in ((0.1, 198), (0.2, 198), (0.3, 272)):
        x = R.leaf_edge_floats(leaf)
        bad = R.mul_div_disagree(x, leaf)
        assert len(x) == 1200 * 9 and int(bad.sum()) == expect, (leaf, int(bad.sum()))
        # the two formulas never disagree by more than one cell
        assert np.all(np.abs(R.build_ref(x, leaf) - R.lookup_ref(x, leaf)) <= 1)
    for leaf in (1.0, 2.0, 5.0):
        assert not R.mul_div_disagree(R.leaf_edge_floats(leaf), leaf).any()


def test_nonfinite_rows_generator():
    p = np.arange(3000 * 4, dtype=F32).reshape(3000, 4)
    out, ok = R.with_nonfinite_rows(p, seed=2)
    fin = R.finite_rows(out)
    np.testing.assert_array_equal(fin, ok)
    assert not fin[0] and not fin[-1] and not fin[256:512].any() and fin[1:256].all() and fin[512:-1].all()
    np.testing.assert_array_equal(out[ok], p)
    vals = out[~ok][:, :3]
    assert np.isnan(vals).any() and np.isposinf(vals).any() and np.isneginf(vals).any()


def test_population_and_degenerate_leaves():
    pts, expect = R.population_leaves(1.0)
    g = R.leaf_geometry(pts, 1.0)
    idx = R.leaf_indices(pts, g)
    leaves, counts = np.unique(idx, return_counts=True)
    assert sorted(counts.tolist()) == sorted(expect.values())
    vm = R.voxel_map_ref(pts, 1.0)
    assert sorted(vm["npts"].tolist()) == [6, 6, 6, 7, 7, 7]
    # identical, collinear and coplanar leaves: the identity start keeps all three; the line and the plane (n = 1000) have
    # their small eigenvalues raised to 0.01 * ev_max, the identical points (covariance I / n) do not
    d = R.degenerate_leaves(2.0, n=1000)
    vm = R.voxel_map_ref(d, 2.0)
    assert len(vm["idx"]) == 3 and np.all(vm["npts"] == 1000)
    ratio = vm["lam_min"] / vm["lam_max"]
    assert ratio[0] > 0.99 and abs(ratio[1] - 0.01) < 1e-12 and abs(ratio[2] - 0.01) < 1e-12


@pytest.mark.parametrize("n_words", [1, 2047, 2048, 2049, 2048 * 1024 - 1, 2048 * 1024 + 1, 3 * 2048 * 1024 + 5])
def test_word_anchors_produce_their_n_words(n_words):
    dims = R.dims_for_words(n_words)
    g = R.leaf_geometry(R.word_anchors(dims), 1.0)
    assert not g["overflow"] and g["n_words"] == n_words and tuple(g["div_b"]) == dims
    assert g["n_cells"] % 32 != 0  # a partly used last word
    idx = R.leaf_indices(R.word_anchors(dims), g)
    assert idx.tolist() == [0, g["n_cells"] - 1]
    tiles = -(-n_words // R.SCAN_TILE_WORDS)
    assert (tiles > R.SCAN_BLOCK_TILES) == (n_words > 2048 * 1024)


def test_overflow_pair():
    # INT32_MAX = 2^31 - 1 is prime: the largest accepted product of float-representable extents is
    # 2147483646 = 1386 * 4681 * 331; the smallest refused one tested is 2^31 = 1024 * 1024 * 2048
    under = R.leaf_geometry(R.word_anchors((1386, 4681, 331)), 1.0)
    assert not under["overflow"] and under["n_cells"] == 2**31 - 2
    over_pts = R.word_anchors((1024, 1024, 2048))
    over = R.leaf_geometry(over_pts, 1.0)
    assert over["overflow"] and np.prod(over["dxyz"]) == 2**31
    out, err = R.voxelgrid_ref(over_pts, 1.0)
    assert err is None and np.array_equal(out[:, :3], over_pts)
    assert R.voxel_map_ref(over_pts, 1.0) is None


def test_overflow_matches_oracle(oracle_mod):
    over_pts = np.concatenate([R.word_anchors((1024, 1024, 2048)), np.full((3, 3), 7.25, F32)])
    np.testing.assert_array_equal(oracle_mod.voxelgrid(over_pts, 1.0)[:, :3], over_pts)
    o = oracle_mod.NDT(resolution=1.0)
    o.set_target(over_pts)
    assert len(o.voxels()["idx"]) == 0


def test_nn_ring_margin_case():
    t, q, want, g = R.nn_ring_margin_case()
    idx, d2 = R.nn1_ref(t, q)
    assert idx[0] == want
    h = float(g["h"])
    cell = lambda x: int(np.floor((F32(x) - g["origin"][0]) * g["inv_h"]))  # noqa: E731
    assert tuple(g["dims"]) == (4, 4, 4) and cell(q[0, 0]) == 2 and cell(t[8, 0]) == 3 and cell(t[9, 0]) == 0
    d2a = float(R._d2(q, t[8:9])[0, 0])
    # the ring-1 candidate A is beyond the exact bound h^2 by less than 1e-4: only a margin below 1 keeps searching
    assert 0.99999 * h * h < d2a <= 1.0001 * h * h and d2[0] < d2a


def test_nn1_ref_matches_oracle(oracle_mod):
    rng = np.random.default_rng(9)
    targets = {
        "planar": np.c_[rng.uniform(-5, 5, (500, 2)), np.full(500, 1.5)],
        "linear": np.c_[rng.uniform(-5, 5, 400), np.zeros(400), np.zeros(400)],
        "single": np.array([[1.0, 2.0, 3.0]]),
        "two": np.array([[0.0, 0, 0], [1.0, 1.0, 1.0]]),
        "identical": np.full((50, 3), 4.25),
        "duplicates": np.repeat(rng.uniform(-3, 3, (40, 3)), 7, axis=0),
        "shifted": R.shifted(rng.uniform(-20, 20, (800, 3)), R.SHIFTS[1]),
    }
    for name, t in targets.items():
        t = t.astype(F32)
        q = R.nn_edge_queries(t, seed=1)
        i, d = R.nn1_ref(t, q)
        io, do = oracle_mod.nn1(t, q)
        np.testing.assert_array_equal(i, io, err_msg=name)
        np.testing.assert_array_equal(d, do, err_msg=name)
    # the query set covers exact hits and the grid's cell faces
    t = targets["planar"].astype(F32)
    q = R.nn_edge_queries(t)
    assert (R.nn1_ref(t, q)[1] == 0).sum() >= 64
    g = R.nn_geometry(t)
    on_face = (q[:, 0] - g["origin"][0]) * g["inv_h"]
    assert (on_face == np.round(on_face)).sum() >= 10


def test_lattice_ties_decide_gicp_covariances(oracle_mod):
    k = 20
    lat = R.lattice((6, 5, 4), (1.0, 1.3, 1.7))
    low, gap = R.gicp_cov_ref(lat, k)
    high, _ = R.gicp_cov_ref(lat, k, higher_index_ties=True)
    well = gap > 1e-3
    changed = np.abs(low - high).max(axis=(1, 2)) > 1e-2
    assert (well & changed).sum() >= 10  # the tie at the k-th distance decides the covariance of these points
    o = oracle_mod.GICP()
    o.set_target(lat)
    o.set_source(lat)
    o.align()
    co = o.covariances("target")
    assert np.abs(co[well] - low[well]).max() < 1e-9
