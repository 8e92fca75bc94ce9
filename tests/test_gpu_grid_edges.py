"""The grid builders and cell lookups at their edges, each kernel against the plain CPU reference of tests/gridref.py:
VoxelGrid (K4, dense and sparse rank index), the NDT voxel map (K3), the solver's cell lookup (K1), the exact-NN grid
(K8) and GICP's k-NN covariances (K5). The clouds are built to reach the places where a grid kernel is wrong without
failing loudly: rank-index scans of one tile, several tiles and more than 1024 tiles, leaf edges where
floor(x * (1 / leaf)) and floor(x / leaf) disagree, non-finite rows, 5/6/7-point and degenerate leaves, the int32 cell
limit, km-scale offsets, NN cell faces and ring bounds, and ties at the k-th neighbour. Run on an H100 with -m gpu."""
import ctypes as C

import numpy as np
import pytest

import gridref as R

pytestmark = pytest.mark.gpu

F32 = np.float32
U64 = 2.0**-53
DEFAULT_DENSE_BUDGET = 4 << 20  # VoxelGridFilter::dense_word_budget
LADDER = [1, 2047, 2048, 2049, 2048 * 1024 - 1, 2048 * 1024 + 1, 3 * 2048 * 1024 + 5]


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


@pytest.fixture
def vg_budget(b200):
    """Sets the word budget up to which VoxelGrid uses the dense rank index (0 forces the sparse one); restores it."""
    from lidarslam_ros2_b200 import _capi

    L = _capi.lib()
    L.b200reg_debug_set_voxelgrid_dense_budget.argtypes = [C.c_size_t]
    yield L.b200reg_debug_set_voxelgrid_dense_budget
    L.b200reg_debug_set_voxelgrid_dense_budget(DEFAULT_DENSE_BUDGET)


def _ladder_cloud(n_words, seed=0):
    """Leaf-1.0 cloud whose grid needs exactly n_words rank words: the two anchors, then 5..9-point leaves at cell 0, the
    last cell, bit 31 of the first and of a middle word, the page edge 1023/1024, the scan-tile edges (word 2047/2048)
    and the edge of the first 1024 tiles, plus 200 random leaves. On the largest rung, 70 000 further single points in
    distinct 1024-cell pages make VoxelGrid's sparse level-2 scan longer than 1024 tiles. Intensity is random."""
    rng = np.random.default_rng(seed + n_words)
    dims = R.dims_for_words(n_words)
    n_cells = dims[0] * dims[1] * dims[2]
    tile = R.SCAN_TILE_WORDS * 32
    special = [0, n_cells - 1, 31, 32 * (n_words // 2) + 31, 1023, 1024, tile - 1, tile, 1024 * tile - 1, 1024 * tile]
    cells = [c for c in special if c < n_cells] + rng.integers(0, n_cells, 200).tolist()
    parts = [R.word_anchors(dims)]
    for j, c in enumerate(cells):
        parts.append(R.cell_points(R.cell_of_index(c, dims), 1.0, (5, 6, 7, 9)[j % 4], rng))
    n_pages = -(-n_cells // R.PAGE_CELLS)
    if n_pages > 65536 * 2:
        pages = rng.choice(n_pages, 70000, replace=False)
        c = np.minimum(pages * R.PAGE_CELLS + rng.integers(0, R.PAGE_CELLS, len(pages)), n_cells - 1)
        parts.append(R.cell_points(R.cell_of_index(c, dims), 1.0, 1, rng))
    p = np.concatenate(parts)
    return np.c_[p, rng.uniform(0, 100, len(p))].astype(F32), dims


def _check_voxelgrid(out, pts, leaf, what):
    ref, err = R.voxelgrid_ref(pts, leaf)
    assert out.shape == ref.shape, (what, out.shape, ref.shape)  # the same leaves ...
    # ... in the same (ascending leaf index) order: every value within one float32 ulp of the float64 centroid (the
    # kernel's final cast) plus err, the bound on what its float64 atomics' summation order can change
    tol = np.spacing(np.abs(ref).astype(F32)).astype(np.float64) + err
    bad = ~(np.abs(out - ref) <= tol)
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5], out[bad][:5], ref[bad][:5])


# ---- VoxelGrid (K4) -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_words", LADDER)
def test_voxelgrid_word_ladder(b200, vg_budget, n_words):
    pts, dims = _ladder_cloud(n_words)
    g = R.leaf_geometry(pts, 1.0)
    assert g["n_words"] == n_words
    for budget, path in ((8 << 20, "dense"), (0, "sparse")):
        vg_budget(budget)
        _check_voxelgrid(b200.voxel_grid_filter(pts, 1.0), pts, 1.0, (n_words, path))
    if n_words > 3 * 2048 * 1024:  # the sparse path's level-2 scan really spans more than 1024 tiles
        n_pages = -(-g["n_cells"] // R.PAGE_CELLS)
        assert min(len(pts), n_pages) * 32 > 1024 * R.SCAN_TILE_WORDS


def test_voxelgrid_drops_nonfinite_rows(b200, vg_budget):
    rng = np.random.default_rng(11)
    scene = np.c_[rng.uniform(-8, 8, (6000, 2)), rng.uniform(-1, 1, 6000), rng.uniform(0, 9, 6000)].astype(F32)
    bad, ok = R.with_nonfinite_rows(scene, seed=3)
    for budget in (DEFAULT_DENSE_BUDGET, 0):
        vg_budget(budget)
        for leaf in (0.5, 0.3):
            out = b200.voxel_grid_filter(bad, leaf)
            _check_voxelgrid(out, bad, leaf, ("nonfinite", budget, leaf))
            _check_voxelgrid(out, scene, leaf, ("finite rows only", budget, leaf))


def test_voxelgrid_overflow_pair(b200):
    # INT32_MAX = 2^31 - 1 is prime and float products cannot land on every integer: the pair is 1386 x 4681 x 331 =
    # 2^31 - 2 cells (accepted, the largest product of float-representable extents below the limit) and
    # 1024 x 1024 x 2048 = 2^31 cells (refused: PCL returns the input unchanged)
    rng = np.random.default_rng(4)
    for dims, accepted in (((1386, 4681, 331), True), ((1024, 1024, 2048), False)):
        cells = rng.integers(0, dims[0] * dims[1] * dims[2], 300)
        p = np.concatenate([R.word_anchors(dims), R.cell_points(R.cell_of_index(cells, dims), 1.0, 3, rng)])
        p = np.c_[p, rng.uniform(0, 10, len(p))].astype(F32)
        out = b200.voxel_grid_filter(p, 1.0)
        if accepted:
            assert not R.leaf_geometry(p, 1.0)["overflow"]
            _check_voxelgrid(out, p, 1.0, dims)
        else:
            np.testing.assert_array_equal(out, p)


# ---- NDT voxel map (K3) ---------------------------------------------------------------------------------------------
def _ndt(b200, res, method=2):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setNeighborhoodSearchMethod(method)
    return g


def _check_voxel_map(v, ref, what):
    np.testing.assert_array_equal(v["idx"], ref["idx"], err_msg=str(what))
    np.testing.assert_array_equal(v["npts"], ref["npts"], err_msg=str(what))
    n = ref["npts"].astype(np.float64)
    X = ref["maxabs"]
    # mean: any float64 summation order of n terms |x| <= X moves sum / n by <= n u X (u = 2^-53), on either side; the
    # record keeps the mean as a float hi + lo pair (2^-48 relative)
    tol_mean = 2 * n[:, None] * U64 * X[:, None] + 2.0**-47 * np.abs(ref["mean"])
    assert np.all(np.abs(v["mean"] - ref["mean"]) <= tol_mean), (what, np.abs(v["mean"] - ref["mean"]).max())
    # icov: the covariance is sxx / n - 2 s mean^T / n + mean mean^T from float64 sums of n products <= X^2. Each side's
    # summation order moves it by <= (3 n + 6) u X^2 (dcov); the eigen-solvers (Jacobi there, LAPACK here) add
    # ~64 u ev_max; raising small eigenvalues to 0.01 ev_max moves the result by no more than its input moved. The
    # inverse then changes by <= |icov| * |dcov| / lam_min (first order, lam_min of the final covariance); x8 for the
    # entry-wise vs. spectral norms. That is the n 2^-52 X^2 / lam_min conditioning of the voxel.
    dcov = 2 * (3 * n + 6) * U64 * X**2 + 64 * U64 * ref["lam_max"]
    scale = np.abs(ref["icov"]).max(axis=(1, 2))
    tol_icov = 8 * scale * dcov / ref["lam_min"]
    err = np.abs(v["icov"] - ref["icov"]).max(axis=(1, 2))
    assert np.all(err <= tol_icov), (what, np.max(err / tol_icov))
    # centroid: (float)sum / (float)n; the float cast of a float64 sum moved by summation order may step one ulp, the
    # division rounds once more: <= 2^-22 relative
    c = ref["centroid"].astype(np.float64)
    assert np.all(np.abs(v["centroid"] - c) <= 2.0**-22 * np.abs(c) + 4 * n[:, None] * U64 * X[:, None]), what


@pytest.mark.parametrize("n_words", LADDER)
def test_voxel_map_word_ladder(b200, n_words):
    pts, _ = _ladder_cloud(n_words, seed=1)
    ref = R.voxel_map_ref(pts, 1.0)
    g = _ndt(b200, 1.0)
    g.setInputTarget(pts)
    assert g.stats()["n_cells"] == R.leaf_geometry(pts, 1.0)["n_cells"]
    v = g.voxels()
    _check_voxel_map(v, ref, n_words)
    assert 0 in v["idx"] and v["idx"][-1] == R.leaf_geometry(pts, 1.0)["n_cells"] - 1


def test_voxel_map_population_degenerate_and_far(b200, oracle_mod):
    rng = np.random.default_rng(8)
    scene = np.c_[rng.uniform(-10, 10, (20000, 2)), rng.uniform(-1.5, 1.5, 20000)].astype(F32)
    pop, _ = R.population_leaves(1.0)
    clouds = [
        ("population", pop, 1.0),
        ("degenerate", R.degenerate_leaves(2.0, n=1000), 2.0),
        ("nonfinite", R.with_nonfinite_rows(scene, seed=5)[0], 1.0),
    ]
    for off in R.SHIFTS:
        clouds += [(("shift", off, res), R.shifted(scene, off), res) for res in (1.0, 2.0)]
        clouds += [(("shift degenerate", off), R.shifted(R.degenerate_leaves(2.0, n=1000), off), 2.0)]
    for what, pts, res in clouds:
        ref = R.voxel_map_ref(pts, res)
        g = _ndt(b200, res)
        g.setInputTarget(pts)
        v = g.voxels()
        _check_voxel_map(v, ref, what)
        o = oracle_mod.NDT(resolution=res)
        o.set_target(np.ascontiguousarray(pts[:, :3]))
        np.testing.assert_array_equal(v["idx"], o.voxels()["idx"], err_msg=str(what))
    assert sorted(R.voxel_map_ref(pop, 1.0)["npts"].tolist()) == [6, 6, 6, 7, 7, 7]


def test_voxel_map_grid_overflow_keeps_the_handle_usable(b200):
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    g = _ndt(b200, 1.0)
    over = np.concatenate([R.word_anchors((1024, 1024, 2048)), np.full((8, 3), 3.5, F32)])
    with pytest.raises(B200RegError) as e:
        g.setInputTarget(over)
    assert e.value.code == _capi.ERR_GRID
    assert len(g.voxels()["idx"]) == 0
    pts, _ = _ladder_cloud(2049, seed=2)
    g.setInputTarget(pts)
    _check_voxel_map(g.voxels(), R.voxel_map_ref(pts, 1.0), "after ERR_GRID")
    src = pts[::3, :3].copy()
    g.setInputSource(src)
    s, grad, H = g.derivatives(np.eye(4, dtype=F32), np.zeros(6))
    assert np.isfinite(s) and np.isfinite(grad).all() and np.isfinite(H).all() and g.stats()["hits"] > 0


# ---- solver cell lookup (K1) ----------------------------------------------------------------------------------------
def _neighbour_offsets(method):
    if method in (2, 3):  # DIRECT7 / DIRECT1
        offs = [(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
        return offs[:1] if method == 3 else offs
    all27 = [(x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]
    return [o for o in all27 if o != (0, 0, 0)] if method == 1 else all27


def _ref_hits(src, res, tgt, ref, method, gpu_centroids):
    """(point, voxel) pairs the solver scores at identity: the cells around lookup_ref(point) that hold a valid voxel
    of the reference map (KDTREE: those whose centroid is closer than the resolution, float32 un-fused distance). All
    these pairs pass the e2 gate because gauss_d2 < 1 at these resolutions."""
    g = R.leaf_geometry(tgt, res)
    ijk = np.stack([R.lookup_ref(src[:, a], res) for a in range(3)], axis=1)
    where = {int(i): r for r, i in enumerate(ref["idx"])}
    r2 = F32(float(F32(res)) * float(F32(res)))
    hits = 0
    for o in _neighbour_offsets(method):
        rel = ijk + np.array(o) - g["min_b"]
        inside = ((rel >= 0) & (rel < g["div_b"])).all(axis=1)
        lin = rel[:, 0] + rel[:, 1] * g["mul"][1] + rel[:, 2] * g["mul"][2]
        for p, l in zip(src[inside], lin[inside]):
            r = where.get(int(l))
            if r is None:
                continue
            if method == 0:
                d = p - gpu_centroids[r]
                if not (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] < r2:
                    continue
            hits += 1
    return hits


@pytest.mark.parametrize("res", [0.3, 0.1])
def test_solver_lookup_on_leaf_edges(b200, oracle_mod, res):
    """Source points exactly on the floats where floor(x * inv_leaf) and floor(x / leaf) disagree, identity transform (the
    transformed point IS the source point), target voxels on both sides of every such edge: the solver must take the
    division's cell like the reference (lookup_cell_fast's fallback)."""
    rng = np.random.default_rng(int(res * 10))
    x = R.leaf_edge_floats(res)
    x = x[R.mul_div_disagree(x, res)]
    assert len(x) >= 150
    cells = np.unique(np.concatenate([R.lookup_ref(x, res), R.build_ref(x, res)]))
    cells = np.unique(np.concatenate([cells - 1, cells, cells + 1]))
    tgt = R.cell_points(np.c_[cells, np.zeros((len(cells), 2))], res, 8, rng)
    yz = (rng.uniform(0.15, 0.85, size=(len(x), 2)) * F32(res)).astype(F32)
    src = np.c_[x, yz].astype(F32)
    assert (R.lookup_ref(yz, res) == 0).all() and (R.build_ref(yz, res) == 0).all()
    ref = R.voxel_map_ref(tgt, res)
    T, p0 = np.eye(4, dtype=F32), np.zeros(6)
    for method in (2, 3, 1, 0):
        g = _ndt(b200, res, method)
        g.setInputTarget(tgt)
        g.setInputSource(src)
        v = g.voxels()
        _check_voxel_map(v, ref, ("lookup", res))
        o = oracle_mod.NDT(resolution=res, search_method=method)
        o.set_target(tgt)
        o.set_source(src)
        sg, gg, Hg = g.derivatives(T, p0, True)
        so, go, Ho = o.derivatives(T, p0, True)
        scale = max(np.abs(Ho).max(), np.abs(go).max(), 1.0)
        assert abs(sg - so) <= 1e-6 * max(1.0, abs(so)), (method, sg, so)
        assert np.abs(gg - go).max() <= 2e-5 * scale, (method, np.abs(gg - go).max() / scale)
        assert np.abs(Hg - Ho).max() <= 2e-5 * scale, (method, np.abs(Hg - Ho).max() / scale)
        assert g.stats()["hits"] == _ref_hits(src, res, tgt, ref, method, v["centroid"]), method


def test_solver_ignores_nonfinite_and_huge_source_points(b200, oracle_mod):
    """NaN, +-inf and |x| = 1e12 rows in the source change nothing: a NaN point lands in the leaf of the origin (floorf(NaN)
    casts to 0 on the GPU), which holds a voxel here, and only the pair gate keeps it out of the sums."""
    rng = np.random.default_rng(21)
    tgt = np.c_[rng.uniform(-6, 6, (20000, 2)), rng.uniform(-1.2, 1.2, 20000)].astype(F32)
    clean = tgt[::4] + F32(0.05)
    bad, ok = R.with_nonfinite_rows(clean, seed=6)
    huge = np.array([[1e12, 0, 0], [-1e12, 1, 1], [0, 1e12, 0], [0, 0, -1e12], [1e12, 1e12, 1e12]], dtype=F32)
    bad = np.concatenate([huge, bad, huge])
    ref = R.voxel_map_ref(tgt, 1.0)
    g0 = R.leaf_geometry(tgt, 1.0)
    origin_leaf = int((-g0["min_b"] * g0["mul"]).sum())
    assert origin_leaf in ref["idx"]
    poses = (np.zeros(6), np.array([0.05, -0.03, 0.02, 0.01, -0.005, 0.02]))
    for method in (2, 3, 1, 0):
        res_ = {}
        for name, src in (("clean", clean), ("bad", bad)):
            g = _ndt(b200, 1.0, method)
            g.setInputTarget(tgt)
            g.setInputSource(src)
            out = []
            for p in poses:
                T = oracle_mod.pose_to_matrix(p)
                s, gr, H = g.derivatives(T, p, True)
                out.append((s, gr, H, g.stats()["hits"]))
            res_[name] = out
        for (s0, g0_, H0, h0), (s1, g1, H1, h1) in zip(res_["clean"], res_["bad"]):
            assert np.isfinite(s1) and np.isfinite(g1).all() and np.isfinite(H1).all(), method
            scale = max(np.abs(H0).max(), np.abs(g0_).max(), 1.0)
            assert h1 == h0 and h0 > 0, (method, h0, h1)
            assert abs(s1 - s0) <= 1e-6 * max(1.0, abs(s0))
            assert np.abs(g1 - g0_).max() <= 2e-5 * scale and np.abs(H1 - H0).max() <= 2e-5 * scale
    guess = oracle_mod.pose_to_matrix(np.array([0.1, -0.05, 0.03, 0.0, 0.0, 0.02]))
    poses_out = []
    for src in (clean, bad):
        g = _ndt(b200, 1.0)
        g.setInputTarget(tgt)
        g.setInputSource(src)
        T = g.align(guess)
        assert np.isfinite(T).all()
        poses_out.append((T, g.getFinalNumIteration(), g.hasConverged()))
    from lidarslam_ros2_b200 import synth

    dt, dr = synth.pose_error(poses_out[0][0], poses_out[1][0])
    assert dt < 1e-3 and dr < 1e-3 and poses_out[0][1:] == poses_out[1][1:], (dt, dr, poses_out)


# ---- exact-NN grid (K8) ---------------------------------------------------------------------------------------------
def _nn_targets():
    rng = np.random.default_rng(9)
    scene = rng.uniform(-20, 20, (3000, 3))
    t = {
        "planar": np.c_[rng.uniform(-5, 5, (500, 2)), np.full(500, 1.5)],
        "linear": np.c_[rng.uniform(-5, 5, 400), np.zeros(400), np.zeros(400)],
        "single": np.array([[1.0, 2.0, 3.0]]),
        "two": np.array([[0.0, 0, 0], [1.0, 1.0, 1.0]]),
        "identical": np.full((50, 3), 4.25),
        "duplicates": np.repeat(rng.uniform(-3, 3, (40, 3)), 7, axis=0)[rng.permutation(280)],
        "nonfinite": R.with_nonfinite_rows(scene.astype(F32), seed=7)[0],
    }
    for off in R.SHIFTS:
        t[("shift", off)] = R.shifted(scene, off)
    return {k: np.ascontiguousarray(v, dtype=F32)[:, :3] for k, v in t.items()}


def test_nn_grid_edges_exact(b200):
    for name, t in _nn_targets().items():
        q = R.nn_edge_queries(t, seed=2)
        g = b200.GeneralizedIterativeClosestPoint()
        g.setInputTarget(t)
        idx, d2 = g.nearest(q)
        ri, rd = R.nn1_ref(t, q)
        np.testing.assert_array_equal(idx, ri, err_msg=str(name))
        np.testing.assert_array_equal(d2, rd, err_msg=str(name))


def test_nn_ring_bound_margin(b200):
    t, q, want, _ = R.nn_ring_margin_case()
    g = b200.GeneralizedIterativeClosestPoint()
    g.setInputTarget(t)
    idx, d2 = g.nearest(q)
    ri, rd = R.nn1_ref(t, q)
    assert idx[0] == want == ri[0] and d2[0] == rd[0]


def test_fitness_max_range_is_inclusive(b200):
    rng = np.random.default_rng(12)
    t = rng.uniform(-5, 5, (2000, 3)).astype(F32)
    s = (t[::5] + rng.normal(0, 0.2, (400, 3))).astype(F32)
    _, d2 = R.nn1_ref(t, s)
    mr = float(np.sort(d2)[200])  # one query's squared distance, exactly
    inclusive, exclusive = d2[d2 <= mr].astype(np.float64), d2[d2 < mr].astype(np.float64)
    assert len(inclusive) == len(exclusive) + 1
    g = b200.GeneralizedIterativeClosestPoint()
    g.setInputTarget(t)
    g.setInputSource(s)  # final transformation: identity
    f = g.getFitnessScore(mr)
    assert abs(f - inclusive.mean()) <= 1e-12 * inclusive.mean()
    assert abs(f - exclusive.mean()) > 1e-9 * inclusive.mean()


# ---- GICP k-NN covariances (K5) -------------------------------------------------------------------------------------
def test_gicp_covariances_at_k_and_with_ties(b200, oracle_mod):
    k = 20
    rng = np.random.default_rng(13)
    clouds = {
        "k": rng.normal(0, 1, (k, 3)) * [3, 1, 0.3],
        "k+1": rng.normal(0, 1, (k + 1, 3)) * [3, 1, 0.3],
        "lattice": R.lattice((6, 5, 4), (1.0, 1.3, 1.7)),
        "lattice shifted": R.shifted(R.lattice((6, 5, 4), (1.0, 1.3, 1.7)), R.SHIFTS[0]),
    }
    for name, c in clouds.items():
        c = np.ascontiguousarray(c, dtype=F32)
        g = b200.GeneralizedIterativeClosestPoint()
        g.setInputTarget(c)
        g.setInputSource(c)
        g.align()
        o = oracle_mod.GICP()
        o.set_target(c)
        o.set_source(c)
        o.align()
        cg, co = g.covariances("target"), o.covariances("target")
        ref, gap = R.gicp_cov_ref(c, k)
        assert cg.shape == co.shape == ref.shape
        # only the smallest-eigenvalue direction enters the covariance: compare where it is well defined
        well = gap > 1e-3
        assert well.sum() >= min(len(c), 10), name
        assert np.abs(cg[well] - co[well]).max() < 1e-6, (name, np.abs(cg[well] - co[well]).max())
        assert np.abs(cg[well] - ref[well]).max() < 1e-6, name


def test_gicp_cloud_smaller_than_k_has_zero_covariances(b200):
    """A cloud with fewer than k points gets no neighbourhoods (pclomp refuses it and leaves the covariances unset): the
    covariances stay all zero, the kernel never runs, and align() with the other cloud's covariances still returns a
    finite pose."""
    rng = np.random.default_rng(14)
    small = rng.normal(0, 1, (19, 3)).astype(F32)
    big = rng.normal(0, 1, (500, 3)).astype(F32)
    g = b200.GeneralizedIterativeClosestPoint()
    g.setInputTarget(small)
    g.setInputSource(big)
    assert np.isfinite(g.align()).all()
    ct, cs = g.covariances("target"), g.covariances("source")
    assert ct.shape == (19, 3, 3) and np.all(ct == 0)
    assert cs.shape == (500, 3, 3) and np.isfinite(cs).all() and np.abs(cs).max() > 0
