"""The NDT solver's derivative evaluation (K1, derivatives()) against the float64 reference of tests/ndtref.py, entry by
entry: the score, the 6 gradient and 21 upper Hessian entries within their own bound, and the hit count exactly. The
fixtures sit where the evaluation can be quietly wrong: every search method with and without the Hessian, large pitch
(where the live table's +sy shows), the 1e-4 angle snap, km-scale coordinates, badly conditioned voxels, scan sizes at
the CTA, unit and shared-memory staging edges (and beyond: points read from global memory, in batch launches at the
host record stride), the rank index in and out of shared memory at the TMA chunk edges, and accumulators left over from
an earlier evaluation. Run on an H100 with -m gpu; each test prints the largest |K1 - ref| / bound it saw."""
import numpy as np
import pytest

import gridref as R
import ndtref as N

pytestmark = pytest.mark.gpu

F32 = np.float32
METHODS = [(2, "DIRECT7"), (3, "DIRECT1"), (1, "DIRECT26"), (0, "KDTREE")]
MODERATE = [np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02]), np.array([-0.4, 0.3, -0.1, 2.9, 0.01, -0.3])]
TILE_OFFSETS = ((0.0, 0.0, 0.0), (0.013, -0.007, 0.005), (-0.011, 0.009, -0.004))


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


@pytest.fixture(scope="module")
def big_pair():
    """The headline target (1M points) and a ~250k-point scan, as a 128-ring sensor produces: the headline scan tiled
    three times with millimetre offsets."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("headline", 2.0)
    big = np.concatenate([src + F32(o) for o in np.array(TILE_OFFSETS, dtype=F32)])[:250_000]
    return np.ascontiguousarray(big, dtype=F32), tgt


def _ndt(b200, tgt, src, res=2.0, method=2):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setNeighborhoodSearchMethod(method)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    return g


def _check(g, src, tgt, res, method, p, hess, n_sms, what, minus_sy=False):
    """derivatives() against the reference at pose p; returns the largest |K1 - ref| / bound."""
    import oracle

    T = oracle.pose_to_matrix(p)
    got = g.derivatives(T, p, hess)
    ref = N.derivatives(src, T[:3], p, res, g.voxels(), R.leaf_geometry(tgt, res), method, compute_hessian=hess,
                        minus_sy=minus_sy, n_sms=n_sms)
    assert ref["near_threshold"] == 0, what
    assert g.stats()["hits"] == ref["hits"], (what, g.stats()["hits"], ref["hits"])
    r = N.within(got, ref)
    assert r["max"] <= 1.0, (what, p, hess, r)
    if not hess:
        assert np.all(got[2] == 0), what
    return r["max"]


def _scenes():
    from lidarslam_ros2_b200 import synth

    small = synth.registration_pair("small", 2.0)[:2]
    out = {"small": (small, (0.0, 0.0, 0.0)), "c1": (synth.registration_pair("c1", 2.0)[:2], (0.0, 0.0, 0.0)),
           "illconditioned": (N.illconditioned_pair(), (0.0, 0.0, 0.0)), "shifted": (N.shifted_pair(*small), N.SHIFT)}
    return out


@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_eval_methods_and_poses(b200, n_sms, method):
    poses = MODERATE + N.pitch_poses() + [p for p, _, _ in N.snap_poses()]
    worst = {}
    for name, ((src, tgt), off) in _scenes().items():
        g = _ndt(b200, tgt, src, 2.0, method)
        for p in (poses if name == "small" else MODERATE + N.pitch_poses()[:2]):
            p = np.array(p, dtype=np.float64)
            p[:3] += off
            for hess in (True, False):
                worst[name] = max(worst.get(name, 0.0), _check(g, src, tgt, 2.0, method, p, hess, n_sms, (name, method)))
    print(f"\nmax |K1 - ref| / bound, method {method}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_oracle_parity_per_entry(b200, oracle_mod, pair_small, n_sms, method):
    """K1 against the oracle's f32 restatement on test_gpu_parity's derivative inputs, each entry within twice its own
    bound (the oracle sums in another order than K1) instead of one tolerance scaled by the largest entry."""
    src, tgt, _ = pair_small
    g = _ndt(b200, tgt, src, 2.0, method)
    o = oracle_mod.NDT(resolution=2.0, search_method=method)
    o.set_target(tgt)
    o.set_source(src)
    geom = R.leaf_geometry(tgt, 2.0)
    for p in MODERATE:
        T = oracle_mod.pose_to_matrix(p)
        for hess in (True, False):
            got = g.derivatives(T, p, hess)
            so, go, Ho = o.derivatives(T, p, hess)
            ref = N.derivatives(src, T[:3], p, 2.0, g.voxels(), geom, method, compute_hessian=hess, n_sms=n_sms)
            assert ref["near_threshold"] == 0 and g.stats()["hits"] == ref["hits"]
            r = N.within(got, dict(ref, score=so, g=go, H=Ho), scale=2.0)
            assert r["max"] <= 1.0, (p, hess, r)


def test_kdtree_dense_target_per_entry(b200, n_sms):
    """KDTREE on test_gpu_parity's dense target (c2), where the handle's centroids differ from the reference's float running
    sums by a few ulp: with the handle's own centroids in the float64 reference the radius test cannot flip, so g and H
    are compared per entry and the hits exactly."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("c2", 2.0)
    g = _ndt(b200, tgt, src, 2.0, 0)
    p = np.array([0.2, -0.1, 0.03, 0.004, -0.003, 0.015])
    print(f"\nmax |K1 - ref| / bound, KDTREE dense target: {_check(g, src, tgt, 2.0, 0, p, True, n_sms, 'c2'):.3g}")


def test_eval_sees_the_live_sy_sign(b200, n_sms):
    """At large pitch K1's H(4,4) is far from the -sy variant of the reference: the suite can tell the two conventions."""
    import oracle
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("small", 2.0)
    g = _ndt(b200, tgt, src)
    for p in N.pitch_poses():
        T = oracle.pose_to_matrix(p)
        _, _, H = g.derivatives(T, p, True)
        ref = N.derivatives(src, T[:3], p, 2.0, g.voxels(), R.leaf_geometry(tgt, 2.0), minus_sy=True, n_sms=n_sms)
        assert abs(H[4, 4] - ref["H"][4, 4]) > 10 * ref["tol_H"][4, 4], p


def test_scan_size_ladder(b200, n_sms, big_pair):
    """Scans at the partition edges (ragged 32-point units, one unit per CTA, all evaluators busy) and at the
    shared-memory staging capacity 768 (SMs - 3): beyond it each thread evaluates a second point read from global memory."""
    src_all, tgt = big_pair
    sizes = N.ladder_sizes(n_sms) + [len(src_all)]
    assert sizes[-2] < len(src_all)
    g = b200.NormalDistributionsTransform()
    g.setResolution(2.0)
    g.setInputTarget(tgt)
    p = MODERATE[1]
    worst = 0.0
    for n in sizes:
        src = np.ascontiguousarray(src_all[:n])
        g.setInputSource(src)
        for hess in ((True, False) if n > sizes[-6] else (True,)):
            worst = max(worst, _check(g, src, tgt, 2.0, 2, p, hess, n_sms, ("ladder", n)))
    print(f"\nmax |K1 - ref| / bound, scan-size ladder: {worst:.3g}")


def test_batch_above_staging_capacity(b200, oracle_mod, n_sms, big_pair):
    """Batch launches read the points beyond the staging capacity from the caller's records at their own stride: host
    records of 12 and 32 bytes and device float4 buffers, on 1, 2 and 3 slots, must give align()'s poses bit for bit."""
    import torch
    from lidarslam_ros2_b200 import synth

    src_all, tgt = big_pair
    cap = 768 * (n_sms - N.CTL_CTAS)
    scans = [np.ascontiguousarray(src_all[:cap + 33]), np.ascontiguousarray(src_all[: len(src_all)])]
    guesses = [synth.pose_matrix((0.3, -0.2, 0.05), (0.002, -0.003, 0.01)).astype(F32),
               synth.pose_matrix((0.1, 0.1, 0.0), (0.0, 0.004, -0.008)).astype(F32)]
    g = b200.NormalDistributionsTransform()
    g.setResolution(2.0)
    g.setMaximumIterations(6)
    g.setInputTarget(tgt)
    ref = []
    for s, gu in zip(scans, guesses):
        g.setInputSource(s)
        ref.append((g.align(gu), g.getFinalNumIteration()))
    wide = []
    for s in scans:
        w = np.zeros((len(s), 8), dtype=F32)
        w[:, :3], w[:, 3], w[:, 5] = s, 1.0, 7.0
        wide.append(w)
    dev = [torch.from_numpy(np.c_[s, np.ones(len(s), F32)]).cuda() for s in scans]
    torch.cuda.synchronize()
    for slots in (1, 2, 3):
        g.setBatchSlots(slots)
        for what, r in (("12 B", g.alignBatch(scans, guesses)), ("32 B", g.alignBatch(wide, guesses)),
                        ("device", g.alignBatchDevice([d.data_ptr() for d in dev], [len(s) for s in scans], guesses))):
            assert np.all(r["status"] == 0), (slots, what)
            for k, (P, it) in enumerate(ref):
                assert np.array_equal(r["pose"][k], P), (slots, what, k, np.abs(r["pose"][k] - P).max())
                assert r["iterations"][k] == it, (slots, what, k)
    o = oracle_mod.NDT(resolution=2.0, max_iterations=6)
    o.set_target(tgt)
    o.set_source(scans[0])
    dt, dr = synth.pose_error(ref[0][0], o.align(guesses[0]))
    assert dt < 1e-3 and dr < 1e-3, (dt, dr)
    assert ref[0][1] == o.iterations


def _index_ladder_pair(n_words, seed=0):
    """Leaf-1.0 target whose rank index has exactly n_words words: 8-point leaves at cell 0, the last cell, both sides of
    each 16 KB TMA chunk edge (word 2048 k) and of the 64 KB limit, and 300 random cells; the source is its points
    jittered by 0.05."""
    rng = np.random.default_rng(seed + n_words)
    dims = R.dims_for_words(n_words)
    n_cells = dims[0] * dims[1] * dims[2]
    edges = [c for w in (2048, 4096, 6144, 8192) for c in (32 * w - 1, 32 * w)]
    cells = [c for c in [0, n_cells - 1] + edges if c < n_cells] + rng.integers(0, n_cells, 300).tolist()
    tgt = np.concatenate([R.word_anchors(dims)] + [R.cell_points(R.cell_of_index(c, dims), 1.0, 8, rng) for c in cells])
    src = (tgt[2:] + rng.normal(0, 0.05, (len(tgt) - 2, 3))).astype(F32)
    return src, tgt.astype(F32)


@pytest.mark.parametrize("n_words", [1, 2047, 2048, 2049, 8192, 8193])
def test_rank_index_ladder(b200, n_sms, n_words):
    """The solver stages the rank index into shared memory in 16 KB TMA chunks up to 64 KB (8192 words) and reads it from
    global memory above that; both must score the same pairs."""
    src, tgt = _index_ladder_pair(n_words)
    assert R.leaf_geometry(tgt, 1.0)["n_words"] == n_words
    worst = 0.0
    for method in (2, 0):
        g = _ndt(b200, tgt, src, 1.0, method)
        for p in (np.zeros(6), np.array([0.02, -0.01, 0.01, 0.0005, -0.0004, 0.0008])):
            worst = max(worst, _check(g, src, tgt, 1.0, method, p, True, n_sms, ("index", n_words, method)))
        assert g.stats()["index_in_smem"] == (1 if n_words <= 8192 else 0), n_words
    print(f"\nmax |K1 - ref| / bound, rank index of {n_words} words: {worst:.3g}")


def test_stale_accumulators(b200, n_sms):
    """One handle evaluates a pose where every CTA hits, then a pose where whole threads and CTAs miss, with the Hessian
    off and on in turn: each result must equal a fresh handle's bit for bit, and a pose where nothing hits gives exact
    zeros."""
    import oracle
    from lidarslam_ros2_b200 import synth

    _, tgt, _ = synth.registration_pair("small", 2.0)
    rng = np.random.default_rng(5)
    src = tgt[rng.choice(len(tgt), 12000, replace=False)]
    src = np.ascontiguousarray(src[np.argsort(src[:, 0])] + rng.normal(0, 0.02, src.shape).astype(F32), dtype=F32)
    span = float(src[:, 0].max() - src[:, 0].min())
    p_in, p_out, p_none = np.zeros(6), np.array([0.8 * span, 0, 0, 0, 0, 0]), np.array([1e4, 0, 0, 0, 0, 0])
    g = _ndt(b200, tgt, src)
    geom, v = R.leaf_geometry(tgt, 2.0), g.voxels()
    rank, tid, rows = N.point_owner(len(src), n_sms)
    per_cta = {}
    for name, p in (("in", p_in), ("out", p_out)):
        hits = N.per_point_hits(src, oracle.pose_to_matrix(p)[:3], 2.0, v, geom)
        per_cta[name] = np.bincount(rank, weights=hits, minlength=rows)
        per_thread = np.bincount(rank * 768 + tid, weights=hits)
        if name == "out":
            assert (per_thread[np.bincount(rank * 768 + tid) > 0] == 0).any()
    assert (per_cta["in"] > 0).all() and (per_cta["out"] == 0).any() and (per_cta["out"] > 0).any()
    seq = [(p_in, True), (p_out, True), (p_out, False), (p_in, False), (p_out, True), (p_none, True), (p_in, True),
           (p_none, False)]
    for p, hess in seq:
        T = oracle.pose_to_matrix(p)
        a = g.derivatives(T, p, hess)
        ha = g.stats()["hits"]
        fresh = _ndt(b200, tgt, src)
        b = fresh.derivatives(T, p, hess)
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), (p, hess)
        assert ha == fresh.stats()["hits"]
        if p is p_none:
            assert a[0] == 0 and np.all(a[1] == 0) and np.all(a[2] == 0) and ha == 0
        else:
            _check(g, src, tgt, 2.0, 2, p, hess, n_sms, ("stale", p[0], hess))
