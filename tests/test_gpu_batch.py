"""GPU tests of the batched NDT entry points (b200reg_ndt_align_batch / _device, b200reg_align_batch) and of
b200reg_get_aligned. A batched registration must be BITWISE the registration b200reg_align performs for the same
(source, guess): the batch kernel keeps the point partition and every summation order of the single launch."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


def _engine(m, tgt, res=2.0, max_it=35):
    g = m.NormalDistributionsTransform()
    g.setResolution(res)
    g.setTransformationEpsilon(0.01)
    g.setMaximumIterations(max_it)
    g.setNeighborhoodSearchMethod(m.DIRECT7)
    g.setInputTarget(tgt)
    return g


def _scans_and_guesses(src, n):
    """n different (scan, guess) problems from one scan: sub-sampled / perturbed copies and perturbed guesses."""
    from lidarslam_ros2_b200 import synth

    rng = np.random.default_rng(7)
    scans, guesses = [], []
    d = np.pi / 180
    for k in range(n):
        keep = rng.random(len(src)) < (1.0 - 0.07 * (k % 4))  # ragged sizes
        s = src[keep].copy()
        s[:, :3] += rng.normal(0, 0.004, size=(len(s), 3)).astype(np.float32)
        scans.append(np.ascontiguousarray(s[:, :3]))
        guesses.append(synth.pose_matrix((0.05 * (k % 3), -0.04 * (k % 2), 0.0), (0, 0, 0.3 * d * (k % 5))).astype(np.float32))
    return scans, guesses


def _single(g, scans, guesses):
    out = []
    for s, T in zip(scans, guesses):
        g.setInputSource(s)
        P = g.align(T)
        out.append((P, g.getFinalNumIteration(), g.hasConverged(), g.getTransformationProbability(), g.stats()["evaluations"]))
    return out


@pytest.mark.parametrize("config,res", [("small", 2.0), ("c1", 5.0)])
def test_batch_equals_single_bitwise(b200, config, res):
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair(config, res)
    g = _engine(b200, tgt, res)
    scans, guesses = _scans_and_guesses(src, 9)
    ref = _single(g, scans, guesses)
    for slots in (3, 2, 1):
        g.setBatchSlots(slots)
        r = g.alignBatch(scans, guesses)
        assert np.all(r["status"] == 0)
        for k, (P, it, conv, tp, ev) in enumerate(ref):
            assert np.array_equal(r["pose"][k], P), (slots, k, np.abs(r["pose"][k] - P).max())
            assert r["iterations"][k] == it and bool(r["converged"][k]) == conv and r["evaluations"][k] == ev
            assert r["trans_probability"][k] == tp
    # the handle's getters describe the last registration of the batch
    assert np.array_equal(g.getFinalTransformation(), ref[-1][0])
    assert g.stats()["evaluations"] == sum(x[4] for x in ref)


def test_batch_device_sources_and_identity_guess(b200):
    import torch

    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("small", 2.0)
    g = _engine(b200, tgt)
    scans, _ = _scans_and_guesses(src, 5)
    ref = _single(g, scans, [None] * len(scans))
    dev = [torch.from_numpy(np.concatenate([s, np.ones((len(s), 1), np.float32)], axis=1)).cuda() for s in scans]
    torch.cuda.synchronize()
    r = g.alignBatchDevice([d.data_ptr() for d in dev], [d.shape[0] for d in dev])
    for k, (P, it, conv, tp, ev) in enumerate(ref):
        assert np.array_equal(r["pose"][k], P) and r["iterations"][k] == it
    # one registration, and an empty batch
    r1 = g.alignBatchDevice([dev[2].data_ptr()], [dev[2].shape[0]])
    assert np.array_equal(r1["pose"][0], ref[2][0])
    r0 = g.alignBatch([])
    assert r0["pose"].shape == (0, 4, 4)


def test_batch_fallback_configurations(b200):
    """step_max <= step_min runs the More-Thuente inner loop (K2 passes): the batch entry serves it one by one."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("tiny", 2.0)
    g = _engine(b200, tgt)
    g.setStepSize(0.004)  # < transformation_epsilon / 2
    scans, guesses = _scans_and_guesses(src, 3)
    ref = _single(g, scans, guesses)
    r = g.alignBatch(scans, guesses)
    for k, (P, it, conv, tp, ev) in enumerate(ref):
        assert np.array_equal(r["pose"][k], P) and r["iterations"][k] == it
    # no target: soft failure like align()
    e = b200.NormalDistributionsTransform()
    r = e.alignBatch(scans[:1])
    assert r["status"][0] != 0 or not r["converged"][0]


def test_align_batch_over_handles(b200, oracle_mod):
    """b200reg_align_batch: independent handles (different targets), every result == the handle's own align()."""
    from lidarslam_ros2_b200 import synth

    engines, refs = [], []
    for cfg, res in (("tiny", 2.0), ("small", 2.0), ("small", 5.0)):
        src, tgt, _ = synth.registration_pair(cfg, 2.0)
        g = _engine(b200, tgt, res)
        g.setInputSource(src)
        refs.append(g.align())
        engines.append(g)
    out = b200.align_batch(engines)
    for k in range(len(engines)):
        assert np.array_equal(out[k], refs[k])
        assert np.array_equal(engines[k].getFinalTransformation(), refs[k])


def test_get_aligned_matches_transformed_source(b200, oracle_mod, pair_small):
    """b200reg_get_aligned = the `output` cloud of align(): source moved by the final transformation in un-fused float
    arithmetic ((m0*x + m1*y) + m2*z) + m3, the solver's own definition of transformPointCloud."""
    src, tgt, _ = pair_small
    g = _engine(b200, tgt)
    g.setInputSource(src)
    T = g.align()
    out = g.getAligned()
    p = src[:, :3].astype(np.float32)
    R, t = T[:3, :3].astype(np.float32), T[:3, 3].astype(np.float32)
    ref = np.empty_like(p)
    for r in range(3):
        ref[:, r] = ((R[r, 0] * p[:, 0] + R[r, 1] * p[:, 1]) + R[r, 2] * p[:, 2]) + t[r]
    assert out.shape == (len(src), 4)
    np.testing.assert_array_equal(out[:, :3], ref)
    assert np.all(out[:, 3] == 1.0)
    # and against the oracle's transformed cloud
    o = oracle_mod.NDT(resolution=2.0, transformation_epsilon=0.01)
    o.set_target(tgt)
    o.set_source(src)
    To = o.align()
    refo = (To[:3, :3].astype(np.float64) @ p.T.astype(np.float64)).T + To[:3, 3]
    assert np.abs(out[:, :3] - refo).max() < 1e-3


def test_sweep_equals_sequential_pairs(b200):
    """b200reg_ndt_sweep (up to four engines / host threads, pairs dealt round-robin) == the same pairs through setInputTarget + setInputSource + align +
    getFitnessScore one after the other, bitwise (each pair is computed by exactly the same kernels on the same inputs)."""
    from lidarslam_ros2_b200 import batch, synth

    srcs, tgts, idx = [], [], []
    for k, (cfg, res) in enumerate((("small", 2.0), ("tiny", 2.0), ("c1", 2.0), ("small", 2.0), ("tiny", 2.0))):
        s, t, _ = synth.registration_pair(cfg, 2.0)
        rng = np.random.default_rng(k)
        srcs.append((s + rng.normal(0, 0.003, size=s.shape)).astype(np.float32))
        tgts.append(t)
        idx.append(10 + k)
    sw = batch.LoopSweep(b200, device=0, resolution=2.0, max_iterations=100)
    a = sw.run_sequential(srcs, tgts, idx)
    for _ in range(2):
        b = sw.run(srcs, tgts, idx)
        np.testing.assert_array_equal(a, b)
    assert sw.run([], [], []).shape == (0, batch.ROW)


def test_comm_all_gather_world1(b200):
    """include/b200comm.h on one GPU: ncclGetUniqueId + ncclCommInitRank(world 1) + ncclAllGather through the C entry points
    (the N > 1 path is the same call; bench.py --gpus N exercises it)."""
    import ctypes as C

    from lidarslam_ros2_b200 import _capi

    L = _capi.lib()
    ident = (C.c_ubyte * 128)()
    assert L.b200comm_unique_id(ident) == 0, L.b200comm_last_error()
    h = C.c_void_p()
    assert L.b200comm_create(ident, 0, 1, 0, C.byref(h)) == 0, L.b200comm_last_error()
    rows = np.arange(3 * 20, dtype=np.float32).reshape(3, 20)
    out = np.zeros_like(rows)
    assert L.b200comm_all_gather_rows(h, rows.ctypes.data, 3, 20, out.ctypes.data) == 0, L.b200comm_last_error()
    np.testing.assert_array_equal(out, rows)
    r, w = C.c_int(-1), C.c_int(-1)
    assert L.b200comm_rank(h, C.byref(r), C.byref(w)) == 0 and (r.value, w.value) == (0, 1)
    assert L.b200comm_destroy(h) == 0


def test_voxelgrid_sparse_index_equals_dense(b200, oracle_mod):
    """pcl::VoxelGrid on a bounding box too large for a dense occupancy bitmap: the two-level sparse rank index (O(points)
    memory) must give the dense path's output — same leaves in the same (ascending leaf index) order — and the oracle's."""
    import ctypes as C

    from lidarslam_ros2_b200 import _capi, synth

    src, _, _ = synth.registration_pair("c1", 2.0)
    pts = np.concatenate([src[:, :3], np.linspace(0, 1, len(src), dtype=np.float32)[:, None]], axis=1)
    L = _capi.lib()
    L.b200reg_debug_set_voxelgrid_dense_budget.argtypes = [C.c_size_t]
    try:
        for leaf in (0.5, 0.05):
            L.b200reg_debug_set_voxelgrid_dense_budget(4 << 20)
            dense = b200.voxel_grid_filter(pts, leaf)
            L.b200reg_debug_set_voxelgrid_dense_budget(0)
            sparse = b200.voxel_grid_filter(pts, leaf)
            assert dense.shape == sparse.shape and len(dense) > 100
            np.testing.assert_allclose(sparse, dense, rtol=0, atol=1e-6)
            ref = oracle_mod.voxelgrid(pts, leaf)
            assert ref.shape == sparse.shape
            np.testing.assert_allclose(sparse, ref, atol=5e-5)
    finally:
        L.b200reg_debug_set_voxelgrid_dense_budget(4 << 20)


def test_nn_far_queries_exact(b200):
    """Exact 1-NN for queries the ring search cannot resolve (far outside the target's bounding box, or deep inside an empty
    region): the coarse-level pass of nn_grid.cu must return the brute-force answer — same index (lower index on ties) and
    the same un-fused float32 squared distance."""
    from lidarslam_ros2_b200 import synth

    _, tgt, _ = synth.registration_pair("small", 2.0)
    tgt = np.ascontiguousarray(tgt[:, :3])
    tgt[100] = tgt[7]  # an exact duplicate: the lower index must win
    rng = np.random.default_rng(3)
    lo, hi = tgt.min(axis=0), tgt.max(axis=0)
    inside = rng.uniform(lo, hi, size=(300, 3))
    inside[:, 2] += 25.0  # high above the scene: empty space, still inside the x/y extent
    outside = rng.uniform(lo - 400.0, hi + 400.0, size=(700, 3))
    near = tgt[rng.integers(0, len(tgt), 200)] + rng.normal(0, 0.05, size=(200, 3))
    q = np.concatenate([inside, outside, near, tgt[7:8]]).astype(np.float32)
    g = b200.NormalDistributionsTransform()
    g.setInputTarget(tgt)
    idx, d2 = g.nearest(q)
    d = q[:, None, :] - tgt[None, :, :]                       # float32, un-fused like FLANN's L2_Simple
    ref = (d[:, :, 0] * d[:, :, 0] + d[:, :, 1] * d[:, :, 1]) + d[:, :, 2] * d[:, :, 2]
    ridx = ref.argmin(axis=1)                                 # first minimum = lowest index
    np.testing.assert_array_equal(idx, ridx)
    np.testing.assert_array_equal(d2, ref[np.arange(len(q)), ridx])
    assert idx[-1] == 7
