"""The NDT batch solver (b200reg_ndt_align_batch / _device) at its scheduling edges, and the pose scorer K12
(b200reg_ndt_score_poses) at its evaluation edges. Run on an H100 with -m gpu.

Batch: every registration of a batch call must be bit for bit the align() of the same (source, guess) on a handle with
the same target and configuration (ndt_solver.cuh): final_T, converged, iterations, evaluations, trans_probability,
hits_total and status. After the call the handle's getters describe the last registration and stats() sums evaluations
and hits over the batch. The fixtures (tests/ndtbatchref.py) put a ladder-top scan next to a 1-point scan on one slot,
equal-size scans with different points one after the other, registrations that leave the fast controller among
ordinary ones, every host record stride with garbage past x, y, z, pinned and pageable sources (one of 9.6 MB), the
streaming upload and the unpack path, calls cut into several launches, a jobs table that grows, a rank index in and out
of shared memory, and the targets that send a batch down the one-by-one path.

K12: every score within the float64 reference's bound (tests/ndtref.py, compute_hessian=False) with the hit count exact
and equal to derivatives()'s at the same pose, over multi-tile scans, km offsets, ill-conditioned voxels, pitch poses,
leaf-edge sources, non-finite and huge rows, and the KDTREE escape and equality fixtures of tests/radiusref.py."""
import numpy as np
import pytest

import gridref as R
import ndtbatchref as B
import ndtctl_ref as X
import ndtref as N
import radiusref as RR
import test_gpu_ndt_controller as TC
import test_gpu_ndt_eval as TE

pytestmark = pytest.mark.gpu

F32 = np.float32
METHODS = [(2, "DIRECT7"), (3, "DIRECT1"), (1, "DIRECT26"), (0, "KDTREE")]


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
def big_scan():
    """The headline target (1M points) and its scan tiled to 305k points."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("headline", 2.0)
    return B.tiled_scan(src, B.PAGEABLE_POINTS + 5000), tgt


def _ndt(b200, tgt, method=2, res=2.0, max_it=10, eps=0.01, step=None):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setTransformationEpsilon(eps)
    g.setMaximumIterations(max_it)
    g.setNeighborhoodSearchMethod(method)
    if step is not None:
        g.setStepSize(step)
    g.setInputTarget(tgt)
    return g


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32)


def _align_rc(g, guess):
    """align() with its status code (the Python wrapper raises on a hard error)."""
    from lidarslam_ros2_b200.registration import B200RegError

    try:
        return g.align(guess), 0
    except B200RegError as e:
        return g.getFinalTransformation(), e.code


def _single(g, jobs):
    """align() of every (points, guess) on g, one after the other."""
    out = []
    for pts, G in jobs:
        g.setInputSource(pts)
        P, rc = _align_rc(g, G)
        st = g.stats()
        out.append(dict(pose=P, iterations=g.getFinalNumIteration(), converged=g.hasConverged(),
                        evaluations=st["evaluations"], tp=g.getTransformationProbability(), hits=st["hits_total"], status=rc))
    return out


def _check(g, r, ref, what):
    """A batch result against align()'s, field by field and bit for bit, and the handle's state after the call."""
    assert len(r["pose"]) == len(ref), what
    for k, a in enumerate(ref):
        w = (what, k)
        assert np.array_equal(_bits(r["pose"][k]), _bits(a["pose"])), (w, np.abs(r["pose"][k] - a["pose"]).max())
        assert r["iterations"][k] == a["iterations"] and bool(r["converged"][k]) == a["converged"], w
        assert r["evaluations"][k] == a["evaluations"] and r["hits_total"][k] == a["hits"], (w, r["hits_total"][k], a["hits"])
        assert _bits(np.float64(r["trans_probability"][k])) == _bits(np.float64(a["tp"])), w
        assert r["status"][k] == a["status"], w
    last = ref[-1]
    assert np.array_equal(_bits(g.getFinalTransformation()), _bits(last["pose"])), what
    assert g.getFinalNumIteration() == last["iterations"] and g.hasConverged() == last["converged"], what
    assert _bits(np.float64(g.getTransformationProbability())) == _bits(np.float64(last["tp"])), what
    st = g.stats()
    assert st["evaluations"] == sum(a["evaluations"] for a in ref), what
    assert st["hits_total"] == sum(a["hits"] for a in ref), what


def _device(clouds):
    import torch

    dev = [torch.from_numpy(np.c_[c[:, :3], np.ones(len(c), F32)]).cuda() for c in clouds]
    torch.cuda.synchronize()
    return dev


def _batch_device(g, dev, guesses):
    return g.alignBatchDevice([d.data_ptr() for d in dev], [d.shape[0] for d in dev], guesses)


# ---- 1. mixed sizes, every method ------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_mixed_sizes_every_method(b200, n_sms, big_scan, method):
    """The size ladder, the top job directly before and after a 1-point job, 65 jobs, on 1 to 4 slots (4 is clamped to
    3), from host records and from device buffers."""
    scan, tgt = big_scan
    sizes = B.size_ladder(n_sms)
    jobs = B.ladder_jobs(scan, sizes, B.ladder_order(sizes), B.ordinary_guesses(7, seed=method))
    assert len(jobs) >= 64
    g = _ndt(b200, tgt, method, max_it=8)
    ref = _single(g, jobs)
    assert all(a["status"] == 0 for a in ref)
    clouds, guesses = [p for p, _ in jobs], [G for _, G in jobs]
    dev = _device(clouds)
    for slots in (1, 2, 3, 4):
        g.setBatchSlots(slots)
        _check(g, g.alignBatch(clouds, guesses), ref, (method, slots, "host"))
        _check(g, _batch_device(g, dev, guesses), ref, (method, slots, "device"))


def test_same_size_jobs_with_different_points(b200, n_sms, big_scan):
    """Each ladder size twice in a row with the same guess, the second scan a jittered or row-rotated copy of the first:
    a slot that kept the first scan's staged points would return the first result for the second."""
    scan, tgt = big_scan
    sizes = B.size_ladder(n_sms)
    pairs = B.same_size_pairs(scan, sizes, seed=5)
    guesses = B.ordinary_guesses(len(pairs), seed=9)
    jobs = [(x, guesses[k]) for k, (a, b) in enumerate(pairs) for x in (a, b)]
    g = _ndt(b200, tgt, 2, max_it=8)
    ref = _single(g, jobs)
    differ = [not np.array_equal(_bits(ref[2 * k]["pose"]), _bits(ref[2 * k + 1]["pose"])) or
              ref[2 * k]["hits"] != ref[2 * k + 1]["hits"] for k in range(len(pairs))]
    # the comparison can see a stale slot: the jittered pairs (and most rotated ones) register differently
    assert all(d for k, d in enumerate(differ) if k % 2 and sizes[k] >= 128) and sum(differ) > len(pairs) // 2, differ
    clouds, gs = [p for p, _ in jobs], [G for _, G in jobs]
    dev = _device(clouds)
    for slots in (1, 2, 3):
        g.setBatchSlots(slots)
        _check(g, g.alignBatch(clouds, gs), ref, ("same size", slots, "host"))
        _check(g, _batch_device(g, dev, gs), ref, ("same size", slots, "device"))


# ---- 2. controller edges inside a batch --------------------------------------------------------------------------------
def _replay(b200, src, tgt, res, guess, cfg, batch_row):
    """Trace the single align() of (src, guess), replay it round by round with test_gpu_ndt_controller's checks, and
    tie the traced result to the batch's."""
    tg = TC._ndt(b200, src, tgt, res, 2, cfg)
    recs = TC._traced_align(tg, guess)
    TC._check_bookkeeping(tg, recs, len(src))
    assert TC._check_control_blocks(recs) == 0
    w, _, _ = TC._check_steps(recs, cfg, guess)
    assert np.array_equal(_bits(tg.getFinalTransformation()), _bits(batch_row["pose"]))
    assert tg.stats()["hits_total"] == batch_row["hits"] and tg.getFinalNumIteration() == batch_row["iterations"]
    return w, recs


def test_controller_edges_inside_a_batch(b200, oracle_mod, golden, pair_small):
    """Zero hits (10 km away), ascent and snap rounds, a singular Hessian (the origin source) and the iteration cap, each
    among ordinary registrations: every slot moves on and every result is align()'s. A sample is traced through align()
    and replayed in float64, which closes the chain batch -> single launch -> replay."""
    cfg = X.config()
    gs, gt = golden["source"], golden["target"]
    edge = B.controller_edge_guesses()
    ordinary = B.ordinary_guesses(len(edge), seed=11)
    guesses = [G for pair in zip(ordinary, edge) for G in pair]
    jobs = [(gs, G) for G in guesses]
    g = _ndt(b200, gt, 2, res=1.0, max_it=cfg["max_iterations"], eps=cfg["trans_eps"], step=cfg["step_size"])
    ref = _single(g, jobs)
    far = ref[2 * (len(edge) - 1) + 1]
    assert far["hits"] == 0 and far["iterations"] == 0 and far["evaluations"] == 1 and far["converged"]
    for slots in (1, 2, 3):
        g.setBatchSlots(slots)
        _check(g, g.alignBatch([p for p, _ in jobs], guesses), ref, ("golden edges", slots))
    o = oracle_mod.NDT(resolution=1.0, num_threads=1)
    o.set_target(gt)
    o.set_source(gs)
    worst = {}
    sample = {"far": B.far_guess(), "ascent": X.first_with(o, cfg, X.ascent_guesses(), len(gs), X.is_ascent_round),
              "snap": X.first_with(o, cfg, X.edge_guesses(), len(gs), X.is_snap_round)}
    for name, G in sample.items():
        assert G is not None, name
        k = next(i for i, x in enumerate(guesses) if np.array_equal(x, G))
        worst[name], _ = _replay(b200, gs, gt, 1.0, G, cfg, ref[k])
    # the origin source (LDL^T refuses, pivoted LU fails) among ordinary registrations on the same target
    osrc, otgt = X.origin_pair()
    rng = np.random.default_rng(4)
    plain = [(otgt[rng.choice(len(otgt), 400, replace=False)] + rng.normal(0, 0.02, (400, 3))).astype(F32) for _ in range(3)]
    ojobs = [(plain[0], np.eye(4, dtype=F32)), (osrc, np.eye(4, dtype=F32)), (plain[1], ordinary[0]),
             (osrc, ordinary[1]), (plain[2], np.eye(4, dtype=F32))]
    go = _ndt(b200, otgt, 2, res=2.0, max_it=cfg["max_iterations"], eps=cfg["trans_eps"], step=cfg["step_size"])
    oref = _single(go, ojobs)
    for slots in (1, 2, 3):
        go.setBatchSlots(slots)
        _check(go, go.alignBatch([p for p, _ in ojobs], [G for _, G in ojobs]), oref, ("origin", slots))
    worst["origin"], recs = _replay(b200, osrc, otgt, 2.0, np.eye(4, dtype=F32), cfg, oref[1])
    assert (recs["fast"] == 0).any()
    # the iteration cap: max_iterations 1 and 2, identity guesses among perturbed ones
    src, tgt, _ = pair_small
    for m in B.EDGE_MAX_ITERATIONS:
        c = X.config(max_iterations=m)
        cg = [np.eye(4, dtype=F32)] + B.ordinary_guesses(4, seed=m) + [np.eye(4, dtype=F32)]
        gm = _ndt(b200, tgt, 2, max_it=m, eps=c["trans_eps"], step=c["step_size"])
        mref = _single(gm, [(src, G) for G in cg])
        assert mref[0]["iterations"] == m + 2 and mref[-1]["iterations"] == m + 2
        for slots in (1, 2, 3):
            gm.setBatchSlots(slots)
            _check(gm, gm.alignBatch([src] * len(cg), cg), mref, ("cap", m, slots))
        worst[f"cap {m}"], _ = _replay(b200, src, tgt, 2.0, np.eye(4, dtype=F32), c, mref[0])
    print("\ncontroller edges in a batch, max step deviation / bound of the replayed align(): "
          + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


# ---- 3. strides and uploads ----------------------------------------------------------------------------------------------
def test_strides_and_uploads(b200, n_sms, big_scan):
    """Every record stride with garbage past x, y, z, pinned and pageable, the 9.6 MB pageable scan (four staging
    threads), the streaming upload (4 registrations, one launch) and the unpack path (6 registrations, two launches),
    device buffers, and a prepared call whose arrays are rewritten in place between two calls."""
    scan, tgt = big_scan
    e = B.n_eval(n_sms)
    cap = B.staging_capacity(e)
    sizes = [B.PAGEABLE_POINTS, 1, 5000, 777, 128 * e + 1, cap + 33]
    clouds = [np.ascontiguousarray(scan[k * 997:k * 997 + n]) for k, n in enumerate(sizes)]
    guesses = B.ordinary_guesses(len(clouds), seed=21)
    max_it = B.CHUNK_MAX_ITERATIONS[4]
    g = _ndt(b200, tgt, 2, max_it=max_it)
    ref = _single(g, list(zip(clouds, guesses)))
    assert all(a["converged"] and a["iterations"] < 100 for a in ref), [a["iterations"] for a in ref]
    pl = B.per_launch(max_it)
    assert len(clouds) > pl == 4
    for stride in B.STRIDES:
        for pinned in (False, True):
            recs = [B.records(c, stride, seed=k, pinned=pinned) for k, c in enumerate(clouds)]
            if not pinned:
                assert recs[0].nbytes >= B.FOUR_THREAD_BYTES or stride < 32
            for n in (pl, len(clouds)):  # streaming, then unpack
                _check(g, g.alignBatch(recs[:n], guesses[:n]), ref[:n], (stride, pinned, n))
    dev = _device(clouds)
    _check(g, _batch_device(g, dev, guesses), ref, "device")
    # prepared calls, arrays rewritten in place: the second call registers the new contents
    new = [b for _, b in B.same_size_pairs(np.concatenate([scan[3:], scan[:3]]), sizes, seed=8)]
    nref = _single(g, list(zip(new, guesses)))
    for stride, pinned in ((32, False), (16, True), (12, False)):
        for n in (pl, len(clouds)):
            recs = [B.records(c, stride, seed=k, pinned=pinned) for k, c in enumerate(clouds[:n])]
            call = g.prepareBatch(recs, guesses[:n])
            _check(g, call(), ref[:n], ("prepared", stride, pinned, n))
            for r, c in zip(recs, new[:n]):
                r[:, :3] = c
            _check(g, call(), nref[:n], ("prepared, rewritten", stride, pinned, n))


# ---- 4. several launches per call -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pl", sorted(B.CHUNK_MAX_ITERATIONS))
def test_several_launches_per_call(b200, pair_small, pl):
    """max_iterations of 14996, 29996 and 59996 cut a call into launches of 4, 2 and 1 registrations: counts one short of,
    at and past a launch, and three launches and one, from host records (streaming up to one launch, unpack beyond)
    and device buffers. The scenes converge long before the cap."""
    src, tgt, _ = pair_small
    max_it = B.CHUNK_MAX_ITERATIONS[pl]
    assert B.per_launch(max_it) == pl
    rng = np.random.default_rng(pl)
    n_jobs = max(B.launch_counts(pl))
    clouds = [np.ascontiguousarray(src[rng.random(len(src)) < 0.7 + 0.05 * (k % 5)] + F32(0.001 * k)) for k in range(n_jobs)]
    guesses = B.ordinary_guesses(n_jobs, seed=30 + pl)
    g = _ndt(b200, tgt, 2, max_it=max_it)
    ref = _single(g, list(zip(clouds, guesses)))
    assert all(a["converged"] and a["iterations"] < 100 for a in ref), [a["iterations"] for a in ref]
    dev = _device(clouds)
    for count in B.launch_counts(pl):
        for slots in (1, 3):
            g.setBatchSlots(slots)
            _check(g, g.alignBatch(clouds[:count], guesses[:count]), ref[:count], (pl, count, slots, "host"))
            _check(g, _batch_device(g, dev[:count], guesses[:count]), ref[:count], (pl, count, slots, "device"))


# ---- 5. handle state ------------------------------------------------------------------------------------------------------
def test_handle_state_between_batches(b200, pair_small):
    """One handle: a batch of 3, of 200 (the jobs table grows), of 3, with align(), derivatives(), scorePoses() and
    setTrace() in between, then targets whose rank index has 8192 and 8193 words (in and out of shared memory): every
    batch equals a fresh handle's bit for bit."""
    import oracle

    src, tgt, _ = pair_small
    rng = np.random.default_rng(12)
    clouds = [np.ascontiguousarray(src[rng.random(len(src)) < 0.8] + F32(0.002 * (k % 7))) for k in range(200)]
    guesses = B.ordinary_guesses(len(clouds), seed=13)

    def fresh(t, cs, gs, res=2.0):
        f = _ndt(b200, t, 2, res=res, max_it=35)
        return f.alignBatch(cs, gs)

    def same(a, b, what):
        for key in ("pose", "iterations", "converged", "evaluations", "hits_total", "status"):
            assert np.array_equal(a[key], b[key]), (what, key)
        assert np.array_equal(_bits(a["trans_probability"]), _bits(b["trans_probability"])), what

    g = _ndt(b200, tgt, 2, max_it=35)
    same(g.alignBatch(clouds[:3], guesses[:3]), fresh(tgt, clouds[:3], guesses[:3]), "3")
    g.setInputSource(src)
    P = g.align(guesses[5])
    p6 = np.array([0.1, -0.05, 0.02, 0.003, -0.002, 0.01])
    g.derivatives(oracle.pose_to_matrix(p6), p6, True)
    g.scorePoses(np.stack([P, np.eye(4, dtype=F32)]))
    g.setTrace(64)
    same(g.alignBatch(clouds, guesses), fresh(tgt, clouds, guesses), "200")
    assert np.array_equal(g.align(guesses[5]), P)  # the handle's own source is still the one it was given
    g.setTrace(0)
    same(g.alignBatch(clouds[-3:], guesses[-3:]), fresh(tgt, clouds[-3:], guesses[-3:]), "3 after 200")
    g.setResolution(1.0)
    for n_words in (8192, 8193):
        s_i, t_i = TE._index_ladder_pair(n_words)
        cs = [np.ascontiguousarray(s_i[k::3]) for k in range(3)]
        gi = B.ordinary_guesses(3, seed=n_words)
        gi = [np.eye(4, dtype=F32)] + [G for G in gi[1:]]
        g.setInputTarget(t_i)
        a = g.alignBatch(cs, gi)
        assert g.stats()["index_in_smem"] == (1 if n_words <= 8192 else 0), n_words
        same(a, fresh(t_i, cs, gi, res=1.0), ("index", n_words))


# ---- 6. the one-by-one path ---------------------------------------------------------------------------------------------------
def test_sequential_fallbacks(b200, pair_small):
    """A target whose leaves all hold fewer than six points (an empty map) and a More-Thuente configuration send a
    batch down the one-by-one path: every result is align()'s, status included, and the handle keeps its own source."""
    src, tgt, _ = pair_small
    rng = np.random.default_rng(14)
    clouds = [np.ascontiguousarray(src[rng.random(len(src)) < 0.6]) for _ in range(4)]
    guesses = B.ordinary_guesses(4, seed=15)
    for what, t, step in (("empty map", tgt[::400][:40] * F32(30.0), None), ("More-Thuente", tgt, 0.004)):
        g = _ndt(b200, t, 2, max_it=6, step=step)
        if what == "empty map":
            assert g.voxels()["idx"].size == 0
        ref = _single(g, list(zip(clouds, guesses)))
        if what == "empty map":
            assert all(np.array_equal(a["pose"], G) and a["converged"] and a["evaluations"] == 1
                       for a, G in zip(ref, guesses))
        g.setInputSource(src)
        own = g.align(guesses[0])
        for slots in (1, 3):
            g.setBatchSlots(slots)
            _check(g, g.alignBatch(clouds, guesses), ref, (what, slots, "host"))
            _check(g, _batch_device(g, _device(clouds), guesses), ref, (what, slots, "device"))
            assert np.array_equal(g.align(guesses[0]), own), what
            assert np.array_equal(g.getAligned()[:, :3], N.transform_points(own[:3], src)), what


# ---- 7. K12 at its edges --------------------------------------------------------------------------------------------------
def _score_check(g, src, tgt, res, method, poses, what, hits_exact=True):
    """scorePoses at each pose against the float64 reference and against derivatives()'s hits; returns the largest
    |score - ref| / bound and the hit counts."""
    import oracle

    poses = [np.asarray(p, dtype=np.float64) for p in poses]
    Ts = np.stack([oracle.pose_to_matrix(p) for p in poses]).astype(F32)
    scores, hits = g.scorePoses(Ts)
    v, geom = g.voxels(), R.leaf_geometry(tgt, res)
    worst = 0.0
    for k, p in enumerate(poses):
        ref = N.derivatives(src, Ts[k][:3], p, res, v, geom, method, compute_hessian=False)
        if hits_exact:
            assert ref["near_threshold"] == 0, (what, k)
            assert hits[k] == ref["hits"], (what, k, hits[k], ref["hits"])
        tol = ref["tol_score"]
        assert scores[k] == ref["score"] or abs(scores[k] - ref["score"]) <= tol, (what, k, scores[k], ref["score"], tol)
        if tol:
            worst = max(worst, abs(scores[k] - ref["score"]) / tol)
        g.derivatives(Ts[k], p, False)
        assert g.stats()["hits"] == hits[k], (what, k)
    return worst, hits


def _scorer(b200, tgt, src, res, method):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setNeighborhoodSearchMethod(method)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    return g


@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_scores_at_the_edges(b200, big_scan, method):
    worst = {}
    poses = [np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02])]
    # scans on both sides of the tile multiples, and about a hundred tiles. The hit counts are compared exactly, so
    # _score_check asserts that the reference finds no pair within a few ulp of the e2 gate or of the KDTREE radius
    # (near_threshold == 0); a scan or pose that put one there would fail loudly, not be skipped.
    scan, tgt = big_scan
    g = None
    for n in B.tile_sizes():
        src = np.ascontiguousarray(scan[:n])
        if g is None:
            g = _scorer(b200, tgt, src, 2.0, method)
        else:
            g.setInputSource(src)
        w, _ = _score_check(g, src, tgt, 2.0, method, poses if n < 10000 else poses[1:], ("tiles", n))
        worst["tiles"] = max(worst.get("tiles", 0.0), w)
    # km offsets and ill-conditioned voxels, with pitch poses
    from lidarslam_ros2_b200 import synth

    s_src, s_tgt = synth.registration_pair("small", 2.0)[:2]
    for name, (src, t), off in (("shifted", N.shifted_pair(s_src, s_tgt), N.SHIFT),
                                ("illconditioned", N.illconditioned_pair(), (0.0, 0.0, 0.0))):
        ps = []
        for p in poses + N.pitch_poses():
            p = np.array(p, dtype=np.float64)
            p[:3] += off
            ps.append(p)
        w, _ = _score_check(_scorer(b200, t, src, 2.0, method), src, t, 2.0, method, ps, name)
        worst[name] = w
    # leaf-edge sources at the identity and one ulp either way
    for res in (0.3, 0.1):
        src, t = B.leaf_edge_source(res)
        for u in (0, -1, 1):
            s = B.nudged(src, u)
            w, h = _score_check(_scorer(b200, t, s, res, method), s, t, res, method, [np.zeros(6)], ("leaf edge", res, u))
            assert h[0] > 0
            worst["leaf edge"] = max(worst.get("leaf edge", 0.0), w)
    # non-finite and +-1e12 rows: the same hits as the clean scan
    clean = np.ascontiguousarray(s_src)
    _, h0 = _score_check(_scorer(b200, s_tgt, clean, 2.0, method), clean, s_tgt, 2.0, method, poses, "clean")
    huge = np.array([[1e12, 0, 0], [-1e12, 1, 1], [0, 1e12, 0], [0, 0, -1e12], [1e12, 1e12, 1e12]], dtype=F32)
    bad, _ = R.with_nonfinite_rows(clean, seed=9)
    bad = np.ascontiguousarray(np.concatenate([huge, bad[:, :3], huge]), dtype=F32)
    w, h = _score_check(_scorer(b200, s_tgt, bad, 2.0, method), bad, s_tgt, 2.0, method, poses, "non-finite")
    assert np.array_equal(h, h0)
    worst["non-finite"] = w
    print(f"\nmax |score - ref| / bound, method {method}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


ESCAPES = [(leaf, axis, d, inside) for leaf in (0.3, 0.9) for axis in (0, 2) for d in (1, -1) for inside in (True, False)]


def test_kdtree_escape_and_equality_scores(b200):
    """K12's KDTREE branch reaches the voxel two lookup cells away (which the 27-cell block misses), and counts a pair
    exactly when its f32 d2 is below res^2."""
    worst = 0.0
    for leaf, axis, d, inside in ESCAPES:
        t, q, _, _, _ = RR.escape_fixture(leaf, axis, d, inside)
        g = _scorer(b200, t, q, leaf, 0)
        assert RR.score(q, leaf, g.voxels(), rule="block27", geom=R.leaf_geometry(t, leaf))["hits"] == 0
        w, h = _score_check(g, q, t, leaf, 0, [np.zeros(6)], ("escape", leaf, axis, d, inside))
        assert h[0] == 1
        worst = max(worst, w)
    for res, (x, y, z) in {1.0: (2.0, 0.5, 0.25), 0.3: (0.75, 0.45, 0.15), 0.6: (1.5, 0.9, 0.3)}.items():
        cen = np.array([x, y, z], dtype=F32)
        t = RR.wall(0, cen[0], (cen[1], cen[2]), res)
        qs = RR.equality_queries(res, cen)
        r2 = RR.radius2(res)
        assert qs[0][1] < r2 <= qs[-1][1]
        for qv, d2 in qs:
            s = qv.reshape(1, 3).astype(F32)
            g = _scorer(b200, t, s, res, 0)
            # the reference's near_threshold flags these pairs by design: the hit is decided by d2 < r2 exactly
            w, h = _score_check(g, s, t, res, 0, [np.zeros(6)], ("equality", res, float(d2)), hits_exact=False)
            assert h[0] == int(d2 < r2), (res, d2)
            worst = max(worst, w)
    print(f"\nmax |score - ref| / bound, KDTREE escape and equality fixtures: {worst:.3g}")
