"""The NDT solver's on-device controller (controller_fast, controller, build_control and the round bookkeeping of
ndt_solver.cu), round by round, through the opt-in trace of align(): every round's step is replayed in float64 by
tests/ndtctl_ref.py from the device's own state and totals, with exact discrete decisions and a bound for every
continuous field; every published control block must be bitwise the host's pose_to_matrix / angle tables at the device's
x_t; the bookkeeping (evaluations, hits, iterations, final pose, transformation probability) must follow from the
records exactly; and on the small scenes every evaluation inside align() is checked against the float64 derivative
reference of tests/ndtref.py. Run on an H100 with -m gpu; each test prints its largest deviation / bound."""
import numpy as np
import pytest

import gridref as R
import ndtctl_ref as X
import ndtref as N
import radiusref as RR

pytestmark = pytest.mark.gpu

F32 = np.float32
U = 2.0**-53
METHODS = [(2, "DIRECT7"), (3, "DIRECT1"), (1, "DIRECT26"), (0, "KDTREE")]
GUESS = np.array([[0.9999, -0.0100, 0.0030, 0.30], [0.0100, 0.9999, -0.0020, -0.20], [-0.0030, 0.0020, 1.0, 0.05],
                  [0, 0, 0, 1]], dtype=F32)
GUESSES = (np.eye(4, dtype=F32), GUESS)
SHIPPED = X.config()
MT = X.config(step_size=0.1, trans_eps=0.2, max_iterations=6)
MT_LONG = X.config(step_size=0.5, trans_eps=1.0, max_iterations=6)
CAP = 4096


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
def scenes(golden):
    from lidarslam_ros2_b200 import synth

    out = {k: synth.registration_pair(k, 2.0)[:2] + (2.0,) for k in ("tiny", "small", "c1", "headline")}
    out["golden"] = (golden["source"], golden["target"], 1.0)
    return out


def _ndt(b200, src, tgt, res, method, cfg, cap=CAP):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setNeighborhoodSearchMethod(method)
    g.setStepSize(cfg["step_size"])
    g.setTransformationEpsilon(cfg["trans_eps"])
    g.setMaximumIterations(cfg["max_iterations"])
    g.setInputTarget(tgt)
    g.setInputSource(src)
    g.setTrace(cap)
    return g


def _traced_align(g, guess):
    g.align(guess)
    recs, n = g.trace()
    assert n == len(recs) > 0, (n, len(recs))
    return recs


def _check_bookkeeping(g, recs, n_src):
    st = g.stats()
    ev = recs[recs["evaluated"] == 1]
    assert len(ev) == st["evaluations"]
    assert int(sum(int(r["tot"][28]) for r in ev)) == st["hits_total"] == int(recs[-1]["hits_total"])
    last = recs[-1]
    assert last["done"] == 1 and last["nr_iterations"] == g.getFinalNumIteration()
    assert bool(last["converged"]) == g.hasConverged()
    F = g.getFinalTransformation()
    built = recs[recs["built"] == 1]
    assert np.array_equal(F.reshape(16), last["final_T"])
    if len(built):
        assert np.array_equal(F[:3].reshape(12), built[-1]["T"])
    assert g.getTransformationProbability() == float(last["score"]) / n_src


def _check_control_blocks(recs):
    """T, jang, hang bitwise the host's at the device's x_t, except entries whose f64 value sits within 2 f64 ulp of a f32
    rounding boundary (counted); jd / hd within a few f64 ulp of the reference's f64 tables. Returns the boundary count."""
    import oracle

    boundary = 0
    for r in recs[recs["built"] == 1]:
        x = np.array(r["x_t"], dtype=np.float64)
        T = oracle.pose_to_matrix(x)[:3].reshape(12)
        j, h = oracle.angle_tables(x)
        _, _, j64, h64 = N.angle_tables(x, f64=True)  # f64 values of the live tables (d1.z = +sy)
        ang = np.array(x[3:6], dtype=F32).astype(np.float64)
        trig = np.concatenate([np.sin(ang), np.cos(ang)])
        if not np.array_equal(r["T"], T):
            assert X.near_f32_boundary(trig).any(), (r["round"], r["T"], T)
            boundary += 1
        for got, want, v64 in ((r["jang"], j.reshape(24), j64.reshape(24)), (r["hang"], h.reshape(45), h64.reshape(45))):
            bad = got != want
            if bad.any():
                assert X.near_f32_boundary(v64[bad]).all(), (r["round"], np.nonzero(bad))
                boundary += int(bad.sum())
        if r["build_f64"]:
            _, _, jd, hd = N.angle_tables(x, minus_sy=True, f64=True)
            assert np.abs(r["jd"] - jd.reshape(24)).max() <= 8 * U and np.abs(r["hd"] - hd.reshape(45)).max() <= 8 * U
    return boundary


def _check_steps(recs, cfg, guess, infos=None):
    """Replay every round from the device's state before it; returns (worst deviation / bound, mt cases, decisions).
    infos (a list) receives the replay's info of every round."""
    s = X.initial_state(guess)
    worst, cases, decisions = 0.0, set(), []
    for r in recs:
        assert s["phase"] == r["phase_before"] or (r["phase_before"] == X.PH_LS_HESSIAN and not r["evaluated"]), r["round"]
        before = dict(s, phase=int(r["phase_before"]))
        ref, info = X.step(before, r["tot"] if r["evaluated"] else None, cfg, H_k2=None if r["evaluated"] else r["H"])
        w, bad = X.compare(r, ref, info, X.is_mt_config(cfg))
        assert not bad, (r["launch"], r["round"], bad)
        assert not info["near"], (r["launch"], r["round"], info["near"])
        b = info["build"]
        assert bool(r["built"]) == (b is not None), r["round"]
        if b:
            assert (int(r["compute_hessian"]), int(r["build_f64"])) == b, r["round"]
        assert int(r["mode"]) == (0 if b else (2 if ref["done"] == 2 else 1))
        if infos is not None:
            infos.append(info)
        worst = max(worst, w)
        if info["mt_case"]:
            cases.add(info["mt_case"])
        decisions.append((int(r["phase_after"]), int(r["done"]), int(r["nr_iterations"]), int(r["evaluations"]),
                          int(r["step_iterations"]), int(r["built"]), int(r["converged"])))
        s = X.state_of(r)
    return worst, cases, decisions


def _check_evaluations(recs, src, tgt, res, method, g, guess, n_sms):
    """Every evaluation of align() against the float64 derivative reference at the control block it was evaluated at."""
    geom, v = R.leaf_geometry(tgt, res), g.voxels()
    T, x, worst = np.asarray(guess, dtype=F32)[:3], X.initial_pose(guess), 0.0
    for r in recs:
        if r["evaluated"]:
            hess = r["phase_before"] != X.PH_LS_ITER
            ref = N.derivatives(src, T, x, res, v, geom, method, compute_hessian=hess, n_sms=n_sms)
            assert ref["near_threshold"] == 0 and int(r["tot"][28]) == ref["hits"], r["round"]
            H = np.zeros((6, 6))
            # Without the Hessian (line-search rounds) the evaluators add to the score and gradient slots only
            # (apply_point<false>), so the Hessian slots carry per-thread sums of an earlier evaluation; the controller
            # discards them (load_totals with_hessian = false) and only score, g and hits are compared.
            for k, (i, j) in enumerate(N.TRI if hess else []):
                H[i, j] = H[j, i] = r["tot"][7 + k]
            q = N.within((r["tot"][0], r["tot"][1:7], H), ref)
            assert q["max"] <= 1.0, (r["round"], q)
            worst = max(worst, q["max"])
        if r["built"]:
            T, x = r["T"].reshape(3, 4), np.array(r["x_t"], dtype=np.float64)
    return worst


@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_controller_rounds_against_the_replay(b200, scenes, n_sms, method):
    worst, worst_eval, boundary, rounds = {}, {}, 0, 0
    for name in ("small", "c1", "golden", "headline"):
        src, tgt, res = scenes[name]
        g = _ndt(b200, src, tgt, res, method, SHIPPED)
        for guess in GUESSES:
            recs = _traced_align(g, guess)
            rounds += len(recs)
            _check_bookkeeping(g, recs, len(src))
            boundary += _check_control_blocks(recs)
            w, _, _ = _check_steps(recs, SHIPPED, guess)
            worst[name] = max(worst.get(name, 0.0), w)
            if name in ("small", "golden"):
                worst_eval[name] = max(worst_eval.get(name, 0.0),
                                       _check_evaluations(recs, src, tgt, res, method, g, guess, n_sms))
    print(f"\nmethod {method}: {rounds} rounds; max step deviation / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items())
          + "; max evaluation deviation / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst_eval.items())
          + f"; control-block entries at a f32 rounding boundary: {boundary}")
    assert boundary == 0


def test_fast_and_scalar_controllers_decide_alike(b200, scenes, monkeypatch):
    """B200REG_SCALAR_CTL=1 routes every round through the scalar controller (pivoted LU / SVD): both traces pass the
    replay and take the same decisions round by round."""
    out = {}
    for scalar in (False, True):
        if scalar:
            monkeypatch.setenv("B200REG_SCALAR_CTL", "1")
        for name in ("small", "c1"):
            src, tgt, res = scenes[name]
            g = _ndt(b200, src, tgt, res, 2, SHIPPED)
            for k, guess in enumerate(GUESSES):
                recs = _traced_align(g, guess)
                assert (recs["fast"] == 0).all() if scalar else (recs["fast"] == 1).any()
                w, _, dec = _check_steps(recs, SHIPPED, guess)
                out[(scalar, name, k)] = (w, dec)
    for key in [k for k in out if not k[0]]:
        assert out[key][1] == out[(True,) + key[1:]][1], key
    print("\nmax step deviation / bound, fast vs scalar: " + ", ".join(f"{k}: {v[0]:.3g}" for k, v in out.items()))


def test_more_thuente_rounds_and_k2_passes(b200, oracle_mod, scenes, n_sms):
    """step_max <= step_min: every More-Thuente round is replayed bit for bit (psi, slopes, interval updates and trial
    values), over fixtures that reach trial cases 1, 2 and 3, the open -> closed flip, closed-interval updates and the
    10-step cap; every evaluation (line-search ones without the Hessian included) is checked against the float64
    derivative reference; the Hessian each K2 pass injects matches the float64 radius reference (tests/radiusref.py) at
    that round's control block entry by entry within its bound, and the solve takes one resumed launch per K2 pass."""
    cases, k2, flips, closed, capped, worst, worst_h, worst_e = set(), 0, 0, 0, 0, 0.0, 0.0, 0.0
    for name, guess, cfg in (("tiny", np.eye(4, dtype=F32), MT_LONG), ("tiny", GUESS, MT_LONG), ("small", GUESS, MT_LONG),
                             ("tiny", GUESS, MT)):
        src, tgt, res = scenes[name]
        g = _ndt(b200, src, tgt, res, 2, cfg)
        recs = _traced_align(g, guess)
        _check_bookkeeping(g, recs, len(src))
        _check_control_blocks(recs)
        infos = []
        w, c, _ = _check_steps(recs, cfg, guess, infos)
        worst, cases = max(worst, w), cases | c
        flips += sum(bool(i["decisions"].get("open_to_closed")) for i in infos)
        closed += sum(i["update_branch"] is not None and not r["open_interval"] for r, i in zip(recs, infos))
        capped += int((recs["step_iterations"] == X.MAX_STEP_ITERATIONS).sum())
        worst_e = max(worst_e, _check_evaluations(recs, src, tgt, res, 2, g, guess, n_sms))
        n_k2 = int((recs["done"] == 2).sum())
        assert int(recs["launch"].max()) == n_k2 == int((recs["evaluated"] == 0).sum())
        k2 += n_k2
        last_built = None
        for r in recs:
            if not r["evaluated"]:
                # the K2 pass ran on the control block's f32 transform with the f64 tables the device built for x_t
                ref = RR.hessian(src, last_built["T"].reshape(3, 4), np.array(last_built["x_t"], dtype=np.float64), res,
                                 g.voxels(), tables=(last_built["jd"], last_built["hd"]))
                assert ref["near_threshold"] == 0 and ref["hits"] > 0, (name, r["launch"])
                d, _ = RR.within_h(r["H"].reshape(6, 6), ref)
                assert d <= 1.0, (name, r["launch"], d)
                worst_h = max(worst_h, d)
            if r["built"]:
                last_built = r
    print(f"\nMore-Thuente: trial cases reached {sorted(cases)}, open->closed flips {flips}, closed-interval updates "
          f"{closed}, 10-step caps {capped}, K2 passes {k2}, near-threshold decisions 0, max step deviation / bound "
          f"{worst:.3g}, max evaluation deviation / bound {worst_e:.3g}, max K2 Hessian deviation / bound {worst_h:.3g}")
    assert cases >= {1, 2, 3} and flips > 0 and closed > 0 and capped > 0 and k2 > 0


def test_edge_generators_on_the_device(b200, oracle_mod, scenes, n_sms):
    """The controller edges of tests/ndtctl_ref.py, each replayed round by round: the origin source (rotation rows of H
    exactly zero: LDL^T refuses, LU fails, the scalar controller's minimum-norm SVD direction is checked against
    oracle.svd6_solve within its bound), an ascent start on the golden PCD (the fast path flips the direction) and a snap
    round (a published angle in [1e-5, 1e-4), its tables bitwise the host's)."""
    osrc, otgt = X.origin_pair()
    g = _ndt(b200, osrc, otgt, 2.0, 2, SHIPPED)
    recs = _traced_align(g, np.eye(4, dtype=F32))
    _check_bookkeeping(g, recs, len(osrc))
    infos = []
    w_o, _, _ = _check_steps(recs, SHIPPED, np.eye(4, dtype=F32), infos)
    solved = [(r, i) for r, i in zip(recs, infos) if "solve" in i]
    assert len(solved) >= 2 and all(r["fast"] == 0 for r, _ in solved)
    assert all(np.all(r["dir"][3:] == 0) and np.any(r["dir"][:3] != 0) for r, _ in solved if r["built"])
    gs, gt, gres = scenes["golden"]
    o = oracle_mod.NDT(resolution=gres, num_threads=1)
    o.set_target(gt)
    o.set_source(gs)
    found = {}
    for what, guesses, pred in (("ascent", X.ascent_guesses(), X.is_ascent_round),
                                ("snap", X.edge_guesses(), X.is_snap_round)):
        G = X.first_with(o, SHIPPED, guesses, len(gs), pred)
        assert G is not None, what
        g = _ndt(b200, gs, gt, gres, 2, SHIPPED)
        recs = _traced_align(g, G)
        _check_bookkeeping(g, recs, len(gs))
        assert _check_control_blocks(recs) == 0
        infos = []
        w, _, _ = _check_steps(recs, SHIPPED, G, infos)
        if what == "ascent":
            hit = [r for r, i in zip(recs, infos) if i["decisions"].get("flip") and r["fast"] == 1]
        else:
            hit = [r for r, i in zip(recs, infos) if X.is_snap_round(r, i)]
        assert hit, what
        found[what] = (len(hit), w)
    print(f"\norigin source: {len(solved)} SVD rounds, max step deviation / bound {w_o:.3g}; ascent: {found['ascent'][0]} "
          f"fast-path flips, {found['ascent'][1]:.3g}; snap: {found['snap'][0]} rounds, {found['snap'][1]:.3g}")


@pytest.mark.parametrize("max_iterations", [0, 1, 2])
def test_iteration_cap(b200, scenes, max_iterations):
    src, tgt, res = scenes["small"]
    cfg = X.config(max_iterations=max_iterations)
    g = _ndt(b200, src, tgt, res, 2, cfg)
    recs = _traced_align(g, np.eye(4, dtype=F32))
    _check_bookkeeping(g, recs, len(src))
    w, _, _ = _check_steps(recs, cfg, np.eye(4, dtype=F32))
    assert g.getFinalNumIteration() == max_iterations + 2 and g.hasConverged()
    print(f"\nmax_iterations {max_iterations}: max step deviation / bound {w:.3g}")


def test_trace_does_not_perturb_the_solve(b200, scenes):
    for name, cfg in (("small", SHIPPED), ("tiny", MT)):
        src, tgt, res = scenes[name]
        g = _ndt(b200, src, tgt, res, 2, cfg, cap=0)
        for guess in GUESSES:
            out = []
            for cap in (0, CAP, 0):
                g.setTrace(cap)
                F = g.align(guess)
                st = g.stats()
                out.append((F, g.getFinalNumIteration(), st["evaluations"], st["hits_total"]))
            for a in out[1:]:
                assert np.array_equal(a[0], out[0][0]) and a[1:] == out[0][1:], (name, a[1:], out[0][1:])


def test_trace_overflow_is_reported(b200, scenes):
    src, tgt, res = scenes["small"]
    g = _ndt(b200, src, tgt, res, 2, SHIPPED, cap=2)
    g.align(GUESS)
    recs, n = g.trace()
    assert len(recs) == 2 and n == g.stats()["evaluations"] > 2


def test_stale_state(b200, scenes):
    """One handle traces a More-Thuente solve (K2 passes, resumed launches), then a shipped-configuration solve on another
    target: the second trace equals a fresh handle's bit for bit."""
    src_x, tgt_x, res_x = scenes["tiny"]
    src_y, tgt_y, res_y = scenes["small"]
    g = _ndt(b200, src_x, tgt_x, res_x, 2, MT)
    _traced_align(g, GUESS)
    g.setStepSize(SHIPPED["step_size"])
    g.setTransformationEpsilon(SHIPPED["trans_eps"])
    g.setMaximumIterations(SHIPPED["max_iterations"])
    g.setInputTarget(tgt_y)
    g.setInputSource(src_y)
    a = _traced_align(g, GUESS)
    b = _traced_align(_ndt(b200, src_y, tgt_y, res_y, 2, SHIPPED), GUESS)
    assert a.tobytes() == b.tobytes()
