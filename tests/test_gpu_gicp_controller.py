"""GICP's optimiser (the device controller of gicp_inner_kernel running Bfgs6T) call by call, through the opt-in trace
of align(): every functor call, BFGS step and outer iteration is replayed bit for bit by the float64 restatement of
tests/gicpctl_ref.py from the recorded (f, g); the bookkeeping must follow from the records exactly; every in-BFGS
evaluation must be a real evaluation, bitwise equal to b200reg_gicp_objective at the recorded x on the correspondences
of its outer iteration, and on the small scenes within the bound of the float64 reference gicpref.objective. Run on an
H100 with -m gpu; each test prints its largest ratio to its bound and the branch counts."""
from collections import Counter

import numpy as np
import pytest

import gicpctl_ref as X
import gicpref as G

pytestmark = pytest.mark.gpu
F32 = np.float32
CAP = 1 << 15
_scenes = {}


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


@pytest.fixture(scope="module")
def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _scene(name):
    from lidarslam_ros2_b200 import synth

    if name not in _scenes:
        _scenes[name] = G.surface_pair() if name == "pair" else synth.registration_pair(name, 2.0)[:2]
    return _scenes[name]


def _cfg(name):
    return dict(trans_eps=1e-8, max_iterations=6) if name == "headline" else {}


def _handle(b200, src, tgt, cfg=None, cap=CAP):
    cfg = cfg or {}
    g = b200.GeneralizedIterativeClosestPoint()
    g.setMaxCorrespondenceDistance(5.0)
    if "trans_eps" in cfg:
        g.setTransformationEpsilon(cfg["trans_eps"])
    if "max_iterations" in cfg:
        g.setMaximumIterations(cfg["max_iterations"])
    g.setInputTarget(tgt)
    g.setInputSource(src)
    if cap:
        g.setTrace(cap)
    return g


def _traced(g, guess):
    T = g.align(guess)
    recs, n = g.trace()
    assert n == len(recs) > 0, (n, len(recs))
    return T, recs


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _replay(g, T, recs, guess, cfg):
    """The replay and the bookkeeping; returns the replay's result."""
    r = X.replay(recs, guess, cfg)
    assert not r["bad"], r["bad"][:3]
    assert r["near"] == 0
    st = g.stats()
    assert st["evaluations"] == r["calls"] == int((recs["type"] == 0).sum())
    last = recs[-1]
    assert last["type"] == 2 and last["last"] == 1
    assert st["iterations"] == r["iterations"] == int(last["nr_iterations"])
    assert g.hasConverged() == r["converged"] == bool(last["converged"])
    F = g.getFinalTransformation()
    assert _bits(F.reshape(16)) == _bits(last["final_T"]) == _bits(r["final_T"].reshape(16))
    assert _bits(F) == _bits(T)
    return r


def _check_evaluations(g, src, tgt, recs, guess, depth=None, stride=1):
    """Every call record against b200reg_gicp_objective on its outer iteration's correspondences (bitwise) and, with
    depth, every stride-th against gicpref.objective; returns the largest ratio to the bound."""
    worst = 0.0
    transformation = np.eye(4, dtype=F32)
    moved = G.transform(np.eye(4, dtype=F32) if guess is None else guess, src)
    for o in recs[recs["type"] == 2]:
        k = int(o["outer"])
        corr, maha, m = g.correspondences(T=transformation, guess=guess)
        assert m == o["m"], (k, m, int(o["m"]))
        calls = recs[(recs["type"] == 0) & (recs["outer"] == k)]
        for j, c in enumerate(calls):
            x = np.array(c["x"])
            f, grad, T = g.objective(x, bool(c["want_grad"]))
            assert _bits(np.float64(f)) == _bits(c["f"]), (k, j, f, c["f"])
            if c["want_grad"]:
                assert _bits(grad) == _bits(c["g"]), (k, j, grad, c["g"])
            assert _bits(T[:3].reshape(12)) == _bits(c["T"]), (k, j)
            if depth is not None and j % stride == 0:
                ref = G.objective(T, x, moved, tgt, corr, maha, depth)
                if c["want_grad"]:
                    rat = [abs(f - ref["f"]) / ref["b_f"]] + list(np.abs(grad - ref["g"]) / ref["b_g"])
                else:
                    rat = [abs(f - ref["f32path"]) / ref["b_f32path"]]
                assert max(rat) <= 1.0, (k, j, rat)
                worst = max(worst, max(rat))
        if o["status"] != X.NOT_STARTED:
            transformation = X._mat4(o["T"])
    return worst


@pytest.mark.parametrize("name", ["pair", "tiny", "small", "c1", "headline"])
def test_trace_replays_and_evaluations_are_real(b200, sms, name):
    src, tgt = _scene(name)
    cfg = _cfg(name)
    depth = None
    if name in ("pair", "tiny", "small"):
        depth = G.depth_device(len(src), sms)
    total, worst_eval, worst_T = Counter(), 0.0, 0.0
    for guess in (None, G.GUESS):
        g = _handle(b200, src, tgt, cfg)
        T, recs = _traced(g, guess)
        r = _replay(g, T, recs, guess, cfg)
        total.update(r["counts"])
        worst_T = max(worst_T, r["worst_T"])
        worst_eval = max(worst_eval, _check_evaluations(g, src, tgt, recs, guess, depth, stride=1 if name != "small" else 3))
    print(f"\n{name}: every record bitwise, largest T / bound {worst_T:.3g}, largest "
          f"evaluation / bound {worst_eval:.3g}; branches {dict(sorted(total.items()))}")


def test_generators(b200):
    """Entry NoProgress with its NaN direction, m = 4, m < 4, the inner cap and a far start, replayed and evaluated."""
    s, t = _scene("small")
    total = Counter()
    fixtures = {"identical": X.identical_pair(t), "m4": (G.exact_m_scan(t, 4), t), "m3": (G.exact_m_scan(t, 3), t),
                "offset_near": X.offset_pair(s, t, (0.3, 0.1, 0.0), (0.0, 0.0, 0.02)),
                "offset_far": X.offset_pair(s, t, (3.0, -2.0, 0.5), (0.0, 0.0, 0.2))}
    for name, (src, tgt) in fixtures.items():
        g = _handle(b200, src, tgt)
        T, recs = _traced(g, None)
        r = _replay(g, T, recs, None, {})
        total.update(r["counts"])
        if name == "identical":
            calls = recs[recs["type"] == 0]
            assert len(calls) == 1 and calls[0]["f"] == 0 and np.all(calls[0]["g"] == 0)
            assert r["counts"]["entry_noprogress"] == 1 and r["iterations"] == 1 and r["converged"]
        elif name == "m4":
            assert np.all(recs[recs["type"] == 2]["m"] == 4)
        elif name == "m3":
            assert len(recs) == 1 and recs[0]["m"] == 3 and recs[0]["status"] == X.NOT_STARTED and not g.hasConverged()
        elif name == "offset_near":
            assert r["counts"]["inner_cap"] > 0
        if name != "m3":
            _check_evaluations(g, src, tgt, recs, None)
    print(f"\ngenerators: branches {dict(sorted(total.items()))}")


def test_evaluator_ladder(b200, sms):
    """One evaluator CTA (n <= 256) and SMs - 1 evaluators: every record and evaluation bitwise."""
    _, tgt = _scene("small")
    for n in (200, 256 * (min(sms, G.GI_MAX_CTAS) - 1)):
        src = G.cloud_of_size(tgt, n, seed=n, T=G.T_OFF)
        g = _handle(b200, src, tgt)
        T, recs = _traced(g, G.GUESS)
        _replay(g, T, recs, G.GUESS, {})
        _check_evaluations(g, src, tgt, recs, G.GUESS)
        print(f"\nladder n = {n}: evaluators {G.evaluator_partition(n, sms)[0]}, {len(recs)} records bitwise")


def test_stale_state(b200):
    """Three different aligns on one handle, each bitwise (trace and result) a fresh handle's."""
    s, t = _scene("small")
    s2, _ = _scene("tiny")
    A = _handle(b200, s, t)
    for src, guess in ((s, G.GUESS), (s, None), (s2, G.GUESS)):
        A.setInputSource(src)
        Ta, ra = _traced(A, guess)
        F = _handle(b200, src, t)
        Tf, rf = _traced(F, guess)
        assert _bits(Ta) == _bits(Tf) and _bits(ra) == _bits(rf)


def test_trace_neutral_and_overflow(b200):
    s, t = _scene("small")
    on, off = _handle(b200, s, t), _handle(b200, s, t, cap=0)
    Ton, recs = _traced(on, G.GUESS)
    Toff = off.align(G.GUESS)
    assert _bits(Ton) == _bits(Toff)
    a, b = on.stats(), off.stats()
    for k in ("iterations", "evaluations"):
        assert a[k] == b[k], k
    assert on.hasConverged() == off.hasConverged()
    small = _handle(b200, s, t, cap=5)
    assert _bits(small.align(G.GUESS)) == _bits(Ton)
    part, n = small.trace()
    assert n == len(recs) and len(part) == 5 and _bits(part) == _bits(recs[:5])
    off.setTrace(0)
    assert off.trace()[1] == 0
