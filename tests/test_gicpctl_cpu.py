"""The float64 optimiser replay of tests/gicpctl_ref.py, checked on the CPU before any GPU comparison: driven by the
oracle's own evaluations it must reproduce oracle.GICP.align exactly (every functor call's kind and x, every step, the
outer loop, the final pose), with no decision near its threshold; the fixture generators must reach the edges they are
named for; and replays of subtly wrong optimisers must fail against at least one oracle trace."""
from collections import Counter

import numpy as np
import pytest

import gicpctl_ref as X
import gicpref as G

F32 = np.float32
_cache = {}


def _scene(name):
    from lidarslam_ros2_b200 import synth

    if name not in _cache:
        _cache[name] = G.surface_pair() if name == "pair" else synth.registration_pair(name, 2.0)[:2]
    return _cache[name]


def _generators():
    s, t = _scene("small")
    return {
        "identical": (X.identical_pair(t), None, {}),
        "offset_far": (X.offset_pair(s, t, (3.0, -2.0, 0.5), (0.0, 0.0, 0.2)), None, {}),
        "offset_near": (X.offset_pair(s, t, (0.3, 0.1, 0.0), (0.0, 0.0, 0.02)), None, {}),  # reaches the inner cap
        "m4": ((G.exact_m_scan(t, 4), t), None, {}),
        "m3": ((G.exact_m_scan(t, 3), t), None, {}),
        "max_iterations_2": ((s, t), G.GUESS, {"max_iterations": 2}),
    }


def _oracle_trace(oracle_mod, src, tgt, guess=None, cfg=None):
    cfg = cfg or {}
    o = oracle_mod.GICP(max_correspondence_distance=5.0, **cfg)
    o.set_target(tgt)
    o.set_source(src)
    o.set_trace(True)
    T = o.align(guess)
    return o, T, o.trace()


def _check(o, T, recs, guess, cfg, label):
    r = X.replay(recs, guess, cfg)
    assert not r["bad"], (label, r["bad"][:3])
    assert r["near"] == 0, label
    assert r["iterations"] == o.iterations and r["converged"] == o.converged, label
    assert np.array_equal(r["final_T"], T), label
    assert r["calls"] == int((recs["type"] == 0).sum()), label
    return r


_traces = {}


def _all_traces(oracle_mod):
    """Oracle traces of the scenes (identity and GUESS) and of the generators: {label: (oracle, T, recs, guess, cfg)}."""
    if not _traces:
        for name in ("pair", "tiny", "small"):
            s, t = _scene(name)
            for gname, guess in (("identity", None), ("guess", G.GUESS)):
                _traces[f"{name}/{gname}"] = _oracle_trace(oracle_mod, s, t, guess) + (guess, {})
        for name, ((s, t), guess, cfg) in _generators().items():
            _traces[name] = _oracle_trace(oracle_mod, s, t, guess, cfg) + (guess, cfg)
    return _traces


def test_replay_reproduces_oracle_align(oracle_mod):
    total = Counter()
    for label, (o, T, recs, guess, cfg) in _all_traces(oracle_mod).items():
        r = _check(o, T, recs, guess, cfg, label)
        total.update(r["counts"])
    print(f"\nbranches over {len(_traces)} oracle aligns: {dict(sorted(total.items()))}")
    for k in ("bracket_f", "bracket_slope", "extrapolate", "bracket_success", "delta_f_neg_start", "section_noprogress",
              "section_f", "section_success", "cubic", "quadratic", "sq_two_roots", "sq_no_root", "inner_cap",
              "gradient_success", "entry_noprogress", "dir_flip"):
        assert total[k] > 0, k


def test_generators_reach_their_edges(oracle_mod):
    tr = _all_traces(oracle_mod)
    # source identical to target at identity: f = g = 0, the direction is NaN, NoProgress at entry, one outer iteration
    o, _, recs, _, _ = tr["identical"]
    calls = recs[recs["type"] == 0]
    assert len(calls) == 1 and calls[0]["f"] == 0 and np.all(calls[0]["g"] == 0)
    steps = recs[recs["type"] == 1]
    assert len(steps) == 1 and steps[0]["status"] == X.NO_PROGRESS
    assert o.iterations == 1 and o.converged
    assert X.replay(recs)["counts"]["entry_noprogress"] == 1
    # exactly four correspondences: the BFGS runs; three: the loop ends before it
    o, _, recs, _, _ = tr["m4"]
    outer = recs[recs["type"] == 2]
    assert np.all(outer["m"] == 4) and np.all(outer["status"] != X.NOT_STARTED)
    o, _, recs, _, _ = tr["m3"]
    assert len(recs) == 1 and recs[0]["m"] == 3 and recs[0]["status"] == X.NOT_STARTED and not o.converged
    # the inner cap
    _, _, recs, guess, cfg = tr["offset_near"]
    assert X.replay(recs, guess, cfg)["counts"]["inner_cap"] > 0
    outer = recs[recs["type"] == 2]
    assert np.any((outer["inner"] == 20) & (outer["status"] == X.RUNNING))
    # a small max_iterations ends the loop by the cap, converged
    o, _, recs, _, _ = tr["max_iterations_2"]
    assert o.iterations == 2 and o.converged and recs[-1]["delta"] >= 1
    # a far start extrapolates and brackets by slope
    _, _, recs, guess, cfg = tr["offset_far"]
    c = X.replay(recs, guess, cfg)["counts"]
    assert c["extrapolate"] > 0 and c["bracket_slope"] > 0 and c["bracket_f"] > 0


@pytest.mark.parametrize("mut", [m for m in X.MUTATIONS if m not in X.UNREACHED])
def test_power_of_the_replay(oracle_mod, mut):
    """A replay of a subtly wrong optimiser fails against at least one oracle trace."""
    failed = [label for label, (_, _, recs, guess, cfg) in _all_traces(oracle_mod).items()
              if X.replay(recs, guess, cfg, mut=(mut,))["bad"]]
    print(f"\n{mut}: fails {len(failed)} of {len(_traces)} traces")
    assert failed, mut
