"""tests/deskewref.py against oracle/deskew.py on the CPU: the replay's decisions and carried pointers equal the literal
restatement of adjustDistortion on every scene of the de-skew edge tests (NaN rays and an IMU clock stepping back
included), its coordinates agree with the oracle to rounding, its float32 replay stays within its own float64 bound, and
the scene generators produce the edges they claim to.

The oracle evaluates atan2 / sin / cos in float32 (numpy), the kernel and the replay in double rounded to float. Here the
oracle runs with the double-then-round functions, so both sides take the same decisions at the planted ties."""
import numpy as np
import pytest

import deskewref as DR
from oracle import deskew

ORACLE_MAX_N = 30000  # the literal oracle is a Python loop per point


def _in_double(fn):
    def g(*args):
        r = fn(*(np.asarray(a).astype(np.float64) for a in args))
        return r.astype(np.float32) if np.asarray(args[0]).dtype == np.float32 else r
    return staticmethod(g)


class _DoubleTrig:
    """numpy, with atan2 / asin / sin / cos of float32 arguments evaluated in double and rounded to float32."""

    def __getattr__(self, name):
        return getattr(np, name)

    arctan2, arcsin, sin, cos = _in_double(np.arctan2), _in_double(np.arcsin), _in_double(np.sin), _in_double(np.cos)


@pytest.fixture
def double_trig(monkeypatch):
    monkeypatch.setattr(deskew, "np", _DoubleTrig())


def _view(r):
    return {k: r.get(k) for k in ("n", "t", "rel", "front", "skip", "k_first", "rounds")} | {"n": r["n"] if r["ran"] else 0}


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


SCENES = DR.all_scenes()


@pytest.mark.parametrize("sc", SCENES, ids=[s.name for s in SCENES])
def test_replay_equals_oracle(sc, double_trig):
    o = deskew.LidarUndistortion(scan_period=sc.scan_period)
    for step in sc.steps:
        if step[0] == "imu":
            DR.feed([o], step[1])
            continue
        _, cloud, st, claim = step
        ring = DR.Ring.from_oracle(o)
        r = DR.replay(cloud, ring, st)
        claim(_view(r), ring)
        assert not r["ambiguous"].any(), np.flatnonzero(r["ambiguous"])[:10]
        if r["ran"]:
            if r["monotone"]:  # the kernel's form equals the walk, and the scan needs the passes it reports
                assert np.array_equal(r["par_front"], r["front"]) and np.array_equal(r["par_skip"], r["skip"])
                assert r["par_ptrs"] == (r["ptr_front"], r["ptr_last_iter"])
            fin = np.isfinite(r["out"][:, :3]) & np.isfinite(r["ref64"])
            assert np.all(np.abs(r["out"][:, :3] - r["ref64"])[fin] <= r["bound"][fin])
        if len(cloud) <= ORACLE_MAX_N:
            a = o.adjust_distortion(cloud, st)
            assert (o.ptr_front, o.ptr_last_iter) == (r["ptr_front"], r["ptr_last_iter"]), sc.name
            assert _same(np.isnan(a), np.isnan(r["out"]))
            untouched = np.all((r["out"][:, :3] == cloud[:, :3]) | np.isnan(cloud[:, :3]), axis=1)
            assert _same(a[untouched], cloud[untouched])
            fin = np.isfinite(a[:, :3]) & np.isfinite(r["ref64"])
            assert np.all(np.abs(a[:, :3] - r["ref64"])[fin] <= 4 * r["bound"][fin] + 1e-6)
        else:
            o.ptr_front, o.ptr_last_iter = r["ptr_front"], r["ptr_last_iter"]


def test_step_back_breaks_the_parallel_form():
    """The clock step back is the case the kernel's parallel form cannot take: the replay shows it differs from the walk."""
    sc = [s for s in DR.stamp_scenes() if s.name == "stamps_clock_step_back"][0]
    o = deskew.LidarUndistortion(scan_period=sc.scan_period)
    DR.feed([o], sc.steps[0][1])
    _, cloud, st, _ = sc.steps[1]
    r = DR.replay(cloud, DR.Ring.from_oracle(o), st)
    assert not r["monotone"]
    assert r["par_ptrs"] != (r["ptr_front"], r["ptr_last_iter"]) or not np.array_equal(r["par_skip"], r["skip"])


@pytest.mark.parametrize("sc", [s for s in SCENES if len(s.steps) == 2], ids=lambda s: s.name)
def test_no_ambiguous_rounding_on_the_device_ring(sc):
    """With the ring getImu builds on the host (glibc atan2f / asinf), no value of the scene lies near a float midpoint."""
    ring = DR.glibc_ring(sc.steps[0][1], sc.scan_period)
    _, cloud, st, _ = sc.steps[1]
    assert not DR.replay(cloud, ring, st)["ambiguous"].any()


def test_generators_reach_their_edges():
    # ties: the planted stamps equal the points' t
    sc, idx = DR.ladder(4097)
    stamps = [m[3] for m in sc.steps[0][1]]
    t = DR.times_of(sc.steps[1][1], sc.steps[1][2], sc.scan_period)["t"]
    per = -(-4097 // 1024)
    assert {per - 1, per, per + 1, 511 * per - 1, 511 * per, 511 * per + 1} <= set(idx)
    assert all(float(t[j]) in stamps for j in idx)
    # the half-turn threshold: fl(a - start) == float(pi) at kf, one float below at kf - 1
    scs, kf = DR.azimuth_scenes()
    c = [s for s in scs if s.name == "az_half_turn_threshold"][0].steps[1][1]
    d = DR.times_of(c, 40.0, 0.1)
    so = d["start_ori"]
    assert DR.F(d["a"][kf] - so) == DR.F(np.pi) and float(DR.F(np.pi)) > np.pi
    assert DR.F(d["a"][kf - 1] - so) == np.nextafter(DR.F(np.pi), DR.F(0)) and d["k_first"] == kf
    # exactly scan_period: fl(|t - s|) == scan_period
    s = DR.stamp_at_period(30.0123456789, 0.125)
    assert abs(30.0123456789 - s) == 0.125
    # the chain seeds need 2 and >= 3 passes (the claims assert it in test_replay_equals_oracle too)
    assert DR.find_chain_seeds(rounds_wanted=(2, 3), tries=30) == DR.CHAIN_SEEDS
