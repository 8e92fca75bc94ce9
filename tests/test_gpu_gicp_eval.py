"""GICP's correspondence pass (K6) and objective evaluation (K7, both the persistent device-BFGS kernel and the host-driven
gicp_cost_kernel) against the float64 reference of tests/gicpref.py, entry by entry: correspondences exactly, Mahalanobis
matrices bit for bit, f / f32path / g within the bound the reference derives for the path's summation order. Each test
prints its largest |kernel - reference| / bound."""
import os

import numpy as np
import pytest

import gicpref as G
import gridref as GR

pytestmark = pytest.mark.gpu
F32 = np.float32
HOST_ENV = "B200REG_GICP_HOST_BFGS"


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


_scenes = {}


def _scene(name):
    from lidarslam_ros2_b200 import synth

    if name not in _scenes:
        if name == "pair":
            _scenes[name] = G.surface_pair()
        else:
            s, t, _ = synth.registration_pair(name, 2.0)
            _scenes[name] = (s, t)
    return _scenes[name]


def _handle(b200, src, tgt, host=False, corr_dist=5.0):
    """A GICP handle; host=True creates it with the host-driven BFGS switch set."""
    if host:
        os.environ[HOST_ENV] = "1"
    try:
        g = b200.GeneralizedIterativeClosestPoint()
    finally:
        os.environ.pop(HOST_ENV, None)
    g.setMaxCorrespondenceDistance(corr_dist)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    return g


def _k6(g, src, tgt, corr_dist=5.0, guess=None, T=None):
    """K6 against the reference: exact corr and m, bitwise maha; returns (reference, maha ratio to the exact bound)."""
    corr, maha, m = g.correspondences(T=T, guess=guess)
    ref = G.correspondences(src, tgt, g.covariances("source"), g.covariances("target"), corr_dist, guess=guess, T=T)
    bad = np.nonzero(corr != ref["corr"])[0]
    assert len(bad) == 0, (len(bad), bad[:5], corr[bad[:5]], ref["corr"][bad[:5]], ref["d2"][bad[:5]])
    assert m == ref["m"]
    sel = corr >= 0
    diff = np.nonzero((maha[sel].view(np.int32) != ref["maha"][sel].view(np.int32)).any(axis=(1, 2)))[0]
    assert len(diff) == 0, (len(diff), maha[sel][diff[:2]], ref["maha"][sel][diff[:2]])
    ratio = 0.0
    if sel.any():
        err = np.abs(maha[sel].astype(np.float64) - ref["maha_exact"][sel]).max(axis=(1, 2))
        ratio = float((err / ref["maha_bound"][sel]).max())
        assert ratio <= 1.0
    ref["maha_kernel"] = maha
    ref["maha_ratio"] = ratio
    return ref


def _k7(g, ref, tgt, x, depth):
    """One fdf and one f-only evaluation against the reference at the transform the path returned; largest ratio."""
    f, grad, T = g.objective(x, True)
    f32, _, T2 = g.objective(x, False)
    assert np.array_equal(T.view(np.int32), T2.view(np.int32))
    r = G.objective(T, x, ref["moved"], tgt, ref["corr"], ref["maha_kernel"], depth)
    rat = [abs(f - r["f"]) / r["b_f"], abs(f32 - r["f32path"]) / r["b_f32path"]]
    rat += list(np.abs(grad - r["g"]) / r["b_g"])
    assert max(rat) <= 1.0, (x, f - r["f"], r["b_f"], f32 - r["f32path"], r["b_f32path"], grad - r["g"], r["b_g"])
    T64, b = G.state_T_bound(x)
    assert np.all(np.abs(T[:3].astype(np.float64) - T64) <= b), (x, T[:3] - T64)
    return max(rat), dict(f=f, f32=f32, g=grad, T=T, bound=r)


# ---- K6 ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pair", "tiny", "small", "c1", "headline"])
def test_k6_matches_reference(b200, name):
    src, tgt = _scene(name)
    g = _handle(b200, src, tgt)
    worst = 0.0
    for guess, T in ((G.GUESS, None), (G.GUESS, G.T_OFF), (None, G.T_OFF)):
        ref = _k6(g, src, tgt, guess=guess, T=T)
        assert ref["m"] > len(src) // 2
        worst = max(worst, ref["maha_ratio"])
    print(f"K6 {name}: corr exact, maha bitwise, m = {ref['m']}, largest maha_exact ratio {worst:.3g}")


def test_k6_gate_edges(b200):
    src, tgt, expect = G.gate_pair(0.5)
    g = _handle(b200, src, tgt, corr_dist=0.5)
    ref = _k6(g, src, tgt, corr_dist=0.5)
    assert np.array_equal(ref["corr"], expect)  # equality rejected, one ulp below accepted, one ulp above rejected
    g.setMaxCorrespondenceDistance(float("inf"))
    ref = _k6(g, src, tgt, corr_dist=float("inf"))
    assert ref["m"] == len(src)
    far = G.exact_m_scan(_scene("tiny")[1], 4, n=300)
    g = _handle(b200, far, _scene("tiny")[1], corr_dist=float("inf"))
    ref = _k6(g, far, _scene("tiny")[1], corr_dist=float("inf"))
    assert ref["m"] == len(far)


def test_k6_far_pass_km_shift_large_rotation(b200):
    src, tgt, cd = G.far_pass_scene()
    g = _handle(b200, src, tgt, corr_dist=cd)
    ref = _k6(g, src, tgt, corr_dist=cd)
    assert np.all(ref["corr"][:200] >= 0)  # answered by the far pass, under the cutoff
    s, t = _scene("small")
    off = (1500.0, -2300.0, 40.0)
    ss, ts = GR.shifted(s, off), GR.shifted(t, off)
    g = _handle(b200, ss, ts)
    _k6(g, ss, ts, guess=G.GUESS, T=G.T_OFF)
    rot = (np.linalg.inv(G.BIG_ROT.astype(np.float64))[:3, :3] @ s.T.astype(np.float64)
           + np.linalg.inv(G.BIG_ROT.astype(np.float64))[:3, 3:]).T.astype(F32)
    g = _handle(b200, rot, t)
    ref = _k6(g, rot, t, guess=G.BIG_ROT, T=G.T_OFF)
    assert ref["m"] > len(s) // 2


# ---- K7 ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_k7_matches_reference(b200, sms, host):
    worst = 0.0
    for name in ("pair", "small"):
        src, tgt = _scene(name)
        g = _handle(b200, src, tgt, host=host)
        ref = _k6(g, src, tgt, guess=G.GUESS, T=G.T_OFF)
        depth = (G.depth_host if host else G.depth_device)(len(src), sms)
        for x in G.STATES.values():
            r, _ = _k7(g, ref, tgt, x, depth)
            worst = max(worst, r)
    print(f"K7 {'host' if host else 'device'}: largest ratio {worst:.3g}")


def test_k7_paths_agree(b200, sms):
    src, tgt = _scene("small")
    gd, gh = _handle(b200, src, tgt), _handle(b200, src, tgt, host=True)
    rd, rh = _k6(gd, src, tgt, guess=G.GUESS), _k6(gh, src, tgt, guess=G.GUESS)
    worst, same_T = 0.0, 0
    for x in G.STATES.values():
        _, a = _k7(gd, rd, tgt, x, G.depth_device(len(src), sms))
        _, b = _k7(gh, rh, tgt, x, G.depth_host(len(src), sms))
        if not np.array_equal(a["T"].view(np.int32), b["T"].view(np.int32)):
            continue  # cosf / sinf of the device and the host may differ in the last bit; each matched the reference
        same_T += 1
        tf = a["bound"]["b_f"] + b["bound"]["b_f"]
        tg = a["bound"]["b_g"] + b["bound"]["b_g"]
        assert abs(a["f"] - b["f"]) <= tf and np.all(np.abs(a["g"] - b["g"]) <= tg)
        worst = max(worst, abs(a["f"] - b["f"]) / tf, float((np.abs(a["g"] - b["g"]) / tg).max()))
    assert same_T >= 1  # x = 0 builds the identity on both
    print(f"K7 device vs host: largest ratio {worst:.3g} over {same_T} states with equal T")


def _ladder_case(b200, src, tgt, host, sms, x=G.STATES["moderate"]):
    g = _handle(b200, src, tgt, host=host)
    ref = _k6(g, src, tgt)
    if ref["m"] < 4:
        return 0.0
    depth = (G.depth_host if host else G.depth_device)(len(src), sms)
    return _k7(g, ref, tgt, x, depth)[0]


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_partition_ladder(b200, sms, host):
    _, tgt = _scene("small")
    worst = {}
    for n in G.ladder(sms, host=host):
        src = G.cloud_of_size(tgt, n, seed=n)
        worst[n] = _ladder_case(b200, src, tgt, host, sms)
    # correspondences confined to one evaluator chunk: the other evaluators contribute exactly +0.0
    n = 256 * (min(sms, G.GI_MAX_CTAS) - 1) + 1
    n_eval, chunk = G.evaluator_partition(n, sms)
    base = G.cloud_of_size(tgt, n, seed=7)
    for which in (0, n_eval // 2, n_eval - 1):
        src, _ = G.confine_to_chunk(base, n_eval, chunk, which)
        worst[f"chunk{which}"] = _ladder_case(b200, src, tgt, host, sms)
    print(f"ladder {'host' if host else 'device'}: largest ratio {max(worst.values()):.3g}", worst)


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_large_scans(b200, sms, host):
    src, tgt = _scene("headline")
    worst = [_ladder_case(b200, src, tgt, host, sms)]
    big = G.cloud_of_size(tgt, 250_000, seed=11)
    worst.append(_ladder_case(b200, big, tgt, host, sms))
    print(f"headline and 250k ({'host' if host else 'device'}): ratios {worst}")


# ---- m at 3 and 4, stale state, end to end ---------------------------------------------------------------------------
@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_three_and_four_correspondences(b200, oracle_mod, sms, host):
    from lidarslam_ros2_b200 import synth
    from lidarslam_ros2_b200.registration import B200RegError

    _, tgt = _scene("tiny")
    for m in (3, 4):
        src = G.exact_m_scan(tgt, m)
        g = _handle(b200, src, tgt, host=host)
        ref = _k6(g, src, tgt)
        assert ref["m"] == m
        if m == 3:
            with pytest.raises(B200RegError) as e:
                g.objective(G.STATES["moderate"])
            assert e.value.code == -1
            o = oracle_mod.GICP(max_correspondence_distance=5.0)
            o.set_target(tgt)
            o.set_source(src)
            dt, dr = synth.pose_error(g.align(G.GUESS), o.align(G.GUESS))
            assert dt < 1e-6 and dr < 1e-6
            assert not g.hasConverged() and not o.converged
        else:
            r, _ = _k7(g, ref, tgt, G.STATES["moderate"], (G.depth_host if host else G.depth_device)(len(src), sms))
            print(f"m = 4 ({'host' if host else 'device'}): ratio {r:.3g}")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def test_stale_state(b200):
    src, tgt = _scene("small")
    src2, _ = _scene("tiny")
    x = G.STATES["moderate"]
    A = _handle(b200, src, tgt)
    assert _bits(A.align(G.GUESS)) == _bits(_handle(b200, src, tgt).align(G.GUESS))
    A.setCorrespondenceRandomness(10)
    F = _handle(b200, src, tgt)
    F.setCorrespondenceRandomness(10)
    a, f = A.correspondences(T=G.T_OFF, guess=G.GUESS), F.correspondences(T=G.T_OFF, guess=G.GUESS)
    assert all(_bits(np.asarray(u)) == _bits(np.asarray(v)) for u, v in zip(a, f))
    assert all(_bits(np.asarray(u)) == _bits(np.asarray(v)) for u, v in zip(A.objective(x), F.objective(x)))
    A.setInputSource(src2)
    F = _handle(b200, src2, tgt)
    F.setCorrespondenceRandomness(10)
    a, f = A.correspondences(guess=G.GUESS), F.correspondences(guess=G.GUESS)
    assert all(_bits(np.asarray(u)) == _bits(np.asarray(v)) for u, v in zip(a, f))
    first = A.objective(x)
    for k in range(300):
        out = A.objective(x, want_grad=bool(k & 1))
        if k & 1:
            assert _bits(np.array([out[0]])) == _bits(np.array([first[0]])) and _bits(out[1]) == _bits(first[1])
    assert _bits(A.align(G.GUESS)) == _bits(F.align(G.GUESS))
    assert A.numCorrespondences() == F.numCorrespondences()


@pytest.mark.parametrize("name", ["pair", "small"])
def test_host_path_align_end_to_end(b200, oracle_mod, name):
    from lidarslam_ros2_b200 import synth

    src, tgt = _scene(name)
    gh, gd = _handle(b200, src, tgt, host=True), _handle(b200, src, tgt)
    o = oracle_mod.GICP(max_correspondence_distance=5.0)
    o.set_target(tgt)
    o.set_source(src)
    To = o.align()
    Th, Td = gh.align(), gd.align()
    dt, dr = synth.pose_error(Th, To)
    assert dt < 1e-3 and dr < 1e-3, (dt, dr)
    assert gh.hasConverged() == o.converged
    sh, sd = gh.stats(), gd.stats()
    print(f"{name}: host path {sh['iterations']} iterations / {sh['evaluations']} evaluations, device path "
          f"{sd['iterations']} / {sd['evaluations']}, oracle {o.iterations} iterations; host vs oracle {dt:.2e} m {dr:.2e} rad")
