"""tests/gicpref.py against the CPU oracle, its power to see the kernel mistakes it exists for, and its fixture
generators. No GPU needed."""
import numpy as np
import pytest

import gicpref as G
import gridref as GR

F32 = np.float32
STATES = [G.STATES["zero"], G.STATES["moderate"], np.array([0.02, 0.01, -0.015, 0.004, 0.003, -0.006])]


def _scene(name):
    from lidarslam_ros2_b200 import synth

    if name == "pair":
        return G.surface_pair()
    s, t, _ = synth.registration_pair(name, 2.0)
    return s, t


_cache = {}


def _oracle_case(oracle_mod, name):
    """The oracle after one outer iteration under G.GUESS (correspondences at transformation_ = I) and the reference's
    correspondences on the oracle's covariances."""
    if name in _cache:
        return _cache[name]
    src, tgt = _scene(name)
    o = oracle_mod.GICP(max_correspondence_distance=5.0, max_iterations=1)
    o.set_target(tgt)
    o.set_source(src)
    o.align(G.GUESS)
    ref = G.correspondences(src, tgt, o.covariances("source"), o.covariances("target"), 5.0, guess=G.GUESS)
    _cache[name] = (o, src, tgt, ref)
    return _cache[name]


def _oracle_maha(o, n):
    s, _, M = o.correspondences()
    full = np.tile(np.eye(3, dtype=F32), (n, 1, 1))
    full[s] = M
    return full


@pytest.mark.parametrize("name", ["pair", "tiny", "small"])
def test_reference_correspondences_match_oracle(oracle_mod, name):
    o, src, tgt, ref = _oracle_case(oracle_mod, name)
    s, t, M = o.correspondences()
    rs = np.nonzero(ref["corr"] >= 0)[0]
    assert np.array_equal(rs, s)
    assert np.array_equal(ref["corr"][rs], t)
    assert ref["m"] == o.num_correspondences() >= 4
    # the oracle's matrix product and inverse round in another order: one f32 ulp apart at most
    km = ref["maha"][rs]
    ulp = np.spacing(np.maximum(np.abs(km), np.abs(M)).astype(F32))
    assert np.all(np.abs(km.astype(np.float64) - M) <= ulp), name
    err = np.abs(km - ref["maha_exact"][rs]).max(axis=(1, 2))
    ratio = float((err / ref["maha_bound"][rs]).max())
    print(f"{name}: m = {ref['m']}, maha_exact max ratio {ratio:.3g}")
    assert ratio <= 1.0


@pytest.mark.parametrize("name", ["pair", "tiny", "small"])
def test_reference_objective_matches_oracle(oracle_mod, name):
    o, src, tgt, ref = _oracle_case(oracle_mod, name)
    maha = _oracle_maha(o, len(src))
    worst = 0.0
    for x in STATES:
        T = o.apply_state(x)
        r = G.objective(T, x, ref["moved"], tgt, ref["corr"], maha, depth=ref["m"])
        fo, go = o.fdf(x)
        f32o = o.f_only(x)
        assert abs(r["f"] - fo) <= 2 * r["b_f"], (name, x, r["f"], fo, r["b_f"])
        assert abs(r["f32path"] - f32o) <= 2 * r["b_f32path"], (name, x, r["f32path"], f32o)
        assert np.all(np.abs(r["g"] - go) <= 2 * r["b_g"]), (name, x, r["g"] - go, r["b_g"])
        worst = max(worst, abs(r["f"] - fo) / r["b_f"], abs(r["f32path"] - f32o) / r["b_f32path"],
                    float((np.abs(r["g"] - go) / r["b_g"]).max()))
    print(f"{name}: largest |oracle - ref| / bound {worst:.3g}")


@pytest.mark.parametrize("name", ["pair", "tiny", "small"])
def test_reference_power(oracle_mod, name):
    """The bounds are tight enough to see: f-only requests served from the f64 path, R[0,1] and R[1,0] swapped, and a
    dropped correspondence."""
    o, src, tgt, ref = _oracle_case(oracle_mod, name)
    maha = _oracle_maha(o, len(src))
    x = G.STATES["moderate"]
    T = o.apply_state(x)
    depth = G.depth_device(len(src), 132)
    r = G.objective(T, x, ref["moved"], tgt, ref["corr"], maha, depth=depth)
    assert abs(r["f32path"] - r["f"]) > 10 * (r["b_f"] + r["b_f32path"]), name
    sw = G.objective(T, x, ref["moved"], tgt, ref["corr"], maha, depth=depth, R_swap=True)
    assert np.max(np.abs(sw["g"][3:] - r["g"][3:]) / r["b_g"][3:]) > 10, name
    fd = r["terms"]["fdf"]
    total = np.abs(fd).sum()
    big = np.abs(fd) >= 1e-9 * total
    moved_by = np.abs(fd[big]) / r["m"]  # dropping term i moves f by term_i / m (the normalisation stays m or moves more)
    assert np.all(moved_by > 10 * r["b_f"]), name
    caught = np.abs(fd) / r["m"] > 10 * r["b_f"]
    print(f"{name}: smallest dropped term caught {np.abs(fd[caught]).min() / total:.3g} of sum|term|")


def test_nn1_candidates_match_brute_force():
    rng = np.random.default_rng(3)
    t = np.concatenate([rng.normal(size=(3000, 3)), GR.lattice((6, 6, 6), (0.5, 0.5, 0.5))]).astype(F32)
    q = np.concatenate([rng.normal(size=(800, 3)) * 1.5, GR.lattice((6, 6, 6), (0.5, 0.5, 0.5), origin=(0.25, 0.0, 0.0)),
                        t[:50]]).astype(F32)
    for pts in (t, GR.shifted(t, (1500.0, -2300.0, 40.0))):
        qq = q if pts is t else GR.shifted(q, (1500.0, -2300.0, 40.0))
        i0, d0 = GR.nn1_ref(pts, qq)
        i1, d1 = G.nn1(pts, qq, brute_limit=0)
        assert np.array_equal(i0, i1) and np.array_equal(d0, d1)


def test_maha_kernel_order_is_the_kernel_arithmetic():
    """Spot-check the vectorised operation order against a scalar restatement of gicp_corr_kernel."""
    rng = np.random.default_rng(5)
    R = G.transform_R(G.BIG_ROT, G.GUESS)
    for _ in range(20):
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        C1 = np.eye(3) - 0.999 * np.outer(u, u)
        v = rng.normal(size=3)
        v /= np.linalg.norm(v)
        C2 = np.eye(3) - 0.999 * np.outer(v, v)
        A = C1.ravel()
        M = [0.0] * 9
        Tm = [0.0] * 9
        r9 = R.ravel()
        for r in range(3):
            for c in range(3):
                M[r * 3 + c] = r9[r * 3] * A[c] + r9[r * 3 + 1] * A[3 + c] + r9[r * 3 + 2] * A[6 + c]
        for r in range(3):
            for c in range(3):
                Tm[r * 3 + c] = M[r * 3] * r9[c * 3] + M[r * 3 + 1] * r9[c * 3 + 1] + M[r * 3 + 2] * r9[c * 3 + 2]
        Tm = [a + b for a, b in zip(Tm, C2.ravel())]
        want = G._inverse3(np.array([Tm])).astype(F32).reshape(3, 3)
        got = G.maha_kernel_order(R, C1[None], C2[None])[0]
        assert np.array_equal(want.view(np.int32), got.view(np.int32))


def test_state_transform_bound_holds_for_the_oracle(oracle_mod):
    o = oracle_mod.GICP()
    for x in G.STATES.values():
        T = o.apply_state(x)
        T64, b = G.state_T_bound(x)
        assert np.all(np.abs(T[:3].astype(np.float64) - T64) <= b), x


def test_generators_produce_their_edges():
    src, tgt, expect = G.gate_pair(0.5)
    idx, d2 = GR.nn1_ref(tgt, src)
    assert d2[0] == F32(0.25) and d2[1] < F32(0.25) < d2[2]
    assert np.array_equal(np.where(d2.astype(np.float64) < 0.25, idx, -1), expect)
    src, tgt, cd = G.far_pass_scene()
    far = G.ring_distance(tgt, src[:200])
    _, d2 = GR.nn1_ref(tgt, src[:200])
    assert far.min() > 3 and d2.max() < cd * cd
    s = G.exact_m_scan(tgt, 4)
    _, d2 = GR.nn1_ref(tgt, s)
    assert int((d2 < 25.0).sum()) == 4
    n = 33537
    n_eval, chunk = G.evaluator_partition(n, 132)
    assert (n_eval, chunk) == (131, 257)
    for which in (0, n_eval // 2, n_eval - 1):
        c, (lo, hi) = G.confine_to_chunk(np.zeros((n, 3), F32), n_eval, chunk, which)
        assert np.all(c[lo:hi, 2] == 0) and np.all(c[:lo, 2] == G.FAR) and np.all(c[hi:, 2] == G.FAR)
    assert hi - lo == n - (n_eval - 1) * chunk < chunk  # the last chunk is ragged
    lad = G.ladder(132, host=True)
    assert 256 * 131 + 1 in lad and 512 * 132 + 1 in lad and 4 in lad
    assert G.depth_device(256 * 131, 132) + 1 == G.depth_device(256 * 131 + 1, 132)  # a thread takes two points
