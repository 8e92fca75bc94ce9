"""The float64 controller replay of tests/ndtctl_ref.py, checked on the CPU before any GPU comparison: driven by the
oracle's derivatives it must reproduce oracle.NDT.align exactly (iterations, evaluations, convergence, final pose) in the
shipped configuration and in More-Thuente configurations, with no decision near its threshold; the fixture generators
(origin source, ascent start, snap round, clamp, iteration cap, More-Thuente edges) must reach their edges; and records
from the replay, mutated the way a subtly wrong controller would mutate them, must fail the comparison."""
import numpy as np
import pytest

import ndtctl_ref as X

F32 = np.float32
GUESS = np.array([[0.9999, -0.0100, 0.0030, 0.30], [0.0100, 0.9999, -0.0020, -0.20], [-0.0030, 0.0020, 1.0, 0.05],
                  [0, 0, 0, 1]], dtype=F32)
ITERATION_CAP = [(0, np.eye(4, dtype=F32)), (1, np.eye(4, dtype=F32)), (2, np.eye(4, dtype=F32))]
CONFIGS = {"shipped": X.config(), "mt": X.config(step_size=0.1, trans_eps=0.2, max_iterations=6),
           "mt_long": X.config(step_size=0.5, trans_eps=1.0, max_iterations=6)}


def _oracle(oracle_mod, src, tgt, res, cfg, method=2):
    o = oracle_mod.NDT(resolution=res, search_method=method, step_size=cfg["step_size"],
                       transformation_epsilon=cfg["trans_eps"], max_iterations=cfg["max_iterations"], num_threads=1)
    o.set_target(tgt)
    o.set_source(src)
    return o


def _replay_records(recs, cfg, guess, infos):
    """Replay every record of drive() from its predecessor's state, with the oracle's own (not quite symmetric) Hessian;
    returns (worst ratio, mismatches, near decisions)."""
    worst, bad, near = 0.0, [], []
    s = X.initial_state(guess)
    for r, inf in zip(recs, infos):
        before = dict(s, phase=int(r["phase_before"]))
        ref, info = X.step(before, None if not r["evaluated"] else r["tot"], cfg,
                           H_k2=None if r["evaluated"] else r["H"], H_full=inf["H_full"])
        w, b = X.compare(r, ref, info, X.is_mt_config(cfg))
        worst, bad, near = max(worst, w), bad + b, near + info["near"]
        s = X.state_of(r)
    return worst, bad, near


@pytest.mark.parametrize("cfg_name", list(CONFIGS))
def test_drive_reproduces_oracle_align(oracle_mod, pair_tiny, pair_small, golden, cfg_name):
    cfg = CONFIGS[cfg_name]
    cases = [("tiny", pair_tiny[0], pair_tiny[1], 2.0), ("small", pair_small[0], pair_small[1], 2.0)]
    if cfg_name != "mt_long":
        cases.append(("golden", golden["source"], golden["target"], 1.0))
    for name, src, tgt, res in cases:
        for guess in (np.eye(4, dtype=F32), GUESS):
            o = _oracle(oracle_mod, src, tgt, res, cfg)
            recs, res_d, infos = X.drive(o, guess, cfg, len(src))
            Tf = o.align(guess)
            assert res_d["iterations"] == o.iterations, (name, cfg_name)
            assert res_d["evaluations"] == o.evaluations, (name, cfg_name)
            assert res_d["converged"] == o.converged, (name, cfg_name)
            assert np.array_equal(res_d["final_T"], Tf), (name, cfg_name, np.abs(res_d["final_T"] - Tf).max())
            assert res_d["trans_probability"] == o.trans_probability
            worst, bad, near = _replay_records(recs, cfg, guess, infos)
            assert not bad, (name, cfg_name, bad[:3])
            assert not near, (name, cfg_name, near)


def test_more_thuente_fixtures_reach_the_loop_edges(oracle_mod, pair_tiny, pair_small):
    """eps >= 2 step_size on the tiny and small pairs: the open -> closed flip, the 10-step cap and at least three of the
    four trial-value cases."""
    cases, flips, closed, capped = set(), 0, 0, 0
    for (src, tgt, _), guess, cfg in ((pair_tiny, np.eye(4, dtype=F32), "mt_long"), (pair_tiny, GUESS, "mt_long"),
                                      (pair_small, GUESS, "mt_long"), (pair_tiny, GUESS, "mt")):
        if True:
            if True:
                o = _oracle(oracle_mod, src, tgt, 2.0, CONFIGS[cfg])
                recs, _, infos = X.drive(o, guess, CONFIGS[cfg], len(src))
                cases |= {i["mt_case"] for i in infos if i["mt_case"]}
                flips += sum(bool(i["decisions"].get("open_to_closed")) for i in infos)
                closed += sum(i["update_branch"] is not None and not r["open_interval"] for r, i in zip(recs, infos))
                capped += sum(int(r["step_iterations"]) == X.MAX_STEP_ITERATIONS for r in recs)
            near = [n for i in infos for n in i["near"]]
            assert not near, near
    print(f"\nMore-Thuente trial cases reached: {sorted(cases)}; open->closed flips {flips}; closed-interval updates "
          f"{closed}; 10-step caps {capped}; near-threshold decisions 0")
    assert cases >= {1, 2, 3} and flips > 0 and closed > 0 and capped > 0


def test_generators_reach_their_edges(oracle_mod, pair_small, golden):
    src, tgt, _ = pair_small
    cfg = CONFIGS["shipped"]
    # origin source: the rotation rows / columns of H and g are exactly zero in every round, LDL^T refuses, pivoted LU
    # fails and the minimum-norm SVD solve gives a translation-only direction
    osrc, otgt = X.origin_pair()
    o = _oracle(oracle_mod, osrc, otgt, 2.0, cfg)
    recs, res, infos = X.drive(o, np.eye(4, dtype=F32), cfg, len(osrc))
    solved = [i for i in infos if "solve" in i]
    assert res["converged"] and len(solved) >= 2
    for i in solved:
        H = i["H_full"]
        assert np.all(H[3:] == 0) and np.all(H[:, 3:] == 0) and np.any(H != 0) and not X.ldlt_accepts(H)
        assert np.all(i["solve"][3:] == 0) and np.any(i["solve"][:3] != 0)
    assert all(np.all(r["x_t"][3:] == 0) for r in recs)
    # ascent and snap rounds on the golden PCD
    gs, gt = golden["source"], golden["target"]
    o = _oracle(oracle_mod, gs, gt, 1.0, cfg)
    assert X.first_with(o, cfg, X.ascent_guesses(), len(gs), X.is_ascent_round) is not None
    assert X.first_with(o, cfg, X.edge_guesses(), len(gs), X.is_snap_round) is not None
    # clamp: the last steps are shorter than step_min = eps / 2, so a_t = eps / 2
    o = _oracle(oracle_mod, src, tgt, 2.0, cfg)
    _, _, infos = X.drive(o, GUESS, cfg, len(src))
    assert any(i["decisions"].get("clamp") == "min" for i in infos)
    # iteration cap: with max_iterations m the solve ends by nr_iterations > m at the latest
    for m, guess in ITERATION_CAP:
        c = X.config(max_iterations=m)
        o = _oracle(oracle_mod, src, tgt, 2.0, c)
        recs, res, _ = X.drive(o, guess, c, len(src))
        assert res["iterations"] == m + 2 and res["converged"], (m, res)


def test_power_of_the_replay_comparison(oracle_mod, pair_small):
    """Records that a subtly wrong controller would publish fail the comparison: the sign flip dropped, dir scaled by
    1 + 2^-20, psi and phi swapped in a closed-interval update, the clamp to step_min missing."""
    src, tgt, _ = pair_small
    cfg = CONFIGS["shipped"]
    o = _oracle(oracle_mod, src, tgt, 2.0, cfg)
    recs, _, infos = X.drive(o, GUESS, cfg, len(src))
    assert not _replay_records(recs, cfg, GUESS, infos)[1]
    k = next(i for i, r in enumerate(recs) if r["built"] and r["phase_after"] == X.PH_LS_FIRST)
    m = recs.copy()
    m[k]["dir"] = m[k]["dir"] * (1 + 2.0**-20)
    assert _replay_records(m, cfg, GUESS, infos)[1]
    m = recs.copy()
    m[k]["dir"], m[k]["d_phi_0"] = -m[k]["dir"], -m[k]["d_phi_0"]
    assert _replay_records(m, cfg, GUESS, infos)[1]
    kc = next(i for i, inf in enumerate(infos) if inf["decisions"].get("clamp") == "min")
    m = recs.copy()
    m[kc]["a_t"] = np.sqrt(np.dot(infos[kc]["solve"], infos[kc]["solve"]))
    assert _replay_records(m, cfg, GUESS, infos)[1]
    # psi / phi swap: a closed-interval update fed (psi, d_psi) instead of (phi, d_phi)
    mt = CONFIGS["mt_long"]
    for src_, tgt_ in ((src, tgt),):
        o = _oracle(oracle_mod, src_, tgt_, 2.0, mt)
        recs, _, infos = X.drive(o, GUESS, mt, len(src_))
        assert not _replay_records(recs, mt, GUESS, infos)[1]
        idx = [i for i, r in enumerate(recs) if r["phase_before"] == X.PH_LS_ITER and not r["open_interval"]
               and not _closed_in(recs, i)]
        assert idx, "no closed-interval update in the More-Thuente fixture"
        i = idx[0]
        m = recs.copy()
        prev = X.state_of(recs[i - 1])
        phi_t = -float(m[i]["tot"][0])
        d_phi_t = -X._dot(m[i]["tot"][1:7], prev["dir"])
        psi_t = phi_t - prev["phi_0"] - X.MU * prev["d_phi_0"] * prev["a_t"]
        d_psi_t = d_phi_t - X.MU * prev["d_phi_0"]
        conv, v = oracle_mod.mt_update(prev["a_l"], prev["f_l"], prev["g_l"], prev["a_u"], prev["f_u"], prev["g_u"],
                                       prev["a_t"], psi_t, d_psi_t)
        for j, name in enumerate(X.MT_FIELDS):
            m[i][name] = v[j]
        assert _replay_records(m, mt, GUESS, infos)[1]


def _closed_in(recs, i):
    """True when record i's round closed the interval itself (its update used the flipped values)."""
    return i > 0 and bool(recs[i - 1]["open_interval"])


def test_near_f32_boundary():
    f = np.float32(1.25)
    mid = (float(f) + float(np.nextafter(f, np.float32(2)))) / 2
    assert X.near_f32_boundary(mid)[0] and X.near_f32_boundary(np.nextafter(mid, 2))[0]
    assert not X.near_f32_boundary(float(f))[0]
