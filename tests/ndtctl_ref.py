"""A float64 replay of the NDT solver's controller, one round at a time, written from pclomp's computeTransformation and
computeStepLengthMT (the Newton loop and the More-Thuente line search) and reusing the oracle's JacobiSVD solve, trial
value, interval update, pose_to_matrix and angle tables. Nothing here needs a GPU.

The solver kernel runs the reference loop as a sequence of rounds: every round consumes the totals of one evaluation
(score, g, the upper Hessian, hits) and either publishes the control block of the next evaluation, finishes, or leaves the
kernel for the f64 radius-Hessian pass (K2). The phase says where in the loop a round resumes:
  PH_INITIAL    the initial computeDerivatives (:119), then the first Newton solve
  PH_LS_FIRST   the first evaluation of computeStepLengthMT (:821)
  PH_LS_ITER    a More-Thuente evaluation (:865, no Hessian)
  PH_LS_HESSIAN the K2 Hessian has been injected (:912-913); the round evaluates nothing
step() takes the state before a round (the previous trace record, or initial_state()) and the totals the round consumed,
and returns the reference's state after it, its discrete decisions, an absolute bound for every continuous field it
recomputed (fields it did not touch must be equal bit for bit) and the decisions whose input lies within its bound of the
threshold (near: such a fixture cannot pin the decision and is moved off the threshold). A decision on a value the
replay reproduces bit for bit (the convergence test on the previous a_t, every More-Thuente test) is exact.

Bounds, u = 2^-53:
  * the Newton direction: the device solves H x = -g by LDL^T (fast path) or pivoted LU / Jacobi SVD (scalar path), the
    reference by JacobiSVD. |d dir_i| <= C_SOLVE kappa u, kappa = s_max / s_min over the singular values the SVD keeps
    (s > 6 eps s_max); the norm moves by the same relative amount.
  * d_phi_0 = -g . dir: |g|_2 sqrt(6) |d dir| plus the dot product's own rounding, 8 u sum |g_i dir_i| (FMA contraction
    included).
  * a_t = clamp(norm): the norm's bound unless a clamp bound it (then exact); x_t = p + dir a_t: |d dir| a_t + |d a_t| plus
    2 u (|p| + |dir a_t|) for the fused or unfused multiply-add; the same 2 u term for p += dir a_t.
  * More-Thuente: the controller spells phi, psi, their slopes, the interval updates and the trial value out un-fused in
    the reference's evaluation order (ndt_math.cuh), and sqrt and division are correctly rounded, so from the same state
    and totals they are bitwise the replay's: bound 0, and every decision on them is exact, ties included. Only x_t =
    p + dir a_t keeps its 2 u term (the multiply-add may be fused).
"""
from __future__ import annotations

import math

import numpy as np

import oracle

U = 2.0**-53
MU, NU = 1.0e-4, 0.9
MAX_STEP_ITERATIONS = 10
C_SOLVE = 64.0
PH_INITIAL, PH_LS_FIRST, PH_LS_ITER, PH_LS_HESSIAN = 0, 1, 2, 3
TRI = [(i, j) for i in range(6) for j in range(i, 6)]
VEC = ("p", "dir", "x_t", "g")
SCALARS = ("a_t", "phi_0", "d_phi_0", "a_l", "f_l", "g_l", "a_u", "f_u", "g_u", "score")
INTS = ("phase", "interval_converged", "open_interval", "step_iterations", "nr_iterations", "evaluations", "converged",
        "done", "hits_total")
MT_FIELDS = ("a_l", "f_l", "g_l", "a_u", "f_u", "g_u")


def config(step_size=0.1, trans_eps=0.1, max_iterations=35):
    """The solver settings the controller reads (the reference constructor's defaults)."""
    return dict(step_size=float(step_size), trans_eps=float(trans_eps), max_iterations=int(max_iterations))


def is_mt_config(cfg):
    """The More-Thuente loop runs only when step_max <= step_min (computeStepLengthMT's interval_converged, :803)."""
    return not (cfg["step_size"] - cfg["trans_eps"] / 2 > 0)


def initial_pose(guess):
    """p of :103-111: the guess's translation and eulerAngles(0, 1, 2) in float, widened to double."""
    T = np.asarray(guess, dtype=np.float32)
    ang = oracle.euler_angles_012(T[:3, :3])
    return np.array([T[0, 3], T[1, 3], T[2, 3], ang[0], ang[1], ang[2]], dtype=np.float64)


def initial_state(guess):
    s = {k: np.zeros(6) for k in VEC}
    s.update({k: 0.0 for k in SCALARS})
    s.update({k: 0 for k in INTS})
    s["p"] = initial_pose(guess)
    s["H"] = np.zeros((6, 6))
    return s


def state_of(rec):
    """The controller state after a trace record's round."""
    s = {k: np.array(rec[k], dtype=np.float64) for k in VEC}
    s.update({k: float(rec[k]) for k in SCALARS})
    s.update({k: int(rec[k]) for k in INTS if k != "phase"})
    s["phase"] = int(rec["phase_after"])
    s["H"] = np.array(rec["H"], dtype=np.float64).reshape(6, 6)
    return s


def totals(score, g, H, hits, hessian=True):
    """The 32-slot reduction vector of one evaluation: score, g, upper H row-major, hits."""
    t = np.zeros(32)
    t[0], t[1:7], t[28] = score, g, hits
    if hessian:
        t[7:28] = [H[i, j] for i, j in TRI]
    return t


def _dot(a, b):
    s = 0.0
    for x, y in zip(a, b):
        s += float(x) * float(y)
    return s


def _kappa(H):
    sv = np.linalg.svd(H, compute_uv=False)
    keep = sv[sv > sv.max() * 6.0 * np.finfo(float).eps] if sv.max() > 0 else sv[:0]
    return float(keep.max() / keep.min()) if len(keep) else math.inf


def mt_case(a_l, f_l, g_l, a_u, f_u, g_u, a_t, f_t, g_t):
    """Which branch trialValueSelectionMT takes (:673-753): 1 f_t > f_l, 2 opposite slopes, 3 |g_t| <= |g_l|, 4 else."""
    if f_t > f_l:
        return 1
    if g_t * g_l < 0:
        return 2
    if abs(g_t) <= abs(g_l):
        return 3
    return 4


def update_branch(a_l, f_l, g_l, a_t, f_t, g_t):
    """Which branch updateIntervalMT takes (:632-670): 1 f_t > f_l, 2 / 3 by the sign of g_t (a_l - a_t), 4 converged."""
    if f_t > f_l:
        return 1
    if g_t * (a_l - a_t) > 0:
        return 2
    if g_t * (a_l - a_t) < 0:
        return 3
    return 4


def step(s, tot, cfg, H_k2=None, H_full=None):
    """One controller round. Returns (state after, info); info holds 'tol' (field -> absolute bound), 'near' (decisions
    within their bound of the threshold), 'decisions', 'build' ((compute_hessian, build_f64) of the block published, or
    None), 'mt_case' and 'update_branch' (or None). H_full replaces the symmetric Hessian the upper totals give: the
    oracle's f32 sums leave its H a few f32 ulp from symmetric, and drive() follows the oracle exactly."""
    s = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in s.items()}
    smax, smin = cfg["step_size"], cfg["trans_eps"] / 2
    tol, near, dec = {}, [], {}
    info = dict(tol=tol, near=near, decisions=dec, build=None, mt_case=None, update_branch=None)
    s["done"] = 0

    def check_near(name, value, bound):
        if abs(value) <= bound:
            near.append(name)

    phase = s["phase"]
    phi_t = d_phi_t = psi_t = d_psi_t = 0.0
    if phase == PH_LS_HESSIAN:
        s["H"] = np.array(H_k2, dtype=np.float64).reshape(6, 6)
        act = "end"
    else:
        tot = np.asarray(tot, dtype=np.float64)
        s["score"], s["g"] = float(tot[0]), tot[1:7].copy()
        H = np.zeros((6, 6))
        if phase != PH_LS_ITER:
            for k, (i, j) in enumerate(TRI):
                H[i, j] = H[j, i] = tot[7 + k]
        s["H"] = H if H_full is None else np.array(H_full, dtype=np.float64)
        s["hits_total"] += int(tot[28] + 0.5)
        s["evaluations"] += 1
        if phase == PH_INITIAL:
            act = "begin"
        else:
            phi_t = -s["score"]
            d_phi_t = -_dot(s["g"], s["dir"])
            psi_t = phi_t - s["phi_0"] - MU * s["d_phi_0"] * s["a_t"]
            d_psi_t = d_phi_t - MU * s["d_phi_0"]
            if phase == PH_LS_ITER:
                if s["open_interval"] and psi_t <= 0 and d_psi_t >= 0:  # :878-889
                    dec["open_to_closed"] = True
                    s["open_interval"] = 0
                    s["f_l"] = s["f_l"] + s["phi_0"] - MU * s["d_phi_0"] * s["a_l"]
                    s["g_l"] = s["g_l"] + MU * s["d_phi_0"]
                    s["f_u"] = s["f_u"] + s["phi_0"] - MU * s["d_phi_0"] * s["a_u"]
                    s["g_u"] = s["g_u"] + MU * s["d_phi_0"]
                f_t, g_t = (psi_t, d_psi_t) if s["open_interval"] else (phi_t, d_phi_t)
                br = update_branch(s["a_l"], s["f_l"], s["g_l"], s["a_t"], f_t, g_t)
                info["update_branch"] = br
                conv, v = oracle.mt_update(s["a_l"], s["f_l"], s["g_l"], s["a_u"], s["f_u"], s["g_u"], s["a_t"], f_t, g_t)
                s["interval_converged"] = int(conv)
                for k, name in enumerate(MT_FIELDS):
                    s[name] = float(v[k])
                s["step_iterations"] += 1
            act = "check"
    for _ in range(8):
        if act == "check":  # :834
            if (not s["interval_converged"] and s["step_iterations"] < MAX_STEP_ITERATIONS
                    and not (psi_t <= 0 and d_phi_t <= -NU * s["d_phi_0"])):
                f_t, g_t = (psi_t, d_psi_t) if s["open_interval"] else (phi_t, d_phi_t)
                args = (s["a_l"], s["f_l"], s["g_l"], s["a_u"], s["f_u"], s["g_u"], s["a_t"], f_t, g_t)
                case = mt_case(*args)
                info["mt_case"] = case
                a = max(min(oracle.mt_trial(*args), smax), smin)
                s["a_t"] = a
                s["x_t"] = s["p"] + s["dir"] * a
                tol["x_t"] = 2 * U * (np.abs(s["p"]) + np.abs(s["dir"] * a))
                s["phase"] = PH_LS_ITER
                info["build"] = (0, 1)
                return s, info
            if s["step_iterations"]:  # :912-913
                s["phase"] = PH_LS_HESSIAN
                s["done"] = 2
                return s, info
            act = "end"
        if act == "end":  # :143-164
            s["p"] = s["p"] + s["dir"] * s["a_t"]
            tol["p"] = 2 * U * (np.abs(s["p"]) + np.abs(s["dir"] * s["a_t"]))
            conv = s["nr_iterations"] > cfg["max_iterations"] or (s["nr_iterations"] and abs(s["a_t"]) < cfg["trans_eps"])
            s["nr_iterations"] += 1
            if conv:
                s["converged"] = 1
                s["done"] = 1
                return s, info
            act = "begin"
        if act == "begin":  # :127-142 and the prologue of computeStepLengthMT :761-821
            g = s["g"]
            dp = oracle.svd6_solve(s["H"], -g)
            norm = math.sqrt(_dot(dp, dp))
            if norm == 0 or norm != norm:
                s["converged"] = int(norm == norm)
                s["done"] = 1
                info["solve"] = dp
                return s, info
            d = dp / norm
            kappa = _kappa(s["H"])
            t_dir = C_SOLVE * kappa * U
            t_norm = t_dir * norm
            info["kappa"], info["solve"] = kappa, dp
            s["phi_0"] = -s["score"]
            d_phi_0 = -_dot(g, d)
            t_dphi = float(np.linalg.norm(g)) * math.sqrt(6) * t_dir + 8 * U * float(np.abs(g * d).sum())
            check_near("d_phi_0 >= 0 (ascent: flip)", d_phi_0, t_dphi)
            dec["flip"] = bool(d_phi_0 > 0)
            if d_phi_0 >= 0:
                if d_phi_0 == 0:
                    s["dir"], s["d_phi_0"], s["a_t"] = d, d_phi_0, 0.0  # :771-772, zero step
                    act = "end"
                    continue
                d_phi_0 = -d_phi_0
                d = -d
            s["dir"], s["d_phi_0"] = d, d_phi_0
            tol["dir"] = np.full(6, t_dir)
            tol["d_phi_0"] = t_dphi
            s["step_iterations"] = 0
            s["a_l"] = s["a_u"] = 0.0
            s["f_l"] = s["phi_0"] - s["phi_0"] - MU * d_phi_0 * 0.0  # psiMT(0, phi_0, phi_0, d_phi_0, mu)
            s["g_l"] = d_phi_0 - MU * d_phi_0
            s["f_u"], s["g_u"] = s["f_l"], s["g_l"]
            tol["g_l"] = tol["g_u"] = 2 * t_dphi
            s["interval_converged"] = int(smax - smin > 0)
            s["open_interval"] = 1
            if smax > smin:  # otherwise a_t = step_min whatever the norm
                check_near("norm > step_max", norm - smax, t_norm)
                check_near("norm < step_min (clamp)", norm - smin, t_norm)
            dec["clamp"] = "max" if norm > smax else ("min" if norm < smin else None)
            a = max(min(norm, smax), smin)
            t_a = 0.0 if a in (smax, smin) else t_norm
            s["a_t"] = a
            s["x_t"] = s["p"] + d * a
            tol["a_t"] = t_a
            tol["x_t"] = t_dir * a + np.abs(d) * t_a + 2 * U * (np.abs(s["p"]) + np.abs(d * a))
            s["phase"] = PH_LS_FIRST
            info["build"] = (1, 0 if s["interval_converged"] else 1)
            return s, info
    s["converged"] = 0
    s["done"] = 1
    return s, info


def compare(rec, ref, info, mt):
    """Largest |device - replay| / bound over the continuous fields of one round, and the list of mismatches (discrete
    fields that differ, continuous fields outside their bound). Fields the round did not recompute must match exactly.
    mt: also compare the More-Thuente interval (the fast path keeps none)."""
    bad, worst = [], 0.0
    for k in INTS:
        got = int(rec["phase_after"]) if k == "phase" else int(rec[k])
        if got != ref[k]:
            bad.append((k, got, ref[k]))
    for k in VEC + SCALARS:
        if k in MT_FIELDS and not mt:
            continue
        got = np.asarray(rec[k], dtype=np.float64)
        t = np.asarray(info["tol"].get(k, 0.0), dtype=np.float64)
        dev = np.abs(got - ref[k])
        if np.any(dev > t):
            bad.append((k, got.tolist(), np.asarray(ref[k]).tolist(), t.tolist()))
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(dev == 0, 0.0, dev / t)
        worst = max(worst, float(np.max(r)))
    return worst, bad


def near_f32_boundary(v64, ulps=2):
    """True where a float64 value lies within `ulps` float64 ulp of a float32 rounding boundary (the midpoint between two
    neighbouring floats): there an f64 error of that size can change the float32 it rounds to."""
    v = np.atleast_1d(np.asarray(v64, dtype=np.float64))
    f = v.astype(np.float32)
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    f64 = f.astype(np.float64)
    d = np.minimum(np.abs(v - (f64 + up) / 2), np.abs(v - (f64 + dn) / 2))
    return d <= ulps * np.spacing(np.abs(v))


def record(s, info, rnd, launch, tot, evaluated, fast=0, hits=None):
    """One trace record (registration.NormalDistributionsTransform.TRACE_DTYPE) of a replayed round."""
    from lidarslam_ros2_b200.registration import NormalDistributionsTransform as NDT

    r = np.zeros((), dtype=NDT.TRACE_DTYPE)
    r["round"], r["launch"], r["fast"], r["evaluated"] = rnd, launch, fast, int(evaluated)
    for k in INTS:
        if k != "phase":
            r[k] = s[k]
    r["phase_after"] = s["phase"]
    for k in VEC + SCALARS:
        r[k] = s[k]
    if tot is not None:
        r["tot"] = tot
    b = info["build"]
    r["mode"] = 0 if b else (2 if s["done"] == 2 else 1)
    if b:
        import ndtref

        r["built"], r["compute_hessian"], r["build_f64"] = 1, b[0], b[1]
        r["T"] = oracle.pose_to_matrix(s["x_t"])[:3].reshape(12)
        j, h = oracle.angle_tables(s["x_t"])
        r["jang"], r["hang"] = j.reshape(24), h.reshape(45)
        if b[1]:
            _, _, j64, h64 = ndtref.angle_tables(s["x_t"], minus_sy=True, f64=True)
            r["jd"], r["hd"] = j64.reshape(24), h64.reshape(45)
    return r


def drive(o, guess, cfg, n_src, max_rounds=5000):
    """A whole solve by the replay with the oracle's derivatives (o: oracle.NDT with the same target, source and
    settings). Returns (records, result) with result = iterations, evaluations, converged, final_T, trans_probability,
    and per round the replay's info (records[i], infos[i])."""
    guess = np.asarray(guess, dtype=np.float32)
    s = initial_state(guess)
    T, x, hess = guess, s["p"].copy(), 1
    recs, infos, launch, rnd = [], [], 0, 0
    for _ in range(max_rounds):
        if s["phase"] == PH_LS_HESSIAN:
            H_k2, tot, evaluated = o.hessian_radius(T, x), None, False
            s_before = dict(s, phase=PH_LS_HESSIAN)
        else:
            score, g, H = o.derivatives(T, x, bool(hess))
            tot, H_k2, evaluated = totals(score, g, H, 0, bool(hess)), None, True
            s_before = s
        H_full = H if evaluated and hess else None
        s, info = step(s_before, tot, cfg, H_k2, H_full=H_full)
        info["H_full"] = H_full
        if not evaluated:
            s["H"] = np.array(H_k2).reshape(6, 6)
        r = record(s, info, rnd, launch, tot, evaluated)
        r["phase_before"] = s_before["phase"]
        r["H"] = s["H"].reshape(36) if not evaluated else 0.0
        recs.append(r)
        infos.append(info)
        rnd += 1
        if s["done"] == 1:
            break
        if s["done"] == 2:
            launch, rnd = launch + 1, 0
            continue
        T = oracle.pose_to_matrix(s["x_t"])
        x, hess = s["x_t"].copy(), info["build"][0]
    F = np.eye(4, dtype=np.float32)
    built = [r for r in recs if r["built"]]
    final_T = np.vstack([built[-1]["T"].reshape(3, 4), [0, 0, 0, 1]]).astype(np.float32) if built else guess
    res = dict(iterations=s["nr_iterations"], evaluations=s["evaluations"], converged=bool(s["converged"]),
               final_T=final_T if built else F @ guess, trans_probability=s["score"] / n_src)
    return np.array(recs), res, infos


# ---- fixtures at the controller's edges -----------------------------------------------------------------------------
def ldlt_accepts(H):
    """Whether the fast path's LDL^T solve (ndt_math.cuh ldlt_solve6_upper) takes H: every pivot above 1e-10 of the
    largest diagonal entry (the f64 elimination here differs from the device's by rounding only)."""
    U_ = np.array(H, dtype=np.float64)
    dmax = np.abs(np.diag(U_)).max()
    if not dmax > 0:
        return False
    for k in range(6):
        if not abs(U_[k, k]) > 1e-10 * dmax:
            return False
        U_[k + 1:, k + 1:] -= np.outer(U_[k + 1:, k], U_[k, k + 1:]) / U_[k, k]
    return True


def origin_pair(n_src=64, n_tgt=3000, seed=0):
    """Source points all exactly at the origin against a blob of target points around it: every point Jacobian and every
    second-derivative vector is (table) . 0 = 0, so the rotation rows and columns of H and g are exactly zero in every
    round. LDL^T refuses, pivoted LU fails, and the minimum-norm SVD solve decides a translation-only step."""
    rng = np.random.default_rng(seed)
    tgt = (np.array([0.4, -0.3, 0.2]) + rng.normal(0, 1, (n_tgt, 3)) * np.array([0.6, 0.4, 0.25])).astype(np.float32)
    return np.zeros((n_src, 3), dtype=np.float32), tgt


def ascent_guesses():
    """Guesses offset from the scene's true pose far enough that H is indefinite at some Newton step."""
    out = []
    for t in (0.6, 0.9, 1.2, 1.5):
        for yaw in (0.0, 0.05, -0.08):
            c, s_ = math.cos(yaw), math.sin(yaw)
            out.append(np.array([[c, -s_, 0, t], [s_, c, 0, -0.5 * t], [0, 0, 1, 0.1], [0, 0, 0, 1]], dtype=np.float32))
    return out


def first_with(o, cfg, guesses, n_src, pred):
    """The first guess whose replayed solve (drive) has a round for which pred(record, info) holds, or None."""
    for G in guesses:
        recs, _, infos = drive(o, G, cfg, n_src)
        if any(pred(r, i) for r, i in zip(recs, infos)):
            return G
    return None


def is_ascent_round(r, info):
    """A Newton step whose d_phi_0 > 0 on a Hessian the fast path's LDL^T takes: the fast path flips the direction."""
    return bool(info["decisions"].get("flip")) and info.get("H_full") is not None and ldlt_accepts(info["H_full"])


def is_snap_round(r, info):
    """A published pose with an angle in [1e-5, 1e-4): the angle tables snap it (ndt_omp_impl.hpp:292-325); a snap
    threshold ten times smaller would not."""
    a = np.abs(np.asarray(r["x_t"])[3:6])
    return bool(r["built"]) and bool(((a >= 1e-5) & (a < 1e-4)).any())


def edge_guesses():
    """The identity and the ascent guesses: on the golden PCD (resolution 1.0) they reach ascent and snap rounds."""
    return [np.eye(4, dtype=np.float32)] + ascent_guesses()
