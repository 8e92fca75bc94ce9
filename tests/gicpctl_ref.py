"""A float64 replay of GICP's optimiser, written from the algorithm and checked against traces of it, with no GPU.

The inner solver of estimateRigidTransformationBFGS (gicp_omp_impl.hpp:180-241) is PCL 1.12 `BFGS<Functor>` (external),
a port of GSL's vector_bfgs2 with Fletcher's bracketing / sectioning line search (multimin/linear_minimize.c), called with
rho = sigma = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, order 3 and step_size 1. It is restated here in plain Python
floats, one operation at a time in the algorithm's order (sequential dot products from +0.0, compound assignments as
written), as a coroutine: `bfgs()` yields ("call", want_grad, x) and receives (f, g), and yields ("step", status, x, f, g,
inner) once per minimizeOneStep. Python floats are IEEE doubles without contraction, and the optimiser uses only + - * /,
sqrt, fabs, fmax, fmin and comparisons, so given the same (f, g) it asks for exactly the same x at every call: a replay
of a trace is compared bit for bit.

`replay()` drives the coroutine with the recorded (f, g) of a trace (the engine's b200reg_gicp_trace_record or the
oracle's GicpTraceRec, the same layout) and checks the outer loop of computeTransformation (:369-515):
  * x0 comes from glibc atan2f / asinf of the f32 transformation: it must be f32-representable and within 1 f32 ulp of
    the f64 value rounded to f32 (the translation entries exactly);
  * transformation_ after applyState comes from host or device cosf / sinf: within gicpref.state_T_bound of x;
  * given the recorded matrices, delta (an f32 subtraction, then the f64 ratio), the delta < 1 / max_iterations / m < 4
    decisions and final_T = previous * guess (f32 products and sums) are exact. A convergence decision whose delta lies
    within its bound (ratio times the transformation's bound) of 1 is counted as near.
It also counts the line-search branches it takes. `MUTATIONS` are subtly wrong optimisers for the power checks.
"""
from __future__ import annotations

import math
from collections import Counter

import numpy as np

import gicpref as G

F32 = np.float32
EPS = 2.220446049250313e-16
NAN = float("nan")
RUNNING, SUCCESS, NO_PROGRESS, NOT_STARTED = -1, 0, 1, -2
RHO, SIGMA, TAU1, TAU2, TAU3, ORDER, STEP_SIZE = 0.01, 0.01, 9.0, 0.05, 0.5, 3, 1.0
BRACKET_ITERS = SECTION_ITERS = 100

# subtly wrong optimisers: each must fail the replay of at least one trace
MUTATIONS = ("tau_swap",      # tau2 and tau3 exchanged in the sectioning interval
             "quad_always",   # the quadratic interpolation even when fpb is finite
             "no_dir",        # the sign flip of the new direction dropped
             "no_floor",      # alpha1 without the 10 eps |f0| floor of delta
             "gt_bracket",    # falpha > falpha_prev instead of >= in the bracketing f test
             "cap19",         # an inner cap of 19
             "fpb_zero",      # fpb = 0 instead of NaN after an f-increase bracket
             "eps_swap")      # rotation and translation epsilon ratios exchanged in the outer loop
# no fixture found so far takes a step short enough for the floor or an exactly repeated f in the bracketing to matter
UNREACHED = ("no_floor", "gt_bracket")


def _div(a, b):
    """IEEE a / b (Python raises on a zero divisor)."""
    if b != 0 or math.isnan(b):
        return a / b
    if a == 0 or math.isnan(a):
        return NAN
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def _sqrt(a):
    return math.sqrt(a) if a >= 0 else NAN


def _fmax(a, b):
    return b if math.isnan(a) else a if math.isnan(b) else (a if a > b else b)


def _fmin(a, b):
    return b if math.isnan(a) else a if math.isnan(b) else (a if a < b else b)


def _dot(a, b):
    s = 0.0
    for u, v in zip(a, b):
        s = s + u * v
    return s


def _norm(a):
    return _sqrt(_dot(a, a))


class _Bfgs:
    """The minimiser's state (vector_bfgs2 + the line search's cached function values)."""

    def __init__(self, mut, counts):
        self.mut, self.c = mut, counts
        self.f, self.gradient = 0.0, [0.0] * 6
        self.delta_f = self.fp0 = self.pnorm = self.g0norm = 0.0
        self.x0, self.g0, self.dx, self.p = [0.0] * 6, [0.0] * 6, [0.0] * 6, [0.0] * 6
        self.f_alpha = self.df_alpha = 0.0
        self.x_alpha, self.g_alpha = [0.0] * 6, [0.0] * 6
        self.f_key = self.df_key = self.x_key = self.g_key = 0.0

    # ---- functor calls ----
    def _fdf(self, x):
        f, g = yield ("call", 1, list(x))
        return float(f), [float(v) for v in g]

    def _f(self, x):
        f, _ = yield ("call", 0, list(x))
        return float(f)

    # ---- vector_bfgs2 ----
    def init(self, x):
        self.delta_f = 0.0
        self.dx = [0.0] * 6
        self.f, self.gradient = yield from self._fdf(x)
        self.x0, self.g0 = list(x), list(self.gradient)
        self.g0norm = _norm(self.g0)
        self.p = [_div(gi * -1, self.g0norm) for gi in self.gradient]
        self.pnorm = _norm(self.p)
        self.fp0 = -self.g0norm
        self._change_direction()

    def step(self, x):
        c = self.c
        alpha = 0.0
        f0 = self.f
        if self.pnorm == 0.0 or self.g0norm == 0.0 or self.fp0 == 0:
            self.dx = [0.0] * 6
            c["entry_noprogress"] += 1
            return NO_PROGRESS
        if self.delta_f < 0:
            c["delta_f_neg_start"] += 1
            d = -self.delta_f if "no_floor" in self.mut else _fmax(-self.delta_f, 10 * EPS * abs(f0))
            alpha1 = _fmin(1.0, _div(2.0 * d, -self.fp0))
        else:
            alpha1 = abs(STEP_SIZE)
        status, alpha = yield from self._line_search(alpha1)
        if status != SUCCESS:
            return status
        yield from self._apply_fdf(alpha)
        self.f = self.f_alpha
        x[:] = self.x_alpha
        self.gradient = list(self.g_alpha)
        self.delta_f = self.f - f0
        dx0 = [x[i] - self.x0[i] for i in range(6)]
        dg0 = [self.gradient[i] - self.g0[i] for i in range(6)]
        self.dx = list(dx0)
        dxg, dgg, dxdg, dgnorm = _dot(dx0, self.gradient), _dot(dg0, self.gradient), _dot(dx0, dg0), _norm(dg0)
        if dxdg != 0:
            B = dxg / dxdg
            A = -(1.0 + dgnorm * dgnorm / dxdg) * B + dgg / dxdg
        else:
            B = A = 0.0
        self.p = [-A * dx0[i] + self.gradient[i] - B * dg0[i] for i in range(6)]
        self.g0, self.x0 = list(self.gradient), list(x)
        self.g0norm = _norm(self.g0)
        self.pnorm = _norm(self.p)
        d = -1.0 if _dot(self.p, self.gradient) > 0 else 1.0
        if "no_dir" in self.mut:
            d = 1.0
        if d < 0:
            c["dir_flip"] += 1
        q = _div(d, self.pnorm)
        self.p = [pi * q for pi in self.p]
        self.pnorm = _norm(self.p)
        self.fp0 = _dot(self.p, self.g0)
        self._change_direction()
        return SUCCESS

    def test_gradient(self, eps):
        return SUCCESS if _norm(self.gradient) < eps else RUNNING

    # ---- cached line function ----
    def _change_direction(self):
        self.x_alpha, self.x_key = list(self.x0), 0.0
        self.f_alpha, self.f_key = self.f, 0.0
        self.g_alpha, self.g_key = list(self.g0), 0.0
        self.df_alpha, self.df_key = self._slope(), 0.0

    def _move_to(self, alpha):
        if alpha == self.x_key:
            return
        self.x_alpha = [self.x0[i] + alpha * self.p[i] for i in range(6)]
        self.x_key = alpha

    def _slope(self):
        return _dot(self.g_alpha, self.p)

    def _apply_f(self, alpha):
        if alpha == self.f_key:
            return self.f_alpha
        self._move_to(alpha)
        self.f_alpha = yield from self._f(self.x_alpha)
        self.f_key = alpha
        return self.f_alpha

    def _apply_df(self, alpha):
        if alpha == self.df_key:
            return self.df_alpha
        self._move_to(alpha)
        if alpha != self.g_key:
            _, self.g_alpha = yield from self._fdf(self.x_alpha)  # df: the f of the call is discarded
            self.g_key = alpha
        self.df_alpha = self._slope()
        self.df_key = alpha
        return self.df_alpha

    def _apply_fdf(self, alpha):
        if alpha == self.f_key and alpha == self.df_key:
            return self.f_alpha, self.df_alpha
        if alpha == self.f_key or alpha == self.df_key:
            fo = yield from self._apply_f(alpha)
            dfo = yield from self._apply_df(alpha)
            return fo, dfo
        self._move_to(alpha)
        self.f_alpha, self.g_alpha = yield from self._fdf(self.x_alpha)
        self.f_key = self.g_key = alpha
        self.df_alpha = self._slope()
        self.df_key = alpha
        return self.f_alpha, self.df_alpha

    # ---- Fletcher's line search ----
    def _line_search(self, alpha1):
        c, mut = self.c, self.mut
        alpha, alpha_prev = alpha1, 0.0
        i = 0
        f0, fp0 = yield from self._apply_fdf(0.0)
        falpha_prev, fpalpha_prev = f0, fp0
        a, b, fa, fb, fpa, fpb = 0.0, alpha, f0, 0.0, fp0, 0.0
        while True:
            go = i < BRACKET_ITERS
            i += 1
            if not go:
                break
            falpha = yield from self._apply_f(alpha)
            same = falpha > falpha_prev if "gt_bracket" in mut else falpha >= falpha_prev
            if falpha > f0 + alpha * RHO * fp0 or same:
                c["bracket_f"] += 1
                if falpha == falpha_prev and not falpha > f0 + alpha * RHO * fp0:
                    c["bracket_f_equal"] += 1
                a, fa, fpa = alpha_prev, falpha_prev, fpalpha_prev
                b, fb, fpb = alpha, falpha, (0.0 if "fpb_zero" in mut else NAN)
                break
            fpalpha = yield from self._apply_df(alpha)
            if abs(fpalpha) <= -SIGMA * fp0:
                c["bracket_success"] += 1
                return SUCCESS, alpha
            if fpalpha >= 0:
                c["bracket_slope"] += 1
                a, fa, fpa = alpha, falpha, fpalpha
                b, fb, fpb = alpha_prev, falpha_prev, fpalpha_prev
                break
            delta = alpha - alpha_prev
            c["extrapolate"] += 1
            alpha_next = self._interpolate(alpha_prev, falpha_prev, fpalpha_prev, alpha, falpha, fpalpha,
                                           alpha + delta, alpha + TAU1 * delta)
            alpha_prev, falpha_prev, fpalpha_prev = alpha, falpha, fpalpha
            alpha = alpha_next
        t2, t3 = (TAU3, TAU2) if "tau_swap" in mut else (TAU2, TAU3)
        while True:
            go = i < SECTION_ITERS
            i += 1
            if not go:
                break
            delta = b - a
            alpha = self._interpolate(a, fa, fpa, b, fb, fpb, a + t2 * delta, b - t3 * delta)
            falpha = yield from self._apply_f(alpha)
            if (a - alpha) * fpa <= EPS:
                c["section_noprogress"] += 1
                return NO_PROGRESS, 0.0
            if falpha > f0 + RHO * alpha * fp0 or falpha >= fa:
                c["section_f"] += 1
                b, fb, fpb = alpha, falpha, NAN
            else:
                fpalpha = yield from self._apply_df(alpha)
                if abs(fpalpha) <= -SIGMA * fp0:
                    c["section_success"] += 1
                    return SUCCESS, alpha
                if ((b - a) >= 0 and fpalpha >= 0) or ((b - a) <= 0 and fpalpha <= 0):
                    c["section_swap"] += 1
                    b, fb, fpb = a, fa, fpa
                a, fa, fpa = alpha, falpha, fpalpha
        c["section_exhausted"] += 1
        return SUCCESS, 0.0

    def _interpolate(self, a, fa, fpa, b, fb, fpb, xmin, xmax):
        ymin, ymax = _div(xmin - a, b - a), _div(xmax - a, b - a)
        if ymin > ymax:
            ymin, ymax = ymax, ymin
        if ORDER > 2 and fpb == fpb and "quad_always" not in self.mut:
            self.c["cubic"] += 1
            y = self._interp_cubic(fa, fpa * (b - a), fb, fpb * (b - a), ymin, ymax)
        else:
            self.c["quadratic"] += 1
            y = self._interp_quad(fa, fpa * (b - a), fb, ymin, ymax)
        return a + y * (b - a)

    @staticmethod
    def _interp_quad(f0, fp0, f1, zl, zh):
        fl = f0 + zl * (fp0 + zl * (f1 - f0 - fp0))
        fh = f0 + zh * (fp0 + zh * (f1 - f0 - fp0))
        c = 2 * (f1 - f0 - fp0)
        zmin, fmin = zl, fl
        if fh < fmin:
            zmin, fmin = zh, fh
        if c > 0:
            z = -fp0 / c
            if z > zl and z < zh:
                fz = f0 + z * (fp0 + z * (f1 - f0 - fp0))
                if fz < fmin:
                    zmin, fmin = z, fz
        return zmin

    def _interp_cubic(self, f0, fp0, f1, fp1, zl, zh):
        eta = 3 * (f1 - f0) - 2 * fp0 - fp1
        xi = fp0 + fp1 - 2 * (f1 - f0)
        c0, c1, c2, c3 = f0, fp0, eta, xi
        cubic = lambda z: c0 + z * (c1 + z * (c2 + z * c3))  # noqa: E731
        zmin, fmin = zl, cubic(zl)
        y = cubic(zh)
        if y < fmin:
            zmin, fmin = zh, y
        n, z0, z1 = self._solve_quadratic(3 * c3, 2 * c2, c1)
        for z, ok in ((z0, n >= 1), (z1, n == 2)):
            if ok and z > zl and z < zh:
                y = cubic(z)
                if y < fmin:
                    zmin, fmin = z, y
        return zmin

    def _solve_quadratic(self, a, b, c):
        k = self.c
        if a == 0:
            if b == 0:
                k["sq_degenerate"] += 1
                return 0, 0.0, 0.0
            k["sq_linear"] += 1
            return 1, -c / b, 0.0
        disc = b * b - 4 * a * c
        if disc > 0:
            if b == 0:
                k["sq_b_zero"] += 1
                r = _sqrt(-c / a)
                return 2, -r, r
            k["sq_two_roots"] += 1
            sgnb = 1.0 if b > 0 else -1.0
            temp = -0.5 * (b + sgnb * _sqrt(disc))
            r1, r2 = _div(temp, a), _div(c, temp)
            return (2, r1, r2) if r1 < r2 else (2, r2, r1)
        if disc == 0:
            k["sq_double_root"] += 1
            return 2, -0.5 * b / a, -0.5 * b / a
        k["sq_no_root"] += 1
        return 0, 0.0, 0.0


def bfgs(x0, max_inner=20, gradient_tol=1e-2, mut=(), counts=None):
    """The inner loop of estimateRigidTransformationBFGS as a coroutine (see the module docstring); returns
    (result, inner, x)."""
    counts = Counter() if counts is None else counts
    mut = frozenset(mut)
    if "cap19" in mut:
        max_inner -= 1
    B = _Bfgs(mut, counts)
    x = [float(v) for v in x0]
    yield from B.init(x)
    inner = 0
    while True:
        inner += 1
        result = yield from B.step(x)
        yield ("step", result, list(x), B.f, list(B.gradient), inner)
        if result:
            break
        result = B.test_gradient(gradient_tol)
        if result == SUCCESS:
            counts["gradient_success"] += 1
        if not (result == RUNNING and inner < max_inner):
            break
    if result == RUNNING and inner == max_inner:
        counts["inner_cap"] += 1
    return result, inner, x


# ---- replay of a trace --------------------------------------------------------------------------------------------
def _bits(v):
    return np.asarray(v, dtype=np.float64).view(np.int64).tolist()


def _f32_near(x0, v64):
    """x0 is an f32 value within 1 f32 ulp of f32(v64)."""
    if float(F32(x0)) != x0:
        return False
    r = F32(v64)
    return x0 in (float(r), float(np.nextafter(r, F32(np.inf))), float(np.nextafter(r, F32(-np.inf))))


def _mat4(T12):
    M = np.eye(4, dtype=F32)
    M[:3] = np.asarray(T12, dtype=F32).reshape(3, 4)
    return M


def replay(recs, guess=None, cfg=None, mut=()):
    """Replay a trace. cfg: max_inner (or max_inner_iterations), max_iterations, rotation_eps, trans_eps, gradient_tol (the shipped defaults).
    Returns dict(bad: mismatches (empty when every record reproduces), near: near-threshold decisions, counts: branch
    counts, calls, iterations, converged, final_T, worst_T: largest |T - T64| / bound)."""
    cfg = dict(dict(max_inner=20, max_iterations=200, rotation_eps=2e-3, trans_eps=5e-4, gradient_tol=1e-2), **(cfg or {}))
    if "max_inner_iterations" in cfg:  # the oracle's / the engine's setter name
        cfg["max_inner"] = cfg["max_inner_iterations"]
    guess = np.eye(4, dtype=F32) if guess is None else np.asarray(guess, dtype=F32)
    mut = frozenset(mut)
    counts, bad, near = Counter(), [], 0
    worst_T = 0.0
    recs = np.asarray(recs)
    outer_idx = np.nonzero(recs["type"] == 2)[0]
    if not len(outer_idx) or outer_idx[-1] != len(recs) - 1:
        return dict(bad=["the trace does not end with an outer record"], near=0, counts=counts)
    transformation = np.eye(4, dtype=F32)
    previous = np.eye(4, dtype=F32)
    start, converged, calls, nr = 0, False, 0, 0
    for k, oi in enumerate(outer_idx):
        o = recs[oi]
        inner_recs = recs[start:oi]
        start = oi + 1
        previous = transformation.copy()
        if int(o["outer"]) != k or (o["status"] == NOT_STARTED and int(o["nr_iterations"]) != nr):
            bad.append((k, "outer index", int(o["outer"]), int(o["nr_iterations"])))
        if o["status"] == NOT_STARTED:  # m < 4: the reference's exception, caught: the loop ends
            if o["m"] >= 4 or len(inner_recs) or k != len(outer_idx) - 1:
                bad.append((k, "m < 4 record", int(o["m"]), len(inner_recs)))
            break
        if o["m"] < 4:
            bad.append((k, "BFGS ran with m < 4", int(o["m"])))
        # x0 from transformation_
        t = transformation.astype(np.float64)
        x0 = [float(v) for v in o["x0"]]
        want = (math.atan2(t[2, 1], t[2, 2]), math.asin(-t[2, 0]), math.atan2(t[1, 0], t[0, 0]))
        if x0[:3] != [t[0, 3], t[1, 3], t[2, 3]] or not all(_f32_near(a, w) for a, w in zip(x0[3:], want)):
            bad.append((k, "x0", x0, want))
        # the inner BFGS, call by call
        gen = bfgs(x0, cfg["max_inner"], cfg["gradient_tol"], mut, counts)
        it = iter(inner_recs)
        msg, ok, n_calls = next(gen), True, 0
        try:
            while True:
                r = next(it, None)
                if r is None:
                    bad.append((k, "trace ends early", msg[:2]))
                    ok = False
                    break
                if msg[0] == "call":
                    n_calls += 1
                    if r["type"] != 0 or r["want_grad"] != msg[1] or _bits(r["x"]) != _bits(msg[2]):
                        bad.append((k, "call", n_calls - 1, msg[:2], int(r["type"]), int(r["want_grad"]), list(r["x"]), msg[2]))
                        ok = False
                        break
                    msg = gen.send((r["f"], list(r["g"])))
                else:
                    _, status, x, f, g, inner = msg
                    if (r["type"] != 1 or r["status"] != status or r["inner"] != inner or _bits(r["x"]) != _bits(x)
                            or _bits(r["f"]) != _bits(f) or _bits(r["g"]) != _bits(g)):
                        bad.append((k, "step", inner, status, int(r["type"]), int(r["status"]), list(r["x"]), x))
                        ok = False
                        break
                    msg = next(gen)
        except StopIteration as e:
            result, inner, x = e.value
            if next(it, None) is not None:
                bad.append((k, "trace has extra records"))
                ok = False
        if not ok:
            break
        calls += n_calls
        if (o["status"] != result or o["inner"] != inner or _bits(o["x"]) != _bits(x)
                or o["evaluation"] != n_calls):
            bad.append((k, "outer result", int(o["status"]), result, int(o["inner"]), inner, int(o["evaluation"]), n_calls))
            break
        if not (result in (NO_PROGRESS, SUCCESS) or inner == cfg["max_inner"]):  # the reference throws: the loop ends
            if k != len(outer_idx) - 1:
                bad.append((k, "loop continued after an unaccepted BFGS result"))
            break
        # transformation_ = applyState(identity, x), within its bound
        T = _mat4(o["T"])
        T64, bT = G.state_T_bound(x)
        dev = np.abs(T[:3].astype(np.float64) - T64)
        if np.any(dev > bT):
            bad.append((k, "T", T[:3], T64))
        with np.errstate(invalid="ignore", divide="ignore"):
            worst_T = max(worst_T, float(np.nanmax(np.where(bT > 0, dev / bT, 0.0))))
        # delta: the f32 difference, then the f64 ratio
        rr, rt = 1.0 / cfg["rotation_eps"], 1.0 / cfg["trans_eps"]
        if "eps_swap" in mut:
            rr, rt = rt, rr
        delta, slack = 0.0, 0.0
        for a in range(4):
            for b_ in range(4):
                ratio = rr if (a < 3 and b_ < 3) else rt
                cd = ratio * float(abs(F32(previous[a, b_]) - F32(T[a, b_])))
                if cd > delta:
                    delta = cd
                if a < 3:
                    slack = max(slack, ratio * float(bT[a, b_]))
        nr += 1
        conv = nr >= cfg["max_iterations"] or delta < 1
        if abs(delta - 1.0) <= slack:
            near += 1
        if _bits(o["delta"]) != _bits(delta) or int(o["nr_iterations"]) != nr or bool(o["converged"]) != conv:
            bad.append((k, "convergence", float(o["delta"]), delta, int(o["nr_iterations"]), nr, int(o["converged"]), conv))
            break
        transformation = T
        if conv:
            previous = T.copy()
            converged = True
            if k != len(outer_idx) - 1:
                bad.append((k, "loop continued after convergence"))
            break
    last = recs[outer_idx[-1]]
    final = np.zeros((4, 4), dtype=F32)
    for i in range(4):
        for j in range(4):
            acc = F32(0)
            for kk in range(4):
                acc = F32(acc + F32(previous[i, kk] * guess[kk, j]))
            final[i, j] = acc
    if not bad:
        if not last["last"] or int(np.sum(recs["last"])) != 1:
            bad.append(("last flag",))
        if _bits(last["final_T"].astype(np.float64)) != _bits(final.reshape(16).astype(np.float64)):
            bad.append(("final_T", last["final_T"], final.reshape(16)))
    return dict(bad=bad, near=near, counts=counts, calls=calls, iterations=nr, converged=converged, final_T=final,
                worst_T=worst_T)


# ---- fixture generators -------------------------------------------------------------------------------------------
def identical_pair(target, n=3000, seed=0):
    """Source = target (a subset of it, as its own target): at identity every residual is exactly 0, so f = g = 0,
    g0norm = 0, p is NaN and minimizeOneStep returns NoProgress at once; the outer loop converges in one iteration."""
    rng = np.random.default_rng(seed)
    t = np.asarray(target, dtype=F32)[:, :3]
    s = t[np.sort(rng.choice(len(t), size=min(n, len(t)), replace=False))]
    return s.copy(), s.copy()


def offset_pair(source, target, t=(0.0, 0.0, 0.0), rpy=(0.0, 0.0, 0.0)):
    """The source moved by a pose (translation t, Euler rpy): with step_size 1 along a unit direction, a far start makes
    the line search extrapolate or bracket by slope, a near one bracket by an f increase."""
    T = G.rpy_f32(t, rpy).astype(np.float64)
    s = np.asarray(source, dtype=np.float64)[:, :3]
    return (s @ T[:3, :3].T + T[:3, 3]).astype(F32), np.asarray(target, dtype=F32)
