"""A float64 reference of GICP's correspondence pass (K6: nn1_query + gicp_corr_kernel) and of one evaluation of its
fixed-correspondence objective (K7: the functor's operator() and fdf), written from gicp_omp_impl.hpp:244-366 and
420-456 and vectorised in numpy, with a bound per entry. Nothing here needs a GPU.

What is computed
  The covariances come from the caller (the handle's own covariances()), so K5 stays out of the comparison.
  * moved = guess * source and the query transformation_ * moved: f32, ((T0 x + T1 y) + T2 z) + T3 un-fused, the order
    of transform_point. gicp.cu is built with -fmad=false and numpy does not contract either, so both are bit-exact.
  * transform_R = transformation_ * guess in f64, in the loop order of GicpSolver::correspondences (products of two
    floats are exact in f64; the sums run k = 0..3 from +0.0).
  * the 1-NN in FLANN L2_Simple f32 order ((dx dx + dy dy) + dz dz), ties to the lower index. Small problems are brute
    force (gridref.nn1_ref). Large ones take candidates from scipy's cKDTree in f64: every target point within
    d_min (1 + 2e-6) of the query. The f32 distance of a point is within 5 * 2^-24 relative of its exact distance (the
    three differences, squares and two sums each round once), so a point outside that radius cannot have an f32 distance
    at or below the f32 distance of the exact nearest point. The candidates are then re-ranked in f32.
  * the gate (double) d2 < corr_dist^2, strict.
  * maha_kernel_order: R A, (R A) R^T, + C2 and inverse3 in gicp_corr_kernel's operation order in f64, then f32. Every
    operation is the kernel's, so this is bitwise the kernel's value.
  * maha_exact: np.linalg.inv(R C1 R^T + C2) in f64. The kernel's f32 matrix is within
        (2^-24 + 64 kappa 2^-53) max|M|
    of it per entry: the f32 rounding, plus the forward error of a cofactor inverse of a matrix of condition kappa
    (the matrix itself is formed with relative error of a few 2^-53, which kappa amplifies the same way).
  * the objective at a given f32 transform T (12 floats), state x, corr and M:
      f32path: the per-correspondence f32 value r^T (M r) of operator(), residual and M r in f32, each widened to f64;
      f, g[0..2], and the nine R sums of fdf: residual widened to f64, temp = M r in f64, r^T temp, temp, p temp^T;
      g[3..5] = sum_ij m1(j, i) R(i, j) of computeRDerivative with m1 = dPhi, dTheta, dPsi.
    Every per-correspondence term is the kernel's bit for bit; only the order of the f64 sums differs. The sums here are
    exact (math.fsum), then divided by m / multiplied by 2 / m like the kernel.

The bound
  A recursive f64 sum whose deepest chain of additions has D steps is within D u sum|term| of the exact sum (u = 2^-53,
  first order). The kernel's chains:
    gicp_inner_kernel: the points a thread takes in its evaluator chunk (ceil(chunk / 256)), the 5-level shuffle tree,
      8 warps, the 10 rows a controller thread sums, the 16 interleaved chains.
  The oracle sums serially: D = m. Each entry's bound is (D + c) u sum|term| scaled like the entry (1 / m or 2 / m), c = 4
  for the final division and multiplication. g[3..5] add sum_ij |m1|(j, i) bound(R(i, j)) and the double sin / cos of
  the device (<= 2 ulp) and host (<= 1 ulp) libraries: each m1 entry is a sum of products of up to three of them, so it
  moves by at most 24 u |m1|(j, i), |m1| formed from absolute values; the nine-term sum adds 9 u.
"""
from __future__ import annotations

import math

import numpy as np

import gridref as GR

F32 = np.float32
U = 2.0**-53
U32 = 2.0**-24
GI_THREADS = 256
GI_MAX_CTAS = 160
C_FINAL = 4
TRIG = 24


# ---- transforms ------------------------------------------------------------------------------------------------------
def transform(T, pts) -> np.ndarray:
    """transform_point: ((T0 x + T1 y) + T2 z) + T3 in f32, un-fused. T: (3|4, 4) or 12 floats, row-major."""
    T = np.asarray(T, dtype=F32).reshape(-1, 4)
    p = np.asarray(pts, dtype=F32)[:, :3]
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def transform_R(transformation, guess) -> np.ndarray:
    """transformation_ * guess in f64, accumulated k = 0..3 from +0.0 (GicpSolver::correspondences); the 3x3 block."""
    t = np.asarray(transformation, dtype=F32).astype(np.float64)
    g = np.asarray(guess, dtype=F32).astype(np.float64)
    R = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            acc = 0.0
            for k in range(4):
                acc = acc + t[i, k] * g[k, j]
            R[i, j] = acc
    return R


def rpy_f32(t, rpy) -> np.ndarray:
    """A float32 pose R = Rz(yaw) Ry(pitch) Rx(roll), translation t (row-major 4x4)."""
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    T = np.eye(4)
    T[:3, :3] = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]]) @ np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]]) @ \
        np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    T[:3, 3] = t
    return T.astype(F32)


# ---- correspondences ------------------------------------------------------------------------------------------------
def nn1(target, queries, brute_limit=4e7):
    """Exact 1-NN in FLANN L2_Simple f32 order, ties to the lower index: (index, d2 float32)."""
    t = np.asarray(target, dtype=F32)[:, :3]
    q = np.asarray(queries, dtype=F32)[:, :3]
    if len(t) * len(q) <= brute_limit:
        return GR.nn1_ref(t, q)
    from scipy.spatial import cKDTree

    tree = cKDTree(t.astype(np.float64))
    d, _ = tree.query(q.astype(np.float64), k=1)
    cand = tree.query_ball_point(q.astype(np.float64), r=d * (1 + 2e-6))
    lens = np.fromiter((len(c) for c in cand), dtype=np.int64, count=len(q))
    qi = np.repeat(np.arange(len(q)), lens)
    ti = np.fromiter((j for c in cand for j in c), dtype=np.int64, count=int(lens.sum()))
    dd = q[qi] - t[ti]
    d2 = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
    order = np.lexsort((ti, d2, qi))  # per query: smallest f32 d2, then the lowest index
    first = np.ones(len(order), bool)
    first[1:] = qi[order][1:] != qi[order][:-1]
    pick = order[first]
    idx = np.full(len(q), -1, dtype=np.int32)
    out = np.full(len(q), np.finfo(F32).max, dtype=F32)
    idx[qi[pick]] = ti[pick]
    out[qi[pick]] = d2[pick]
    return idx, out


def _inverse3(m):
    """gicp.cu inverse3, operation by operation; m (n, 9) f64."""
    c00 = m[:, 4] * m[:, 8] - m[:, 5] * m[:, 7]
    c01 = m[:, 5] * m[:, 6] - m[:, 3] * m[:, 8]
    c02 = m[:, 3] * m[:, 7] - m[:, 4] * m[:, 6]
    idt = 1.0 / ((m[:, 0] * c00 + m[:, 1] * c01) + m[:, 2] * c02)
    return np.stack([c00 * idt, (m[:, 2] * m[:, 7] - m[:, 1] * m[:, 8]) * idt, (m[:, 1] * m[:, 5] - m[:, 2] * m[:, 4]) * idt,
                     c01 * idt, (m[:, 0] * m[:, 8] - m[:, 2] * m[:, 6]) * idt, (m[:, 2] * m[:, 3] - m[:, 0] * m[:, 5]) * idt,
                     c02 * idt, (m[:, 1] * m[:, 6] - m[:, 0] * m[:, 7]) * idt, (m[:, 0] * m[:, 4] - m[:, 1] * m[:, 3]) * idt],
                    axis=1)


def maha_kernel_order(R, C1, C2) -> np.ndarray:
    """(R C1 R^T + C2)^-1 in gicp_corr_kernel's operation order, then f32: (n, 3, 3)."""
    A = np.asarray(C1, dtype=np.float64).reshape(-1, 9)
    B = np.asarray(C2, dtype=np.float64).reshape(-1, 9)
    R = np.asarray(R, dtype=np.float64).reshape(9)
    M = np.stack([(R[r * 3] * A[:, c] + R[r * 3 + 1] * A[:, 3 + c]) + R[r * 3 + 2] * A[:, 6 + c]
                  for r in range(3) for c in range(3)], axis=1)
    Tm = np.stack([(M[:, r * 3] * R[c * 3] + M[:, r * 3 + 1] * R[c * 3 + 1]) + M[:, r * 3 + 2] * R[c * 3 + 2]
                   for r in range(3) for c in range(3)], axis=1)
    Tm = Tm + B
    return _inverse3(Tm).astype(F32).reshape(-1, 3, 3)


def maha_exact(R, C1, C2):
    """np.linalg.inv(R C1 R^T + C2) in f64 and the per-matrix bound on the kernel's f32 entries: (M (n,3,3), bound (n,))."""
    R = np.asarray(R, dtype=np.float64).reshape(3, 3)
    A = R[None] @ np.asarray(C1, dtype=np.float64).reshape(-1, 3, 3) @ R.T[None] + np.asarray(C2, dtype=np.float64).reshape(-1, 3, 3)
    M = np.linalg.inv(A)
    kappa = np.linalg.cond(A)
    return M, (U32 + 64 * kappa * U) * np.abs(M).max(axis=(1, 2))


def correspondences(source, target, cov_src, cov_tgt, corr_dist, guess=None, T=None):
    """K6 at transformation_ = T: dict(corr (n,) -1 = none, m, d2, moved, R, maha (n,3,3) f32 kernel order (identity where
    corr < 0), maha_exact, maha_bound)."""
    guess = np.eye(4, dtype=F32) if guess is None else np.asarray(guess, dtype=F32)
    T = np.eye(4, dtype=F32) if T is None else np.asarray(T, dtype=F32)
    moved = transform(guess, source)
    q = transform(T, moved)
    idx, d2 = nn1(target, q)
    thr = float(corr_dist) * float(corr_dist)
    ok = (idx >= 0) & (d2.astype(np.float64) < thr)
    corr = np.where(ok, idx, -1).astype(np.int32)
    R = transform_R(T, guess)
    sel = np.nonzero(ok)[0]
    maha = np.tile(np.eye(3, dtype=F32), (len(corr), 1, 1))
    mex = np.tile(np.eye(3), (len(corr), 1, 1))
    mb = np.zeros(len(corr))
    if len(sel):
        c1 = np.asarray(cov_src).reshape(-1, 3, 3)[sel]
        c2 = np.asarray(cov_tgt).reshape(-1, 3, 3)[idx[sel]]
        maha[sel] = maha_kernel_order(R, c1, c2)
        mex[sel], mb[sel] = maha_exact(R, c1, c2)
    return dict(corr=corr, m=int(ok.sum()), d2=d2, moved=moved, R=R, maha=maha, maha_exact=mex, maha_bound=mb)


# ---- objective ------------------------------------------------------------------------------------------------------
def _dmats(x, absolute=False):
    """dPhi, dTheta, dPsi of computeRDerivative (row-major 3x3 each); absolute: the same sums of |products|."""
    phi, theta, psi = x[3], x[4], x[5]
    cphi, sphi, cth, sth, cpsi, spsi = math.cos(phi), math.sin(phi), math.cos(theta), math.sin(theta), math.cos(psi), math.sin(psi)
    if absolute:
        cphi, sphi, cth, sth, cpsi, spsi = map(abs, (cphi, sphi, cth, sth, cpsi, spsi))
        a = lambda *t: sum(t)  # noqa: E731  (the factors are already absolute values)
        dPhi = [0, a(sphi * spsi, cphi * cpsi * sth), a(cphi * spsi, cpsi * sphi * sth),
                0, a(cpsi * sphi, cphi * spsi * sth), a(cphi * cpsi, sphi * spsi * sth),
                0, cphi * cth, cth * sphi]
        dTheta = [cpsi * sth, cpsi * cth * sphi, cphi * cpsi * cth, spsi * sth, cth * sphi * spsi, cphi * cth * spsi,
                  cth, sphi * sth, cphi * sth]
        dPsi = [cth * spsi, a(cphi * cpsi, sphi * spsi * sth), a(cpsi * sphi, cphi * spsi * sth),
                cpsi * cth, a(cphi * spsi, cpsi * sphi * sth), a(sphi * spsi, cphi * cpsi * sth), 0, 0, 0]
    else:
        dPhi = [0, sphi * spsi + cphi * cpsi * sth, cphi * spsi - cpsi * sphi * sth,
                0, -cpsi * sphi + cphi * spsi * sth, -cphi * cpsi - sphi * spsi * sth,
                0, cphi * cth, -cth * sphi]
        dTheta = [-cpsi * sth, cpsi * cth * sphi, cphi * cpsi * cth, -spsi * sth, cth * sphi * spsi, cphi * cth * spsi,
                  -cth, -sphi * sth, -cphi * sth]
        dPsi = [-cth * spsi, -cphi * cpsi - sphi * spsi * sth, cpsi * sphi - cphi * spsi * sth,
                cpsi * cth, -cphi * spsi + cpsi * sphi * sth, sphi * spsi + cphi * cpsi * sth, 0, 0, 0]
    return [np.array(m, dtype=np.float64).reshape(3, 3) for m in (dPhi, dTheta, dPsi)]


def r_derivative(x, R):
    """g[3..5] = sum_ij m1(j, i) R(i, j) (matricesInnerProd) for m1 = dPhi, dTheta, dPsi."""
    return np.array([math.fsum((m1.T * R).ravel()) for m1 in _dmats(x)])


def terms(T, moved, target, corr, maha):
    """Per-correspondence terms, bit-exact with cost_point: dict(f32path (m,), fdf (m,), t (m,3), P (m,9) = p_r temp_c)."""
    sel = np.nonzero(np.asarray(corr) >= 0)[0]
    ps = np.asarray(moved, dtype=F32)[sel]
    pt = np.asarray(target, dtype=F32)[:, :3][np.asarray(corr)[sel]]
    M = np.asarray(maha, dtype=F32).reshape(-1, 9)[sel]
    q = transform(T, ps)
    r = q - pt
    r0, r1, r2 = r[:, 0], r[:, 1], r[:, 2]
    mr = [(M[:, 3 * k] * r0 + M[:, 3 * k + 1] * r1) + M[:, 3 * k + 2] * r2 for k in range(3)]
    f32 = ((r0 * mr[0] + r1 * mr[1]) + r2 * mr[2]).astype(np.float64)
    d = r.astype(np.float64)
    Md = M.astype(np.float64)
    t = np.stack([(Md[:, 3 * k] * d[:, 0] + Md[:, 3 * k + 1] * d[:, 1]) + Md[:, 3 * k + 2] * d[:, 2] for k in range(3)], axis=1)
    fd = (d[:, 0] * t[:, 0] + d[:, 1] * t[:, 1]) + d[:, 2] * t[:, 2]
    b = ps.astype(np.float64)
    P = np.stack([b[:, rr] * t[:, c] for rr in range(3) for c in range(3)], axis=1)
    return dict(f32path=f32, fdf=fd, t=t, P=P, src=sel)


def depth_device(n, sm_count):
    """Deepest f64 summation chain of gicp_inner_kernel for n source points on sm_count SMs."""
    n_eval = max(1, min(-(-n // GI_THREADS), min(sm_count, GI_MAX_CTAS) - 1))
    chunk = -(-n // n_eval)
    return -(-chunk // GI_THREADS) + 5 + 8 + GI_MAX_CTAS // 16 + 16


def evaluator_partition(n, sm_count):
    """(n_eval, chunk) of the persistent kernel: the evaluator CTA k takes points [k chunk, min(n, (k + 1) chunk))."""
    n_eval = max(1, min(-(-n // GI_THREADS), min(sm_count, GI_MAX_CTAS) - 1))
    return n_eval, -(-n // n_eval)


def objective(T, x, moved, target, corr, maha, depth, R_swap=False):
    """Exact sums of the functor at transform T (12 or 16 f32, row-major) and state x: dict(f32path, f, g (6,), R (3,3),
    bounds b_f32path, b_f, b_g (6,), and the terms). depth: the D of the summation compared with (depth_device, or
    m for the oracle). R_swap exchanges R[0,1] and R[1,0] (a power check)."""
    tm = terms(T, moved, target, corr, maha)
    m = len(tm["fdf"])
    k = (depth + C_FINAL) * U
    S = lambda a: math.fsum(a.tolist())  # noqa: E731
    A = lambda a: math.fsum(np.abs(a).tolist())  # noqa: E731
    f32path = S(tm["f32path"]) / m
    f = S(tm["fdf"]) / m
    g = np.zeros(6)
    bg = np.zeros(6)
    for c in range(3):
        g[c] = S(tm["t"][:, c]) * (2.0 / m)
        bg[c] = k * A(tm["t"][:, c]) * (2.0 / m)
    R = np.array([S(tm["P"][:, j]) for j in range(9)]).reshape(3, 3) * (2.0 / m)
    bR = np.array([k * A(tm["P"][:, j]) for j in range(9)]).reshape(3, 3) * (2.0 / m)
    if R_swap:
        R[0, 1], R[1, 0] = R[1, 0], R[0, 1]
    g[3:] = r_derivative(x, R)
    for j, m1a in enumerate(_dmats(x, absolute=True)):
        bg[3 + j] = float(((m1a.T * bR).sum()) + (TRIG + 9) * U * (m1a.T * np.abs(R)).sum())
    return dict(f32path=f32path, f=f, g=g, R=R, m=m, terms=tm,
                b_f32path=k * A(tm["f32path"]) / m, b_f=k * A(tm["fdf"]) / m, b_g=bg)


def rotation_f64(x):
    """R64 = Rz Ry Rx of the f32-rounded angles in f64 and |Rz| |Ry| |Rx| (applyState's order)."""
    a = [float(F32(v)) for v in x[3:6]]
    cx, sx, cy, sy, cz, sz = math.cos(a[0]), math.sin(a[0]), math.cos(a[1]), math.sin(a[1]), math.cos(a[2]), math.sin(a[2])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    return Rz @ Ry @ Rx, np.abs(Rz) @ np.abs(Ry) @ np.abs(Rx)


def state_T_bound(x):
    """(T64 (3, 4), bound (3, 4)) for the f32 transform apply_state builds from x: each f32 sin / cos within 2 ulp
    (<= 4 * 2^-24 relative), an entry a sum of products of up to three of them (12) plus the f32 products and sums of
    the two 3x3 products (4 roundings) and the final rounding: 17 * 2^-24 * (|Rz| |Ry| |Rx|). The translation is f32(x)."""
    R, Ra = rotation_f64(x)
    T = np.zeros((3, 4))
    T[:, :3] = R
    T[:, 3] = [float(F32(v)) for v in x[:3]]
    b = np.zeros((3, 4))
    b[:, :3] = 17 * U32 * Ra
    return T, b


# ---- fixture generators ---------------------------------------------------------------------------------------------
FAR = 1.0e3  # how far the generators move points that must not find a correspondence


def confine_to_chunk(source, n_eval, chunk, which):
    """The source with every point outside evaluator chunk `which` (0, a middle one or the ragged last) moved FAR along z,
    beyond any corr_dist: only that chunk's evaluator sees correspondences, the others contribute +0.0."""
    s = np.asarray(source, dtype=F32).copy()
    lo, hi = which * chunk, min(len(s), (which + 1) * chunk)
    out = np.ones(len(s), bool)
    out[lo:hi] = False
    s[out, 2] += F32(FAR)
    return s, (lo, hi)


def exact_m_scan(target, m, n=64, seed=0):
    """A source of n points of which exactly m lie within 0.05 of a target point; the rest are FAR away."""
    rng = np.random.default_rng(seed)
    t = np.asarray(target, dtype=F32)[:, :3]
    pick = rng.choice(len(t), size=n, replace=False)
    s = t[pick] + rng.uniform(-0.02, 0.02, size=(n, 3)).astype(F32)
    s[m:, 2] += F32(FAR)
    return s.astype(F32)


def gate_pair(corr_dist=0.5):
    """Target: a 5 x 5 x 5 lattice of spacing 4 at (8, 8, 8). Source queries at +x offsets from lattice points: exactly
    corr_dist (f32 d2 == corr_dist^2 exactly), one ulp below and one ulp above, and four exact hits. Returns (source,
    target, expected corr: -1 where the gate must reject)."""
    t = GR.lattice((5, 5, 5), (4.0, 4.0, 4.0), origin=(8.0, 8.0, 8.0))
    base = t[[31, 62, 93]]  # interior lattice points
    q = base.copy()
    q[0, 0] = base[0, 0] + F32(corr_dist)  # on the gate
    q[1, 0] = np.nextafter(base[1, 0] + F32(corr_dist), F32(-np.inf), dtype=F32)  # one ulp inside
    q[2, 0] = np.nextafter(base[2, 0] + F32(corr_dist), F32(np.inf), dtype=F32)  # one ulp outside
    exact = t[[0, 40, 80, 124]]
    src = np.concatenate([q, exact]).astype(F32)
    expect = np.array([-1, 62, -1, 0, 40, 80, 124], dtype=np.int32)
    return src, t, expect


def far_pass_scene(seed=0):
    """Two dense blobs 40 m apart and queries in the empty space between them, 15-20 m from any target point: inside
    corr_dist = 25 but more than three NN-grid rings from every occupied cell, so nn1_query answers them in its far pass
    under the cutoff. Returns (source, target, corr_dist); the source also holds blob points (ordinary queries)."""
    rng = np.random.default_rng(seed)
    blob = lambda c, n: (np.asarray(c) + rng.normal(scale=0.6, size=(n, 3))).astype(F32)  # noqa: E731
    t = np.concatenate([blob((0, 0, 0), 3000), blob((40, 0, 0), 3000)])
    far = np.stack([rng.uniform(17, 23, 200), rng.uniform(-3, 3, 200), rng.uniform(-3, 3, 200)], axis=1).astype(F32)
    near = t[rng.choice(len(t), 300, replace=False)] + rng.normal(scale=0.05, size=(300, 3)).astype(F32)
    return np.concatenate([far, near]).astype(F32), t, 25.0


def ring_distance(target, queries):
    """Chebyshev distance in NN-grid cells from each query's cell to the nearest occupied cell."""
    g = GR.nn_geometry(target)
    t = np.asarray(target, dtype=F32)[:, :3]
    cell = lambda p: np.clip(np.floor((p - g["origin"]) * g["inv_h"]).astype(np.int64), 0, g["dims"] - 1)  # noqa: E731
    occ = np.unique(cell(t), axis=0)
    qc = cell(np.asarray(queries, dtype=F32)[:, :3])
    return np.array([np.abs(occ - c).max(axis=1).min() for c in qc])


def cloud_of_size(target, n, seed=0, T=None):
    """n source points drawn from the target (with replacement past its size), jittered by 2 cm and moved by T^-1."""
    rng = np.random.default_rng(seed)
    t = np.asarray(target, dtype=F32)[:, :3]
    pick = rng.choice(len(t), size=n, replace=n > len(t))
    p = t[pick].astype(np.float64) + rng.normal(scale=0.02, size=(n, 3))
    if T is not None:
        Ti = np.linalg.inv(np.asarray(T, dtype=np.float64))
        p = p @ Ti[:3, :3].T + Ti[:3, 3]
    return p.astype(F32)


def ladder(sm_count):
    """Source sizes at the evaluator partition's edges."""
    e = min(sm_count, GI_MAX_CTAS) - 1
    return sorted({4, 5, 255, 256, 257, 256 * e - 1, 256 * e, 256 * e + 1})


def surface_pair(seed=17):
    """test_gpu_gicp's small pair: a smooth surface and a wall, source = every other point moved by T_gt^-1."""
    rng = np.random.default_rng(seed)
    n = 6000
    u = rng.uniform(-3, 3, size=(n, 2))
    z = 0.3 * np.sin(u[:, 0]) + 0.2 * np.cos(1.7 * u[:, 1])
    wall = rng.uniform(-3, 3, size=(n // 3, 2))
    a = np.stack([u[:, 0], u[:, 1], z], axis=1)
    b = np.stack([wall[:, 0], np.full(len(wall), 3.0) + 0.05 * np.sin(3 * wall[:, 0]), 1.5 + 0.5 * wall[:, 1]], axis=1)
    tgt = np.concatenate([a, b]).astype(F32)
    T_gt = rpy_f32((0.08, -0.05, 0.03), (0.01, -0.015, 0.02)).astype(np.float64)
    Ti = np.linalg.inv(T_gt)
    src = (tgt[::2].astype(np.float64) @ Ti[:3, :3].T + Ti[:3, 3]).astype(F32)
    return src, tgt


GUESS = rpy_f32((0.05, -0.02, 0.01), (0.002, -0.004, 0.01))
T_OFF = rpy_f32((-0.03, 0.02, 0.005), (0.003, 0.001, -0.006))
BIG_ROT = rpy_f32((0.3, -0.2, 0.1), (0.2, 1.2, 2.9))
STATES = {"zero": np.zeros(6), "moderate": np.array([0.05, -0.03, 0.02, 0.01, -0.02, 0.03]),
          "large": np.array([0.8, -1.1, 0.4, 0.6, -0.9, 2.5])}
