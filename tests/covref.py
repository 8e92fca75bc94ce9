"""A float64 reference of GICP's k-NN covariances (K5, gicp_cov_kernel) with a bound per point, a numpy restatement of
the exact-NN grid's ring search and its stop rule, and seeded generators of the clouds where K5 and the ring searches go
wrong. Nothing here needs a GPU.

What is computed
  * the k nearest neighbours of every finite row over the finite rows, in lexicographic (f32 L2_Simple d2, index)
    order. Small clouds are brute force. Large ones take k + m candidates from a float64 cKDTree and re-rank them by
    (f32 d2, index); the set is complete when the (k+m)-th float64 distance D satisfies D^2 (1 - 2^-20) > d2_k, the f32
    k-th distance: the f32 d2 of any point is within 5 * 2^-24 relative of its exact square distance (three differences,
    three squares and two sums each round once), so no point outside the candidates can rank at or before the k-th.
    Otherwise m grows.
  * the moments as the kernel forms them: f32 products (x*x with float operands), float64 sums in ascending (d2, index)
    order, one explicit sequential add per neighbour, the mean and the second moments divided by k, then c/k - m_a m_b.
    gicp.cu is built with -fmad=false, so the last line is a rounded division, a rounded product and a rounded
    subtraction (the DFMAs in gicp_cov_kernel's SASS are the refinement steps of the IEEE division and square root); numpy
    rounds the same three operations. The moments here are therefore the kernel's bit for bit.
  * u, the eigenvector of the eigenvalue of smallest |lambda| (numpy.linalg.eigh), and cov = I - (1 - eps) u u^T.

The bound
  Both sides start from the same C. The kernel's cyclic Jacobi stops with off-diagonal mass <= 1e-17 ||C|| and applies
  at most a few sweeps of three rotations, each with a backward error of a few u ||C|| (u = 2^-53); LAPACK's symmetric
  eigensolver is backward stable with a comparable constant. C_EIG = 64 (in units of 2^-52 ||C||) covers both with a
  margin of about two. An eigenvector moves by at most ||E|| / gap under a symmetric perturbation E, where
  gap = |lambda_2| - |lambda_1| (eigenvalues ordered by |lambda|) is not larger than the distance of lambda_1 to the
  others; u u^T then moves by at most twice that, and cov by (1 - eps) times that:
      |dcov| <= 2 (1 - eps) (C_EIG 2^-52 ||C|| + |dC|) / gap + 8 * 2^-53   (|dC| = 0: the moments are exact)
  where the last term is the rounding of 1 - w u_a u_b. Where that bound exceeds AMBIGUOUS (1e-6), u is not determined
  by C to the precision worth testing, and the check switches to invariants that need no unique u: (I - cov) / (1 - eps)
  is a unit rank-1 projector, and its direction v has v^T C v within |lambda_2 - lambda_1| + 2 C_EIG 2^-52 ||C|| of
  lambda_1. Where C is diagonal as far as the kernel's Jacobi can tell (its first-sweep stop test holds, so nothing is
  rotated), u is the unit vector of the column Eigen's JacobiSVD puts last: its sort takes the first maximum of the
  remaining |diag| and swaps only when that is not already in place, and stops at a zero maximum.
"""
from __future__ import annotations

import numpy as np

import gridref as GR

F32 = np.float32
U = 2.0**-53
C_EIG = 64
AMBIGUOUS = 1e-6
FORM = 8 * U
FLT_MAX = float(np.finfo(F32).max)


# ---- k nearest neighbours -------------------------------------------------------------------------------------------
def d2_rows(q, t) -> np.ndarray:
    """FLANN L2_Simple in f32, un-fused, of matching rows: ((dx dx + dy dy) + dz dz)."""
    d = np.asarray(q, dtype=F32) - np.asarray(t, dtype=F32)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _lex_rows(cand, d2, higher_index_ties=False):
    """Per row, the candidates in (d2, index) order (index descending on ties when higher_index_ties)."""
    key = -cand if higher_index_ties else cand
    o = np.argsort(key, axis=1, kind="stable")
    cand, d2 = np.take_along_axis(cand, o, 1), np.take_along_axis(d2, o, 1)
    o = np.argsort(d2, axis=1, kind="stable")
    return np.take_along_axis(cand, o, 1), np.take_along_axis(d2, o, 1)


def knn(cloud, k, higher_index_ties=False, brute_limit=4e6):
    """Exact k-NN of every row of `cloud` over its finite rows: (I (n, k) int64, D (n, k) f32), rows of non-finite points
    (and every row when fewer than k rows are finite) are -1 / inf."""
    p = np.asarray(cloud, dtype=F32)[:, :3]
    ok = GR.finite_rows(p)
    fin = np.flatnonzero(ok)
    n = len(p)
    I = np.full((n, k), -1, dtype=np.int64)
    D = np.full((n, k), np.inf, dtype=F32)
    if len(fin) < k:
        return I, D
    t = p[fin]
    if len(fin) * len(fin) <= brute_limit:
        for lo in range(0, len(fin), 512):
            q = t[lo:lo + 512]
            d = GR._d2(q, t)
            cand = np.broadcast_to(np.arange(len(t)), d.shape)
            ci, cd = _lex_rows(cand, d, higher_index_ties)
            I[fin[lo:lo + 512]] = fin[ci[:, :k]]
            D[fin[lo:lo + 512]] = cd[:, :k]
        return I, D
    from scipy.spatial import cKDTree

    tree = cKDTree(t.astype(np.float64))
    pending = np.arange(len(t))
    m = 8
    while len(pending):
        kk = min(k + m, len(t))
        dd, ii = tree.query(t[pending].astype(np.float64), k=kk, workers=-1)
        ii = ii.astype(np.int64)
        d2 = d2_rows(t[pending][:, None, :], t[ii])
        ci, cd = _lex_rows(ii, d2, higher_index_ties)
        done = np.ones(len(pending), bool) if kk == len(t) else dd[:, -1] ** 2 * (1 - 2.0**-20) > cd[:, k - 1]
        rows = pending[done]
        I[fin[rows]] = fin[ci[done, :k]]
        D[fin[rows]] = cd[done, :k]
        pending = pending[~done]
        m *= 4
    return I, D


# ---- the ring search (nn_search.cuh, gicp_cov_kernel) ---------------------------------------------------------------
def cells(points, g) -> np.ndarray:
    """nn_cell_coord: floor(f32(f32(v - o) * inv_h)), clamped to the grid; (n, 3)."""
    p = np.asarray(points, dtype=F32)[:, :3]
    with np.errstate(invalid="ignore"):
        c = np.floor((p - g["origin"].astype(F32)) * F32(g["inv_h"]))
    c = np.nan_to_num(c, nan=0.0, posinf=2.0**31, neginf=-2.0**31)
    return np.clip(c, 0, g["dims"] - 1).astype(np.int64)


def ring_b2(r, g, rule) -> F32:
    """The squared radius the search trusts after ring r. "old": (r h)^2 0.99999; "sound": the same with r reduced by
    delta = max dim 2^-20 cells, the f32 cell-assignment error of query and point together (nn_search.cuh)."""
    h = F32(g["h"])
    rr = F32(r)
    if rule == "sound":
        rr = max(F32(rr - F32(float(max(g["dims"]))) * F32(2.0**-20)), F32(0))
    bound = F32(rr * h)
    return F32(F32(bound * bound) * F32(0.99999))


def ring_search(target, query, k, rule="old", max_d2=FLT_MAX, max_rings=None):
    """The ring walk of nn1_search (k = 1) and gicp_cov_kernel for one query, restated: after each ring the k best
    (d2, index) of the visited points; stop when k are known and the k-th is <= ring_b2, or (k = 1) when ring_b2 >
    max_d2. Returns (indices, d2) of what the search holds when it stops (fewer than k when it stopped without them)."""
    t = np.asarray(target, dtype=F32)[:, :3]
    ok = GR.finite_rows(t)
    g = GR.nn_geometry(t[ok])
    ct = cells(t[ok], g)
    cq = cells(np.asarray(query, dtype=F32).reshape(1, 3), g)[0]
    ring = np.abs(ct - cq).max(axis=1)
    d2 = d2_rows(np.asarray(query, dtype=F32).reshape(1, 3), t[ok])
    idx = np.flatnonzero(ok)
    top = int(g["dims"].max()) if max_rings is None else max_rings
    for r in range(top + 1):
        vis = ring <= r
        o = np.lexsort((idx[vis], d2[vis]))[:k]
        bi, bd = idx[vis][o], d2[vis][o]
        b2 = ring_b2(r, g, rule)
        if len(bi) == k and bd[-1] <= b2:
            break
        if k == 1 and b2 > F32(max_d2):
            break
    return bi, bd


def knn_by_rings(cloud, k, rule="old"):
    """k-NN of every finite row by the restated ring search (small clouds only)."""
    p = np.asarray(cloud, dtype=F32)[:, :3]
    I = np.full((len(p), k), -1, dtype=np.int64)
    for i in np.flatnonzero(GR.finite_rows(p)):
        bi, _ = ring_search(p, p[i], k, rule)
        I[i, :len(bi)] = bi
    return I


# ---- moments and covariance -----------------------------------------------------------------------------------------
def moments(cloud, I, k, f64_products=False, divisor=None):
    """The kernel's C (n, 6: xx xy xz yy yz zz) from the neighbours I (ascending (d2, index) order)."""
    p = np.asarray(cloud, dtype=F32)[:, :3]
    rows = (I >= 0).all(axis=1)
    nb = p[np.where(I >= 0, I, 0)]
    mean = np.zeros((len(p), 3))
    c = np.zeros((len(p), 6))
    pairs = ((0, 0), (1, 0), (2, 0), (1, 1), (2, 1), (2, 2))
    for s in range(k):  # one rounded add per neighbour, in order (a numpy axis sum would be pairwise)
        x = nb[:, s]
        mean = mean + x.astype(np.float64)
        if f64_products:
            x = x.astype(np.float64)
        c = c + np.stack([(x[:, a] * x[:, b]).astype(np.float64) for a, b in pairs], axis=1)
    kk = float(k if divisor is None else divisor)
    with np.errstate(invalid="ignore"):  # rows without a neighbourhood are dropped by the caller
        mean = mean / kk
        c = c / kk - np.stack([mean[:, a] * mean[:, b] for a, b in pairs], axis=1)
    return c, rows


def sym(c6) -> np.ndarray:
    c = np.asarray(c6)
    return np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], axis=1)


def eigen_last_column(diag_abs) -> int:
    """Which column of an unrotated U Eigen's JacobiSVD puts last: selection sort of the singular values, descending,
    first maximum, swap only when it is not in place, stop at a zero maximum."""
    s, col = [float(v) for v in diag_abs], [0, 1, 2]
    for i in range(3):
        j = i + int(np.argmax(s[i:]))
        if s[j] == 0.0:
            break
        if j != i:
            s[i], s[j] = s[j], s[i]
            col[i], col[j] = col[j], col[i]
    return col[2]


def completion_last_column(diag_abs) -> int:
    """The column oracle/linalg.hpp's JacobiSVD puts last for an unrotated diagonal: a stable descending sort, with the
    columns of zero singular values completed by Gram-Schmidt on e_0, e_1, e_2. It differs from Eigen's only when two
    values are exactly zero and the nonzero one is not first (diag(0, 0, s): Eigen's swap leaves x last, this y)."""
    d = [float(v) for v in diag_abs]
    nz = [j for j in sorted(range(3), key=lambda j: -d[j]) if d[j] > 0]
    return (nz + [e for e in range(3) if e not in nz])[2]


def unrotated(c6) -> np.ndarray:
    """Where sym_eig_smallest's first-sweep stop test holds: no rotation, U = I."""
    c = np.asarray(c6)
    off = c[:, 1] * c[:, 1] + c[:, 2] * c[:, 2] + c[:, 4] * c[:, 4]
    diag = c[:, 0] * c[:, 0] + c[:, 3] * c[:, 3] + c[:, 5] * c[:, 5]
    return (off == 0.0) | (off <= 1e-34 * diag)


def cov_from_moments(c6, eps, column="eigen", eps_column="smallest"):
    """cov = I - (1 - eps) u u^T per point, and what the check needs: (cov (n, 3, 3), info dict)."""
    C = sym(c6)
    lam, V = np.linalg.eigh(C)
    order = np.argsort(np.abs(lam), axis=1, kind="stable")
    n = len(C)
    pick = order[:, 2] if eps_column == "largest" else order[:, 0]
    u = V[np.arange(n), :, pick]
    flat = unrotated(c6)
    for i in np.flatnonzero(flat):
        d = np.abs(np.asarray(c6)[i, [0, 3, 5]])
        if eps_column == "largest":
            m = int(np.argmax(d))
        elif column == "eigen":
            m = eigen_last_column(d)
        elif column == "completion":
            m = completion_last_column(d)
        else:  # the first minimum
            m = int(np.argmin(d))
        u[i] = np.eye(3)[m]
    w = 1.0 - eps
    cov = np.eye(3)[None] - w * u[:, :, None] * u[:, None, :]
    la = np.take_along_axis(lam, order, 1)
    norm = np.abs(la[:, 2])
    gap = np.abs(la[:, 1]) - np.abs(la[:, 0])
    with np.errstate(divide="ignore", invalid="ignore"):
        bound = 2.0 * w * C_EIG * 2.0**-52 * norm / gap + FORM
    bound = np.where(np.isfinite(bound), bound, np.inf)
    bound[flat] = FORM
    return cov, dict(C=C, lam=la, norm=norm, bound=bound, flat=flat, eps=eps)


def reference(cloud, k, eps=1e-3, **mut):
    """K5 restated for every row: (cov (n, 3, 3), info). Rows without a k-neighbourhood (non-finite, or fewer than k
    finite rows) are zero in cov and marked info["rows"] False; a cloud of fewer than k rows is all zero (the kernel is
    not launched). mut: higher_index_ties, stop_rule ("old"/"sound": the ring search instead of the exact k-NN),
    f64_products, column ("first"), eps_column ("largest"), divisor."""
    p = np.asarray(cloud, dtype=F32)[:, :3]
    if len(p) < k:
        return np.zeros((len(p), 3, 3)), dict(rows=np.zeros(len(p), bool))
    if mut.get("stop_rule"):
        I = knn_by_rings(p, k, mut["stop_rule"])
    else:
        I, _ = knn(p, k, higher_index_ties=mut.get("higher_index_ties", False))
    c6, rows = moments(p, I, k, mut.get("f64_products", False), mut.get("divisor"))
    cov, info = cov_from_moments(np.where(rows[:, None], c6, 0.0), eps, mut.get("column", "eigen"),
                                 mut.get("eps_column", "smallest"))
    cov[~rows] = 0.0
    info["rows"] = rows
    info["I"] = I
    return cov, info


def check(got, cov, info):
    """Per point: (bad mask over the rows with a neighbourhood, worst ratio |dcov| / bound over the pointwise-checked
    points, number of points checked by invariants)."""
    got = np.asarray(got, dtype=np.float64)
    rows = info["rows"]
    if "bound" not in info:  # fewer than k rows: no covariance is computed, all stay zero
        return ~(got == 0).all(axis=(1, 2)), 0.0, 0
    err = np.abs(got - cov).max(axis=(1, 2))
    bound = info["bound"]
    point = rows & (bound <= AMBIGUOUS)
    bad = point & ~(err <= bound)
    inv = rows & ~point
    if inv.any():
        w = 1.0 - info["eps"]
        P = (np.eye(3)[None] - got[inv]) / w
        ev, V = np.linalg.eigh(P)
        v = V[:, :, 2]
        proj = (np.abs(P - np.swapaxes(P, 1, 2)).max(axis=(1, 2)) <= 1e-12) & \
               (np.abs(ev - [0.0, 0.0, 1.0]).max(axis=1) <= 1e-12)
        C, lam, norm = info["C"][inv], info["lam"][inv], info["norm"][inv]
        ray = np.einsum("ni,nij,nj->n", v, C, v)
        tol = np.abs(lam[:, 1] - lam[:, 0]) + 2 * C_EIG * 2.0**-52 * norm
        bad[inv] = ~(proj & (np.abs(ray - lam[:, 0]) <= tol))
    ratio = float(np.max(err[point] / bound[point])) if point.any() else 0.0
    return bad, ratio, int(inv.sum())


# ---- fixture generators ---------------------------------------------------------------------------------------------
def box_corners(L, w):
    return np.array([[x, y, z] for x in (0.0, L) for y in (0.0, w) for z in (0.0, w)])


def _first_float_of_cell(c, inv_h):
    """Per cell index c (array), the smallest f32 x >= 0 with floor(f32(x * inv_h)) >= c (origin 0)."""
    cell = lambda v: np.floor(v * F32(inv_h))  # noqa: E731
    x = (np.asarray(c, dtype=np.float64) / float(inv_h)).astype(F32)
    for _ in range(64):
        lo = cell(x) >= c
        prev = np.nextafter(x, F32(-np.inf), dtype=F32)
        down = lo & (cell(prev) >= c)
        up = ~lo
        if not (down.any() or up.any()):
            return x
        x = np.where(down, prev, np.where(up, np.nextafter(x, F32(np.inf), dtype=F32), x))
    raise RuntimeError("cell face search did not settle")


def _a_offset(q, ax, y0, dB, b2_lo, b2):
    """A = (ax, y0 + dy, y0) with dB < d2(q, A) <= b2 and d2(q, A) > b2_lo, or None. The window between d2(q, B) and the
    bound is far narrower than the step one ulp of x makes in d2; the y offset tunes d2(q, A) in steps below it."""
    qq = np.array([q, y0, y0], dtype=F32)
    dax = float(d2_rows(qq, np.array([ax, y0, y0], dtype=F32)))
    for f in (0.0, 0.5, 0.25, 0.75, 0.1, 0.9):
        dy = F32(np.sqrt(max(float(dB) - dax, 0.0) + f * max(float(b2) - max(float(dB), dax), 0.0)))
        for _ in range(8):
            a = np.array([ax, y0 + dy, y0], dtype=F32)
            dA = d2_rows(qq, a)
            if dB < dA <= b2 and dA > b2_lo:
                return a
            dy = np.nextafter(dy, F32(np.inf), dtype=F32)
    return None


def far_face(kind, k=1, L=3000.0, w=0.5, max_j=48):
    """A query q at the low face of cell t of a long 1-D grid (the 8 corners of [0, L] x [0, w]^2 fix the geometry),
    B the last float of cell t - 2 (ring 2) on the line y = z = w / 5 through q and, for kind "1nn" / "knn", A in cell
    t - 1 (ring 1), 0.3 off that line in y, its x and y tuned so that d2(q, A) lies between d2(q, B) and the old bound.
    f32 cell rounding puts B closer to q than (h^2 0.99999) although two cells lie between them. Cells are searched from
    the far end of the axis until:
      "1nn":   d2(q, B) < d2(q, A) <= (h^2 0.99999): a search that trusts (r h)^2 stops after ring 1 with A;
      "knn":   the same with k - 2 further points in q's cell, off the line in y and z (closer than A and B), so the k-th
               neighbour of q is B and the old rule stops with A;
      "gated": no A, and d2(q, B) * 1.0001 < (h^2 0.99999): a caller radius max_d2 = d2(q, B) * 1.0001 (the slack of
               getFitnessScore and of the correspondence search) ends the search after ring 1 with nothing found.
    Returns dict(target, query (1, 3), want (index of B), d2 (f32 d2(q, B)), geometry, t)."""
    y0 = F32(w / 5)
    n = 8 + {"1nn": 2, "knn": k + 1, "gated": 1}[kind]  # fixed before h: h depends on n
    box = box_corners(L, w)
    g = GR.nn_geometry(np.concatenate([box, np.full((n - 8, 3), w / 5)]).astype(F32))
    h, inv_h, dims = F32(g["h"]), F32(g["inv_h"]), int(g["dims"][0])
    assert g["dims"][1] == g["dims"][2] == 1
    b2_old, b2_sound = ring_b2(1, g, "old"), ring_b2(1, g, "sound")
    ts = np.arange(dims - 3, max(dims // 8, 3), -1)
    x_t = _first_float_of_cell(ts, inv_h)
    B = np.nextafter(_first_float_of_cell(ts - 1, inv_h), F32(-np.inf), dtype=F32)
    q = x_t.copy()
    for j in range(max_j):
        ok = (np.floor(q * inv_h) == ts) & (np.floor(B * inv_h) == ts - 2)
        dB = F32(q - B) * F32(q - B)
        if kind == "gated":
            hit = ok & (F32(F32(dB) * F32(1.0001)) + F32(1e-30) < b2_old)
        else:
            hit = ok & (dB < b2_old)
        for i in np.flatnonzero(hit):
            a = None
            if kind != "gated":
                ax = F32(q[i] - F32(np.sqrt(max(float(dB[i]) - 0.09, 0.0))))
                if abs(int(np.floor(ax * inv_h)) - int(ts[i])) > 1:
                    continue
                a = _a_offset(q[i], ax, y0, dB[i], b2_sound, b2_old)
                if a is None:
                    continue
            qq = np.array([[q[i], y0, y0]], dtype=F32)
            parts = [box.astype(F32)]
            if kind == "knn":
                jj = np.arange(k - 2)
                extra = np.stack([np.full(k - 2, q[i]), y0 + F32(0.05) * (1 + jj % 6), y0 + F32(0.05) * (1 + jj // 6)], 1)
                parts += [qq, extra.astype(F32)]
            if a is not None:
                parts.append(a[None])
            parts.append(np.array([[B[i], y0, y0]], dtype=F32))
            tgt = np.concatenate(parts).astype(F32)
            assert len(tgt) == n
            g2 = GR.nn_geometry(tgt)
            assert g2["h"] == h and (g2["dims"] == g["dims"]).all()
            return dict(target=tgt, query=qq, want=len(tgt) - 1, d2=F32(dB[i]), geometry=g2, t=int(ts[i]))
        q = np.nextafter(q, F32(np.inf), dtype=F32)
    raise LookupError((kind, k, L, w))


def far_face_case(kind, k=1, L=3000.0, w=0.5, tries=64):
    """far_face on the first of the boxes L (1 + 0.0131 i) x w x w that has such a cell: whether one exists depends on
    how h's mantissa meets the f32 spacing of the far cells' coordinates."""
    for i in range(tries):
        try:
            return far_face(kind, k, L=round(L * (1 + 0.0131 * i), 3), w=w)
        except LookupError:
            continue
    raise LookupError((kind, k, L, w))


def far_face_gated():
    """The gated case needs d2(q, B) below 0.99989 h^2: more than 5e-5 cells of f32 cell rounding, which the 1 130-cell
    box of the 1-NN case never reaches (one ulp of a coordinate there is 4.6e-5 cells of 2.66 m). A 40 km x 5 cm box
    has 28 000 cells of 1.4 m, and its far cells do."""
    return far_face_case("gated", L=40000.0, w=0.05)


def face_queries(target, seed=0, axes_min_cells=1000):
    """Queries on every cell face (and one ulp either side) of each axis with at least axes_min_cells cells, up to the
    last face; the other two coordinates from random target points."""
    rng = np.random.default_rng(seed)
    t = np.asarray(target, dtype=F32)[:, :3]
    t = t[GR.finite_rows(t)]
    g = GR.nn_geometry(t)
    out = []
    for a in range(3):
        if g["dims"][a] < axes_min_cells:
            continue
        faces = (g["origin"][a] + np.arange(int(g["dims"][a]) + 1) * np.float64(g["h"])).astype(F32)
        for u in (-1, 0, 1):
            q = t[rng.integers(len(t), size=len(faces))].copy()
            q[:, a] = faces if u == 0 else np.nextafter(faces, F32(u * np.inf), dtype=F32)
            out.append(q)
    return np.concatenate(out).astype(F32)


def corridor(n=20000, seed=0):
    """A 2 km x 20 m x 5 m corridor: an NN grid with about 1 500 cells along x."""
    rng = np.random.default_rng(seed)
    return np.c_[rng.uniform(0, 2000, n), rng.uniform(0, 20, n), rng.uniform(0, 5, n)].astype(F32)


def dyadic_duplicates(k, groups=4):
    """groups of k + 3 identical points at dyadic positions far apart: every neighbourhood is one position, C = 0."""
    c = np.array([[4.25, -1.5, 0.75], [40.5, 2.0, -3.25], [-17.0, 30.125, 8.0], [0.0, 0.0, 0.0]])[:groups]
    return np.repeat(c, k + 3, axis=0).astype(F32)


def axis_line(axis, n=64, step=0.25):
    """n points at dyadic spacing along one axis through the origin: C = diag with two exact zeros."""
    p = np.zeros((n, 3))
    p[:, axis] = np.arange(n) * step - 4.0
    return p.astype(F32)


def axis_plane(normal, n_side=12, step=0.5, height=1.5):
    """An n_side^2 lattice in the plane {x_normal = height}: one zero eigenvalue, ties in every neighbourhood."""
    a, b = [i for i in range(3) if i != normal]
    ii, jj = np.meshgrid(np.arange(n_side), np.arange(n_side), indexing="ij")
    p = np.zeros((n_side * n_side, 3))
    p[:, a], p[:, b], p[:, normal] = ii.ravel() * step, jj.ravel() * step * 1.25, height
    return p.astype(F32)


def scene(n=3000, seed=0):
    """Two noisy surfaces and a wall, 20 m across: ordinary anisotropic neighbourhoods."""
    rng = np.random.default_rng(seed)
    u = rng.uniform(-10, 10, size=(n, 2))
    z = 0.5 * np.sin(0.4 * u[:, 0]) + 0.2 * np.cos(0.7 * u[:, 1]) + rng.normal(0, 0.02, n)
    wall = np.c_[rng.uniform(-10, 10, n // 3), np.full(n // 3, 10.0) + rng.normal(0, 0.02, n // 3),
                 rng.uniform(0, 3, n // 3)]
    return np.concatenate([np.c_[u, z], wall]).astype(F32)


def cov_fixtures(k):
    """The K5 clouds for k neighbours: name -> (n, 3) f32."""
    rng = np.random.default_rng(100 + k)
    aniso = lambda m: (rng.normal(0, 1, (m, 3)) * [3, 1, 0.3]).astype(F32)  # noqa: E731
    out = {
        "far-face knn": far_face_case("knn", k)["target"],
        "far-face 1nn": far_face_case("1nn")["target"],
        "lattice": GR.lattice((6, 5, 4), (1.0, 1.3, 1.7)),
        "cubic lattice": GR.lattice((5, 5, 5), (0.5, 0.5, 0.5)),
        "dyadic duplicates": dyadic_duplicates(k),
        "identical": np.full((50, 3), 4.25, F32),
        "line x": axis_line(0), "line y": axis_line(1), "line z": axis_line(2),
        "plane z": axis_plane(2), "plane x": axis_plane(0),
        "nonfinite": GR.with_nonfinite_rows(scene(800, seed=k), seed=k)[0][:, :3],
        "n = k": aniso(k), "n = k+1": aniso(k + 1), "n = 2k": aniso(2 * k),
    }
    for off in GR.SHIFTS:
        out[("shift", off)] = GR.shifted(scene(1500, seed=k), off)
    return {name: np.ascontiguousarray(c, dtype=F32)[:, :3] for name, c in out.items()}
