"""Exact Python replay of csrc/map_consistency.hpp (the map consistency of b200sm_build_map_consistency): float32 transforms
one rounding per operation, fixed point, cells and every moment sum in int64 integers (exact: no sum can overflow), and
the per-query covariance, determinant, logarithm and Jacobi sweeps as IEEE doubles in the header's order, vectorised with
numpy (elementwise, no fused operations). `mut` names a deliberate deviation, so the tests can show the replay tells each
of them apart."""
import math

import numpy as np

F32 = np.float32
ONE = 1 << 16
COORD_LIMIT = 2.0 ** 46
RADIUS2 = 1 << 32
MAX_POINTS = (1 << 31) - 1
MAX_CELLS = (1 << 31) - 1
NAN_BITS = 0x7FF8000000000000
NAN = np.array([NAN_BITS], dtype=np.uint64).view(np.float64)[0]
H_SCALE = 2.0 ** 24
PLANE_SCALE = 2.0 ** 30
SWEEPS = 6
TWO_PI_E = float.fromhex("0x1.114580b45d475p+4")
LN2_HI = float.fromhex("0x1.62e42fee00000p-1")
LN2_LO = float.fromhex("0x1.a39ef35793c76p-33")
SQRT2 = float.fromhex("0x1.6a09e667f3bcdp+0")
LOG_C = [2.0 / (2 * k + 1) for k in range(1, 12)]  # 2/3 ... 2/23, each correctly rounded

MUTATIONS = ("lt_radius", "cells26", "cov_n1", "drop_self", "trunc")

DEFAULTS = dict(radius=0.5, min_neighbors=10, query_stride=1)


def params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    return p


class Refused(Exception):
    """The build is refused; .code is the host harness's return code."""

    def __init__(self, code, why):
        super().__init__(why)
        self.code = code


def mc_log(x):
    """The header's mc_log, elementwise over a float64 array (positive normal values)."""
    x = np.asarray(x, dtype=np.float64)
    b = x.view(np.uint64)
    e = ((b >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64) - 1023
    m = ((b & np.uint64(0xFFFFFFFFFFFFF)) | np.uint64(0x3FF0000000000000)).view(np.float64)
    big = m > SQRT2
    m = np.where(big, m * 0.5, m)
    e = e + big
    f = m - 1.0
    s = f / (2.0 + f)
    z = s * s
    R = np.full_like(z, LOG_C[10])
    for k in range(9, -1, -1):
        R = LOG_C[k] + z * R
    R = z * R
    lnm = f - s * (f - R)
    de = e.astype(np.float64)
    return de * LN2_HI + (lnm + de * LN2_LO)


def _rotate(app, aqq, apq, arp, arq):
    with np.errstate(all="ignore"):
        theta = (aqq - app) / (2.0 * apq)
        at = np.abs(theta)
        t = 1.0 / (at + np.sqrt(theta * theta + 1.0))
        t = np.where(theta < 0.0, -t, t)
        c = 1.0 / np.sqrt(t * t + 1.0)
        s = t * c
        tp = t * apq
        napp, naqq = app - tp, aqq + tp
        narp = c * arp - s * arq
        narq = s * arp + c * arq
    skip = apq == 0.0
    return (np.where(skip, app, napp), np.where(skip, aqq, naqq), np.where(skip, apq, 0.0), np.where(skip, arp, narp),
            np.where(skip, arq, narq))


def lambda_min(a00, a01, a02, a11, a12, a22):
    """The header's mc_lambda_min, elementwise."""
    a00, a01, a02, a11, a12, a22 = (np.array(v, dtype=np.float64, copy=True) for v in (a00, a01, a02, a11, a12, a22))
    for _ in range(SWEEPS):
        a00, a11, a01, a02, a12 = _rotate(a00, a11, a01, a02, a12)
        a00, a22, a02, a01, a12 = _rotate(a00, a22, a02, a01, a12)
        a11, a22, a12, a01, a02 = _rotate(a11, a22, a12, a01, a02)
    m = np.where(a00 < a11, a00, a11)
    return np.where(m < a22, m, a22)


def det3(c00, c01, c02, c11, c12, c22):
    m0 = c11 * c22 - c12 * c12
    m1 = c01 * c22 - c12 * c02
    m2 = c01 * c12 - c11 * c02
    return (c00 * m0 - c01 * m1) + c02 * m2


def prepare(p):
    r = p["radius"]
    if not (0.01 <= r <= 100.0):
        raise Refused(-1, "radius")
    if p["min_neighbors"] < 4:
        raise Refused(-1, "min_neighbors")
    if p["query_stride"] < 1:
        raise Refused(-1, "query_stride")
    S = 65536.0 / r
    c0 = float(3.0 * mc_log(np.array([TWO_PI_E]))[0] - 6.0 * mc_log(np.array([S]))[0])
    return dict(S=S, S2=S * S, r2=r * r, c0=c0, min_neighbors=int(p["min_neighbors"]), stride=int(p["query_stride"]))


def box(lo, hi):
    """sm_box: the dims of inclusive cell bounds, or None beyond 2^31 - 1 cells."""
    dims, n = [], 1
    for a in range(3):
        w = int(hi[a]) - int(lo[a]) + 1
        if w < 1 or w > MAX_CELLS:
            return None
        dims.append(w)
        n *= w
        if n > MAX_CELLS:
            return None
    return dims


def pose_f(P):
    P = np.asarray(P, dtype=np.float64)
    return [F32(P[r, c]) for r in range(3) for c in range(4)]


def transform(T, pts):
    x, y, z = (np.asarray(pts[:, a], dtype=F32) for a in range(3))
    with np.errstate(all="ignore"):
        return np.stack([((T[4 * r] * x + T[4 * r + 1] * y) + T[4 * r + 2] * z) + T[4 * r + 3] for r in range(3)], axis=1)


def quantise(c, e, mut=None):
    """(X int64 (n, 3), ok bool (n,)); Refused(-3) when a non-skipped product is not inside (-2^46, 2^46)."""
    ok = np.all(np.isfinite(e), axis=1)
    with np.errstate(all="ignore"):
        prod = e.astype(np.float64) * c["S"]
    if np.any(ok & ~np.all((prod > -COORD_LIMIT) & (prod < COORD_LIMIT), axis=1)):
        raise Refused(-3, "coordinate range")
    prod = np.where(ok[:, None], prod, 0.0)
    X = (np.trunc(prod) if mut == "trunc" else np.floor(prod)).astype(np.int64)
    return X, ok


def values(c, mom, mut=None):
    """(valid, h, plane_var, qh, ql) of the queries' moments (n, sx, sy, sz, sxx, sxy, sxz, syy, syz, szz: int64 arrays)."""
    n, sx, sy, sz, sxx, sxy, sxz, syy, syz, szz = (np.asarray(v, dtype=np.int64).astype(np.float64) for v in mom)
    nn = n - 1.0 if mut == "cov_n1" else n
    with np.errstate(all="ignore"):
        def cov(sab, sa, sb):
            return (sab - (sa * sb) / n) / nn

        c00, c01, c02 = cov(sxx, sx, sx), cov(sxy, sx, sy), cov(sxz, sx, sz)
        c11, c12, c22 = cov(syy, sy, sy), cov(syz, sy, sz), cov(szz, sz, sz)
        det = det3(c00, c01, c02, c11, c12, c22)
        valid = (np.asarray(mom[0]) >= c["min_neighbors"]) & (det >= 1.0)
        safe = np.where(valid, det, 1.0)
        h = 0.5 * (c["c0"] + mc_log(safe))
        pv = lambda_min(c00, c01, c02, c11, c12, c22) / c["S2"]
        qh = np.rint(h * H_SCALE)
        ql = np.rint((pv / c["r2"]) * PLANE_SCALE)
    h = np.where(valid, h, NAN)
    pv = np.where(valid, pv, NAN)
    qh = np.where(valid, qh, 0).astype(np.int64)
    ql = np.where(valid, ql, 0).astype(np.int64)
    return valid, h, pv, qh, ql


def offsets27(mut=None):
    offs = [(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    return offs[:-1] if mut == "cells26" else offs


def mme(sum_h, valid):
    return (float(sum_h) * (1.0 / H_SCALE)) / float(valid) if valid else NAN


def mpv(c, sum_plane, valid):
    return ((float(sum_plane) * (1.0 / PLANE_SCALE)) * c["r2"]) / float(valid) if valid else NAN


def build(submaps, p=None, mut=None):
    """submaps: [(points (n, >= 3) float32, pose 4x4)]. The build's layers, rows and info as a dict; Refused on a
    refusal."""
    p = params(**(p or {}))
    c = prepare(p)
    if not submaps:
        raise Refused(-2, "no submaps")
    E, sub_of = [], []
    for k, (pts, P) in enumerate(submaps):
        pts = np.asarray(pts, dtype=F32).reshape(len(pts), -1) if len(pts) else np.zeros((0, 3), F32)
        E.append(transform(pose_f(P), pts))
        sub_of.append(np.full(len(pts), k, dtype=np.int64))
    e = np.concatenate(E) if E else np.zeros((0, 3), F32)
    sub_of = np.concatenate(sub_of)
    total = len(e)
    if total > MAX_POINTS:
        raise Refused(-5, "points")
    X, ok = quantise(c, e, mut)
    cell = X >> 16
    n_used = int(ok.sum())
    out_n = np.zeros(total, dtype=np.uint32)
    out_h = np.full(total, NAN)
    out_pv = np.full(total, NAN)
    n_sub = len(submaps)
    rows = dict(n_points=np.array([len(s[0]) for s in submaps], dtype=np.int64), n_queries=np.zeros(n_sub, np.int64),
                n_valid=np.zeros(n_sub, np.int64), n_neighbors=np.zeros(n_sub, np.int64), sum_h_q=np.zeros(n_sub, np.int64),
                sum_plane_q=np.zeros(n_sub, np.int64))
    info = dict(n_points=total, n_skipped=total - n_used, n_cells=0, n_candidates=0, box_origin=(0, 0, 0), box_dims=(0, 0, 0))
    if n_used:
        used = np.flatnonzero(ok)
        lo = cell[used].min(axis=0)
        hi = cell[used].max(axis=0)
        dims = box(lo, hi)
        if dims is None:
            raise Refused(-4, "box")
        info["box_origin"] = tuple(int(v) for v in lo)
        info["box_dims"] = tuple(dims)
        W, H = dims[0], dims[1]

        def lin(cc):
            return ((cc[:, 2] - lo[2]) * H + (cc[:, 1] - lo[1])) * W + (cc[:, 0] - lo[0])

        key = lin(cell[used])
        order = np.argsort(key, kind="stable")
        skey, sidx = key[order], used[order]
        info["n_cells"] = int(len(np.unique(skey)))
        q = used[used % c["stride"] == 0]
        mom = [np.zeros(len(q), np.int64) for _ in range(10)]
        cand = 0
        for d in offsets27(mut):
            nc = cell[q] + np.array(d, dtype=np.int64)
            inside = np.all((nc >= lo) & (nc <= hi), axis=1)
            k = np.where(inside, lin(np.where(inside[:, None], nc, lo)), -1)
            a = np.searchsorted(skey, k, side="left")
            b = np.searchsorted(skey, k, side="right")
            cnt = np.where(inside, b - a, 0)
            cand += int(cnt.sum())
            qi = np.repeat(np.arange(len(q)), cnt)
            start = np.repeat(a - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
            j = sidx[start + np.arange(len(qi))] if len(qi) else np.zeros(0, np.int64)
            D = X[j] - X[q[qi]]
            d2 = (D * D).sum(axis=1)
            acc = d2 < RADIUS2 if mut == "lt_radius" else d2 <= RADIUS2
            if mut == "drop_self":
                acc &= j != q[qi]
            qi, D = qi[acc], D[acc]
            terms = [np.ones(len(qi), np.int64), D[:, 0], D[:, 1], D[:, 2], D[:, 0] * D[:, 0], D[:, 0] * D[:, 1],
                     D[:, 0] * D[:, 2], D[:, 1] * D[:, 1], D[:, 1] * D[:, 2], D[:, 2] * D[:, 2]]
            for t in range(10):
                np.add.at(mom[t], qi, terms[t])
        info["n_candidates"] = cand
        valid, h, pv, qh, ql = values(c, mom, mut)
        out_n[q] = mom[0].astype(np.uint32)
        out_h[q] = h
        out_pv[q] = pv
        s = sub_of[q]
        np.add.at(rows["n_queries"], s, 1)
        np.add.at(rows["n_valid"], s, valid.astype(np.int64))
        np.add.at(rows["n_neighbors"], s, mom[0])
        np.add.at(rows["sum_h_q"], s, qh)
        np.add.at(rows["sum_plane_q"], s, ql)
    rows["mme"] = np.array([mme(rows["sum_h_q"][k], rows["n_valid"][k]) for k in range(n_sub)])
    rows["mpv"] = np.array([mpv(c, rows["sum_plane_q"][k], rows["n_valid"][k]) for k in range(n_sub)])
    for k in ("n_queries", "n_valid", "n_neighbors", "sum_h_q", "sum_plane_q"):
        info[k] = int(rows[k].sum())
    info["mme"] = mme(info["sum_h_q"], info["n_valid"])
    info["mpv"] = mpv(c, info["sum_plane_q"], info["n_valid"])
    return dict(n=out_n, h=out_h, plane_var=out_pv, rows=rows, info=info, c=c)
