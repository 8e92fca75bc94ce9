"""A float64 reference of the NDT radius paths, written from the algorithm: the radius neighbourhood of
VoxelGridCovariance::radiusSearch (every voxel centroid, no cells), computeHessian / updateHessian (ndt_omp_impl.hpp:538-629,
the K2 pass) and calculateScore (:919-953), each with a per-entry bound on how far the device's float64 evaluation may be
from it; and the fixtures where a cell-based neighbourhood goes wrong. Nothing here needs a GPU.

What is computed
  The voxels come from the caller (the handle's own voxels(): leaf index, mean as record_mean returns it, the f64 icov,
  the f32 centroid), so the voxel map builder stays out of the comparison.
  * neighbourhood: every voxel whose f32 centroid c passes ((dx*dx + dy*dy) + dz*dz) < f32(res^2), un-fused f32 with
    d = f32(x_t) - c. A cKDTree over the centroids gives a superset (radius res (1 + 1e-6)); the f32 test decides.
    Rows that are not finite have no neighbour (a FLANN query with NaN / inf finds none). near_threshold counts pairs
    whose d2 is within 4 f32 ulp of r^2: an exact-hit assertion against a differently rounded centroid is only valid
    where it is zero. rule="block27" restricts the candidates to the 27 cells around floor(x / leaf) (the rule the
    device used to have), only to show that the fixtures below tell the two apart.
  * x_t: ndtref.transform_points, the f32 transform of the live path (ground truth: both sides transform in float).
  * Hessian, per pair, as updateHessian spells it: x' = f64(x_t) - mean, Cx = C x', e = d2 exp(-d2 x'.Cx / 2), the pair
    dropped when e > 1, e < 0 or NaN, e *= d1; for a <= b:
        H_ab += e (-d2 (x'.C J_a)(x'.C J_b) + x'.C h_ab + J_b.C J_a)
    with J (3 x 6) and h_ab (a, b >= 3) formed in float64 from the source point and the f64 angle tables the host hands
    the K2 pass (ndtref.angle_tables(p, minus_sy=True, f64=True): d1.z = -sy, the f64 convention of
    ndt_omp_impl.hpp:359), d1 and d2 float64.
  * calculateScore: sum over points of (sum over its neighbours of (-d1 exp(-d2 q / 2) - d3)) / |nb|, divided by the
    number of rows n. Rows without a neighbour (non-finite ones included) add nothing but count in n; n = 0 is 0 / 0.

The bound (u = 2^-53)
  tol_k = u sum_p (gamma + sigma_p) a_pk, a_pk the pair's contribution with every factor replaced by its absolute value
  (|x'|, |C|, |J| = |table| . |x|, d2 |x'.C J_a| |x'.C J_b| -> d2 (|x'||C||J_a|)(|x'||C||J_b|)).
    sigma_p, the sensitivity of e: the f64 q = x'.C x' is within 6 u A_p (A_p = |x'| |C| |x'|), which moves exp by
      d2 / 2 6 u A_p relative; the rounding of the argument adds |d2 q / 2| u; exp (1 ulp on either side), e = d2 ex and
      e d1 a few more: sigma_p = 3 d2 A_p + |d2 q / 2| + 8. x' is the same f64 subtraction on both sides.
    gamma, the depth of the sums an entry passes through: the per-pair products (J from the tables 3, C J 3, the dots 3,
      the three terms and e: 32 with an ulp of the host's trigonometry in the tables); the pairs one thread adds in
      sequence (the most pairs of a point times the points one thread takes in the grid-stride loop of 128-thread
      blocks over min(ceil(n / 128), 132 * 8) blocks); 5 shuffle levels; and one atomicAdd per warp, in any order.
      A serial sum (the oracle's) has the total number of pairs instead.
  Score: tol = u / n sum_p (sigma_p |d1 ex| + (|d1 ex| + |d3|)(|nb| + 3 + D)) / |nb| (D: the points per thread, shuffles
  and warps, or the total pair count of a serial sum), plus the final division.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

import gridref as R
import ndtref as N

F32 = np.float32
U = 2.0**-53
H100_SMS = 132  # the radius kernels' grid: min(ceil(n / 128), H100_SMS * 8) blocks of 128 threads
PAIR_DEPTH = 32
TRI = N.TRI


def gauss_constants(outlier_ratio, resolution):
    """(d1, d2, d3) in float64 with the resolution as float (ndt_omp_impl.hpp:88-93)."""
    import math

    res = float(F32(resolution))
    c1 = 10 * (1 - outlier_ratio)
    c2 = outlier_ratio / res**3
    d3 = -math.log(c2)
    d1 = -math.log(c1 + c2) - d3
    d2 = -2 * math.log((-math.log(c1 * math.exp(-0.5) + c2) - d3) / d1)
    return d1, d2, d3


def radius2(res):
    return F32(float(F32(res)) * float(F32(res)))


def f32_d2(xt, c):
    """The un-fused f32 squared distance of the device and of FLANN's L2_Simple."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = np.asarray(xt, dtype=F32) - np.asarray(c, dtype=F32)
        return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def neighbours(xt, res, voxels, rule="all", strict=True, geom=None):
    """(point, voxel) pairs of the radius rule, ordered by point; near: pairs within 4 ulp of r^2 (all candidates)."""
    xt = np.asarray(xt, dtype=F32)
    cen = np.asarray(voxels["centroid"], dtype=F32).reshape(-1, 3)
    r2 = radius2(res)
    if len(cen) == 0 or len(xt) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), 0
    ok = np.nonzero(np.isfinite(xt).all(axis=1) & (np.abs(xt) < 1e30).all(axis=1))[0]
    if rule == "all":
        tree = cKDTree(cen.astype(np.float64))
        lists = tree.query_ball_point(xt[ok].astype(np.float64), r=float(F32(res)) * (1 + 1e-6))
        pi = np.repeat(ok, [len(l) for l in lists]).astype(np.int64)
        vi = np.array([v for l in lists for v in l], dtype=np.int64)
    else:  # the 27 cells around the lookup cell floor(x / leaf), within the grid
        vidx = np.asarray(voxels["idx"], dtype=np.int64)
        ijk = np.stack([R.lookup_ref(xt[ok, a], res) for a in range(3)], axis=1) - geom["min_b"]
        P, V = [], []
        for o in N.offsets(N.KDTREE):
            c = ijk + np.array(o)
            inside = ((c >= 0) & (c < geom["div_b"])).all(axis=1)
            lin = c[:, 0] + c[:, 1] * geom["mul"][1] + c[:, 2] * geom["mul"][2]
            k = np.minimum(np.searchsorted(vidx, lin), len(vidx) - 1)
            hit = inside & (vidx[k] == lin)
            P.append(ok[hit])
            V.append(k[hit])
        pi, vi = np.concatenate(P), np.concatenate(V)
    if len(pi) == 0:
        return pi, vi, 0
    d2 = f32_d2(xt[pi], cen[vi])
    near = int((np.abs(d2.astype(np.float64) - float(r2)) <= 4 * float(np.spacing(r2))).sum())
    keep = (d2 < r2) if strict else (d2 <= r2)
    pi, vi = pi[keep], vi[keep]
    order = np.lexsort((vi, pi))
    return pi[order], vi[order], near


def kernel_depth(n, max_pairs):
    """Summation depth of the radius kernels over n rows: pairs per thread, 5 shuffle levels, one atomicAdd per warp."""
    blocks = max(1, min(-(-n // 128), H100_SMS * 8))
    per_thread = max(1, -(-n // (blocks * 128)))
    return max(1, max_pairs) * per_thread + 5 + 4 * blocks


def _pair_terms(xt, pi, vi, voxels, d2, icov_f32):
    mean = np.asarray(voxels["mean"], dtype=np.float64).reshape(-1, 3)
    C = np.asarray(voxels["icov"], dtype=np.float64).reshape(-1, 3, 3)
    if icov_f32:
        C = C.astype(F32).astype(np.float64)
    xp = xt[pi].astype(np.float64) - mean[vi]
    C = C[vi]
    Cx = np.einsum("pij,pj->pi", C, xp)
    q = np.einsum("pi,pi->p", xp, Cx)
    A = np.einsum("pi,pij,pj->p", np.abs(xp), np.abs(C), np.abs(xp))
    sigma = 3 * d2 * A + np.abs(d2 * q / 2) + 8
    return xp, C, q, sigma


def hessian(src, T, p6, res, voxels, outlier_ratio=0.55, tables=None, minus_sy=True, icov_f32=False, rule="all",
            strict=True, e_guard=True, serial=False, geom=None):
    """computeHessian over the radius neighbourhood. Returns a dict: H (6, 6), tol (6, 6), hits, near_threshold.
    tables: (jd (24,), hd (45,)) f64 tables to use instead of ndtref's (the device's own, from a trace); serial=True
    bounds a serial f64 sum over all pairs (the oracle's) instead of the kernel's."""
    src = np.asarray(src, dtype=F32)[:, :3]
    d1, d2, _ = gauss_constants(outlier_ratio, res)
    if tables is None:
        _, _, jd, hd = N.angle_tables(p6, minus_sy=minus_sy, f64=True)
    else:
        jd, hd = (np.asarray(t, dtype=np.float64).reshape(-1, 3) for t in tables)
    xt = N.transform_points(T, src)
    pi, vi, near = neighbours(xt, res, voxels, rule, strict, geom)
    out = dict(H=np.zeros((6, 6)), tol=np.zeros((6, 6)), hits=0, near_threshold=near, pairs=len(pi))
    if len(pi) == 0:
        return out
    xp, C, q, sigma = _pair_terms(xt, pi, vi, voxels, d2, icov_f32)
    with np.errstate(over="ignore", invalid="ignore"):
        e = d2 * np.exp(-d2 * q / 2)
    if e_guard:
        with np.errstate(invalid="ignore"):
            ok = ~((e > 1) | (e < 0) | np.isnan(e))
        pi, xp, C, q, sigma, e = pi[ok], xp[ok], C[ok], q[ok], sigma[ok], e[ok]
    out["near_threshold"] += int((np.abs(e - 1) <= 64 * U).sum())
    e = e * d1
    out["hits"] = len(pi)
    x = src[pi].astype(np.float64)
    J, Ja = np.zeros((len(pi), 3, 6)), np.zeros((len(pi), 3, 6))
    jv, jva = x @ jd.T, np.abs(x) @ np.abs(jd).T  # (P, 8)
    for M, v in ((J, jv), (Ja, jva)):
        M[:, 0, 0] = M[:, 1, 1] = M[:, 2, 2] = 1.0
        M[:, 1, 3], M[:, 2, 3] = v[:, 0], v[:, 1]
        M[:, :, 4] = v[:, 2:5]
        M[:, :, 5] = v[:, 5:8]
    hv, hva = x @ hd.T, np.abs(x) @ np.abs(hd).T  # (P, 15)
    Hv, Hva = np.zeros((len(pi), 6, 6, 3)), np.zeros((len(pi), 6, 6, 3))
    for M, v in ((Hv, hv), (Hva, hva)):
        z = np.zeros(len(pi))
        vecs = (np.stack([z, v[:, 0], v[:, 1]], 1), np.stack([z, v[:, 2], v[:, 3]], 1), np.stack([z, v[:, 4], v[:, 5]], 1),
                v[:, 6:9], v[:, 9:12], v[:, 12:15])
        for (a, b), vec in zip(((3, 3), (3, 4), (3, 5), (4, 4), (4, 5), (5, 5)), vecs):
            M[:, a, b] = M[:, b, a] = vec
    Ca, xa = np.abs(C), np.abs(xp)
    CJ = np.einsum("pij,pjk->pik", C, J)
    CJa = np.einsum("pij,pjk->pik", Ca, Ja)
    xCJ = np.einsum("pi,pik->pk", xp, CJ)
    xCJa = np.einsum("pi,pik->pk", xa, CJa)
    xC = np.einsum("pi,pij->pj", xp, C)
    xCa = np.einsum("pi,pij->pj", xa, Ca)
    h = -d2 * xCJ[:, :, None] * xCJ[:, None, :] + np.einsum("pc,pabc->pab", xC, Hv) + np.einsum("pcb,pca->pab", J, CJ)
    ha = d2 * xCJa[:, :, None] * xCJa[:, None, :] + np.einsum("pc,pabc->pab", xCa, Hva) + np.einsum("pcb,pca->pab", Ja, CJa)
    if serial:
        gamma = len(pi) + PAIR_DEPTH
    else:
        gamma = kernel_depth(len(src), int(np.bincount(pi).max())) + PAIR_DEPTH
    out["H"] = np.einsum("p,pab->ab", e, h)
    out["tol"] = U * np.einsum("p,pab->ab", (gamma + sigma) * np.abs(e), ha)
    il = np.tril_indices(6, -1)  # the kernels form the upper triangle and mirror it
    out["H"][il] = out["H"].T[il]
    out["tol"][il] = out["tol"].T[il]
    return out


def score(cloud, res, voxels, outlier_ratio=0.55, rule="all", strict=True, average="point", serial=False, geom=None):
    """calculateScore of an already transformed cloud. Returns a dict: score, tol, hits, near_threshold, n.
    average="global" (a mutation) divides the sum over all pairs by the number of pairs instead."""
    xt = np.asarray(cloud, dtype=F32)[:, :3]
    n = len(xt)
    d1, d2, d3 = gauss_constants(outlier_ratio, res)
    pi, vi, near = neighbours(xt, res, voxels, rule, strict, geom)
    out = dict(score=np.nan if n == 0 else 0.0, tol=0.0, hits=len(pi), near_threshold=near, n=n)
    if len(pi) == 0:
        return out
    xp, C, q, sigma = _pair_terms(xt, pi, vi, voxels, d2, False)
    ex = np.exp(-d2 * q / 2)
    t = -d1 * ex - d3
    nb = np.bincount(pi, minlength=n)
    if average == "global":
        out["score"] = float(t.sum() / len(pi))
    else:
        out["score"] = float((np.bincount(pi, weights=t, minlength=n)[nb > 0] / nb[nb > 0]).sum() / n)
    D = (len(pi) if serial else kernel_depth(n, int(nb.max())))
    maj = (sigma * np.abs(d1 * ex) + (np.abs(d1 * ex) + abs(d3)) * (nb[pi] + 3 + D)) / nb[pi]
    out["tol"] = U * float(maj.sum()) / n + 2 * U * abs(out["score"])
    return out


def within_h(H, ref, scale=1.0):
    """Per upper entry |H - ref| / (scale tol) (0 where equal); the largest."""
    r = np.array([0.0 if H[i, j] == ref["H"][i, j] else abs(H[i, j] - ref["H"][i, j]) / (scale * ref["tol"][i, j])
                  for i, j in TRI])
    return float(r.max()), r


def within_score(s, ref, scale=1.0):
    if s == ref["score"]:
        return 0.0
    return abs(s - ref["score"]) / (scale * ref["tol"]) if ref["tol"] else np.inf


# ---- fixtures where a cell-based neighbourhood goes wrong ----------------------------------------------------------
def _floats_near(v, ulps=12):
    v = F32(v)
    lo = v
    for _ in range(ulps):
        lo = np.nextafter(lo, F32(-np.inf), dtype=F32)
    out = [lo]
    for _ in range(2 * ulps):
        out.append(np.nextafter(out[-1], F32(np.inf), dtype=F32))
    return np.array(out, dtype=F32)


def escape_pairs(leaf, direction, k_range=range(-700, 700), limit=4):
    """(w, q): a wall coordinate w in build cell k = floor(fl(w * inv_leaf)) and a query q two LOOKUP cells from it
    (floor(q / leaf) = k - 2 for direction +1: the wall above the query; k + 2 for -1) with f32 (q - w)^2 < res^2 by more
    than 4 ulp. The first `limit` found, scanning k."""
    leaf = F32(leaf)
    r2 = radius2(leaf)
    found = []
    for k in k_range:
        edge = k if direction > 0 else k + 1
        w_c = _floats_near(edge * float(leaf))
        w_c = w_c[R.build_ref(w_c, leaf) == k]
        q_edge = (k - 1) if direction > 0 else (k + 2)
        q_c = _floats_near(q_edge * float(leaf))
        q_c = q_c[R.lookup_ref(q_c, leaf) == k - 2 * direction]
        if len(w_c) == 0 or len(q_c) == 0:
            continue
        w =w_c.min() if direction > 0 else w_c.max()
        q = q_c.max() if direction > 0 else q_c.min()
        dx = F32(q - w)
        d2 = F32(dx * dx)
        if d2 < r2 and float(r2) - float(d2) > 4 * float(np.spacing(r2)):
            found.append((w, q))
            if len(found) >= limit:
                break
    return found


def wall(axis, w, centre, leaf):
    """8 points at coordinate w on `axis`, +-leaf/8 and +-leaf/16 around `centre` on the other two axes: the f64 sum and
    the division by 8 are exact, so the centroid is (w, centre) exactly (centre exact in f32). The identity start of the
    covariance (the reference's cov_ = Identity quirk) keeps the flat leaf a valid voxel."""
    o = [a for a in range(3) if a != axis]
    pts = np.zeros((8, 3), dtype=F32)
    t1, t2 = F32(leaf / 8), F32(leaf / 16)
    offs = [(t1, t2), (-t1, -t2), (t1, -t2), (-t1, t2), (t2, t1), (-t2, -t1), (t2, -t1), (-t2, t1)]
    for i, (a, b) in enumerate(offs):
        pts[i, axis] = w
        pts[i, o[0]] = F32(centre[0]) + a
        pts[i, o[1]] = F32(centre[1]) + b
    return pts


def escape_fixture(leaf, axis, direction, inside=True, case=0, seed=0):
    """A target holding one wall voxel whose centroid is within the radius of a query two lookup cells away on `axis`.
    inside=True adds a floor of ordinary voxels 6 cells away on another axis, spanning the query, so the query lies inside
    the grid; inside=False leaves the wall alone: the query is then two cells outside the grid bounds.
    Returns (target, query (1, 3), the wall's centroid, w, q)."""
    w, q = escape_pairs(leaf, direction)[case]
    o = [a for a in range(3) if a != axis]
    k = int(R.build_ref(np.array([w]), leaf)[0])
    centre_cells = (3, -2)
    centre = [F32((c + 0.5) * float(F32(leaf))) for c in centre_cells]
    tgt = [wall(axis, w, centre, leaf)]
    if inside:
        rng = np.random.default_rng(seed)
        cells = []
        for a in range(k - 5, k + 6):
            c = [0, 0, 0]
            c[axis], c[o[0]], c[o[1]] = a, centre_cells[0] + 6, centre_cells[1]
            cells.append(c)
        tgt.append(R.cell_points(cells, float(F32(leaf)), 10, rng).astype(F32))
    query = np.zeros((1, 3), dtype=F32)
    query[0, axis], query[0, o[0]], query[0, o[1]] = q, centre[0], centre[1]
    cen = np.zeros(3, dtype=F32)
    cen[axis], cen[o[0]], cen[o[1]] = w, centre[0], centre[1]
    return np.concatenate(tgt).astype(F32), query, cen, w, q


def equality_queries(res, centroid, axis=0):
    """Queries displaced from `centroid` along `axis` whose f32 d2 is r^2 exactly and the nearest attainable values below
    and above it: [(query (3,), d2)], d2 ascending."""
    r2 = radius2(res)
    c = np.asarray(centroid, dtype=F32)
    cand = _floats_near(F32(c[axis]) + F32(res), ulps=64)
    qs = np.repeat(c[None, :], len(cand), axis=0)
    qs[:, axis] = cand
    d2 = f32_d2(qs, c[None, :])
    below = d2 < r2
    eq = d2 == r2
    above = d2 > r2
    out = []
    if below.any():
        i = np.nonzero(below)[0][np.argmax(d2[below])]
        out.append((qs[i], d2[i]))
    if eq.any():
        i = np.nonzero(eq)[0][0]
        out.append((qs[i], d2[i]))
    if above.any():
        i = np.nonzero(above)[0][np.argmin(d2[above])]
        out.append((qs[i], d2[i]))
    return out


def huge_rows(points, values=(1e30, -1e30, 3e38, -3e38)):
    """The cloud with rows at each huge value on each axis (the other coordinates from the first rows); returns
    (cloud, ordinary-row mask)."""
    p = np.asarray(points, dtype=F32)
    extra = []
    for a in range(3):
        for i, v in enumerate(values):
            r = p[i % len(p)].copy()
            r[a] = F32(v)
            extra.append(r)
    extra = np.array(extra, dtype=F32)
    half = len(p) // 2
    out = np.concatenate([extra[:6], p[:half], extra[6:], p[half:]])
    ok = np.concatenate([np.zeros(6, bool), np.ones(half, bool), np.zeros(len(extra) - 6, bool), np.ones(len(p) - half, bool)])
    return out, ok
