"""A float64 reference of one NDT derivative pass (computeDerivatives / updateDerivatives of pclomp), written from the
algorithm and vectorised in numpy, with a per-entry bound on how far the f32 evaluation of the solver (K1) or of the
oracle may be from it. Nothing here needs a GPU.

What is computed
  The voxels come from the caller (the handle's own voxels(): leaf index, mean, icov, centroid) and the grid geometry from
  gridref.leaf_geometry, so the voxel map builder (K3) stays out of the comparison.
  * transformed point: the solver's f32 transform, ((T0 x + T1 y) + T2 z) + T3 un-fused. The reference transforms in float
    too (pcl::transformPointCloud), so this is ground truth, not an approximation; cells and hits follow from it exactly.
  * neighbourhood: the cell floor(f32(x) / f32(leaf)) (gridref.lookup_ref), then DIRECT7: centre plus the six face
    neighbours, DIRECT1: centre, DIRECT26: the 26 cells around the centre without it; every neighbour is tested against
    the grid bounds per axis. KDTREE has no cells: every voxel whose centroid's un-fused f32 squared distance is below
    f32(res^2) (radiusref.neighbours). It is not confined to the 27 cells around the lookup cell: the builder's cell
    floor(x * inv_leaf) and the lookup's floor(x / leaf) disagree near a face, so a hit can lie two lookup cells away.
  * each pair in float64: x' = f64(x_t) - mean, C = f64(f32(icov)), s = C x', q = x'^T s, ex = exp(-d2 q / 2),
    e2 = d2 ex, score increment -d1 ex, the pair dropped (score included) when e2 > 1, e2 < 0 or NaN, e = d1 e2;
    gradient e s^T J_k, Hessian e (-d2 (s^T J_i)(s^T J_j) + s^T H_ij + J_i^T C J_j). d1 is float64, d2 the float32 value
    the f32 path uses. J and H_ij are formed from the float32 angle tables (the values the live path multiplies with,
    d1.z = +sy and the 1e-4 snap); minus_sy=True switches d1.z to -sy (the f64 convention), to show a test can see it.

The bound
  Let u = 2^-24. Per pair p and entry k, a_pk is the contribution with every factor replaced by its absolute value (|s| by
  |C| |x'|, J and H_ij by |table| . |x|, C by |C|, W = M - d2 Q by |M| + d2 |Q|): the largest value any rounding of the
  terms inside the entry can scale. The accepted deviation of entry k is

      tol_k = u * sum_p (gamma + sigma_p) a_pk                            (= gamma u B_k, B_k = sum_p (1 + sigma_p / gamma) a_pk)

  sigma_p, the sensitivity of the pair's inputs, in units of u:
    * x': the kernel forms (x_t - mean_hi) - mean_lo in f32. It is within 1 ulp of f32(f64(x_t) - mean) (not always
      equal), so within 1.5 ulp <= 3u |x'_i| of x'. Through s = C x' (and its own f32 rounding, 3 terms) |ds_i| <= 6u (|C||x'|)_i;
      the product of two s-factors in the Hessian doubles that: 12.
    * q: 2 x'^T C dx' + x'^T ds + the rounding of the f32 dot give |dq| <= 12u A_p, A_p = sum |x'_i C_ij x'_j|; ex moves by
      d2/2 |dq| relative: 6 d2 A_p.
    * expf (2 ulp), the rounding of its argument (|d2 q / 2| u, relative to ex) and the f32 products e2 = d2 ex, e = e2 d1
      with d1 rounded to float: 8 + 2 |d2 q / 2|.
    * the angle tables: the f32 table values are the definition of the live path (both sides multiply with them), so they
      add nothing beyond the f32 products J x and H_ij x, which are counted in gamma.
  gamma, the depth of the f32 sums an entry passes through: the pairs of a point (DIRECT7 7, DIRECT1 1, DIRECT26 26,
  KDTREE 27 or the most any point of the scan has), the per-point J / H_E products (j = table . x, three terms, W = M - d2 Q, W J, J^T W J, s^T H_ij: 10), the
  points one thread accumulates (one per 768 staged points, more than one above the staging capacity), and the 4-term
  f32 pre-sum of the warp reduction (2). Everything after that is float64, fixed order, and a few 2^-53 at most.
  The oracle (one f32 contribution per pair, summed in float64) stays inside the same bound: its per-pair product depth
  (about 12) is below gamma.
  Score: tol = u * sum_p (n_pairs + 4 + sigma_p) |d1 ex|. Hits are exact.
  near_threshold counts pairs whose discard test or KDTREE radius test sits within a few ulp of flipping; an exact-hit
  assertion is only valid where it is zero.
"""
from __future__ import annotations

import math

import numpy as np

import gridref as R

F32 = np.float32
U32 = 2.0**-24
KDTREE, DIRECT26, DIRECT7, DIRECT1 = 0, 1, 2, 3
MAX_PAIRS = {KDTREE: 27, DIRECT26: 26, DIRECT7: 7, DIRECT1: 1}
SMEM_POINTS = 768  # source points an evaluator CTA stages in shared memory
SOLVER_THREADS = 768
CTL_CTAS = 3  # SMs kept for controller CTAs in every solver launch (NDT_MAX_SLOTS)
JH_DEPTH = 10
PRESUM_DEPTH = 2
TRI = [(i, j) for i in range(6) for j in range(i, 6)]  # the 21 upper-triangular entries, row-major


def gauss_constants(outlier_ratio, resolution):
    """(d1, d2) of ndt_omp_impl.hpp:88-93 with the resolution as float."""
    res = float(F32(resolution))
    c1 = 10 * (1 - outlier_ratio)
    c2 = outlier_ratio / res**3
    d3 = -math.log(c2)
    d1 = -math.log(c1 + c2) - d3
    d2 = -2 * math.log((-math.log(c1 * math.exp(-0.5) + c2) - d3) / d1)
    return d1, d2


def angle_tables(p6, minus_sy=False, f64=False):
    """computeAngleDerivatives (ndt_omp_impl.hpp:287-393): the float32 tables (8 x 3 for J's angular columns a..h,
    15 x 3 for the second derivatives a2 a3 b2 b3 c2 c3 d1 d2 d3 e1 e2 e3 f1 f2 f3), angles below 1e-4 snapped to
    (cos, sin) = (1, 0). The live f32 table keeps +sy in d1.z; minus_sy gives the f64 convention. f64=True also returns
    the float64 values before the cast (J64, H64), the values the K2 pass reads and that decide float32 rounding."""
    def cs(a):
        return (1.0, 0.0) if abs(a) < 10e-5 else (math.cos(a), math.sin(a))

    (cx, sx), (cy, sy), (cz, sz) = cs(p6[3]), cs(p6[4]), cs(p6[5])
    J = [[-sx * sz + cx * sy * cz, -sx * cz - cx * sy * sz, -cx * cy],
         [cx * sz + sx * sy * cz, cx * cz - sx * sy * sz, -sx * cy],
         [-sy * cz, sy * sz, cy],
         [sx * cy * cz, -sx * cy * sz, sx * sy],
         [-cx * cy * cz, cx * cy * sz, -cx * sy],
         [-cy * sz, -cy * cz, 0.0],
         [cx * cz - sx * sy * sz, -cx * sz - sx * sy * cz, 0.0],
         [sx * cz + cx * sy * sz, cx * sy * cz - sx * sz, 0.0]]
    H = [[-cx * sz - sx * sy * cz, -cx * cz + sx * sy * sz, sx * cy],
         [-sx * sz + cx * sy * cz, -cx * sy * sz - sx * cz, -cx * cy],
         [cx * cy * cz, -cx * cy * sz, cx * sy],
         [sx * cy * cz, -sx * cy * sz, sx * sy],
         [-sx * cz - cx * sy * sz, sx * sz - cx * sy * cz, 0.0],
         [cx * cz - sx * sy * sz, -sx * sy * cz - cx * sz, 0.0],
         [-cy * cz, cy * sz, -sy if minus_sy else sy],
         [-sx * sy * cz, sx * sy * sz, sx * cy],
         [cx * sy * cz, -cx * sy * sz, -cx * cy],
         [sy * sz, sy * cz, 0.0],
         [-sx * cy * sz, -sx * cy * cz, 0.0],
         [cx * cy * sz, cx * cy * cz, 0.0],
         [-cy * cz, cy * sz, 0.0],
         [-cx * sz - sx * sy * cz, -cx * cz + sx * sy * sz, 0.0],
         [-sx * sz + cx * sy * cz, -cx * sy * sz - sx * cz, 0.0]]
    if f64:
        return np.array(J, dtype=F32), np.array(H, dtype=F32), np.array(J), np.array(H)
    return np.array(J, dtype=F32), np.array(H, dtype=F32)


def transform_points(T, src):
    """The solver's f32 transform, ((T0 x + T1 y) + T2 z) + T3, un-fused (numpy float32 arithmetic does not contract)."""
    T = np.asarray(T, dtype=F32)
    p = np.asarray(src, dtype=F32)[:, :3]
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def split_mean(mean):
    """The voxel record's float-float mean: hi = f32(mean), lo = f32(mean - hi)."""
    m = np.asarray(mean, dtype=np.float64)
    hi = m.astype(F32)
    return hi, (m - hi.astype(np.float64)).astype(F32)


def kernel_xprime(xt, mean):
    """x' as the kernel forms it: (x_t - mean_hi) - mean_lo in f32."""
    hi, lo = split_mean(mean)
    return (np.asarray(xt, dtype=F32) - hi) - lo


def offsets(method):
    if method in (DIRECT7, DIRECT1):
        o = [(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
        return o[:1] if method == DIRECT1 else o
    o = [(x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]
    return [d for d in o if d != (0, 0, 0)] if method == DIRECT26 else o


def points_per_thread(n_src, n_sms):
    """Most points one solver thread accumulates in f32 for a scan of n_src points on a GPU with n_sms SMs (rows_for):
    32-point units dealt round-robin over min(ceil(n / 128), SMs - 3) evaluator CTAs of 768 threads."""
    n_eval = max(1, n_sms - CTL_CTAS)
    rows = max(1, min((n_src + 127) // 128, n_eval))
    units = (n_src + 31) // 32
    return max(1, -(-(-(-units // rows) * 32) // SOLVER_THREADS))


def _pairs(xt, g, res, method, vidx, centroid):
    """(point, voxel) candidate pairs of the neighbourhood rule; near: pairs within 4 ulp of the KDTREE radius."""
    if method == KDTREE:  # every centroid, no cells (radiusref.neighbours)
        import radiusref

        return radiusref.neighbours(xt, res, dict(idx=vidx, centroid=centroid))
    ijk = np.stack([R.lookup_ref(xt[:, a], res) for a in range(3)], axis=1) - g["min_b"]
    P, V = [], []
    for o in offsets(method):
        c = ijk + np.array(o)
        inside = ((c >= 0) & (c < g["div_b"])).all(axis=1)
        pi = np.nonzero(inside)[0]
        lin = c[pi, 0] + c[pi, 1] * g["mul"][1] + c[pi, 2] * g["mul"][2]
        k = np.minimum(np.searchsorted(vidx, lin), len(vidx) - 1)
        hit = vidx[k] == lin
        P.append(pi[hit])
        V.append(k[hit])
    return np.concatenate(P), np.concatenate(V), 0


def derivatives(src, T, p6, res, voxels, geom, method=DIRECT7, outlier_ratio=0.55, compute_hessian=True,
                minus_sy=False, n_sms=132, chunk=16384):
    """One derivative pass in float64. Returns a dict: score, g (6,), H (6, 6), hits, near_threshold, and the bounds
    tol_score, tol_g (6,), tol_H (6, 6) (zero where compute_hessian is False: H is then all zero)."""
    src = np.asarray(src, dtype=F32)[:, :3]
    d1, d2 = gauss_constants(outlier_ratio, res)
    d2 = float(F32(d2))
    jt, ht = angle_tables(p6, minus_sy)
    jt64, ht64 = jt.astype(np.float64), ht.astype(np.float64)
    vidx = np.asarray(voxels["idx"], dtype=np.int64)
    mean = np.asarray(voxels["mean"], dtype=np.float64)
    C_all = np.asarray(voxels["icov"], dtype=np.float64).astype(F32).astype(np.float64)
    cen = np.asarray(voxels["centroid"], dtype=F32)
    max_pairs = MAX_PAIRS[method]
    if method == KDTREE and len(vidx):  # a radius neighbourhood can exceed 27 voxels (it spans up to 4 cells per axis)
        for lo in range(0, len(src), chunk):
            pi = _pairs(transform_points(T, src[lo:lo + chunk]), geom, res, method, vidx, cen)[0]
            max_pairs = max(max_pairs, int(np.bincount(pi).max()) if len(pi) else 0)
    gamma = max_pairs + JH_DEPTH + points_per_thread(len(src), n_sms) + PRESUM_DEPTH
    out = dict(score=0.0, g=np.zeros(6), H=np.zeros((6, 6)), hits=0, near_threshold=0, tol_score=0.0,
               tol_g=np.zeros(6), tol_H=np.zeros((6, 6)))
    if len(vidx) == 0:
        return out
    for lo in range(0, len(src), chunk):
        x32 = src[lo:lo + chunk]
        xt = transform_points(T, x32)
        pi, vi, near = _pairs(xt, geom, res, method, vidx, cen)
        out["near_threshold"] += near
        if len(pi) == 0:
            continue
        xp = xt[pi].astype(np.float64) - mean[vi]
        C = C_all[vi]
        Ca = np.abs(C)
        s = np.einsum("pij,pj->pi", C, xp)
        q = np.einsum("pi,pi->p", xp, s)
        ex = np.exp(-d2 * q / 2)
        e2 = d2 * ex
        with np.errstate(invalid="ignore"):
            ok = ~((e2 > 1) | (e2 < 0) | np.isnan(e2))
        out["near_threshold"] += int((np.abs(e2 - 1) <= 64 * U32).sum())
        pi, vi, xp, C, Ca, s, q, ex = pi[ok], vi[ok], xp[ok], C[ok], Ca[ok], s[ok], q[ok], ex[ok]
        e = d1 * d2 * ex
        out["hits"] += len(pi)
        # sensitivity of each pair (units of u)
        sabs = np.einsum("pij,pj->pi", Ca, np.abs(xp))
        A = np.einsum("pi,pi->p", np.abs(xp), sabs)
        sig_e = 6 * d2 * A + 2 * np.abs(d2 * q / 2) + 8
        sigma = sig_e + 12
        n_pairs = np.bincount(pi, minlength=len(x32))[pi]
        out["score"] += float((-d1 * ex).sum())
        out["tol_score"] += U32 * float(((n_pairs + 4 + sig_e) * np.abs(d1 * ex)).sum())
        # point Jacobian: J (P, 3, 6) with columns 3..5 from the f32 table times the source point
        x = x32[pi].astype(np.float64)
        xa = np.abs(x)
        jv, jva = x @ jt64.T, xa @ np.abs(jt64).T  # (P, 8)
        J = np.zeros((len(pi), 3, 6))
        Ja = np.zeros((len(pi), 3, 6))
        J[:, 0, 0] = J[:, 1, 1] = J[:, 2, 2] = 1.0
        Ja[:, 0, 0] = Ja[:, 1, 1] = Ja[:, 2, 2] = 1.0
        for M, v in ((J, jv), (Ja, jva)):
            M[:, 1, 3], M[:, 2, 3] = v[:, 0], v[:, 1]
            M[:, :, 4] = v[:, 2:5]
            M[:, :, 5] = v[:, 5:8]
        sJ = np.einsum("pi,pik->pk", s, J)
        sJa = np.einsum("pi,pik->pk", sabs, Ja)
        w = (gamma + sigma) * U32
        out["g"] += np.einsum("p,pk->k", e, sJ)
        out["tol_g"] += np.einsum("p,pk->k", w * np.abs(e), sJa)
        if not compute_hessian:
            continue
        hv, hva = x @ ht64.T, xa @ np.abs(ht64).T  # (P, 15)
        Hv = np.zeros((len(pi), 6, 6, 3))
        Hva = np.zeros((len(pi), 6, 6, 3))
        for M, v in ((Hv, hv), (Hva, hva)):
            a = np.stack([np.zeros(len(pi)), v[:, 0], v[:, 1]], axis=1)
            b = np.stack([np.zeros(len(pi)), v[:, 2], v[:, 3]], axis=1)
            c = np.stack([np.zeros(len(pi)), v[:, 4], v[:, 5]], axis=1)
            dd, ee, ff = v[:, 6:9], v[:, 9:12], v[:, 12:15]
            for (i, j), vec in (((3, 3), a), ((3, 4), b), ((3, 5), c), ((4, 4), dd), ((4, 5), ee), ((5, 5), ff)):
                M[:, i, j] = M[:, j, i] = vec
        CJ = np.einsum("pij,pjk->pik", C, J)
        CJa = np.einsum("pij,pjk->pik", Ca, Ja)
        h = -d2 * sJ[:, :, None] * sJ[:, None, :] + np.einsum("pc,pijc->pij", s, Hv) + np.einsum("pci,pcj->pij", J, CJ)
        ha = d2 * sJa[:, :, None] * sJa[:, None, :] + np.einsum("pc,pijc->pij", sabs, Hva) + np.einsum("pci,pcj->pij", Ja, CJa)
        out["H"] += np.einsum("p,pij->ij", e, h)
        out["tol_H"] += np.einsum("p,pij->ij", w * np.abs(e), ha)
    return out


def within(gpu, ref, scale=1.0):
    """Largest |gpu - ref| / (scale * tol) over score, g and the 21 upper H entries, plus the per-entry ratios.
    gpu: (score, g, H) as derivatives() returns them."""
    s, g, H = gpu
    if s == ref["score"]:
        r = {"score": 0.0}
    else:
        r = {"score": abs(s - ref["score"]) / (scale * ref["tol_score"]) if ref["tol_score"] else np.inf}
    with np.errstate(divide="ignore", invalid="ignore"):
        rg = np.abs(np.asarray(g) - ref["g"]) / (scale * ref["tol_g"])
        rg[(np.asarray(g) == ref["g"])] = 0.0
        rh = np.array([abs(H[i, j] - ref["H"][i, j]) / (scale * ref["tol_H"][i, j]) if H[i, j] != ref["H"][i, j] else 0.0
                       for i, j in TRI])
    r["g"], r["H"] = rg, rh
    r["max"] = max(r["score"], float(rg.max()), float(rh.max()) if len(rh) else 0.0)
    return r


# ---- fixtures where the evaluation goes wrong -----------------------------------------------------------------------
SHIFT = (3000.0, -2000.0, 50.0)


def snap_poses(base=(0.21, -0.13, 0.04, 0.006, -0.004, 0.02)):
    """Each angle at +-1e-4 and one float64 ulp either side of it: the angle tables snap (cos, sin) to (1, 0) below 1e-4
    (ndt_omp_impl.hpp:292-325). Returns [(axis, angle, snapped)]."""
    out = []
    for axis in (3, 4, 5):
        for sign in (1.0, -1.0):
            edge = sign * 10e-5
            for a, snapped in ((edge, False), (np.nextafter(edge, 0.0), True), (np.nextafter(edge, 2 * edge), False)):
                p = np.array(base, dtype=np.float64)
                p[axis] = a
                out.append((p, axis, snapped))
    return out


def pitch_poses():
    return [np.array([0.1, 0.2, 0.0, 0.05, b, -0.1]) for b in (0.6, -0.6, 1.2, -1.2)]


def illconditioned_pair(res=2.0, seed=0):
    """A target of degenerate leaves (identical, collinear, coplanar points: icov with eigenvalues raised to 1 / 0.01 of
    the largest) and of 5/6/7-point leaves (only >= 6 become voxels), and a source of points near all of them."""
    rng = np.random.default_rng(seed)
    deg = R.degenerate_leaves(res, n=200, seed=seed)
    pop, _ = R.population_leaves(res, seed=seed)
    pop = R.shifted(pop, (0.0, 2 * res, 0.0))
    tgt = np.concatenate([deg, pop]).astype(F32)
    src = (tgt[rng.integers(0, len(tgt), 3000)] + rng.normal(0, 0.15 * res, (3000, 3))).astype(F32)
    return src, tgt


def shifted_pair(src, tgt, offset=SHIFT):
    """The target moved by `offset` (km scale: x_t - mean loses the low bits of both), the source left in the sensor
    frame; a pose p maps to p + offset in translation."""
    return src, R.shifted(tgt, offset)


def ladder_sizes(n_sms):
    """Scan sizes at the partition and staging edges of a GPU with n_sms SMs: ragged units, one and two units per CTA, the
    last size that spreads over fewer than all evaluators, and the shared-memory staging capacity."""
    n_eval = n_sms - CTL_CTAS
    cap = SMEM_POINTS * n_eval
    return [1, 31, 32, 33, 127, 128, 129, 128 * n_eval, 128 * n_eval + 1, cap - 1, cap, cap + 1, cap + 32, cap + 33]


def point_owner(n_src, n_sms):
    """(evaluator CTA, thread) that evaluates each point of a scan (units of 32 dealt round-robin over rows_for CTAs,
    local slot j evaluated by thread j mod 768)."""
    n_eval = max(1, n_sms - CTL_CTAS)
    rows = max(1, min((n_src + 127) // 128, n_eval))
    gi = np.arange(n_src)
    unit = gi // 32
    rank = unit % rows
    local = (unit // rows) * 32 + gi % 32
    return rank, local % SOLVER_THREADS, rows


def per_point_hits(src, T, res, voxels, geom, method=DIRECT7):
    """Number of (point, voxel) candidate pairs of each point (before the e2 gate)."""
    xt = transform_points(T, src)
    pi, _, _ = _pairs(xt, geom, res, method, np.asarray(voxels["idx"], np.int64), np.asarray(voxels["centroid"], F32))
    return np.bincount(pi, minlength=len(src))
