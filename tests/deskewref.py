"""A replay of the IMU de-skew (K9, csrc/deskew.cu) written from LidarUndistortion::adjustDistortion
(lidar_undistortion.hpp:110-226), point by point, with a float64 reference of the same formula and a bound per point.
Nothing here needs a GPU.

What is computed
  * The discrete decisions, exactly: ori = -(float)atan2((double)y, (double)x); formula A before the half turn and B
    after it, with the reference's float / double promotions; k_first, the first index whose formula-A azimuth is more
    than pi past the start (it still uses formula A itself); rel_time = (float)((double)((ori_h - start) / ori_diff)
    * scan_period) and t = scan_time + (double)rel_time; the ring index the reference's walk stops at, the skip flag
    (`continue`) and the final imu_ptr_front_ / imu_ptr_last_iter_.
    - `walk_literal` is the truth: the loop of :151-158 and the carry of :223.
    - `walk_parallel` is the kernel's form: a lower bound per point (first window position whose stamp is not <= t under
      the walk's own test `t < stamp`, clamped to the newest sample), the exclusive prefix max over the non-skipped
      points, and the Jacobi fix point of the skipped set from "nothing skipped". It returns the number of passes, which
      the kernel runs too. It is exact only while the window's stamps never decrease.
  * `replay` (out): the kernel's arithmetic, one float32 operation at a time (numpy elementwise, never a matrix product):
    rf = (float)((t - t_b) / (t_f - t_b)), rb = (float)(1.0 - rf), mix = vf rf + vb rb; half angles h = 0.5f ang with
    sin / cos evaluated in double and rounded; Eigen's quaternion products and toRotationMatrix; the rows of R p as
    (r0 x + r1 y) + r2 z; shift_from_start = (shift - shift0) - velo0 rel; r_s_i as the transpose of the first point's R.
    The kernel evaluates atan2 / sin / cos in double with CUDA's libdevice (<= 2 ulp) and rounds to float; numpy's
    double functions are within 1 ulp. The two can round to different floats only when the double value lies within
    a few double ulps of a float rounding midpoint: `ambiguous` flags every point with such a value (4 double ulps).
    The scenes of the tests contain none, so the kernel must equal this replay bit for bit.
  * `replay` (ref64, bound): the same formula in float64 at the same decisions, rel_time and t, with exact sin / cos and a general
    3x3 inverse for r_s_i.

The bound (|float32 result - float64 reference| per point and coordinate)
  Running error analysis over the float32 replay: every value v carries e >= |v - exact|, where "exact" is the formula
  evaluated in real arithmetic on the same inputs (the ring entries, p, rel_time and t are shared exactly).
    rounding to float of an exact a:  |fl(a) - a| <= u |fl(a)| + 2^-150 with u = 2^-24 / (1 - 2^-24)
    add / sub:  e = e_a + e_b + round(v)
    mul:        e = |a| e_b + |b| e_a + e_a e_b + round(v)
    rf:         one double division (2^-53 relative) then the float rounding; rb = 1 - rf adds e_rf, 2^-53 and a rounding
    sin / cos:  Lipschitz 1 in the angle: e = e_h + 4 * 2^-53 |v| + round(v); h = 0.5f ang: e_h = 0.5 e_ang + round(h)
  The chain is the kernel's: 2 mul + 1 add per interpolated entry; 2 sin/cos per axis; 2 quaternion products of 4 mul
  and 3 add/sub per component; toRotationMatrix (3 doublings, 9 products, 12 add/sub); R p (3 mul, 2 add); sfs (2 sub,
  1 mul); v = R p + sfs; r_s_i v (3 mul, 2 add). r_s_i is the transpose of the first point's float R, whose entries carry
  their own e; the float64 reference inverts its exact R0, which differs from the transpose by < 16 * 2^-53. The float64
  reference's own error is below 2^-40 (|out| + 1), added to the bound.
"""
from __future__ import annotations

import math

import numpy as np

F = np.float32
QUE = 200
PI = math.pi
U = 2.0**-24 / (1 - 2.0**-24)
ETA = 2.0**-150
UD = 2.0**-53


# ---- rounding helpers ------------------------------------------------------------------------------------------------
def near_float_midpoint(x, ulps: int = 4) -> np.ndarray:
    """True where the float64 value x lies within `ulps` double ulps of a float32 rounding midpoint: there a library
    whose double result is a few ulps off could round to the other float."""
    x = np.asarray(x, dtype=np.float64)
    out = np.zeros(x.shape, dtype=bool)
    fin = np.isfinite(x)
    xf = x[fin]
    f = xf.astype(F)
    tol = ulps * np.spacing(np.abs(xf))
    hit = np.zeros(xf.shape, dtype=bool)
    for d in (np.inf, -np.inf):
        nb = np.nextafter(f, F(d))
        mid = (f.astype(np.float64) + nb.astype(np.float64)) * 0.5
        hit |= np.abs(xf - mid) <= tol
    out[fin] = hit
    return out


def neg_atan2(y, x):
    """-(float)atan2((double)y, (double)x) and whether its rounding is ambiguous."""
    a = np.arctan2(np.asarray(y, dtype=F).astype(np.float64), np.asarray(x, dtype=F).astype(np.float64))
    return -(a.astype(F)), near_float_midpoint(a)


# ---- the ring --------------------------------------------------------------------------------------------------------
class Ring:
    """The LidarUndistortion members adjustDistortion reads (and the two pointers it writes)."""

    def __init__(self, time, rpy, shift, velo, ptr_front, ptr_last, ptr_last_iter, scan_period):
        self.time = np.array(time, dtype=np.float64)
        self.rpy = np.array(rpy, dtype=F).reshape(QUE, 3)
        self.shift = np.array(shift, dtype=F).reshape(QUE, 3)
        self.velo = np.array(velo, dtype=F).reshape(QUE, 3)
        self.ptr_front, self.ptr_last, self.ptr_last_iter = int(ptr_front), int(ptr_last), int(ptr_last_iter)
        self.scan_period = float(scan_period)

    @classmethod
    def from_oracle(cls, o):
        rpy = np.stack([o.roll, o.pitch, o.yaw], axis=1)
        return cls(o.time, rpy, o.shift, o.velo, o.ptr_front, o.ptr_last, o.ptr_last_iter, o.scan_period)

    @classmethod
    def from_device(cls, g, scan_period):
        """From scanmatcher.LidarUndistortion: pointers() and sample(k)."""
        time, rpy, sh, ve = np.zeros(QUE), np.zeros((QUE, 3), F), np.zeros((QUE, 3), F), np.zeros((QUE, 3), F)
        for k in range(QUE):
            time[k], rpy[k], sh[k], ve[k] = g.sample(k)
        pf, pl, pi = g.pointers()
        return cls(time, rpy, sh, ve, pf, pl, pi, scan_period)

    def window(self):
        """(base, span, stamps of positions 0..span): the ring indices the walk can visit, in its order."""
        base = self.ptr_last_iter
        span = (self.ptr_last - base) % QUE
        return base, span, self.time[(base + np.arange(span + 1)) % QUE]


# ---- decisions -------------------------------------------------------------------------------------------------------
def orientation_range(cloud):
    """start_ori, end_ori, ori_diff of :115-123 (host arithmetic of adjust_distortion)."""
    c = np.asarray(cloud, dtype=F)
    s, _ = neg_atan2(c[0, 1], c[0, 0])
    e, _ = neg_atan2(c[-1, 1], c[-1, 0])
    s, e = F(s), F(e)
    if float(F(e - s)) > 3 * PI:
        e = F(float(e) - 2 * PI)
    elif float(F(e - s)) < PI:
        e = F(float(e) + 2 * PI)
    return s, e, F(e - s)


def times_of(cloud, scan_time: float, scan_period: float):
    """Per point: ori, formula-A azimuth, k_first, ori_h, rel_time (float32), t (float64), atan2 ambiguity."""
    c = np.asarray(cloud, dtype=F)
    n = len(c)
    so, eo, od = orientation_range(c)
    ori, amb = neg_atan2(c[:, 1], c[:, 0])
    sod, eod = float(so), float(eo)
    a = ori.copy()
    lo = a.astype(np.float64) < sod - PI * 0.5
    hi = ~lo & (a.astype(np.float64) > sod + PI * 1.5)
    a[lo] = (a[lo].astype(np.float64) + 2 * PI).astype(F)
    a[hi] = (a[hi].astype(np.float64) - 2 * PI).astype(F)
    fires = (a - so).astype(F).astype(np.float64) > PI
    k_first = int(np.argmax(fires)) if fires.any() else n
    b = (ori.astype(np.float64) + 2 * PI).astype(F)
    lo = b.astype(np.float64) < eod - 1.5 * PI
    hi = ~lo & (b.astype(np.float64) > eod + 0.5 * PI)
    b[lo] = (b[lo].astype(np.float64) + 2 * PI).astype(F)
    b[hi] = (b[hi].astype(np.float64) - 2 * PI).astype(F)
    ori_h = np.where(np.arange(n) <= k_first, a, b).astype(F)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        q = ((ori_h - so).astype(F) / od).astype(F)
        rel = (q.astype(np.float64) * scan_period).astype(F)
    t = scan_time + rel.astype(np.float64)
    return {"start_ori": so, "end_ori": eo, "ori_diff": od, "ori": ori, "a": a, "k_first": k_first, "ori_h": ori_h,
            "rel": rel, "t": t, "ambiguous": amb}


def walk_literal(ring: Ring, t):
    """:151-158 and :223 literally. Returns ring-index front per point, skip flags, final (ptr_front, ptr_last_iter)."""
    n = len(t)
    front = np.zeros(n, dtype=np.int64)
    skip = np.zeros(n, dtype=bool)
    pf, pli = ring.ptr_front, ring.ptr_last_iter
    if ring.ptr_last <= 0:
        return None, None, (pf, pf if n else pli)
    time, last, sp = ring.time.tolist(), ring.ptr_last, ring.scan_period
    for i, ti in enumerate(t.tolist()):
        f = pli
        while f != last:
            if ti < time[f]:
                break
            f = (f + 1) % QUE
        pf = f
        front[i] = f
        if abs(ti - time[f]) > sp:
            skip[i] = True
            continue
        pli = pf
    return front, skip, (pf, pli)


def walk_parallel(ring: Ring, t):
    """The kernel's form: lower bounds, exclusive prefix max over the non-skipped points, Jacobi from nothing skipped.
    Returns (front ring index, skip, (ptr_front, ptr_last_iter), passes, lower bound positions)."""
    n = len(t)
    base, span, times = ring.window()
    lb = np.minimum(np.searchsorted(times, t, side="right"), span)  # NaN sorts last: `t < stamp` is false for all
    skipped = np.zeros(n, dtype=bool)
    rounds = 0
    for _ in range(n + 1):
        rounds += 1
        contrib = np.where(skipped, -1, lb)
        carried = np.maximum.accumulate(np.concatenate([[0], contrib[:-1]]))
        pos = np.maximum(carried, lb)
        with np.errstate(invalid="ignore"):
            new = np.abs(t - times[pos]) > ring.scan_period
        if np.array_equal(new, skipped):
            break
        skipped = new
    front = (base + pos) % QUE
    ok = np.flatnonzero(~skipped)
    pli = int(front[ok[-1]]) if len(ok) else ring.ptr_last_iter
    return front, skipped, (int(front[-1]), pli), rounds, lb


def window_monotone(ring: Ring) -> bool:
    _, _, times = ring.window()
    return bool(np.all(times[1:] >= times[:-1]))


# ---- tracked float32 arithmetic --------------------------------------------------------------------------------------
class E:
    """A float32 array with a bound e >= |v - exact| per entry."""

    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, dtype=F)
        self.e = np.zeros(self.v.shape) if e is None else np.asarray(e, dtype=np.float64)

    @staticmethod
    def _r(v):
        return U * np.abs(v.astype(np.float64)) + ETA

    def __add__(self, o):
        v = (self.v + o.v).astype(F)
        return E(v, self.e + o.e + E._r(v))

    def __sub__(self, o):
        v = (self.v - o.v).astype(F)
        return E(v, self.e + o.e + E._r(v))

    def __mul__(self, o):
        v = (self.v * o.v).astype(F)
        a, b = np.abs(self.v.astype(np.float64)), np.abs(o.v.astype(np.float64))
        return E(v, a * o.e + b * self.e + self.e * o.e + E._r(v))


def _const(c, shape):
    return E(np.full(shape, c, dtype=F))


def _half_sincos(ang: E, amb):
    h = _const(0.5, ang.v.shape) * ang
    hd = h.v.astype(np.float64)
    out = []
    for fn in (np.sin, np.cos):
        d = fn(hd)
        amb |= near_float_midpoint(d)
        v = d.astype(F)
        out.append(E(v, h.e + 4 * UD * np.abs(d) + E._r(v)))
    return out


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [((aw * bx) + (ax * bw)) + (ay * bz) - (az * by),
            ((aw * by) + (ay * bw)) + (az * bx) - (ax * bz),
            ((aw * bz) + (az * bw)) + (ax * by) - (ay * bx),
            ((aw * bw) - (ax * bx)) - (ay * by) - (az * bz)]


def rot_zyx_f32(roll: E, pitch: E, yaw: E, amb):
    """(AngleAxisf(yaw, Z) * AngleAxisf(pitch, Y) * AngleAxisf(roll, X)).toRotationMatrix(), row-major list of 9 E."""
    shape = roll.v.shape
    z = _const(0.0, shape)
    sz, cz = _half_sincos(yaw, amb)
    sy, cy = _half_sincos(pitch, amb)
    sx, cx = _half_sincos(roll, amb)
    q = _qmul(_qmul([z, z, sz, cz], [z, sy, z, cy]), [sx, z, z, cx])
    x, y, zz, w = q
    two, one = _const(2.0, shape), _const(1.0, shape)
    tx, ty, tz = two * x, two * y, two * zz
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * zz
    return [one - (tyy + tzz), txy - twz, txz + twy,
            txy + twz, one - (txx + tzz), tyz - twx,
            txz - twy, tyz + twx, one - (txx + tyy)]


def _interp_f32(ring: Ring, front, t):
    """rpy / shift / velo at t with the pointer at `front` (:169-197), as E arrays of shape (m,) each."""
    f = front
    b = (front - 1 + QUE) % QUE
    tf, tb = ring.time[f], ring.time[b]
    past = t > tf
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        rd = (t - tb) / (tf - tb)
        rf = rd.astype(F)
        rb = (1.0 - rf.astype(np.float64)).astype(F)
    e_rf = UD * np.abs(rd) + E._r(rf)
    e_rb = e_rf + UD + E._r(rb)
    RF, RB = E(rf, e_rf), E(rb, e_rb)
    out = []
    for arr in (ring.rpy, ring.shift, ring.velo):
        comps = []
        for c in range(3):
            vf, vb = E(arr[f, c]), E(arr[b, c])
            m = (vf * RF) + (vb * RB)
            v = np.where(past, arr[f, c], m.v).astype(F)
            e = np.where(past, 0.0, m.e)
            comps.append(E(v, e))
        out.append(comps)
    return out


def _interp_f64(ring: Ring, front, t):
    f = front
    b = (front - 1 + QUE) % QUE
    tf, tb = ring.time[f], ring.time[b]
    past = (t > tf)[:, None]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        rf = ((t - tb) / (tf - tb))[:, None]
        res = []
        for arr in (ring.rpy, ring.shift, ring.velo):
            A, B = arr[f].astype(np.float64), arr[b].astype(np.float64)
            res.append(np.where(past, A, A * rf + B * (1.0 - rf)))
    return res


def _rot_zyx_f64(rpy):
    def q(ang, axis):
        h = 0.5 * ang
        out = np.zeros(ang.shape + (4,))
        out[..., axis] = np.sin(h)
        out[..., 3] = np.cos(h)
        return out

    def qm(a, b):
        ax, ay, az, aw = (a[..., k] for k in range(4))
        bx, by, bz, bw = (b[..., k] for k in range(4))
        return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                         aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], axis=-1)

    qq = qm(qm(q(rpy[:, 2], 2), q(rpy[:, 1], 1)), q(rpy[:, 0], 0))
    x, y, z, w = (qq[:, k] for k in range(4))
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=-1).reshape(-1, 3, 3)


# ---- the whole call --------------------------------------------------------------------------------------------------
def replay(cloud, ring: Ring, scan_time: float):
    """adjust_distortion on a copy: decisions (literal and parallel), the float32 replay of the corrected coordinates,
    the float64 reference and the bound. `ring` is not modified; the pointers after the call are returned."""
    c = np.array(cloud, dtype=F, copy=True)
    n = len(c)
    r = {"n": n, "out": c.copy(), "ptr_front": ring.ptr_front, "ptr_last_iter": ring.ptr_last_iter, "ran": False}
    if n == 0:
        return r
    d = times_of(c, scan_time, ring.scan_period)
    r.update(d)
    front, skip, ptrs = walk_literal(ring, d["t"])
    r["ptr_front"], r["ptr_last_iter"] = ptrs
    r["ambiguous"] = d["ambiguous"].copy()
    if front is None:  # imu_ptr_last_ <= 0: nothing runs
        r["ref64"] = c[:, :3].astype(np.float64)
        r["bound"] = np.zeros((n, 3))
        return r
    r["ran"] = True
    r["front"], r["skip"] = front, skip
    r["monotone"] = window_monotone(ring)
    pf, ps, pptr, rounds, lb = walk_parallel(ring, d["t"])
    r["par_front"], r["par_skip"], r["par_ptrs"], r["par_rounds"], r["lb"] = pf, ps, pptr, rounds, lb
    r["rounds"] = rounds if r["monotone"] else 0  # the kernel walks literally then and runs no fix point
    r["base"], r["span"], _ = ring.window()
    ref = c[:, :3].astype(np.float64)
    bound = np.zeros((n, 3))
    if skip[0]:  # no start pose: no point is corrected (the reference would read an uninitialised r_s_i)
        r["ref64"], r["bound"] = ref, bound
        return r
    sel = np.flatnonzero(~skip)
    amb = np.zeros(len(sel), dtype=bool)
    t = d["t"][sel]
    rpy, shift, velo = _interp_f32(ring, front[sel], t)
    R = rot_zyx_f32(*rpy, amb)
    # point 0 (sel[0] == 0): the start pose, broadcast
    S = [E(np.full(len(sel), R[k].v[0], dtype=F), np.full(len(sel), R[k].e[0])) for k in range(9)]
    S = [S[3 * (k % 3) + k // 3] for k in range(9)]  # transpose
    for k in range(9):
        S[k].e = S[k].e + 16 * UD
    sh0 = [E(np.full(len(sel), s.v[0], dtype=F), np.full(len(sel), s.e[0])) for s in shift]
    ve0 = [E(np.full(len(sel), s.v[0], dtype=F), np.full(len(sel), s.e[0])) for s in velo]
    rel = E(d["rel"][sel])
    p = [E(c[sel, k]) for k in range(3)]
    v = []
    for row in range(3):
        sfs = (shift[row] - sh0[row]) - (ve0[row] * rel)
        rp = ((R[3 * row] * p[0]) + (R[3 * row + 1] * p[1])) + (R[3 * row + 2] * p[2])
        v.append(rp + sfs)
    outs = [((S[3 * row] * v[0]) + (S[3 * row + 1] * v[1])) + (S[3 * row + 2] * v[2]) for row in range(3)]
    moved = sel[1:]
    for k in range(3):
        r["out"][moved, k] = outs[k].v[1:]
    # float64 reference at the same decisions
    rpy64, sh64, ve64 = _interp_f64(ring, front[sel], t)
    R64 = _rot_zyx_f64(rpy64)
    with np.errstate(invalid="ignore", over="ignore"):
        Sinv = np.linalg.inv(R64[0]) if np.all(np.isfinite(R64[0])) else np.full((3, 3), np.nan)
        sfs64 = sh64 - sh64[0] - ve64[0] * d["rel"][sel].astype(np.float64)[:, None]
        v64 = np.einsum("nij,nj->ni", R64, c[sel, :3].astype(np.float64)) + sfs64
        o64 = v64 @ Sinv.T
    ref[moved] = o64[1:]
    for k in range(3):
        bound[moved, k] = outs[k].e[1:] + 2.0**-40 * (np.abs(o64[1:, k]) + 1)
    r["ambiguous"][sel] |= amb
    r["ambiguous"][moved] |= amb[0]  # the start pose's sin / cos feed every moved point
    r["ref64"], r["bound"] = ref, bound
    return r


def advance(ring: Ring, r) -> Ring:
    """The ring after the call: only the two pointers change."""
    out = Ring(ring.time, ring.rpy, ring.shift, ring.velo, r["ptr_front"], ring.ptr_last, r["ptr_last_iter"],
               ring.scan_period)
    return out


# ---- scenes ----------------------------------------------------------------------------------------------------------
def sweep_scan(n: int, rings: int = 16, turn: float = 2 * PI - 0.1, start: float = -0.05, direction: int = 1, seed: int = 0):
    """n points in firing order, one azimuth per point: direction 1 is a clockwise sweep (ori = -atan2 increases),
    -1 counter-clockwise. `turn` is the swept angle; `start` the first point's atan2 azimuth."""
    rng = np.random.default_rng(seed)
    az = start - direction * turn * (np.arange(n) / max(n - 1, 1))
    d = 5.0 + 20.0 * rng.random(n)
    el = np.deg2rad(-15 + 30 * (np.arange(n) % rings) / max(rings - 1, 1))
    pts = np.stack([d * np.cos(el) * np.cos(az), d * np.cos(el) * np.sin(az), d * np.sin(el), rng.random(n)], axis=1)
    return pts.astype(F)


def random_order_scan(n: int, seed: int = 0):
    """Livox-like: the azimuths of a full turn in random firing order (the first and last points stay the ends of a
    clockwise turn, so start / end are those of a spinning scan)."""
    pts = sweep_scan(n, seed=seed)
    rng = np.random.default_rng(seed + 1)
    mid = 1 + rng.permutation(n - 2)
    return np.concatenate([pts[:1], pts[mid], pts[-1:]])


def imu_messages(stamps, seed: int = 0, yaw_rate: float = 0.4):
    """(angular velocity, acceleration, quaternion xyzw, stamp) per stamp, a smooth yawing motion."""
    rng = np.random.default_rng(seed)
    out = []
    for k, s in enumerate(stamps):
        yaw = yaw_rate * (s % 1000.0)
        q = np.array([0.01 * np.sin(0.1 * k), 0.02 * np.cos(0.07 * k), np.sin(yaw / 2), np.cos(yaw / 2)])
        q /= np.linalg.norm(q)
        w = np.array([0.02, -0.01, yaw_rate]) + 0.01 * rng.normal(size=3)
        a = np.array([0.5, 0.1, 9.8]) + 0.05 * rng.normal(size=3)
        out.append((w, a, q, float(s)))
    return out


def feed(objs, msgs):
    for w, a, q, s in msgs:
        for o in objs:
            (o.get_imu if hasattr(o, "get_imu") else o.getImu)(w, a, q, s)


def planted_stamps(t, indices, background):
    """Stamps exactly on the given points' times (ties: t == stamp, the walk passes the stamp) plus a background grid,
    sorted and unique."""
    s = [float(t[i]) for i in indices] + [float(b) for b in background]
    return sorted(set(s))


def stamp_at_period(t_i: float, scan_period: float, after: bool = True) -> float:
    """A stamp s with fl(|t_i - s|) == scan_period exactly (the skip test's boundary: not skipped)."""
    s = t_i + scan_period if after else t_i - scan_period
    for _ in range(64):
        d = abs(t_i - s)
        if d == scan_period:
            return s
        s = np.nextafter(s, -np.inf if (d > scan_period) == after else np.inf)
    raise ValueError("no stamp at exactly scan_period")


def point_with_ori(target, r: float = 10.0, z: float = 0.5):
    """A float32 point whose ori = -(float)atan2(y, x) equals the float `target` exactly."""
    target = F(target)
    th = -float(target)
    for k in range(4000):
        x, y = F(r * math.cos(th)), F(r * math.sin(th))
        o, _ = neg_atan2(y, x)
        if F(o) == target:
            return np.array([x, y, z, 0.25], dtype=F)
        th += (float(o) - float(target)) * 0.5 + (1e-9 if k % 2 else -1e-9)
    raise ValueError(f"no float point with ori {target!r}")


def ori_for_half_turn(cloud, diff):
    """An ori whose formula-A azimuth a satisfies fl(a - start_ori) == diff exactly (the half-turn test :136)."""
    so, od = orientation_range(cloud)[0], F(diff)
    o = F(float(so) + float(od) - 2 * PI)
    for _ in range(64):
        a = o
        if float(a) < float(so) - PI * 0.5:
            a = F(float(a) + 2 * PI)
        d = F(a - so)
        if d == od:
            return o
        o = np.nextafter(o, F(np.inf) if d < od else F(-np.inf))
    raise ValueError("no ori at that half-turn difference")


# ---- scenarios: IMU pushes and scans, with the property each exists for ----------------------------------------------
class Scenario:
    """steps: ("imu", messages) or ("scan", cloud, scan_time, claim); claim(view, ring) asserts the property the scan is
    for on a view with keys n, t, rel, front, skip, k_first, rounds (the replay's or the device trace's) and the ring
    before the call."""

    def __init__(self, name, scan_period, steps):
        self.name, self.scan_period, self.steps = name, scan_period, steps

    def scans(self):
        return [s for s in self.steps if s[0] == "scan"]


def _grid(t0, t1, dt=0.01):
    return list(t0 + dt * np.arange(int(round((t1 - t0) / dt)) + 1))


def ladder(n: int, sp: float = 0.125, st: float = 100.0, seed=None):
    """Lower-bound steps on the deskew_scan chunk edges q per - 1, q per, q per + 1 (per = ceil(n / 1024)), each a tie:
    the stamp equals the point's t, so the walk passes it and the step lies exactly at that index."""
    seed = n if seed is None else seed
    c = sweep_scan(n, seed=seed)
    t = times_of(c, st, sp)["t"]
    per = -(-n // 1024)
    idx = sorted({j for q in (1, 2, 511, 1023) for j in (q * per - 1, q * per, q * per + 1) if 1 <= j < n})
    idx = [j for j in idx if t[j] > t[j - 1]]
    stamps = planted_stamps(t, idx, _grid(st - 0.3, st + 0.2, 0.02))

    def claim(v, ring):
        assert v["rounds"] == 1 and not v["skip"].any()
        for j in idx:  # a tie at j: t == stamp, so j stands past it and j - 1 before it
            k = int(np.flatnonzero(ring.time == v["t"][j])[0])
            assert v["front"][j] != k and v["front"][j - 1] == k, j
    return Scenario(f"ladder_{n}", sp, [("imu", imu_messages(stamps, seed=seed)), ("scan", c, st, claim)]), idx


def chains(seed: int, n: int = 4000, sp: float = 0.125, st: float = 50.0, want: int = 3):
    """A random-order scan against sparse stamps: late and early times alternate, so a point carried past a far stamp
    skips later points whose own lower bound would keep them. The Jacobi fix point then needs several passes."""
    rng = np.random.default_rng(seed)
    c = random_order_scan(n, seed=seed)
    stamps = sorted(set(list(st - 0.5 + 0.05 * np.arange(10)) + list(st + sp * rng.random(3)) + [st + 0.3, st + 0.6]))

    def claim(v, ring):
        assert (v["rounds"] >= 3 if want >= 3 else v["rounds"] == want) and v["skip"].any() and not v["skip"].all()
    return Scenario(f"chains_{seed}", sp, [("imu", imu_messages(stamps, seed=seed)), ("scan", c, st, claim)])


CHAIN_SEEDS = {2: 25, 3: 0}
LADDER_SCAN_TIME = {262147: 100.25}  # at 100.0 one sin / cos of this scene lies near a float midpoint (glibc_ring)


def glibc_ring(msgs, scan_period):
    """The ring getImu builds (deskew.cu ImuDeskew::get_imu): glibc's atan2f / asinf, float rotation and acceleration
    ((R0 a0 + R1 a1) + R2 a2), shift / velo in double stored as float. Fresh ring, no scan in between."""
    import ctypes
    import ctypes.util

    from oracle import deskew

    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.atan2f.restype = libm.asinf.restype = ctypes.c_float
    libm.atan2f.argtypes = [ctypes.c_float, ctypes.c_float]
    libm.asinf.argtypes = [ctypes.c_float]
    time, rpy = np.zeros(QUE), np.zeros((QUE, 3), F)
    shift, velo = np.zeros((QUE, 3), F), np.zeros((QUE, 3), F)
    last, front = -1, 0
    for w, a, q, stamp in msgs:
        R = deskew._quat_to_matrix_f(np.asarray(q, dtype=F))
        last = (last + 1) % QUE
        if (last + 1) % QUE == front:
            front = (front + 1) % QUE
        time[last] = stamp
        rpy[last] = [libm.atan2f(R[2, 1], R[2, 2]), libm.asinf(-R[2, 0]), libm.atan2f(R[1, 0], R[0, 0])]
        af = np.asarray(a, dtype=F)
        acc = np.array([(R[i, 0] * af[0] + R[i, 1] * af[1]) + R[i, 2] * af[2] for i in range(3)], dtype=F)
        back = (last - 1) % QUE
        dt = time[last] - time[back]
        if dt < scan_period:
            shift[last] = (shift[back].astype(np.float64) + velo[back].astype(np.float64) * dt
                           + acc.astype(np.float64) * dt * dt * 0.5).astype(F)
            velo[last] = (velo[back].astype(np.float64) + acc.astype(np.float64) * dt).astype(F)
    return Ring(time, rpy, shift, velo, front, last, 0, scan_period)  # find_chain_seeds(): two passes, three or more


def _ok(v, ring):
    assert v["n"] > 0


def ring_scenes(sp: float = 0.125):
    out = []
    # the window crosses index 199 -> 0; then a second scan with no push in between (span == 0); three scans carried
    T = 20.0
    c = sweep_scan(3000, seed=7)
    first = imu_messages(T + 0.01 * np.arange(191), seed=7)
    more = imu_messages(T + 1.90 + 0.01 * np.arange(1, 21), seed=8)
    last = imu_messages(T + 2.10 + 0.01 * np.arange(1, 16), seed=9)

    def at_190(v, ring):
        assert ring.ptr_last == 190 and not v["skip"][-1] and v["front"][-1] == 190

    def wraps(v, ring):
        assert ring.ptr_last_iter == 190 and ring.ptr_last == 10 and (v["front"] < 100).any() and (v["front"] >= 190).any()

    def span0(v, ring):
        assert ring.ptr_last_iter == ring.ptr_last == 10 and (v["front"] == 10).all()

    out.append(Scenario("ring_wrap_span0_carry", sp, [
        ("imu", first), ("scan", c, T + 1.90 - 0.02, at_190), ("imu", more), ("scan", c, T + 1.98, wraps),
        ("scan", c, T + 2.05, span0), ("imu", last), ("scan", c, T + 2.12, _ok)]))

    # span == 199: 200 pushes and no scan; then ptr_last == 0 after a wrap (the whole scan is skipped)
    def span199(v, ring):
        assert (ring.ptr_last - ring.ptr_last_iter) % QUE == 199

    def no_run(v, ring):
        assert ring.ptr_last == 0 and v["n"] == 0
    out.append(Scenario("ring_span199_then_ptr_last0", sp, [
        ("imu", imu_messages(T + 0.005 * np.arange(200), seed=3)), ("scan", c, T + 0.9, span199),
        ("imu", imu_messages([T + 1.0], seed=4)), ("scan", c, T + 1.0, no_run)]))

    # front at window position 0: the scan starts before the first stamp; the back sample (ring[199]) was never written
    def front0(v, ring):
        assert ring.ptr_last_iter == 0 and v["front"][0] == 0 and not v["skip"][0] and ring.time[199] == 0.0
    out.append(Scenario("ring_front_at_position0", sp, [
        ("imu", imu_messages(T + 0.05 + 0.01 * np.arange(30), seed=5)), ("scan", c, T, front0)]))

    # an IMU gap longer than scan_period: the slot after the gap keeps stale shift / velo (getImu skips the update)
    gap = list(T + 0.01 * np.arange(10)) + list(T + 0.3 + 0.01 * np.arange(20))

    def stale(v, ring):
        k = int(np.flatnonzero(ring.time == T + 0.3)[0])
        assert ring.time[k] - ring.time[k - 1] > sp and (ring.shift[k] == 0).all() and (v["front"] == k).any()
    out.append(Scenario("ring_gap_stale_slot", sp, [("imu", imu_messages(gap, seed=6)), ("scan", c, T + 0.22, stale)]))
    return out


def stamp_scenes(sp: float = 0.125):
    out = []
    T = 30.0
    c = sweep_scan(2000, seed=11)
    t = times_of(c, T, sp)["t"]
    # duplicate stamps; the newest sample duplicated and tied with the last point's t (rf = 0 / 0)
    dup = sorted(list(T - 0.2 + 0.02 * np.arange(10)) + [float(t[700])] * 2 + [T + 0.05] * 2)
    dup = dup + [float(t[-1]), float(t[-1])]

    def dups(v, ring):
        assert v["t"][-1] == ring.time[ring.ptr_last] == ring.time[ring.ptr_last - 1]
    out.append(Scenario("stamps_duplicate", sp, [("imu", imu_messages(dup, seed=12)), ("scan", c, T, dups)]))

    # exactly scan_period away: no stamp in (t_i, t_i + sp) and one at fl(|t_i - s|) == sp (kept); earlier points skipped
    i = 1200
    s = stamp_at_period(float(t[i]), sp)
    per = list(T - 0.3 + 0.01 * np.arange(36)) + [s]
    per = [x for x in per if x <= float(t[i]) - 0.001 or x == s]

    def period(v, ring):
        k = ring.ptr_last
        assert abs(v["t"][i] - ring.time[k]) == sp and v["front"][i] == k and not v["skip"][i] and v["skip"][i - 1]
    out.append(Scenario("stamps_exactly_scan_period", sp, [("imu", imu_messages(sorted(per), seed=13)), ("scan", c, T, period)]))

    # the IMU clock steps back by 0.3 s inside the window (a bag replayed in a loop): T - 0.2 .. T + 0.2, then T - 0.1 ..
    back = list(T - 0.2 + 0.01 * np.arange(41)) + list(T - 0.1 + 0.01 * np.arange(41))

    def stepback(v, ring):
        _, _, w = ring.window()
        assert (np.diff(w) < 0).any() and v["rounds"] == 0
    out.append(Scenario("stamps_clock_step_back", sp, [("imu", imu_messages(back, seed=14)), ("scan", c, T, stepback),
                                                       ("scan", c, T + 0.1, _ok)]))
    return out


def azimuth_scenes(sp: float = 0.1):
    out = []
    T = 40.0
    imu = imu_messages(T - 0.3 + 0.01 * np.arange(60), seed=21)

    def scene(name, c, claim=_ok):
        out.append(Scenario(name, sp, [("imu", imu), ("scan", c, T, claim)]))

    def has_k(v, ring):
        assert v["k_first"] < v["n"]
    scene("az_clockwise", sweep_scan(5000, seed=21), has_k)
    scene("az_counter_clockwise", sweep_scan(5000, direction=-1, seed=22))
    scene("az_sector", sweep_scan(5000, turn=PI * 0.6, seed=23))
    scene("az_random_order", random_order_scan(5000, seed=24), has_k)
    scene("az_start_near_plus_pi", sweep_scan(5000, start=PI - 1e-3, seed=25), has_k)
    scene("az_start_near_minus_pi", sweep_scan(5000, start=-PI + 1e-3, seed=26), has_k)
    # y = +-0.0 with x < 0 (ori = -+pi), x = y = 0 (ori = -0 / 0 of atan2(+-0, +-0))
    c = sweep_scan(3000, seed=27)
    special = np.array([[-7, 0.0, 1, 0.5], [-7, -0.0, 1, 0.5], [0.0, 0.0, 1, 0.5], [-0.0, 0.0, 1, 0.5],
                        [0.0, -0.0, 1, 0.5], [-0.0, -0.0, 1, 0.5]], dtype=F)
    for j, p in zip((400, 1500, 1501, 1502, 2200, 2201), special):
        c[j] = p
    scene("az_signed_zero_y", c)
    # the half-turn switch: a - start_ori == float(pi) (fires: float(pi) > pi) at index kf, one ulp below just before it
    c = sweep_scan(3000, seed=28)
    kf = 1100
    c[kf - 1] = point_with_ori(ori_for_half_turn(c, np.nextafter(F(np.pi), F(0))))
    c[kf] = point_with_ori(ori_for_half_turn(c, F(np.pi)))

    def half(v, ring):
        assert v["k_first"] == kf
    scene("az_half_turn_threshold", c, half)
    return out, kf


def nonfinite_scenes(sp: float = 0.1):
    T = 60.0
    imu = imu_messages(T - 0.3 + 0.01 * np.arange(60), seed=31)
    out = []
    for name, rows in (("nan_ray_mid", [700]), ("nan_ray_last", [-1]), ("nan_ray_first", [0]), ("nan_rays_many", [5, 700, 701, 1999])):
        c = sweep_scan(2400, seed=32)
        c[rows, :3] = np.nan

        def nan_claim(v, ring, rows=rows):
            assert np.isnan(v["t"][rows]).all()  # a NaN ray walks to the newest sample and is not skipped (:153-162)
            assert (v["front"][rows] == ring.ptr_last).all() and not v["skip"][rows].any()
        out.append(Scenario(name, sp, [("imu", imu), ("scan", c, T + 0.2, nan_claim), ("scan", c, T + 0.25, _ok)]))
    c = sweep_scan(2400, seed=33)
    c[100, 0] = np.inf
    c[900, 1] = -np.inf
    c[1500, 2] = np.inf
    c[1600, :2] = [np.inf, np.inf]
    out.append(Scenario("inf_coordinates", sp, [("imu", imu), ("scan", c, T + 0.2, _ok)]))
    return out


def all_scenes():
    ladder_ns = (1, 2, 31, 1023, 1024, 1025, 2047, 4097, 60000, 262147)
    scs = [ladder(n, st=LADDER_SCAN_TIME.get(n, 100.0))[0] for n in ladder_ns]
    scs += [chains(CHAIN_SEEDS[2], want=2), chains(CHAIN_SEEDS[3], want=3)]
    scs += ring_scenes() + stamp_scenes() + azimuth_scenes()[0] + nonfinite_scenes()
    return scs


def find_chain_seeds(rounds_wanted=(1, 2, 3), n: int = 4000, tries: int = 400):
    """Seeds of `chains` whose scan needs exactly 1, 2 and >= 3 passes (searched on the CPU, deterministic)."""
    from oracle import deskew

    found = {}
    for seed in range(tries):
        sc = chains(seed, n)
        o = deskew.LidarUndistortion(scan_period=sc.scan_period)
        feed([o], sc.steps[0][1])
        _, cloud, st, _ = sc.steps[1]
        r = replay(cloud, Ring.from_oracle(o), st)
        k = min(r["rounds"], 3)
        if k in rounds_wanted and k not in found and r["skip"].any() and not r["skip"].all():
            found[k] = seed
        if len(found) == len(rounds_wanted):
            break
    return found
