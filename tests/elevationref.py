"""Exact Python replay of csrc/elevation_map.hpp (the elevation / traversability map of b200sm_build_elevation_map):
float32 transforms one rounding per operation, fixed point and every statistic and moment sum in Python integers, and the
plane solve, residuals and ratios as IEEE doubles in the header's order. Small inputs only: it is the definition, not a
fast path. `mut` names a deliberate deviation, so the tests can show the replay tells each of them apart."""
import math

import numpy as np

F32 = np.float32
COORD_LIMIT = 2.0 ** 52
ORIGIN_LIMIT = 2.0 ** 46
RANGE_LIMIT = 1 << 30
MAX_CELLS = 1 << 28
HEIGHT_EXTENT = 1 << 40
LO_EMPTY = 0x7F7F7F7F7F7F7F7F
TOP_EMPTY = -0x7F7F7F7F7F7F7F80  # 0x8080808080808080 as int64

MUTATIONS = ("surface_strict", "observed_gt", "step_ge", "round_trunc", "skip_range_ge")

DEFAULTS = dict(resolution=0.1, max_range=100.0, sensor_origin=(0.0, 0.0, 0.0), clearance=2.0, min_points=2, window_cells=3,
                min_cells=6, max_slope=20.0, max_step=0.15, max_roughness=0.05, occupied_thresh=0.65, free_thresh=0.25)


def params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    p["sensor_origin"] = tuple(float(v) for v in p["sensor_origin"])
    return p


class Refused(Exception):
    """The build is refused; .code is the host harness's return code."""

    def __init__(self, code, why):
        super().__init__(why)
        self.code = code


def fixed(v, S, limit):
    """floor(v * S) when |v * S| < limit, else None."""
    prod = float(v) * S
    if not (-limit < prod < limit):
        return None
    return math.floor(prod)


def prepare(p):
    """The header's el_prepare: the constants, or Refused(-1)."""
    def bad(why):
        raise Refused(-1, why)

    res = p["resolution"]
    if not (math.isfinite(res) and res > 0):
        bad("resolution")
    S = 65536.0 / res
    if not math.isfinite(S):
        bad("resolution too small")
    mr = p["max_range"]
    if not (math.isfinite(mr) and mr > 0):
        bad("max_range")
    Rd = mr * S
    if not (Rd <= float(RANGE_LIMIT)):
        bad("max_range / resolution")
    if not all(math.isfinite(v) for v in p["sensor_origin"]):
        bad("sensor_origin")
    C = fixed(p["clearance"], S, COORD_LIMIT) if p["clearance"] >= 0 else None
    if C is None:
        bad("clearance")
    if p["min_points"] < 1:
        bad("min_points")
    r = p["window_cells"]
    if not (1 <= r <= 8):
        bad("window_cells")
    if not (3 <= p["min_cells"] <= (2 * r + 1) ** 2):
        bad("min_cells")
    if not (0 < p["max_slope"] < 90):
        bad("max_slope")
    K = fixed(p["max_step"], S, COORD_LIMIT) if p["max_step"] > 0 else None
    if K is None or K < 1:
        bad("max_step")
    mrough = p["max_roughness"]
    if not (math.isfinite(mrough) and mrough > 0):
        bad("max_roughness")
    if not (0 <= p["free_thresh"] < p["occupied_thresh"] <= 1):
        bad("thresholds")
    G = math.tan(p["max_slope"] * (math.pi / 180.0)) * 65536.0
    if not G > 0:
        bad("max_slope")
    return dict(S=S, R=math.floor(Rd), C=C, K=K, G=G, G2=G * G, max_roughness=mrough, r=r, min_points=p["min_points"],
                min_cells=p["min_cells"], occ=int(np.rint(p["occupied_thresh"] * 100.0)),
                free=int(np.rint(p["free_thresh"] * 100.0)))


def pose_f(P):
    P = np.asarray(P, dtype=np.float64)
    return [F32(P[r, c]) for r in range(3) for c in range(4)]


def transform(T, x, y, z):
    x, y, z = F32(x), F32(y), F32(z)
    with np.errstate(all="ignore"):
        return [((T[4 * r] * x + T[4 * r + 1] * y) + T[4 * r + 2] * z) + T[4 * r + 3] for r in range(3)]


def point(c, xo, yo, e, mut=None):
    """(cell x, cell y, Z) of a transformed point, None when skipped (occupancy's og_ray rule)."""
    X, Y, Z = (fixed(v, c["S"], COORD_LIMIT) for v in e)
    if X is None or Y is None or Z is None:
        return None
    dx, dy, R = X - xo, Y - yo, c["R"]
    if abs(dx) > R or abs(dy) > R:
        return None
    d2 = dx * dx + dy * dy
    if d2 > R * R or (mut == "skip_range_ge" and d2 >= R * R):
        return None
    return X >> 16, Y >> 16, Z


def window(c, h, mut=None, detail=None):
    """(value, step_m, tan_slope, roughness) of one cell; h(u, v) -> surface height or None. Floats are float32 or nan.
    detail (a dict), when given, receives the doubles a, b, s2 and roughness."""
    nan = F32("nan")
    hc = h(0, 0)
    if hc is None:
        return -1, nan, nan, nan
    r = c["r"]
    m = su = sv = suu = suv = svv = sz = suz = svz = 0
    zmin = zmax = hc
    cells = []
    for v in range(-r, r + 1):
        for u in range(-r, r + 1):
            hz = h(u, v)
            if hz is None:
                continue
            z = hz - hc
            cells.append((u, v, z))
            m += 1
            su += u
            sv += v
            suu += u * u
            suv += u * v
            svv += v * v
            sz += z
            suz += u * z
            svz += v * z
            zmin, zmax = min(zmin, hz), max(zmax, hz)
    for s in (sz, suz, svz):
        assert abs(s) < 2 ** 53
    if m < c["min_cells"]:
        return -1, nan, nan, nan
    A, B, Cc = m * suu - su * su, m * suv - su * sv, m * svv - sv * sv
    D = A * Cc - B * B
    if D == 0:
        return -1, nan, nan, nan
    P, Q = m * suz - su * sz, m * svz - sv * sz
    assert abs(P) < 2 ** 63 and abs(Q) < 2 ** 63 and abs(D) < 2 ** 53
    dP, dQ, dA, dB, dC, dD = float(P), float(Q), float(A), float(B), float(Cc), float(D)
    a = (dP * dC - dQ * dB) / dD
    b = (dQ * dA - dP * dB) / dD
    d = ((float(sz) - a * float(su)) - b * float(sv)) / float(m)
    s2 = a * a + b * b
    acc = 0.0
    for u, v, z in cells:
        e = float(z) - ((a * float(u) + b * float(v)) + d)
        acc = acc + e * e
    rough = math.sqrt(acc / float(m)) / c["S"]
    step = zmax - zmin
    root = math.sqrt(s2)
    out = (F32(float(step) / c["S"]), F32(root / 65536.0), F32(rough))
    if detail is not None:
        detail.update(a=a, b=b, s2=s2, roughness=rough)
    lethal_step = step >= c["K"] if mut == "step_ge" else step > c["K"]
    if lethal_step or s2 > c["G2"] or rough > c["max_roughness"]:
        return (100,) + out
    x = float(step) / float(c["K"])
    xs, xr = root / c["G"], rough / c["max_roughness"]
    x = max(x, xs, xr)
    value = math.floor(99.0 * x) if mut == "round_trunc" else math.floor(99.0 * x + 0.5)
    return (min(value, 99),) + out


def pixel(v, occ, free):
    if v < 0:
        return 205
    if v >= occ:
        return 0
    if v <= free:
        return 254
    return 205


def build(submaps, p=None, mut=None):
    """submaps: [(points (N, 3+), pose 4x4)]. The map as a dict of (H, W) arrays and counts; raises Refused."""
    p = params(**(p or {}))
    c = prepare(p)
    if not submaps:
        raise Refused(-4, "no submaps")
    S = c["S"]
    pts = []
    any_points = False
    for P_, Pose in submaps:
        P_ = np.asarray(P_, dtype=F32).reshape(len(P_), -1) if len(P_) else np.zeros((0, 3), F32)
        T = pose_f(Pose)
        if len(P_) == 0:
            continue
        any_points = True
        o = transform(T, *p["sensor_origin"])
        xo, yo = fixed(o[0], S, ORIGIN_LIMIT), fixed(o[1], S, ORIGIN_LIMIT)
        if xo is None or yo is None:
            raise Refused(-2, "origin")
        for row in P_:
            pts.append(point(c, xo, yo, transform(T, row[0], row[1], row[2]), mut))
    if not any_points:
        raise Refused(-5, "no points")
    used = [q for q in pts if q is not None]
    if not used:
        raise Refused(-5, "every point skipped")
    x0, x1 = min(q[0] for q in used), max(q[0] for q in used)
    y0, y1 = min(q[1] for q in used), max(q[1] for q in used)
    W, H = x1 - x0 + 1, y1 - y0 + 1
    if W * H > MAX_CELLS:
        raise Refused(-3, "cells")
    zs = [q[2] for q in used]
    if max(zs) - min(zs) >= HEIGHT_EXTENT:
        raise Refused(-6, "height extent")
    n = np.zeros((H, W), dtype=np.uint32)
    lo = np.full((H, W), LO_EMPTY, dtype=np.int64)
    top = np.full((H, W), TOP_EMPTY, dtype=np.int64)
    for x, y, Z in used:
        n[y - y0, x - x0] += 1
        lo[y - y0, x - x0] = min(int(lo[y - y0, x - x0]), Z)
    over = 0
    for x, y, Z in used:
        limit = int(lo[y - y0, x - x0]) + c["C"]
        if Z > limit or (mut == "surface_strict" and Z == limit):
            over += 1
        else:
            top[y - y0, x - x0] = max(int(top[y - y0, x - x0]), Z)
    mp = c["min_points"]
    obs = (n > mp) if mut == "observed_gt" else (n >= mp)
    out = dict(step=np.zeros((H, W), F32), tan_slope=np.zeros((H, W), F32), roughness=np.zeros((H, W), F32),
               value=np.zeros((H, W), np.int8))
    img = np.zeros((H, W), np.uint8)
    for y in range(H):
        for x in range(W):
            def h(u, v, x=x, y=y):
                gx, gy = x + u, y + v
                if 0 <= gx < W and 0 <= gy < H and obs[gy, gx]:
                    return int(top[gy, gx])
                return None

            v, s, t, g = window(c, h, mut)
            out["value"][y, x], out["step"][y, x], out["tan_slope"][y, x], out["roughness"][y, x] = v, s, t, g
            img[H - 1 - y, x] = pixel(v, c["occ"], c["free"])
    vals = out["value"]
    return dict(width=W, height=H, origin=(x0 * p["resolution"], y0 * p["resolution"]), n=n, h=top, lo=lo, pgm=img.tobytes(),
                n_points=len(used), n_skipped=len(pts) - len(used), n_overhang=over, n_observed=int(obs.sum()),
                n_lethal=int((vals == 100).sum()), n_traversable=int(((vals >= 0) & (vals < 100)).sum()),
                n_unknown=int((vals < 0).sum()), p=p, **out)
