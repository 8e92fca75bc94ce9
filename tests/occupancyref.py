"""An exact replay of the occupancy grid of b200sm_build_occupancy_grid (csrc/occupancy_grid.hpp) in Python integers: the
float32 transform of each point (numpy float32 scalars, one rounding per operation in transform_point's order), one double
multiply per coordinate into fixed point, then integer arithmetic only — the range test, the band clip by floor division,
the Amanatides-Woo walk with its cross-multiplied comparison, the per-submap hit-wins update, the values, the row-flipped
trinary image and the two files.

MUTATIONS names subtly wrong variants, each of which tests/test_occupancy_cpu.py shows changes an outcome:
  y_first    at an exact corner the walk steps y before x
  no_clip    the segment is not clipped to the height band (only the endpoint's hit still needs the band)
  trunc      fixed point and cells by truncation toward zero instead of floor
  free_wins  a cell both hit and freed by one submap also counts as freed by it
  no_flip    image rows run from the bottom (smallest y) up
"""
from __future__ import annotations

import math
import os

import numpy as np

MUTATIONS = ("y_first", "no_clip", "trunc", "free_wins", "no_flip")
F = 16
ONE = 1 << F
COORD_LIMIT = 2.0 ** 52
ORIGIN_LIMIT = 2.0 ** 46
RANGE_LIMIT = 1 << 30
BAND_REACH = 1 << 32
MAX_CELLS = 1 << 28
DEFAULTS = dict(resolution=0.05, z_min=0.2, z_max=2.0, max_range=100.0, sensor_origin=(0.0, 0.0, 0.0), occupied_thresh=0.65,
                free_thresh=0.25)
F32 = np.float32


class Refused(Exception):
    """What the session refuses with B200REG_ERR_ARG; .code is the host compile's return code."""

    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


def params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    return p


def fixed(v, S, limit, mut=()):
    """floor((double)v * S) when |v * S| < limit, else None."""
    p = float(v) * S
    if not (-limit < p < limit):
        return None
    return int(p) if "trunc" in mut else math.floor(p)


def cell(V, mut=()):
    if "trunc" in mut:
        return V >> F if V >= 0 else -((-V) >> F)
    return V >> F


def floor_div(a, b):
    return a // b  # Python's // is floor division for integers of either sign


def prepare(p):
    res = float(p["resolution"])
    if not (math.isfinite(res) and res > 0):
        raise Refused(-1, "resolution")
    S = 65536.0 / res
    if not math.isfinite(S):
        raise Refused(-1, "resolution")
    zmin, zmax = float(p["z_min"]), float(p["z_max"])
    if not (math.isfinite(zmin) and math.isfinite(zmax) and zmin < zmax):
        raise Refused(-1, "band")
    mr = float(p["max_range"])
    if not (math.isfinite(mr) and mr > 0):
        raise Refused(-1, "max_range")
    Rd = mr * S
    if not (Rd <= RANGE_LIMIT):
        raise Refused(-1, "max_range / resolution")
    if not all(math.isfinite(float(v)) for v in p["sensor_origin"]):
        raise Refused(-1, "sensor_origin")
    occ, fr = float(p["occupied_thresh"]), float(p["free_thresh"])
    if not (fr >= 0 and fr < occ and occ <= 1):
        raise Refused(-1, "thresholds")
    zlo, zhi = fixed(zmin, S, ORIGIN_LIMIT), fixed(zmax, S, ORIGIN_LIMIT)
    if zlo is None or zhi is None:
        raise Refused(-1, "band range")
    # round() of a Python float is round-half-even, as rint in the default rounding mode
    return dict(S=S, R=math.floor(Rd), zlo=zlo, zhi=zhi, occ=int(round(occ * 100.0)), free=int(round(fr * 100.0)))


def pose_f(P):
    """The float pose, 3x4 row-major float32 scalars."""
    P = np.asarray(P, dtype=np.float64)
    return [[F32(P[r, c]) for c in range(4)] for r in range(3)]


def transform(T, x, y, z):
    x, y, z = F32(x), F32(y), F32(z)
    with np.errstate(all="ignore"):
        return [((T[r][0] * x + T[r][1] * y) + T[r][2] * z) + T[r][3] for r in range(3)]


def origin(c, p, T):
    so = [F32(float(v)) for v in p["sensor_origin"]]
    o = transform(T, *so)
    O = [fixed(v, c["S"], ORIGIN_LIMIT) for v in o]
    if any(v is None for v in O) or abs(c["zlo"] - O[2]) > BAND_REACH or abs(c["zhi"] - O[2]) > BAND_REACH:
        raise Refused(-2, "origin")
    return O


def ray(c, O, e, mut=()):
    """None when skipped, else (hit: bool, endpoint cell (x, y), clipped segment ((xa, ya), (xb, yb)) or None)."""
    X = [fixed(v, c["S"], COORD_LIMIT, mut) for v in e]
    if any(v is None for v in X):
        return None
    xo, yo, zo = O
    xe, ye, ze = X
    dx, dy = xe - xo, ye - yo
    R = c["R"]
    if abs(dx) > R or abs(dy) > R or dx * dx + dy * dy > R * R:
        return None
    zlo, zhi = c["zlo"], c["zhi"]
    hit = zlo <= ze <= zhi
    end = (cell(xe, mut), cell(ye, mut))
    if "no_clip" in mut:
        return hit, end, ((xo, yo), (xe, ye))
    dz = ze - zo
    na = nb = None
    if dz == 0:
        if zo < zlo or zo > zhi:
            return hit, end, None
    elif dz > 0:
        if zo > zhi or ze < zlo:
            return hit, end, None
        if zo < zlo:
            na = zlo - zo
        if ze > zhi:
            nb = zhi - zo
    else:
        if zo < zlo or ze > zhi:
            return hit, end, None
        if zo > zhi:
            na = zhi - zo
        if ze < zlo:
            nb = zlo - zo
    a = (xo + floor_div(dx * na, dz), yo + floor_div(dy * na, dz)) if na is not None else (xo, yo)
    b = (xo + floor_div(dx * nb, dz), yo + floor_div(dy * nb, dz)) if nb is not None else (xe, ye)
    return hit, end, (a, b)


def walk(a, b, mut=()):
    """The cells of the 4-connected walk from a to b (fixed point), both ends included."""
    (xa, ya), (xb, yb) = a, b
    cx, cy = cell(xa, mut), cell(ya, mut)
    ex, ey = cell(xb, mut), cell(yb, mut)
    ax, ay = abs(xb - xa), abs(yb - ya)
    sx, sy = (1 if ex > cx else -1), (1 if ey > cy else -1)
    nx, ny = abs(ex - cx), abs(ey - cy)
    out = [(cx, cy)]
    while nx + ny > 0:
        if nx == 0:
            step_x = False
        elif ny == 0:
            step_x = True
        else:
            bx = (cx + 1) * ONE - xa if sx > 0 else xa - cx * ONE
            by = (cy + 1) * ONE - ya if sy > 0 else ya - cy * ONE
            step_x = bx * ay < by * ax if "y_first" in mut else bx * ay <= by * ax
        if step_x:
            cx += sx
            nx -= 1
        else:
            cy += sy
            ny -= 1
        out.append((cx, cy))
    return out


def value(h, f):
    n = h + f
    return -1 if n == 0 else (200 * h + n) // (2 * n)


def pixel(v, occ, fr):
    if v < 0:
        return 205
    if v >= occ:
        return 0
    if v <= fr:
        return 254
    return 205


def build(submaps, p=None, mut=()):
    """submaps: list of (points (n, >= 3) float32, pose 4x4 float64). Returns the grid as a dict: width, height, origin,
    hits, frees (uint32, (height, width)), values (int8), pgm (bytes, top row first), n_rays, n_skipped, n_occupied, n_free,
    n_unknown, and p / c for the files."""
    p = params(**(p or {}))
    c = prepare(p)
    if not submaps:
        raise Refused(-4, "no submaps")
    Ts = [pose_f(P) for _, P in submaps]
    Os = [origin(c, p, T) for T in Ts]
    rays = []
    n_rays = n_skipped = 0
    xs = [cell(O[0], mut) for O in Os]
    ys = [cell(O[1], mut) for O in Os]
    for (pts, _), T, O in zip(submaps, Ts, Os):
        rs = []
        for row in np.asarray(pts, dtype=np.float32):
            r = ray(c, O, transform(T, row[0], row[1], row[2]), mut)
            if r is None:
                n_skipped += 1
                continue
            n_rays += 1
            xs.append(r[1][0])
            ys.append(r[1][1])
            rs.append(r)
        rays.append(rs)
    x0, x1, y0, y1 = min(xs), max(xs), min(ys), max(ys)
    W, H = x1 - x0 + 1, y1 - y0 + 1
    if W * H > MAX_CELLS:
        raise Refused(-3, f"{W} x {H} cells")
    hits = np.zeros((H, W), dtype=np.uint32)
    frees = np.zeros((H, W), dtype=np.uint32)
    for rs in rays:
        hit, fre = set(), set()
        for h, end, seg in rs:
            if h:
                hit.add(end)
            if seg is not None:
                fre.update(walk(seg[0], seg[1], mut))
        for (x, y) in hit:
            hits[y - y0, x - x0] += 1
        for (x, y) in (fre if "free_wins" in mut else fre - hit):
            frees[y - y0, x - x0] += 1
    values = np.full((H, W), -1, dtype=np.int8)
    pix = np.zeros((H, W), dtype=np.uint8)
    n_occ = n_free = n_unk = 0
    for y in range(H):
        for x in range(W):
            v = value(int(hits[y, x]), int(frees[y, x]))
            values[y, x] = v
            px = pixel(v, c["occ"], c["free"])
            pix[y, x] = px
            n_unk += v < 0
            n_occ += v >= 0 and px == 0
            n_free += v >= 0 and px == 254
    img = pix if "no_flip" in mut else pix[::-1]
    return dict(width=W, height=H, origin=(float(x0) * float(p["resolution"]), float(y0) * float(p["resolution"])), hits=hits,
                frees=frees, values=values, pgm=img.tobytes(), n_rays=n_rays, n_skipped=n_skipped, n_occupied=n_occ,
                n_free=n_free, n_unknown=n_unk, p=p, c=c, cells0=(x0, y0))


def number(v):
    """The header's og_number: the fewest significant digits (<= 17) that read back to v, '.0' before a bare exponent."""
    for prec in range(1, 18):
        s = "%.*g" % (prec, v)
        if float(s) == v:
            break
    if "e" in s and "." not in s:
        s = s.replace("e", ".0e")
    return s


def pgm_bytes(g):
    head = f"P5\n# CREATOR: lidarslam_ros2_b200 occupancy grid {number(g['p']['resolution'])} m/pix\n{g['width']} {g['height']}\n255\n"
    return head.encode() + g["pgm"]


def yaml_quote(name: bytes) -> str:
    """The header's og_yaml_quote on the name's bytes (as UTF-8 text)."""
    out = bytearray(b'"')
    for ch in name:
        if ch in (0x5C, 0x22):
            out += bytes((0x5C, ch))
        elif ch < 0x20 or ch == 0x7F:
            out += b"\\x%02X" % ch
        else:
            out.append(ch)
    return (out + b'"').decode()


def yaml_text(g, pgm_path):
    p = g["p"]
    return (f"image: {yaml_quote(os.path.basename(os.fsencode(pgm_path)))}\nmode: trinary\nresolution: {number(p['resolution'])}\n"
            f"origin: [{number(g['origin'][0])}, {number(g['origin'][1])}, 0]\nnegate: 0\n"
            f"occupied_thresh: {number(p['occupied_thresh'])}\nfree_thresh: {number(p['free_thresh'])}\n")
