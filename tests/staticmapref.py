"""An exact replay of the static map of b200sm_build_static_map (csrc/static_map.hpp) in Python integers: the float32
transform of each point (numpy float32 scalars, one rounding per operation in transform_point's order), one double multiply
per coordinate into fixed point, then integer arithmetic only — the range test, the shortened segment by an arithmetic
shift, the 6-connected Amanatides-Woo walk with its cross-multiplied comparisons, the per-submap hit-wins update, the
classification and the static map. The fixed point, transform and value are occupancyref's.

MUTATIONS names subtly wrong variants, each of which tests/test_static_map_cpu.py shows changes an outcome:
  y_first       at a tie between x and y the walk steps y first
  trunc         E' = O + trunc(d q / 2^16) (toward zero) instead of the floor
  free_wins     a voxel both hit and freed by one submap also counts as freed by it
  count_rays    hits and frees count rays, not submaps
  drop_skipped  skipped points are dropped from the static map too
"""
from __future__ import annotations

import math

import numpy as np

import occupancyref as O

MUTATIONS = ("y_first", "trunc", "free_wins", "count_rays", "drop_skipped")
F = O.F
ONE = O.ONE
MAX_CELLS = (1 << 31) - 1
DEFAULTS = dict(resolution=0.2, max_range=100.0, sensor_origin=(0.0, 0.0, 0.0), ray_fraction=0.85, min_frees=2,
                dynamic_thresh=0.4)
Refused = O.Refused


def params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    return p


def prepare(p):
    res = float(p["resolution"])
    if not (math.isfinite(res) and res > 0):
        raise Refused(-1, "resolution")
    S = 65536.0 / res
    if not math.isfinite(S):
        raise Refused(-1, "resolution")
    mr = float(p["max_range"])
    if not (math.isfinite(mr) and mr > 0):
        raise Refused(-1, "max_range")
    Rd = mr * S
    if not (Rd <= O.RANGE_LIMIT):
        raise Refused(-1, "max_range / resolution")
    if not all(math.isfinite(float(v)) for v in p["sensor_origin"]):
        raise Refused(-1, "sensor_origin")
    rf = float(p["ray_fraction"])
    if not (rf > 0 and rf <= 1):
        raise Refused(-1, "ray_fraction")
    mf = int(p["min_frees"])
    if mf < 1:
        raise Refused(-1, "min_frees")
    dt = float(p["dynamic_thresh"])
    if not (dt >= 0 and dt <= 1):
        raise Refused(-1, "dynamic_thresh")
    q = int(round(rf * 65536.0))  # round-half-even, as rint
    if q < 1:
        raise Refused(-1, "ray_fraction")
    return dict(S=S, R=math.floor(Rd), q=q, min_frees=mf, dyn=int(round(dt * 100.0)))


def origin(c, p, T):
    so = [O.F32(float(v)) for v in p["sensor_origin"]]
    o = O.transform(T, *so)
    V = [O.fixed(v, c["S"], O.ORIGIN_LIMIT) for v in o]
    if any(v is None for v in V):
        raise Refused(-2, "origin")
    return V


def ray(c, o, e, mut=()):
    """None when skipped, else (endpoint voxel (x, y, z), E' (fixed point))."""
    X = [O.fixed(v, c["S"], O.COORD_LIMIT) for v in e]
    if any(v is None for v in X):
        return None
    d = [X[a] - o[a] for a in range(3)]
    R = c["R"]
    if any(abs(v) > R for v in d) or d[0] * d[0] + d[1] * d[1] + d[2] * d[2] > R * R:
        return None
    q = c["q"]
    if "trunc" in mut:
        end = tuple(o[a] + (abs(d[a] * q) >> F) * (1 if d[a] >= 0 else -1) for a in range(3))
    else:
        end = tuple(o[a] + ((d[a] * q) >> F) for a in range(3))
    return tuple(v >> F for v in X), end


def walk(a, b, mut=()):
    """The voxels of the 6-connected walk from a to b (fixed point), both ends included."""
    c = [v >> F for v in a]
    e = [v >> F for v in b]
    u = [abs(b[k] - a[k]) for k in range(3)]
    s = [1 if e[k] > c[k] else -1 for k in range(3)]
    n = [abs(e[k] - c[k]) for k in range(3)]
    order = (1, 0, 2) if "y_first" in mut else (0, 1, 2)
    out = [tuple(c)]
    while sum(n) > 0:
        bnd = [((c[k] + 1) * ONE - a[k]) if s[k] > 0 else (a[k] - c[k] * ONE) for k in range(3)]
        best = None
        for k in order:
            if n[k] == 0:
                continue
            assert 0 <= bnd[k] <= u[k]  # the header's bound: B_a <= |u_a| on an axis with a step left
            if best is None or bnd[k] * u[best] < bnd[best] * u[k]:
                best = k
        c[best] += s[best]
        n[best] -= 1
        out.append(tuple(c))
    return out


def dynamic(h, f, c):
    return f >= c["min_frees"] and O.value(h, f) <= c["dyn"]


def box_cells(lo, hi):
    """The box's cell count, or None when it has more than 2^31 - 1 cells."""
    n = 1
    for a in range(3):
        w = hi[a] - lo[a] + 1
        if w < 1:
            return None
        n *= w
    return n if n <= MAX_CELLS else None


def build(submaps, p=None, mut=()):
    """submaps: list of (points (n, >= 3) float32, pose 4x4 float64). Returns a dict: lo, dims, n_rays, n_skipped, ijk
    ((V, 3) int32, rank order), hits, frees (uint32), dynamic (uint8), keep (per point, bool), offsets (n_sub + 1),
    n_voxels, n_dynamic, n_points, n_static, and the assembled points (M, 4) float32."""
    p = params(**(p or {}))
    c = prepare(p)
    if not submaps:
        raise Refused(-4, "no submaps")
    Ts = [O.pose_f(P) for _, P in submaps]
    Os = [origin(c, p, T) for T in Ts]
    rays = []
    moved = []
    n_rays = n_skipped = 0
    for (pts, _), T, o in zip(submaps, Ts, Os):
        rs = []
        for row in np.asarray(pts, dtype=np.float32):
            e = O.transform(T, row[0], row[1], row[2])
            moved.append((e[0], e[1], e[2], np.float32(row[3]) if len(row) > 3 else np.float32(0)))
            r = ray(c, o, e, mut)
            rs.append(r)
            if r is None:
                n_skipped += 1
            else:
                n_rays += 1
        rays.append(rs)
    ends = [r[0] for rs in rays for r in rs if r is not None]
    if ends:
        lo = tuple(min(v[a] for v in ends) for a in range(3))
        hi = tuple(max(v[a] for v in ends) for a in range(3))
        if box_cells(lo, hi) is None:
            raise Refused(-3, "box")
        dims = tuple(hi[a] - lo[a] + 1 for a in range(3))
    else:
        lo, dims = (0, 0, 0), (0, 0, 0)

    def lin(v):
        return ((v[2] - lo[2]) * dims[1] + (v[1] - lo[1])) * dims[0] + (v[0] - lo[0])

    occupied = sorted(set(ends), key=lin)
    rank = {v: r for r, v in enumerate(occupied)}
    hits = np.zeros(len(occupied), dtype=np.uint32)
    frees = np.zeros(len(occupied), dtype=np.uint32)
    for rs, o in zip(rays, Os):
        hit, fre = {}, {}
        for r in rs:
            if r is None:
                continue
            hit[r[0]] = hit.get(r[0], 0) + 1
            crossed = {v for v in walk(tuple(o), r[1], mut) if v in rank}
            for v in crossed:
                fre[v] = fre.get(v, 0) + 1
        for v, m in hit.items():
            hits[rank[v]] += m if "count_rays" in mut else 1
        for v, m in fre.items():
            if v in hit and "free_wins" not in mut:
                continue
            frees[rank[v]] += m if "count_rays" in mut else 1
    dyn = np.array([dynamic(int(h), int(f), c) for h, f in zip(hits, frees)], dtype=np.uint8)
    keep, offsets = [], [0]
    for rs in rays:
        for r in rs:
            if r is None:
                keep.append("drop_skipped" not in mut)
            else:
                keep.append(not dyn[rank[r[0]]])
        offsets.append(offsets[-1] + sum(keep[len(keep) - len(rs):]))
    return dict(lo=lo, dims=dims, n_rays=n_rays, n_skipped=n_skipped,
                ijk=np.array(occupied, dtype=np.int32).reshape(-1, 3), hits=hits, frees=frees, dynamic=dyn,
                keep=np.array(keep, dtype=bool), offsets=np.array(offsets, dtype=np.int64), n_voxels=len(occupied),
                n_dynamic=int(dyn.sum()), n_points=len(keep), n_static=int(sum(keep)),
                points=np.array(moved, dtype=np.float32).reshape(-1, 4), p=p, c=c)
