"""A ray-cast drive over analytic outdoor terrain, every point labelled with the solid it hit: flat ground, a 10 degree and a
30 degree ramp beside the road, a 0.2 m curb, a wall, and a bridge deck 3 m above the road (an overhang the sensor drives
under). A 32-line sensor 1.8 m above the road drives along y = 0 from x = 0 to x = 50, one scan per metre; each scan is a
submap in the sensor frame at its exact pose. Solids are convex (an intersection of half-spaces), so each ray is clipped
against each exactly (Cyrus-Beck) and the nearest entry wins."""
import math

import numpy as np

HEIGHT = 1.8
TAN10, TAN30 = math.tan(math.radians(10.0)), math.tan(math.radians(30.0))
GROUND, RAMP10, RAMP30, CURB, WALL, DECK = range(6)
NAMES = ("ground", "ramp10", "ramp30", "curb", "wall", "deck")


def _box(x0, x1, y0, y1, z0, z1):
    return [((1, 0, 0), x1), ((-1, 0, 0), -x0), ((0, 1, 0), y1), ((0, -1, 0), -y0), ((0, 0, 1), z1), ((0, 0, -1), -z0)]


# label -> half-spaces n . p <= c
SOLIDS = [
    (GROUND, _box(-1e3, 1e3, -1e3, 1e3, -10.0, 0.0)),
    # rising with y from the road's edge at y = 3 to a 1.06 m plateau at y = 9 (the plateau ends at y = 12)
    (RAMP10, _box(5.0, 25.0, 3.0, 12.0, -10.0, 6.0 * TAN10)[:5] + [((0, 0, -1), 10.0), ((0, -TAN10, 1), -3.0 * TAN10)]),
    # rising with -y from y = -3 to 3.46 m at y = -9
    (RAMP30, _box(5.0, 25.0, -9.0, -3.0, -10.0, 6.0 * TAN30) + [((0, TAN30, 1), -3.0 * TAN30)]),
    (CURB, _box(35.0, 55.0, 3.0, 10.0, -10.0, 0.2)),
    (WALL, _box(35.0, 55.0, -5.0, -4.6, -10.0, 3.0)),
    (DECK, _box(28.0, 32.0, -8.0, 8.0, 3.0, 3.3)),
]


def surface(x, y):
    """The terrain's analytic height under (x, y) ignoring the deck (an overhang)."""
    z = np.zeros(np.broadcast(x, y).shape)
    inx = (x >= 5.0) & (x <= 25.0)
    z = np.where(inx & (y >= 3.0) & (y <= 12.0), np.minimum(y - 3.0, 6.0) * TAN10, z)
    z = np.where(inx & (y >= -9.0) & (y <= -3.0), (-3.0 - y) * TAN30, z)
    z = np.where((x >= 35.0) & (x <= 55.0) & (y >= 3.0) & (y <= 10.0), 0.2, z)
    z = np.where((x >= 35.0) & (x <= 55.0) & (y >= -5.0) & (y <= -4.6), 3.0, z)
    return z


def _rays(lines=32, azimuths=1800, lo=-22.0, hi=9.0):
    el = np.radians(np.linspace(lo, hi, lines))
    az = np.radians(np.arange(azimuths) * (360.0 / azimuths))
    E, A = np.meshgrid(el, az, indexing="ij")
    return np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], axis=-1).reshape(-1, 3)


def scan(sx, sy=0.0, max_range=40.0):
    """(points (N, 3) float32 in the sensor frame, labels (N,)) from a sensor at (sx, sy, HEIGHT)."""
    d = _rays()
    o = np.array([sx, sy, HEIGHT])
    best = np.full(len(d), np.inf)
    label = np.full(len(d), -1)
    for lab, planes in SOLIDS:
        t0 = np.zeros(len(d))
        t1 = np.full(len(d), np.inf)
        ok = np.ones(len(d), dtype=bool)
        for n, c in planes:
            n = np.asarray(n, dtype=np.float64)
            nd = d @ n
            num = c - o @ n
            with np.errstate(divide="ignore", invalid="ignore"):
                t = num / nd
            t0 = np.where(nd < 0, np.maximum(t0, t), t0)
            t1 = np.where(nd > 0, np.minimum(t1, t), t1)
            ok &= ~((nd == 0) & (num < 0))
        hit = ok & (t0 <= t1) & (t0 > 0) & (t0 < best)
        best = np.where(hit, t0, best)
        label = np.where(hit, lab, label)
    keep = best <= max_range
    pts = (d[keep] * best[keep, None]).astype(np.float32)
    return pts, label[keep]


def pose(sx, sy=0.0):
    P = np.eye(4)
    P[:3, 3] = (sx, sy, HEIGHT)
    return P


def drive(step=1.0, x_end=50.0):
    """[(points, pose)], [labels] over the drive."""
    subs, labels = [], []
    for sx in np.arange(0.0, x_end + 1e-9, step):
        p, lab = scan(float(sx))
        subs.append((p, pose(float(sx))))
        labels.append(lab)
    return subs, labels
