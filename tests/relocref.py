"""TEST INFRASTRUCTURE. A replay of the relocalisation search of b200sm_relocalize (csrc/relocalize.hpp states the
definitions) in Python integers, float64 and numpy float32: every float32 operation of a scan point's rotation is one
numpy float32 operation, rounded on its own, and every product into a cell one float64 multiply, so the tests compare the
header's host compile and the device with this replay bit for bit.

Every function takes `mut`, a set of mutation names (MUTATIONS): a replay of a subtly wrong search, used by
tests/test_relocalize_cpu.py to show that the fixtures tell it from the right one. Nothing here needs a GPU.
"""
from __future__ import annotations

import math

import numpy as np

import sessionref as S

F32 = np.float32
LIM = 1 << 30
MAX_CELLS, MAX_PYRAMID, MAX_LEAVES, MAX_ROOTS = 1 << 28, 1 << 32, 1 << 40, 1 << 32
MAX_OFFSETS, MAX_POINTS, MAX_FRONTIER = 1 << 26, (1 << 24) - 1, 1 << 26
MASK = (1 << 40) - 1
DEFAULTS = dict(resolution=0.25, z_min=0.3, z_max=3.0, yaw_steps=360, num_levels=6, min_score=0.3, top_k=4, accept_fitness=1.0)

MUTATIONS = (
    "window_closed",  # level h is the max over [i, i + 2^h] x [j, j + 2^h] instead of the half-open window
    "trunc",          # truncation toward zero instead of floor, for map cells and scan offsets
    "prune_gt",       # nodes expanded and leaves kept on score > T instead of >= T
    "tie_reversed",   # the higher leaf index wins a tie
    "clamp",          # out-of-grid reads clamped to the nearest stored cell instead of 0
)


def _floor(v, mut):
    return np.trunc(v) if "trunc" in mut else np.floor(v)


def rotations(position, quat, yaw_steps):
    """R_k (yaw_steps, 3, 3): float64 as global_yaw_rotations computes them, and their float32 casts."""
    M = S.pose_matrix(position, quat)
    out = np.zeros((yaw_steps, 3, 3))
    for k in range(yaw_steps):
        th = 2.0 * math.pi * k / yaw_steps
        c, s = math.cos(th), math.sin(th)
        Rz = ((c, -s, 0.0), (s, c, 0.0), (0.0, 0.0, 1.0))
        for r in range(3):
            for col in range(3):
                out[k, r, col] = Rz[r][0] * M[0, col] + Rz[r][1] * M[1, col] + Rz[r][2] * M[2, col]
    return out, out.astype(F32)


def project_map(map4, p, mut=()):
    """(cells (n, 2) int64 of the projected rows)"""
    inv = 1.0 / p["resolution"]
    x, y, z = (np.asarray(map4[:, c], dtype=F32) for c in range(3))
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
        zd = z.astype(np.float64)
        ok &= (p["z_min"] <= zd) & (zd <= p["z_max"])
        fx, fy = _floor(x.astype(np.float64) * inv, mut), _floor(y.astype(np.float64) * inv, mut)
        ok &= (fx >= -LIM) & (fx <= LIM) & (fy >= -LIM) & (fy <= LIM)
    return np.stack([fx[ok], fy[ok]], axis=1).astype(np.int64)


def grid_of(cells, p):
    """dict(i0, j0, W, H, L, S, TW, TH, Y) or None when no row is projected; raises ValueError at a limit."""
    if len(cells) == 0:
        return None
    i0, j0 = int(cells[:, 0].min()), int(cells[:, 1].min())
    W, H = int(cells[:, 0].max()) - i0 + 1, int(cells[:, 1].max()) - j0 + 1
    L, Y = p["num_levels"], p["yaw_steps"]
    S_ = 1 << (L - 1)
    g = dict(i0=i0, j0=j0, W=W, H=H, L=L, S=S_, TW=-(-W // S_), TH=-(-H // S_), Y=Y)
    if W * H > MAX_CELLS:
        raise ValueError("cells")
    if sum((W + (1 << h) - 1) * (H + (1 << h) - 1) for h in range(L)) > MAX_PYRAMID:
        raise ValueError("pyramid")
    if Y * W * H >= MAX_LEAVES:
        raise ValueError("leaves")
    if Y * g["TW"] * g["TH"] > MAX_ROOTS:
        raise ValueError("roots")
    return g


def _window_max(g0, W, H, h, size):
    """level h's stored array (rows j from 1 - 2^h, columns i from 1 - 2^h) as the max of g_0 over size x size windows"""
    e = (1 << h) - 1
    pad = np.zeros((H + e + size, W + e + size), dtype=np.uint8)
    pad[e:e + H, e:e + W] = g0
    out = np.zeros((H + e, W + e), dtype=np.uint8)
    for b in range(size):
        for a in range(size):
            np.maximum(out, pad[b:b + H + e, a:a + W + e], out=out)
    return out


def pyramid(map4, p, mut=()):
    """(grid, [level arrays]) or (None, []) for an empty grid"""
    cells = project_map(map4, p, mut)
    g = grid_of(cells, p)
    if g is None:
        return None, []
    W, H = g["W"], g["H"]
    g0 = np.zeros((H, W), dtype=np.uint8)
    g0[cells[:, 1] - g["j0"], cells[:, 0] - g["i0"]] = 1
    levels = [g0]
    for h in range(1, g["L"]):
        if "window_closed" in mut:
            levels.append(_window_max(g0, W, H, h, (1 << h) + 1))
            continue
        s, e, pe = 1 << (h - 1), (1 << h) - 1, (1 << (h - 1)) - 1
        prev = levels[-1]
        pad = np.zeros((H + e + s, W + e + s), dtype=np.uint8)  # row r, column c hold cell (c - e, r - e)
        pad[e - pe:e - pe + prev.shape[0], e - pe:e - pe + prev.shape[1]] = prev
        lh, lw = H + e, W + e
        levels.append(np.maximum(np.maximum(pad[:lh, :lw], pad[:lh, s:s + lw]), np.maximum(pad[s:s + lh, :lw], pad[s:s + lh, s:s + lw])))
    return g, levels


def offsets(scan4, rot_f, z0, p, mut=()):
    """(offs (Y, m, 2) int64, m)"""
    inv = 1.0 / p["resolution"]
    x, y, z = (np.asarray(scan4[:, c], dtype=F32) for c in range(3))

    def row(R, r):
        return (R[r, 0] * x + R[r, 1] * y) + R[r, 2] * z  # float32, one rounding per operation

    with np.errstate(invalid="ignore", over="ignore"):
        hz = row(rot_f[0], 2).astype(np.float64) + z0
        keep = (p["z_min"] <= hz) & (hz <= p["z_max"])
        Y = len(rot_f)
        out = np.zeros((Y, int(keep.sum()), 2), dtype=np.int64)
        for k in range(Y):
            for c in range(2):
                f = _floor(row(rot_f[k], c)[keep].astype(np.float64) * inv, mut)
                f = np.where(np.isnan(f) | (f < -LIM), -LIM, np.where(f > LIM, LIM, f))
                out[k, :, c] = f.astype(np.int64)
    return out, int(keep.sum())


def scores(levels, g, offs, h, nodes, mut=()):
    """score_h of nodes (N, 3) int64 (k, i, j)"""
    nodes = np.asarray(nodes, dtype=np.int64).reshape(-1, 3)
    if len(nodes) == 0 or offs.shape[1] == 0:
        return np.zeros(len(nodes), dtype=np.int64)
    lvl = levels[h]
    e = (1 << h) - 1
    o = offs[nodes[:, 0]]  # (N, m, 2)
    c = nodes[:, 1:2] + o[:, :, 0] + e
    r = nodes[:, 2:3] + o[:, :, 1] + e
    lh, lw = lvl.shape
    if "clamp" in mut:
        return lvl[np.clip(r, 0, lh - 1), np.clip(c, 0, lw - 1)].astype(np.int64).sum(axis=1)
    ok = (c >= 0) & (c < lw) & (r >= 0) & (r < lh)
    return np.where(ok, lvl[np.where(ok, r, 0), np.where(ok, c, 0)], 0).astype(np.int64).sum(axis=1)


def key(score, idx, mut=()):
    return (int(score) << 40) | (int(idx) if "tie_reversed" in mut else MASK - int(idx))


def key_index(k, mut=()):
    return (k & MASK) if "tie_reversed" in mut else MASK - (k & MASK)


def leaf_index(g, k, i, j):
    return (int(k) * g["H"] + int(j)) * g["W"] + int(i)


def tile_of(g, i, j):
    return (int(j) // g["S"]) * g["TW"] + int(i) // g["S"]


def children(g, nodes, h):
    """children of level-h nodes (dj outer, di inner), kept inside the grid, in node order"""
    s = 1 << (h - 1)
    out = []
    for k, i, j in np.asarray(nodes, dtype=np.int64).reshape(-1, 3):
        for c in range(4):
            ci, cj = i + (c & 1) * s, j + (c >> 1) * s
            if ci < g["W"] and cj < g["H"]:
                out.append((k, ci, cj))
    return np.array(out, dtype=np.int64).reshape(-1, 3)


def roots(g):
    r = np.arange(g["Y"] * g["TW"] * g["TH"], dtype=np.int64)
    per = g["TW"] * g["TH"]
    rem = r % per
    return np.stack([r // per, (rem % g["TW"]) * g["S"], (rem // g["TW"]) * g["S"]], axis=1)


def t0_of(min_score, m):
    return max(1, math.ceil(min_score * m))


def rank(tile_keys, t0, top_k):
    t = [q for q, k in tile_keys.items() if (k >> 40) >= t0]
    t.sort(key=lambda q: -tile_keys[q])
    return t[:top_k]


def search(levels, g, offs, m, p, exhaustive=False, mut=()):
    """dict(t0, t, nodes (16), tiles, keys) or ValueError("frontier") at the frontier cap"""
    res = dict(t0=t0_of(p["min_score"], m), t=0, nodes=[0] * 16, tiles=[], keys=[])
    if m == 0 or g is None:
        return res
    L, top_k = g["L"], p["top_k"]
    leaf_keys = {}

    def fold(nodes, sc, T):
        for (k, i, j), s in zip(nodes, sc):
            if (s > T) if "prune_gt" in mut else (s >= T):
                q = tile_of(g, i, j)
                leaf_keys[q] = max(leaf_keys.get(q, 0), key(s, leaf_index(g, k, i, j), mut))

    if exhaustive:
        Y, W, H = g["Y"], g["W"], g["H"]
        kk, jj, ii = np.meshgrid(np.arange(Y), np.arange(H), np.arange(W), indexing="ij")
        nodes = np.stack([kk.ravel(), ii.ravel(), jj.ravel()], axis=1)
        fold(nodes, scores(levels, g, offs, 0, nodes, mut), -1 if "prune_gt" in mut else 0)
        res["t"] = res["t0"]
        res["nodes"][0] = len(nodes)
    else:
        R = roots(g)
        res["nodes"][L - 1] = len(R)
        rs = scores(levels, g, offs, L - 1, R, mut)
        root_keys = {}
        for (k, i, j), s in zip(R, rs):
            q = tile_of(g, i, j)
            root_keys[q] = max(root_keys.get(q, 0), key(s, leaf_index(g, k, i, j), mut))
        starts = sorted(root_keys, key=lambda q: -root_keys[q])[:top_k]
        dives = []
        for q in starts:
            idx = key_index(root_keys[q], mut)
            node = np.array([[idx // (g["W"] * g["H"]), idx % g["W"], (idx // g["W"]) % g["H"]]])
            score = root_keys[q] >> 40
            for h in range(L - 1, 0, -1):
                ch = children(g, node, h)
                sc = scores(levels, g, offs, h - 1, ch, mut)
                ks = [key(s, leaf_index(g, *c), mut) for c, s in zip(ch, sc)]
                b = int(np.argmax(ks))
                node, score = ch[b:b + 1], ks[b] >> 40
            dives.append(score)
        T = res["t0"] if len(dives) < top_k else max(res["t0"], sorted(dives, reverse=True)[top_k - 1])
        res["t"] = T

        def keep(sc):
            return (sc > T) if "prune_gt" in mut else (sc >= T)

        if L == 1:
            fold(R, rs, T)
        else:
            front, fs, h_front = R, rs, L - 1
            for h in range(L - 2, -1, -1):
                ch = children(g, front[keep(fs)], h_front)
                if len(ch) > MAX_FRONTIER:
                    raise ValueError("frontier")
                res["nodes"][h] = len(ch)
                front, h_front = ch, h
                fs = scores(levels, g, offs, h, front, mut)
                if h == 0:
                    fold(front, fs, T)
    res["tiles"] = rank(leaf_keys, res["t0"], top_k)
    res["keys"] = [leaf_keys[q] for q in res["tiles"]]
    return res
