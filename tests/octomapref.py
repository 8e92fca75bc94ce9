"""An exact replay of the OctoMap of b200sm_build_octomap (csrc/octomap.hpp) in Python integers: the voxel states from the
static map's rays, walks and counts (staticmapref), the tree built level by level from dicts of keys (not from pointers,
as the host compile builds it), the .bt encoder, and an independent .bt decoder that reads a file back into leaves.

MUTATIONS names subtly wrong variants, each of which tests/test_octomap_cpu.py shows changes an outcome:
  swap_codes       FREE leaves written as 2 and OCCUPIED leaves as 1
  no_prune         8 leaf children of one state are not collapsed
  child_axis       the child index takes x from bit 2 and z from bit 0
  size_no_leaves   the header's size counts inner nodes only
"""
from __future__ import annotations


import numpy as np

import staticmapref as R

MUTATIONS = ("swap_codes", "no_prune", "child_axis", "size_no_leaves")
UNKNOWN, FREE, OCCUPIED, INNER = 0, 1, 2, 3
DEPTH = 16
KEY = 32768
Refused = R.Refused


def resolution_exact(res):
    return float("%g" % res) == res


def header(size, res):
    return ("# Octomap OcTree binary file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
            "id OcTree\nsize %d\nres %g\ndata\n" % (size, res)).encode()


def states(submaps, p=None):
    """The box and its voxel states: dict(lo, dims, states (D, H, W) uint8, n_rays, n_skipped, n_dynamic), or Refused
    (-3 box, -5 key range, -6 resolution, and the static map's)."""
    sm = R.build(submaps, p)  # refuses what the static map refuses (a box over 2^31 - 1 voxels included)
    c, p = sm["c"], sm["p"]
    if not resolution_exact(float(p["resolution"])):
        raise Refused(-6, "resolution")
    Ts = [R.O.pose_f(P) for _, P in submaps]
    Os = [R.origin(c, p, T) for T in Ts]
    walks, pts = [], []
    for (pts_k, _), T, o in zip(submaps, Ts, Os):
        any_ray = False
        for row in np.asarray(pts_k, dtype=np.float32):
            r = R.ray(c, o, R.O.transform(T, row[0], row[1], row[2]))
            if r is None:
                continue
            any_ray = True
            pts.append(r[0])
            walks.append((tuple(o), r[1]))
        if any_ray:
            pts.append(tuple(v >> R.F for v in o))
    if not walks:
        return dict(lo=(0, 0, 0), dims=(0, 0, 0), states=np.zeros((0, 0, 0), np.uint8), n_rays=0, n_skipped=sm["n_skipped"],
                    n_dynamic=0)
    lo = tuple(min(v[a] for v in pts) for a in range(3))
    hi = tuple(max(v[a] for v in pts) for a in range(3))
    if R.box_cells(lo, hi) is None:
        raise Refused(-3, "box")
    if any(lo[a] < -KEY or hi[a] > KEY - 1 for a in range(3)):
        raise Refused(-5, "key range")
    dims = tuple(hi[a] - lo[a] + 1 for a in range(3))
    S = np.zeros(dims[::-1], dtype=np.uint8)
    for o, e in walks:
        for x, y, z in R.walk(o, e):
            S[z - lo[2], y - lo[1], x - lo[0]] = FREE
    for (x, y, z), d in zip(map(tuple, sm["ijk"].tolist()), sm["dynamic"]):
        S[z - lo[2], y - lo[1], x - lo[0]] = FREE if d else OCCUPIED
    return dict(lo=lo, dims=dims, states=S, n_rays=sm["n_rays"], n_skipped=sm["n_skipped"], n_dynamic=int(sm["n_dynamic"]))


def child_index(kx, ky, kz, l, mut=()):
    b = l - 1
    bx, by, bz = (kx >> b) & 1, (ky >> b) & 1, (kz >> b) & 1
    if "child_axis" in mut:
        bx, bz = bz, bx
    return bx | (by << 1) | (bz << 2)


def tree(lo, S, mut=()):
    """levels[l]: dict key-triple >> l -> code (FREE / OCCUPIED leaf, INNER), l = 0 .. 16, from the known voxels."""
    D, H, W = S.shape
    zz, yy, xx = np.nonzero(S)
    level = {(int(x) + lo[0] + KEY, int(y) + lo[1] + KEY, int(z) + lo[2] + KEY): int(S[z, y, x]) for z, y, x in zip(zz, yy, xx)}
    levels = [level]
    for l in range(1, DEPTH + 1):
        groups = {}
        for k, v in levels[-1].items():
            groups.setdefault((k[0] >> 1, k[1] >> 1, k[2] >> 1), []).append(v)
        nxt = {}
        for k, vs in groups.items():
            leaf = len(vs) == 8 and vs[0] in (FREE, OCCUPIED) and all(v == vs[0] for v in vs)
            nxt[k] = vs[0] if leaf and "no_prune" not in mut else INNER
        levels.append(nxt)
    return levels


def encode(lo, S, res, mut=()):
    """The .bt bytes of a labelled box (S indexed [z, y, x]) and the counts dict(inner, occupied_leaves, free_leaves, size)."""
    levels = tree(lo, S, mut)
    data = bytearray()
    counts = dict(inner=0, occupied_leaves=0, free_leaves=0)

    def children(l, k):
        codes, keys = [UNKNOWN] * 8, [None] * 8
        for i in range(8):
            ck = (2 * k[0] + (i & 1), 2 * k[1] + ((i >> 1) & 1), 2 * k[2] + ((i >> 2) & 1))
            j = child_index(ck[0] << (l - 1), ck[1] << (l - 1), ck[2] << (l - 1), l, mut)  # full keys
            codes[j], keys[j] = levels[l - 1].get(ck, UNKNOWN), ck
        return codes, keys

    def node(l, k):
        codes, keys = children(l, k)
        counts["inner"] += 1
        b = [0, 0]
        for i, v in enumerate(codes):
            if l == 1 and v == INNER:
                raise AssertionError("a voxel is not inner")
            w = v
            if "swap_codes" in mut and v in (FREE, OCCUPIED):
                w = FREE + OCCUPIED - v
            b[i // 4] |= w << (2 * (i % 4))
            if v == OCCUPIED:
                counts["occupied_leaves"] += 1
            elif v == FREE:
                counts["free_leaves"] += 1
        data.extend(b)
        for i, v in enumerate(codes):
            if v == INNER:
                node(l - 1, keys[i])

    if levels[DEPTH]:
        node(DEPTH, (0, 0, 0))
    size = counts["inner"] + (0 if "size_no_leaves" in mut else counts["occupied_leaves"] + counts["free_leaves"])
    counts["size"] = counts["inner"] + counts["occupied_leaves"] + counts["free_leaves"]
    return header(size, res) + bytes(data), counts


def build(submaps, p=None, mut=()):
    """states() and the file: dict(lo, dims, states, n_rays, n_skipped, n_dynamic, bytes, inner, occupied_leaves,
    free_leaves, size, n_occupied, n_free)."""
    g = states(submaps, p)
    res = float(R.params(**(p or {}))["resolution"])
    g["bytes"], counts = encode(g["lo"], g["states"], res, mut)
    g.update(counts)
    g["n_occupied"] = int((g["states"] == OCCUPIED).sum())
    g["n_free"] = int((g["states"] == FREE).sum())
    return g


def decode(data):
    """An independent reader of a .bt file: (resolution, size, leaves) with leaves a list of (level, kx, ky, kz, state)
    (the keys of a level-l leaf are its lowest voxel's). Raises ValueError on a malformed file."""
    lines = []
    pos = 0
    while True:
        e = data.index(b"\n", pos)
        line = data[pos:e].decode()
        pos = e + 1
        if line.startswith("#"):
            continue
        lines.append(line)
        if line == "data":
            break
    fields = dict(l.split(" ", 1) for l in lines[:-1])
    if fields.get("id") != "OcTree":
        raise ValueError("not an OcTree")
    size, res = int(fields["size"]), float(fields["res"])
    leaves = []
    nodes = [0]

    def read(l, k):
        nonlocal pos
        b0, b1 = data[pos], data[pos + 1]
        pos += 2
        codes = [(b0 >> (2 * i)) & 3 for i in range(4)] + [(b1 >> (2 * i)) & 3 for i in range(4)]
        for i, v in enumerate(codes):
            if v == UNKNOWN:
                continue
            nodes[0] += 1
            ck = (2 * k[0] + (i & 1), 2 * k[1] + ((i >> 1) & 1), 2 * k[2] + ((i >> 2) & 1))
            if v == INNER:
                if l == 1:
                    raise ValueError("an inner voxel")
                read(l - 1, ck)
            else:
                leaves.append((l - 1, ck[0] << (l - 1), ck[1] << (l - 1), ck[2] << (l - 1), v))

    if size:
        nodes[0] = 1
        read(DEPTH, (0, 0, 0))
    if pos != len(data):
        raise ValueError("trailing bytes")
    if nodes[0] != size:
        raise ValueError("size %d, nodes %d" % (size, nodes[0]))
    return res, size, leaves


def expand(leaves, lo, dims):
    """The (D, H, W) state grid of the box from decoded leaves, leaf by leaf; a leaf voxel outside the box raises."""
    S = np.zeros(dims[::-1], dtype=np.uint8)
    for l, kx, ky, kz, v in leaves:
        n = 1 << l
        x0, y0, z0 = kx - KEY - lo[0], ky - KEY - lo[1], kz - KEY - lo[2]
        if x0 < 0 or y0 < 0 or z0 < 0 or x0 + n > dims[0] or y0 + n > dims[1] or z0 + n > dims[2]:
            raise ValueError("a leaf outside the box")
        S[z0:z0 + n, y0:y0 + n, x0:x0 + n] = v
    return S
