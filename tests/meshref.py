"""An exact replay of the surface mesh of b200sm_build_mesh (csrc/mesh.hpp) in Python integers and IEEE doubles (Python
floats, one rounding per operation in the header's order): the rays, walks and box are staticmapref's; then the band
segment, the signed distances, the fused sums and weights, the ACTIVE cells, the surface-nets vertices and the faces.

MUTATIONS names subtly wrong variants, each of which tests/test_mesh_cpu.py shows changes an outcome:
  zero_neg           a sum of exactly 0 is NEG
  ceil_off           the band offset rounds up (ceil) instead of down
  centre_vertex      the vertex sits at the cell's centre instead of the crossings' mean
  flip_y             the quads of y-edges are wound the other way
  three_active       an edge whose four cells include exactly three ACTIVE ones gives the triangle of those three
  weight_per_submap  a voxel's weight counts the submaps that walk it, not the rays
"""
from __future__ import annotations

import math

import numpy as np

import occupancyref as O
import staticmapref as SM

MUTATIONS = ("zero_neg", "ceil_off", "centre_vertex", "flip_y", "three_active", "weight_per_submap")
F = O.F
ONE = O.ONE
MAX_CELLS = SM.MAX_CELLS
DEFAULTS = dict(resolution=0.2, truncation=0.6, max_range=100.0, sensor_origin=(0.0, 0.0, 0.0), min_weight=2)
Refused = O.Refused
EDGES = ((0, 1, 0), (2, 3, 0), (4, 5, 0), (6, 7, 0), (0, 2, 1), (1, 3, 1), (4, 6, 1), (5, 7, 1),
         (0, 4, 2), (1, 5, 2), (2, 6, 2), (3, 7, 2))  # (p, q, axis) in the contract's order


def params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    return p


def prepare(p):
    smp = SM.params(resolution=p["resolution"], max_range=p["max_range"], sensor_origin=p["sensor_origin"], ray_fraction=1.0)
    c = SM.prepare(smp)
    ratio = float(p["truncation"]) / float(p["resolution"])
    if not (math.isfinite(float(p["truncation"])) and ratio >= 1.0 and ratio <= 16.0):
        raise Refused(-1, "truncation / resolution")
    if int(p["min_weight"]) < 1:
        raise Refused(-1, "min_weight")
    T = math.floor(float(p["truncation"]) * c["S"])
    return dict(c, T=T, r=(T >> F) + 1, min_weight=int(p["min_weight"]), resolution=float(p["resolution"]), sm=smp)


def band(T, o, E, mut=()):
    """(A, B, L) of the ray o -> E, or None for a zero-length ray."""
    d = [E[a] - o[a] for a in range(3)]
    dd = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
    if dd == 0:
        return None
    L = math.sqrt(float(dd))
    k = float(T) / L
    rnd = math.ceil if "ceil_off" in mut else math.floor
    off = [rnd(float(d[a]) * k) for a in range(3)]
    B = tuple(E[a] + off[a] for a in range(3))
    A = tuple(o) if L <= float(T) else tuple(E[a] - off[a] for a in range(3))
    return A, B, L


def sdf(T, E, d, L, v):
    dot = sum((E[a] - (v[a] * ONE + ONE // 2)) * d[a] for a in range(3))
    s = math.floor(float(dot) / L)
    return max(-T, min(T, s))


def box(lo, hi, r):
    """(lower corner, dims) of the band box, or None when it has more than 2^31 - 1 voxels."""
    wlo = tuple(lo[a] - r for a in range(3))
    whi = tuple(hi[a] + r for a in range(3))
    if SM.box_cells(wlo, whi) is None:
        return None
    return wlo, tuple(whi[a] - wlo[a] + 1 for a in range(3))


def neg(s, mut=()):
    return s <= 0 if "zero_neg" in mut else s < 0


def vertex(D, ng, ijk, res, mut=()):
    if "centre_vertex" in mut:
        u = (0.5, 0.5, 0.5)
    else:
        sx = sy = sz = 0.0
        n = 0
        for p, q, axis in EDGES:
            if ng[p] == ng[q]:
                continue
            t = D[p] / (D[p] - D[q])
            sx += t if axis == 0 else float(p & 1)
            sy += t if axis == 1 else float((p >> 1) & 1)
            sz += t if axis == 2 else float((p >> 2) & 1)
            n += 1
        u = (sx / float(n), sy / float(n), sz / float(n))
    return tuple(np.float32(((float(ijk[a]) + 0.5) + u[a]) * res) for a in range(3))


def edge_cell(a, S, T, v):
    i, j, k = v
    if a == 0:
        return (i, j - 1 + S, k - 1 + T)
    if a == 1:
        return (i - 1 + T, j, k - 1 + S)
    return (i - 1 + S, j - 1 + T, k)


def quad(ids, v_neg, axis, mut=()):
    c00, c10, c01, c11 = ids
    if "flip_y" in mut and axis == 1:
        v_neg = not v_neg
    if v_neg:
        return [(c00, c10, c11), (c00, c11, c01)]
    return [(c00, c11, c10), (c00, c01, c11)]


def extract(band_voxels, sums, weights, res, min_weight, mut=()):
    """Vertices (V, 3) float32 and faces (F, 3) uint32 of band voxels given in rank order (a list of (i, j, k)), with
    their sums and weights."""
    rank = {v: r for r, v in enumerate(band_voxels)}

    def observed(v):
        r = rank.get(v)
        return r if r is not None and weights[r] >= min_weight else None

    vid, verts = {}, []
    for v in band_voxels:
        D, ng, ok = [], [], True
        for m in range(8):
            r = observed((v[0] + (m & 1), v[1] + ((m >> 1) & 1), v[2] + ((m >> 2) & 1)))
            if r is None:
                ok = False
                break
            D.append(float(sums[r]) / float(weights[r]))
            ng.append(neg(int(sums[r]), mut))
        if not ok or all(ng) or not any(ng):
            continue
        vid[v] = len(verts)
        verts.append(vertex(D, ng, v, res, mut))
    faces = []
    for v in band_voxels:
        r = observed(v)
        if r is None:
            continue
        vn = neg(int(sums[r]), mut)
        for a in range(3):
            w = observed(tuple(v[b] + (b == a) for b in range(3)))
            if w is None or neg(int(sums[w]), mut) == vn:
                continue
            cells = [edge_cell(a, m & 1, m >> 1, v) for m in range(4)]
            have = [c in vid for c in cells]
            if all(have):
                faces += quad([vid[c] for c in cells], vn, a, mut)
            elif "three_active" in mut and sum(have) == 3:
                faces.append(tuple(vid[c] for c in cells if c in vid))
    return (np.array(verts, dtype=np.float32).reshape(-1, 3), np.array(faces, dtype=np.uint32).reshape(-1, 3))


def build(submaps, p=None, mut=()):
    """submaps: list of (points (n, >= 3) float32, pose 4x4 float64). Returns a dict: lo, dims (the band box), n_points,
    n_rays, n_skipped, n_walked, ijk ((B, 3) int32, rank order), sum (int64), weight (uint32), n_band_voxels,
    n_observed_voxels, vertices (V, 3) float32, faces (F, 3) uint32, n_vertices, n_faces."""
    p = params(**(p or {}))
    c = prepare(p)
    if not submaps:
        raise Refused(-4, "no submaps")
    Ts = [O.pose_f(P) for _, P in submaps]
    Os = [SM.origin(c, c["sm"], T) for T in Ts]
    rays = []
    n_rays = n_skipped = n_points = 0
    for (pts, _), T, o in zip(submaps, Ts, Os):
        rs = []
        for row in np.asarray(pts, dtype=np.float32):
            n_points += 1
            r = SM.ray(c, o, O.transform(T, row[0], row[1], row[2]))
            if r is None:
                n_skipped += 1
            else:
                n_rays += 1
                rs.append(r)
        rays.append(rs)
    ends = [r[0] for rs in rays for r in rs]
    if ends:
        lo = tuple(min(v[a] for v in ends) for a in range(3))
        hi = tuple(max(v[a] for v in ends) for a in range(3))
        b = box(lo, hi, c["r"])
        if b is None:
            raise Refused(-3, "box")
        lo, dims = b
    else:
        lo, dims = (0, 0, 0), (0, 0, 0)
    T = c["T"]
    field = {}  # voxel -> [sum, weight, last submap]
    n_walked = 0
    for k, (rs, o) in enumerate(zip(rays, Os)):
        for _, E in rs:
            seg = band(T, o, E, mut)
            if seg is None:
                continue
            A, B, L = seg
            d = [E[a] - o[a] for a in range(3)]
            for v in SM.walk(A, B):
                assert all(lo[a] <= v[a] < lo[a] + dims[a] for a in range(3))  # the header's bound
                s = sdf(T, E, d, L, v)
                f = field.setdefault(v, [0, 0, -1])
                f[0] += s
                if "weight_per_submap" not in mut or f[2] != k:
                    f[1] += 1
                f[2] = k
                n_walked += 1

    def lin(v):
        return ((v[2] - lo[2]) * dims[1] + (v[1] - lo[1])) * dims[0] + (v[0] - lo[0])

    vox = sorted(field, key=lin)
    sums = np.array([field[v][0] for v in vox], dtype=np.int64)
    weights = np.array([field[v][1] for v in vox], dtype=np.uint32)
    verts, faces = extract(vox, sums, weights, c["resolution"], c["min_weight"], mut)
    return dict(lo=lo, dims=dims, n_points=n_points, n_rays=n_rays, n_skipped=n_skipped, n_walked=n_walked,
                ijk=np.array(vox, dtype=np.int32).reshape(-1, 3), sum=sums, weight=weights, n_band_voxels=len(vox),
                n_observed_voxels=int((weights >= c["min_weight"]).sum()), vertices=verts, faces=faces,
                n_vertices=len(verts), n_faces=len(faces), p=p, c=c)


def ply_bytes(vertices, faces):
    """The PLY file of the contract, restated with struct."""
    import struct

    head = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(vertices)}\nproperty float x\nproperty float y\n"
            f"property float z\nelement face {len(faces)}\nproperty list uchar uint vertex_indices\nend_header\n").encode()
    body = b"".join(struct.pack("<fff", *map(float, v)) for v in np.asarray(vertices, dtype=np.float32))
    body += b"".join(struct.pack("<BIII", 3, *map(int, f)) for f in np.asarray(faces, dtype=np.uint32))
    return head + body
