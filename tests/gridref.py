"""Plain CPU references of the grid builders and cell lookups (voxel map K3, VoxelGrid K4, exact-NN grid K6/K8, GICP
k-NN K5), written from the algorithm, and seeded generators of the clouds where grid kernels go wrong.

float32 where the kernels' result is defined by float32 arithmetic (leaf geometry, leaf indices, squared distances),
float64 where the kernels accumulate in float64 (moments, centroids). Nothing here needs a GPU.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32
INT32_MAX = 2**31 - 1
U64 = 2.0**-53  # unit roundoff of float64
SCAN_TILE_WORDS = 2048  # words per tile of the rank-index scan (grid_index.cu: 256 threads x 8)
SCAN_BLOCK_TILES = 1024  # tile sums one pass of scan_tile_sums_kernel covers
PAGE_CELLS = 1024  # cells per page of VoxelGrid's sparse index (voxelgrid.cu)
SHIFTS = ((3000.0, -4500.0, 120.0), (-2.0e4, 1.0e4, 0.0))


# ---- grid geometry --------------------------------------------------------------------------------------------------
def finite_rows(points) -> np.ndarray:
    p = np.asarray(points)
    return np.isfinite(p[:, :3]).all(axis=1)


def leaf_geometry(points, leaf):
    """PCL voxel-grid geometry as make_grid_geom computes it: bounds of the finite points, float32 products, int64 casts.
    Returns None when the cloud has no finite point, else a dict; dict["overflow"] says the int32 guard refused it."""
    p = np.asarray(points, dtype=F32)[:, :3]
    p = p[finite_rows(p)]
    if len(p) == 0:
        return None
    mn, mx = p.min(axis=0), p.max(axis=0)
    leaf = F32(leaf)
    inv = F32(1.0) / leaf
    with np.errstate(over="ignore"):
        span = [F32(F32(mx[a] - mn[a]) * inv) for a in range(3)]
        # a float product of 2^31 or more (inf near FLT_MAX), or a bound whose leaf index is not an int, overflows the
        # grid before any cast
        if not all(s < 2.0**31 and abs(F32(mn[a] * inv)) < 2.0**31 and abs(F32(mx[a] * inv)) < 2.0**31
                   for a, s in enumerate(span)):
            return dict(leaf=leaf, inv_leaf=inv, mn=mn, mx=mx, dxyz=None, overflow=True)
    d = [int(s) + 1 for s in span]  # float product, truncating int64 cast
    g = dict(leaf=leaf, inv_leaf=inv, mn=mn, mx=mx, dxyz=tuple(d), overflow=d[0] * d[1] * d[2] > INT32_MAX)
    if g["overflow"]:
        return g
    min_b = np.array([int(math.floor(F32(mn[a] * inv))) for a in range(3)], dtype=np.int64)
    max_b = np.array([int(math.floor(F32(mx[a] * inv))) for a in range(3)], dtype=np.int64)
    div_b = max_b - min_b + 1
    n_cells = int(div_b[0] * div_b[1] * div_b[2])
    g.update(min_b=min_b, max_b=max_b, div_b=div_b, mul=np.array([1, div_b[0], div_b[0] * div_b[1]], dtype=np.int64),
             n_cells=n_cells, n_words=(n_cells + 31) // 32, overflow=n_cells > INT32_MAX)
    return g


def leaf_indices(points, g) -> np.ndarray:
    """Build-side leaf index of each point, (int)(floorf(x * inv_leaf) - (float)min_b) per axis; -1 for non-finite rows."""
    p = np.asarray(points, dtype=F32)[:, :3]
    ok = finite_rows(p)
    out = np.full(len(p), -1, dtype=np.int64)
    q = p[ok]
    ijk = [(np.floor(q[:, a] * g["inv_leaf"]) - F32(g["min_b"][a])).astype(np.int64) for a in range(3)]
    out[ok] = ijk[0] + ijk[1] * g["mul"][1] + ijk[2] * g["mul"][2]
    return out


def lookup_ref(x, leaf) -> np.ndarray:
    """The solver's cell of a transformed coordinate: floor(float32(x) / float32(leaf)) with an IEEE division."""
    return np.floor(np.asarray(x, dtype=F32) / F32(leaf)).astype(np.int64)


def build_ref(x, leaf) -> np.ndarray:
    """The builder's cell of a coordinate: floor(float32(x) * (1 / float32(leaf)))."""
    return np.floor(np.asarray(x, dtype=F32) * (F32(1.0) / F32(leaf))).astype(np.int64)


# ---- VoxelGrid ------------------------------------------------------------------------------------------------------
def _with_intensity(points) -> np.ndarray:
    p = np.asarray(points, dtype=F32)
    if p.shape[1] >= 4:
        return np.ascontiguousarray(p[:, :4])
    return np.concatenate([p[:, :3], np.zeros((len(p), 1), F32)], axis=1)


def voxelgrid_ref(points, leaf):
    """pcl::VoxelGrid centroids: one float64 mean of (x, y, z, intensity) per occupied leaf, ascending leaf index,
    non-finite rows dropped. Returns (centroids (M, 4) float64, err (M, 4)) where err bounds how far any float64
    summation order (the kernel's atomics) can move the mean: (n + 1) * 2^-53 * mean|value|, doubled for this side's own
    sum. On int32 overflow PCL returns the input unchanged: (input as float32 (N, 4), None)."""
    p = _with_intensity(points)
    g = leaf_geometry(p, leaf)
    if g is None:
        return np.zeros((0, 4)), np.zeros((0, 4))
    if g["overflow"]:
        return p.copy(), None
    idx = leaf_indices(p, g)
    ok = idx >= 0
    leaves, inv = np.unique(idx[ok], return_inverse=True)
    v = p[ok].astype(np.float64)
    n = np.bincount(inv, minlength=len(leaves)).astype(np.float64)
    sums = np.stack([np.bincount(inv, weights=v[:, c], minlength=len(leaves)) for c in range(4)], axis=1)
    abss = np.stack([np.bincount(inv, weights=np.abs(v[:, c]), minlength=len(leaves)) for c in range(4)], axis=1)
    cen = sums / n[:, None]
    err = 2.0 * (n[:, None] + 1.0) * U64 * abss / n[:, None]
    return cen, err


# ---- NDT voxel map --------------------------------------------------------------------------------------------------
def voxel_map_ref(points, leaf, min_points=6, eig_mult=0.01):
    """VoxelGridCovariance::applyFilter: float64 moments per leaf, covariance started at the identity (the reference's
    cov_ = Identity quirk), the (n - 1) / n factor, small eigenvalues raised to eig_mult * ev_max, leaves with ev <= 0 or a
    non-finite inverse rejected, and only leaves with >= min_points points kept. Returns the shape of NDT.voxels():
    idx, npts, mean, icov, centroid, plus per voxel the largest |coordinate| of its points ("maxabs") and the extreme
    eigenvalues of the final covariance ("lam_min", "lam_max") the tolerances derive from. None on int32 overflow."""
    p = np.asarray(points, dtype=F32)[:, :3]
    empty = dict(idx=np.zeros(0, np.int32), npts=np.zeros(0, np.int32), mean=np.zeros((0, 3)), icov=np.zeros((0, 3, 3)),
                 centroid=np.zeros((0, 3), F32), maxabs=np.zeros(0), lam_min=np.zeros(0), lam_max=np.zeros(0))
    g = leaf_geometry(p, leaf)
    if g is None:
        return empty
    if g["overflow"]:
        return None
    idx = leaf_indices(p, g)
    ok = idx >= 0
    leaves, inv = np.unique(idx[ok], return_inverse=True)
    x = p[ok].astype(np.float64)
    L = len(leaves)
    cnt = np.bincount(inv, minlength=L)
    s = np.stack([np.bincount(inv, weights=x[:, a], minlength=L) for a in range(3)], axis=1)
    sxx = np.empty((L, 3, 3))
    for a in range(3):
        for b in range(3):
            sxx[:, a, b] = np.bincount(inv, weights=x[:, a] * x[:, b], minlength=L)
    maxabs = np.zeros(L)
    np.maximum.at(maxabs, inv, np.abs(x).max(axis=1))
    keep = cnt >= min_points
    leaves, cnt, s, sxx, maxabs = leaves[keep], cnt[keep], s[keep], sxx[keep], maxabs[keep]
    n = cnt.astype(np.float64)
    mean = s / n[:, None]
    cov = ((sxx + np.eye(3)) - 2.0 * (s[:, :, None] * mean[:, None, :])) / n[:, None, None] + mean[:, :, None] * mean[:, None, :]
    cov *= ((n - 1.0) / n)[:, None, None]
    ev, V = np.linalg.eigh(cov)
    valid = (ev[:, 0] >= 0) & (ev[:, 1] >= 0) & (ev[:, 2] > 0)
    min_ev = eig_mult * ev[:, 2]
    raise0 = ev[:, 0] < min_ev
    ev = ev.copy()
    ev[raise0, 0] = min_ev[raise0]
    r1 = raise0 & (ev[:, 1] < min_ev)
    ev[r1, 1] = min_ev[r1]
    cov = np.where(raise0[:, None, None], V @ (ev[:, :, None] * np.swapaxes(V, 1, 2)), cov)
    with np.errstate(all="ignore"):
        icov = np.linalg.inv(np.where(valid[:, None, None], cov, np.eye(3)))
    valid &= np.isfinite(icov).all(axis=(1, 2))
    cen = (s.astype(F32) / n.astype(F32)[:, None]).astype(F32)  # (float)sum / (float)n
    return dict(idx=leaves[valid].astype(np.int32), npts=cnt[valid].astype(np.int32), mean=mean[valid], icov=icov[valid],
                centroid=cen[valid], maxabs=maxabs[valid], lam_min=ev[valid, 0], lam_max=ev[valid, 2])


# ---- nearest neighbours ---------------------------------------------------------------------------------------------
def _d2(q, t) -> np.ndarray:
    """FLANN L2_Simple in float32, un-fused: ((dx*dx + dy*dy) + dz*dz), queries x targets."""
    d = q[:, None, :] - t[None, :, :]
    return (d[:, :, 0] * d[:, :, 0] + d[:, :, 1] * d[:, :, 1]) + d[:, :, 2] * d[:, :, 2]


def nn1_ref(target, queries, chunk=2048):
    """Exact 1-NN over the finite target rows by brute force: (index, d2 float32), ties to the lower index; (-1, FLT_MAX)
    when the target has no finite row."""
    t = np.asarray(target, dtype=F32)[:, :3]
    q = np.asarray(queries, dtype=F32)[:, :3]
    bad = ~finite_rows(t)
    idx = np.full(len(q), -1, dtype=np.int32)
    d2 = np.full(len(q), np.finfo(F32).max, dtype=F32)
    if bad.all():
        return idx, d2
    for lo in range(0, len(q), chunk):
        d = _d2(q[lo:lo + chunk], t)
        d[:, bad] = np.inf
        i = d.argmin(axis=1)  # first minimum = lowest index
        idx[lo:lo + chunk] = i
        d2[lo:lo + chunk] = d[np.arange(len(i)), i]
    return idx, d2


def knn_ref(target, queries, k, chunk=512, higher_index_ties=False):
    """Exact k-NN by brute force, lexicographic (d2, index) order: (indices (Q, k), d2 (Q, k)). higher_index_ties flips
    the tie-break to the higher index (only to show that a cloud has ties that matter)."""
    t = np.asarray(target, dtype=F32)[:, :3]
    q = np.asarray(queries, dtype=F32)[:, :3]
    key = -np.arange(len(t)) if higher_index_ties else np.arange(len(t))
    I = np.empty((len(q), k), dtype=np.int64)
    D = np.empty((len(q), k), dtype=F32)
    for lo in range(0, len(q), chunk):
        d = _d2(q[lo:lo + chunk], t)
        for r in range(len(d)):
            o = np.lexsort((key, d[r]))[:k]
            I[lo + r], D[lo + r] = o, d[r][o]
    return I, D


def gicp_cov_ref(cloud, k, eps=1e-3, higher_index_ties=False):
    """GICP point covariance from its k nearest neighbours: float64 mean and second moments of the float32 products
    (x*x formed in float), then I - (1 - eps) u u^T with u the smallest-eigenvalue direction. Also returns the gap
    between the two smallest eigenvalues relative to the largest: u is well defined only when it is not tiny."""
    p = np.asarray(cloud, dtype=F32)[:, :3]
    I, _ = knn_ref(p, p, k, higher_index_ties=higher_index_ties)
    nb = p[I]  # (n, k, 3) float32
    mean = nb.astype(np.float64).sum(axis=1) / k
    prod = (nb[:, :, :, None] * nb[:, :, None, :]).astype(np.float64).sum(axis=1) / k  # float products, f64 sums
    c = prod - mean[:, :, None] * mean[:, None, :]
    ev, V = np.linalg.eigh(c)
    a = np.abs(ev)
    m = a.argmin(axis=1)
    u = V[np.arange(len(p)), :, m]
    cov = np.eye(3)[None] - (1.0 - eps) * u[:, :, None] * u[:, None, :]
    s = np.sort(a, axis=1)
    gap = (s[:, 1] - s[:, 0]) / np.maximum(s[:, 2], 1e-300)
    return cov, gap


def nn_geometry(points):
    """The exact-NN grid's geometry (NnGrid::build): origin = min of the finite points, extent clamped to >= 1e-3, cell
    edge h = cbrt(volume / (4 n)) >= 1e-3 grown by 1.26 until the grid has <= 2^28 cells."""
    p = np.asarray(points, dtype=F32)[:, :3]
    f = p[finite_rows(p)]
    mn, mx = f.min(axis=0), f.max(axis=0)
    ext = np.maximum(1e-3, mx.astype(np.float64) - mn.astype(np.float64))
    hh = max(np.cbrt(ext.prod() / (4.0 * len(p))), 1e-3)
    while np.prod(np.floor(ext / hh) + 1) > 268435456.0:
        hh *= 1.26
    h = F32(hh)
    dims = (np.floor(ext / hh) + 1).astype(np.int64)
    return dict(origin=mn, h=h, inv_h=F32(1.0) / h, dims=dims)


# ---- edge-cloud generators ------------------------------------------------------------------------------------------
def _nudge(x, steps):
    x = F32(x)
    for _ in range(abs(steps)):
        x = np.nextafter(x, F32(np.inf if steps > 0 else -np.inf), dtype=F32)
    return x


def leaf_edge_floats(leaf, n_leaves=600, ulps=4):
    """Every float32 within `ulps` ulp of each leaf edge k * leaf, 0 < |k| <= n_leaves (the edge at 0 is left out: it is
    all subnormals)."""
    leaf = F32(leaf)
    out = [_nudge(F32(k * leaf), u) for k in range(-n_leaves, n_leaves + 1) if k for u in range(-ulps, ulps + 1)]
    return np.unique(np.array(out, dtype=F32))


def mul_div_disagree(x, leaf) -> np.ndarray:
    """Where the builder's floor(x * inv_leaf) and the solver's floor(x / leaf) name different cells."""
    return build_ref(x, leaf) != lookup_ref(x, leaf)


def with_nonfinite_rows(points, seed=0, block=256):
    """The cloud with NaN / +-inf rows added at the first row, the last row and filling the whole thread block of rows
    [block, 2 * block). Returns (cloud, finite-row mask); the finite rows keep their order."""
    p = np.asarray(points, dtype=F32)
    rng = np.random.default_rng(seed)
    bad_vals = np.array([np.nan, np.inf, -np.inf], dtype=F32)

    def bad_rows(m):
        r = rng.normal(size=(m, p.shape[1])).astype(F32)
        for i in range(m):  # one to three non-finite coordinates per row
            cols = rng.choice(3, size=1 + i % 3, replace=False)
            r[i, cols] = bad_vals[(i + cols) % 3]
        return r

    head, body = p[: block - 1], p[block - 1:]
    out = np.concatenate([bad_rows(1), head, bad_rows(block), body, bad_rows(1)])
    ok = np.concatenate([np.zeros(1, bool), np.ones(len(head), bool), np.zeros(block, bool), np.ones(len(body), bool),
                         np.zeros(1, bool)])
    assert len(head) == block - 1 and out.shape[0] > 2 * block
    return out, ok


def cell_points(cells, leaf, count, rng, spread=0.35):
    """`count` points strictly inside each absolute cell (i, j, k) of edge `leaf`: centre +- spread * leaf, far from every
    leaf edge so the multiply and divide cells agree."""
    c = np.asarray(cells, dtype=np.float64).reshape(-1, 3)
    pts = (c[:, None, :] + 0.5 + rng.uniform(-spread, spread, size=(len(c), count, 3))) * float(leaf)
    return pts.reshape(-1, 3).astype(F32)


def population_leaves(leaf, seed=0):
    """Leaves holding exactly 5, 6 and 7 points (the voxel map keeps >= 6), three of each, at absolute cells along x."""
    rng = np.random.default_rng(seed)
    parts, expect = [], {}
    for j, n in enumerate((5, 6, 7, 5, 6, 7, 5, 6, 7)):
        cell = (2 * j, 0, 0)
        parts.append(cell_points([cell], leaf, n, rng))
        expect[cell] = n
    return np.concatenate(parts), expect


def degenerate_leaves(leaf, n=40, seed=0):
    """Three leaves of n points: all identical, collinear (on a tilted line) and coplanar (on a tilted plane)."""
    rng = np.random.default_rng(seed)
    L = float(leaf)
    c0 = np.array([0.5, 0.5, 0.5]) * L
    same = np.repeat(c0[None] + [0.01 * L, -0.02 * L, 0.03 * L], n, axis=0)
    t = rng.uniform(-0.3, 0.3, size=(n, 1)) * L
    line = (np.array([2.5, 0.5, 0.5]) * L) + t * np.array([0.8, 0.5, 0.33])
    uv = rng.uniform(-0.3, 0.3, size=(n, 2)) * L
    plane = (np.array([4.5, 0.5, 0.5]) * L) + uv[:, :1] * np.array([0.7, 0.7, 0.1]) + uv[:, 1:] * np.array([-0.1, 0.2, 0.95])
    return np.concatenate([same, line, plane]).astype(F32)


def dims_for_words(n_words, partial=True):
    """Grid dimensions (a, b, c), every axis <= 2^16, whose cell count needs exactly n_words rank words, as many cells as
    that allows; with partial=True the last word is one cell short of full."""
    lo, hi = 32 * (n_words - 1) + 1, 32 * n_words
    if partial:
        hi -= 1
    for c in range(1, 65537):
        for b in range(1, 65537):
            bc = b * c
            a = hi // bc
            if a <= 65536 and a * bc >= lo:
                return a, b, c
            if bc > hi:
                break
    raise ValueError(n_words)


def word_anchors(dims):
    """Two points that pin the bounding box of a leaf-1.0 grid to `dims` cells: the centres of cell 0 and of the last
    cell (min_b = 0, so leaf index = absolute cell index)."""
    a, b, c = dims
    return np.array([[0.5, 0.5, 0.5], [a - 0.5, b - 0.5, c - 0.5]], dtype=F32)


def cell_of_index(idx, dims):
    idx = np.asarray(idx, dtype=np.int64)
    a, b, _ = dims
    return np.stack([idx % a, (idx // a) % b, idx // (a * b)], axis=-1)


def shifted(points, offset):
    p = np.asarray(points, dtype=F32).copy()
    p[:, :3] = (p[:, :3].astype(np.float64) + np.asarray(offset, dtype=np.float64)).astype(F32)
    return p


def nn_ring_margin_case():
    """A 1-NN query whose answer lies one Chebyshev ring beyond the ring that first holds a candidate, with the two
    squared distances within 1e-4 relative of each other and of the ring bound (r h)^2: the ring search may stop after
    ring 1 only if its margin is below 1. Returns (target, query (1, 3), index of the true nearest point, geometry).
    Target: the 8 corners of [0, 40]^3 (they fix a 4 x 4 x 4 grid) plus A (+x, ring 1) and B (-x, ring 2, closer)."""
    box = np.array([[x, y, z] for x in (0, 40) for y in (0, 40) for z in (0, 40)], dtype=np.float64)
    g = nn_geometry(np.concatenate([box, np.zeros((2, 3))]).astype(F32))
    h = float(g["h"])
    qx = 2.0 * h * (1 + 2e-6)  # just inside the left face of cell 2
    q = np.array([[qx, 20.0, 20.0]])
    a = q + [h * (1 + 3e-5), 0, 0]  # in cell 3: found in ring 1
    b = q - [h * (1 + 1e-5), 0, 0]  # in cell 0: only ring 2 reaches it, and it is closer
    t = np.concatenate([box, a, b]).astype(F32)
    return t, q.astype(F32), 9, nn_geometry(t)


def nn_edge_queries(target, seed=0):
    """Queries at the NN grid's edges: on every interior and outer cell face of each axis (and one ulp either side),
    beyond every face, edge and corner of the bounding box at distances from just outside to 1e4 extents, and exactly at
    target points."""
    rng = np.random.default_rng(seed)
    t = np.asarray(target, dtype=F32)[:, :3]
    t = t[finite_rows(t)]
    g = nn_geometry(t)
    mn, mx = t.min(axis=0).astype(np.float64), t.max(axis=0).astype(np.float64)
    mid, half = (mn + mx) / 2, np.maximum((mx - mn) / 2, 1e-3)
    out = []
    for a in range(3):
        faces = g["origin"][a] + np.arange(int(g["dims"][a]) + 1) * np.float64(g["h"])
        for f in faces[:64]:
            for u in (-1, 0, 1):
                q = t[rng.integers(len(t))].astype(np.float64)
                q[a] = _nudge(F32(f), u)
                out.append(q)
    for d in np.array([[x, y, z] for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]):
        for m in (1e-4, 0.5, 3.0, 1e4):
            out.append(mid + d * (half + m * np.maximum(half, float(g["h"]))))
        out.append(np.where(d > 0, mx, np.where(d < 0, mn, mid)))  # on the clamped outer face / edge / corner
    out.extend(t[rng.integers(0, len(t), size=min(len(t), 64))].astype(np.float64))
    return np.asarray(out).astype(F32)


def lattice(shape, spacing, origin=(0.0, 0.0, 0.0)):
    """Points of a regular lattice, x fastest: every point has neighbour shells of tied distances."""
    ii = np.stack(np.meshgrid(np.arange(shape[2]), np.arange(shape[1]), np.arange(shape[0]), indexing="ij"), axis=-1)
    ii = ii.reshape(-1, 3)[:, ::-1]
    return (np.asarray(origin) + ii * np.asarray(spacing)).astype(F32)
