"""The relocalisation search of b200sm_relocalize on the CPU: the product's header csrc/relocalize.hpp compiled with g++
-ffp-contract=off (tests/hostmath/relocalize_host.cpp, the pruned search run serially) against the replay tests/relocref.py
bit for bit on hand-built cases (negative coordinates, band edges at equality, points on cell boundaries, scans reaching
past every side of the grid, a 1 x 1 grid, W and H not multiples of the tile, one heading, 1 and 16 levels, ties); the
pruned answer against the exhaustive definition on hundreds of random small maps; the bound property; the caps at the
limit and one below; and the replay told apart from subtly wrong ones (relocref.MUTATIONS). Needs no GPU."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import relocref as R
from lidarslam_ros2_b200 import _capi

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "relocalize_host.cpp")
F32 = np.float32


def build_host_lib(out_dir):
    """the harness, compiled into out_dir (a temporary directory: the tree may be read-only)"""
    lib = os.path.join(str(out_dir), "librelocalize_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    lib = C.CDLL(lib)
    vp, ll = C.c_void_p, C.c_longlong
    lib.rl_valid.argtypes = [vp]
    lib.rl_set_map.argtypes = [vp, C.c_size_t, vp, vp, C.c_char_p, C.c_int]
    lib.rl_level.argtypes = [C.c_int, vp, C.c_size_t, C.POINTER(ll), C.POINTER(ll)]
    lib.rl_set_scan.restype = ll
    lib.rl_set_scan.argtypes = [vp, C.c_size_t, vp, vp, C.c_char_p, C.c_int]
    lib.rl_offsets.argtypes = [vp]
    lib.rl_scores.argtypes = [C.c_int, ll, vp, vp]
    lib.rl_search.argtypes = [C.c_int, vp, vp, vp, vp, C.c_char_p, C.c_int]
    lib.rl_guess_of.argtypes = [vp, vp, C.c_int, ll, ll, vp]
    lib.rl_grid_limit.argtypes = [ll, ll, ll, ll, vp]
    lib.rl_points_limit.argtypes = [ll, C.c_int]
    lib.rl_set_yaw_steps.argtypes = [C.c_int]
    return lib


@pytest.fixture(scope="module")
def rl(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("rl"))


def params(**kw):
    return dict(R.DEFAULTS, **kw)


def _cp(p):
    return _capi.SmRelocalizeParams(*(p[k] for k in ("resolution", "z_min", "z_max", "yaw_steps", "num_levels", "min_score", "top_k",
                                                       "accept_fitness")))


def _yaw_quat(yaw):
    return (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))


class Host:
    """the header's serial search on one map and one scan"""

    def __init__(self, rl, map4, p):
        self.rl, self.p = rl, p
        self.map4 = np.ascontiguousarray(map4, dtype=F32)
        self.cp = _cp(p)
        g6 = np.zeros(6, dtype=np.int64)
        err = C.create_string_buffer(256)
        self.refused = rl.rl_set_map(self.map4.ctypes.data, len(self.map4), C.byref(self.cp), g6.ctypes.data, err, 256) != 0
        self.err = err.value.decode()
        self.grid = None if self.refused or g6[2] == 0 else dict(i0=int(g6[0]), j0=int(g6[1]), W=int(g6[2]), H=int(g6[3]),
                                                                   TW=int(g6[4]), TH=int(g6[5]))

    def level(self, h):
        w, hh = C.c_longlong(0), C.c_longlong(0)
        self.rl.rl_level(h, None, 0, C.byref(w), C.byref(hh))
        out = np.zeros((hh.value, w.value), dtype=np.uint8)
        self.rl.rl_level(h, out.ctypes.data, out.size, C.byref(w), C.byref(hh))
        return out

    def set_scan(self, scan4, position, quat):
        self.scan4 = np.ascontiguousarray(scan4, dtype=F32)
        self.pos = np.ascontiguousarray(position, dtype=np.float64)
        self.quat = np.ascontiguousarray(quat, dtype=np.float64)
        err = C.create_string_buffer(256)
        self.m = self.rl.rl_set_scan(self.scan4.ctypes.data, len(self.scan4), self.pos.ctypes.data, self.quat.ctypes.data, err, 256)
        return self.m

    def offsets(self):
        out = np.zeros((self.p["yaw_steps"], max(self.m, 0), 2), dtype=np.int32)
        self.rl.rl_offsets(out.ctypes.data)
        return out

    def scores(self, h, nodes):
        kij = np.ascontiguousarray(np.asarray(nodes, dtype=np.int32).reshape(-1, 3))
        out = np.zeros(len(kij), dtype=np.int64)
        self.rl.rl_scores(h, len(kij), kij.ctypes.data, out.ctypes.data)
        return out

    def search(self, exhaustive=False):
        info, nodes = np.zeros(3, dtype=np.int64), np.zeros(16, dtype=np.int64)
        tiles, keys = np.zeros(64, dtype=np.int64), np.zeros(64, dtype=np.uint64)
        err = C.create_string_buffer(256)
        if self.rl.rl_search(int(exhaustive), info.ctypes.data, nodes.ctypes.data, tiles.ctypes.data, keys.ctypes.data, err, 256):
            return dict(error=err.value.decode())
        n = int(info[2])
        return dict(t0=int(info[0]), t=int(info[1]), nodes=[int(v) for v in nodes], tiles=[int(v) for v in tiles[:n]],
                    keys=[int(v) for v in keys[:n]])

    def guess(self, k, i, j):
        out = np.zeros(16, dtype=F32)
        self.rl.rl_guess_of(self.pos.ctypes.data, self.quat.ctypes.data, k, i, j, out.ctypes.data)
        return out.reshape(4, 4).T


def replay(map4, scan4, position, quat, p, mut=()):
    g, levels = R.pyramid(np.asarray(map4, dtype=F32), p, mut)
    _, rot_f = R.rotations(position, quat, p["yaw_steps"])
    offs, m = R.offsets(np.asarray(scan4, dtype=F32), rot_f, float(position[2]), p, mut)
    return g, levels, offs, m


def _probe_nodes(g, Y, rng, n=60):
    """nodes inside and outside the grid on every side"""
    k = rng.integers(0, Y, n)
    i = rng.integers(-g["W"] - 3, 2 * g["W"] + 3, n)
    j = rng.integers(-g["H"] - 3, 2 * g["H"] + 3, n)
    return np.stack([k, i, j], axis=1)


def check_case(rl, map4, scan4, position, quat, p, seed=0, exhaustive=True):
    """host compile == replay: grid, levels, offsets, node scores, pruned and exhaustive searches; returns the host search"""
    host = Host(rl, map4, p)
    assert not host.refused, host.err
    g, levels, offs, m = replay(map4, scan4, position, quat, p)
    if g is None:
        assert host.grid is None
    else:
        assert host.grid == {k: g[k] for k in ("i0", "j0", "W", "H", "TW", "TH")}
        for h in range(p["num_levels"]):
            assert np.array_equal(host.level(h), levels[h]), h
    assert host.set_scan(scan4, position, quat) == m
    assert np.array_equal(host.offsets(), offs)
    if g is not None and m:
        rng = np.random.default_rng(seed)
        for h in range(p["num_levels"]):
            nodes = _probe_nodes(g, p["yaw_steps"], rng)
            assert np.array_equal(host.scores(h, nodes), R.scores(levels, g, offs, h, nodes)), h
    got = host.search()
    want = R.search(levels, g, offs, m, p)
    assert got == want
    if exhaustive:
        full = host.search(exhaustive=True)
        assert full["tiles"] == got["tiles"] and full["keys"] == got["keys"]
        assert full == R.search(levels, g, offs, m, p, exhaustive=True)
    return host, got


# ---- hand-built cases -------------------------------------------------------------------------------------------------
def _scene(rng, n, lo, hi, z=(0.0, 3.5)):
    pts = np.zeros((n, 4), dtype=F32)
    pts[:, 0] = rng.uniform(lo[0], hi[0], n)
    pts[:, 1] = rng.uniform(lo[1], hi[1], n)
    pts[:, 2] = rng.uniform(z[0], z[1], n)
    return pts


def _scan_of(map4, position, yaw, rng, n=80, noise=0.02):
    """map rows seen from the pose: the rows moved into its frame, some noise, a few strays"""
    pick = map4[rng.choice(len(map4), min(n, len(map4)), replace=False)]
    c, s = math.cos(yaw), math.sin(yaw)
    dx, dy = pick[:, 0] - position[0], pick[:, 1] - position[1]
    out = np.zeros_like(pick)
    out[:, 0] = c * dx + s * dy + rng.normal(0, noise, len(pick))
    out[:, 1] = -s * dx + c * dy + rng.normal(0, noise, len(pick))
    out[:, 2] = pick[:, 2] - position[2]
    return out.astype(F32)


def _hand_cases():
    rng = np.random.default_rng(11)
    cases = []
    # negative coordinates, several headings
    m = _scene(rng, 300, (-9.0, -7.0), (-2.0, -1.5))
    cases.append(("negative", m, _scan_of(m, (-5.0, -4.0, 0.0), 0.3, rng), (-6.0, -3.0, 0.0), 1.1, params(resolution=0.5, yaw_steps=8, num_levels=3, top_k=3, min_score=0.1)))
    # band edges at equality and one float either side; points exactly on cell boundaries (multiples of 0.25, negative too)
    zs = [0.5, 2.0, np.nextafter(F32(0.5), F32(0)), np.nextafter(F32(2.0), F32(3))]
    m = np.array([[x, y, z, 0.0] for x in (-1.0, -0.25, 0.0, 0.25, 1.5) for y in (-0.5, 0.0, 0.75) for z in zs], dtype=F32)
    s = np.array([[x, y, z, 0.0] for x in (-0.5, 0.0, 0.25, 1.0) for y in (-0.25, 0.0, 0.5) for z in (0.5, 2.0, 0.25, 2.25)], dtype=F32)
    cases.append(("band_and_boundaries", m, s, (0.0, 0.0, 0.0), 0.0, params(resolution=0.25, z_min=0.5, z_max=2.0, yaw_steps=4, num_levels=3, top_k=5, min_score=0.0)))
    # a scan reaching past every side of a small grid
    m = _scene(rng, 120, (0.0, 0.0), (3.0, 2.0))
    s = np.concatenate([_scan_of(m, (1.5, 1.0, 0.0), 0.0, rng, 60),
                        np.array([[x, y, 1.0, 0.0] for x in (-40.0, 40.0, 0.0) for y in (-40.0, 40.0, 0.0)], dtype=F32)])
    cases.append(("past_every_side", m, s, (1.5, 1.0, 0.0), 0.0, params(resolution=0.5, yaw_steps=6, num_levels=4, top_k=4, min_score=0.05)))
    # a 1 x 1 grid
    m = np.array([[0.1, 0.1, 1.0, 0.0], [0.2, 0.15, 2.0, 0.0], [0.05, 0.2, 0.4, 0.0]], dtype=F32)
    s = np.array([[0.0, 0.0, 1.0, 0.0], [0.3, 0.0, 1.0, 0.0], [-0.3, 0.1, 1.5, 0.0]], dtype=F32)
    for L in (1, 2, 16):
        cases.append((f"one_cell_L{L}", m, s, (0.0, 0.0, 0.0), 0.0, params(resolution=0.25, yaw_steps=3, num_levels=L, top_k=2, min_score=0.0)))
    # W and H not multiples of the tile (13 x 7 cells, tiles of 4)
    m = _scene(rng, 200, (0.0, 0.0), (6.4, 3.4))
    cases.append(("ragged_tiles", m, _scan_of(m, (3.0, 1.5, 0.0), 0.7, rng), (2.0, 1.0, 0.0), 0.0, params(resolution=0.5, yaw_steps=5, num_levels=3, top_k=6, min_score=0.2)))
    # one heading; 1 and 16 levels
    for L in (1, 16):
        cases.append((f"yaw1_L{L}", m, _scan_of(m, (3.0, 1.5, 0.0), 0.0, rng), (3.0, 1.5, 0.0), 0.0, params(resolution=0.5, yaw_steps=1, num_levels=L, top_k=3, min_score=0.1)))
    # ties: a periodic map, the same view everywhere
    m = np.array([[x + 0.1, y + 0.1, 1.0, 0.0] for x in np.arange(0.0, 8.0, 2.0) for y in np.arange(0.0, 6.0, 2.0)], dtype=F32)
    s = np.array([[0.0, 0.0, 1.0, 0.0], [2.0, 0.0, 1.0, 0.0], [0.0, 2.0, 1.0, 0.0]], dtype=F32)
    cases.append(("ties", m, s, (0.0, 0.0, 0.0), 0.0, params(resolution=0.5, yaw_steps=4, num_levels=3, top_k=8, min_score=0.3)))
    # heights: a tilted pose moves the band
    m = _scene(rng, 250, (-3.0, -3.0), (3.0, 3.0), (-1.0, 4.0))
    cases.append(("tilted_high", m, _scan_of(m, (0.0, 0.0, 1.2), 0.0, rng), (0.5, -0.5, 1.2), 2.0, params(resolution=0.4, yaw_steps=7, num_levels=3, top_k=3, min_score=0.0)))
    return cases


HAND = _hand_cases()


@pytest.mark.parametrize("case", HAND, ids=[c[0] for c in HAND])
def test_hand_cases_equal_replay(rl, case):
    name, m, s, pos, yaw, p = case
    quat = _yaw_quat(yaw)
    if name == "tilted_high":
        quat = (0.05, -0.03, math.sin(yaw / 2), math.cos(yaw / 2))
        n = math.sqrt(sum(v * v for v in quat))
        quat = tuple(v / n for v in quat)
    host, got = check_case(rl, m, s, pos, quat, p)
    if name == "band_and_boundaries":
        assert host.grid["W"] == 11 and host.grid["H"] == 6  # x -1 .. 1.5 and y -0.5 .. 0.75 at 0.25: the boundary rows count
    if name.startswith("one_cell"):
        assert host.grid["W"] == 1 and host.grid["H"] == 1
    if name == "ties":
        assert len(set(k >> 40 for k in got["keys"])) < len(got["keys"])  # equal scores, ranked by leaf index


def test_guess_is_the_cell_corner(rl):
    m = _scene(np.random.default_rng(3), 50, (-2.0, -1.0), (2.0, 1.0))
    p = params(resolution=0.5, yaw_steps=8, num_levels=2, top_k=2)
    host = Host(rl, m, p)
    pos, quat = (0.3, -0.2, 0.7), _yaw_quat(0.4)
    host.set_scan(m, pos, quat)
    G = host.guess(3, 2, 1)
    rot_d, _ = R.rotations(pos, quat, 8)
    assert np.array_equal(G[:3, :3], rot_d[3].astype(F32))
    assert G[0, 3] == F32((host.grid["i0"] + 2) * 0.5) and G[1, 3] == F32((host.grid["j0"] + 1) * 0.5) and G[2, 3] == F32(0.7)


# ---- random small maps: the pruned search is the definition ---------------------------------------------------------------
def _random_case(seed):
    rng = np.random.default_rng(seed)
    res = float(rng.choice([0.25, 0.5, 0.75]))
    lo = rng.uniform(-6, 2, 2)
    m = _scene(rng, int(rng.integers(1, 160)), lo, lo + rng.uniform(0.3, 6, 2))
    pos = (float(rng.uniform(lo[0], lo[0] + 4)), float(rng.uniform(lo[1], lo[1] + 4)), float(rng.uniform(-0.5, 0.5)))
    yaw = float(rng.uniform(-math.pi, math.pi))
    s = _scan_of(m, pos, yaw, rng, int(rng.integers(1, 60)), noise=float(rng.choice([0.0, 0.05, 0.3])))
    p = params(resolution=res, yaw_steps=int(rng.integers(1, 9)), num_levels=int(rng.integers(1, 6)), top_k=int(rng.integers(1, 7)),
               min_score=float(rng.choice([0.0, 0.1, 0.3, 0.6])))
    return m, s, pos, _yaw_quat(float(rng.uniform(-math.pi, math.pi))), p


def test_pruned_equals_exhaustive_on_random_maps(rl):
    expanded = 0
    for seed in range(300):
        m, s, pos, quat, p = _random_case(seed)
        host = Host(rl, m, p)
        host.set_scan(s, pos, quat)
        got, full = host.search(), host.search(exhaustive=True)
        assert got["tiles"] == full["tiles"] and got["keys"] == full["keys"], seed
        assert got["t"] >= got["t0"] or host.m == 0 or host.grid is None  # (no search: T stays 0)
        if host.grid and host.grid["W"] * host.grid["H"] > 1:
            expanded += 1
    assert expanded > 200


def test_random_maps_equal_replay(rl):
    for seed in range(0, 300, 5):
        m, s, pos, quat, p = _random_case(seed)
        check_case(rl, m, s, pos, quat, p, seed=seed, exhaustive=False)


def test_every_bound_covers_its_leaves(rl):
    for seed in range(40):
        m, s, pos, quat, p = _random_case(1000 + seed)
        p["num_levels"] = 4
        g, levels, offs, mm = replay(m, s, pos, quat, p)
        if g is None or mm == 0:
            continue
        host = Host(rl, m, p)
        host.set_scan(s, pos, quat)
        rng = np.random.default_rng(seed)
        for h in range(1, 4):
            w = 1 << h
            for _ in range(10):
                k, i, j = int(rng.integers(0, p["yaw_steps"])), int(rng.integers(-w, g["W"] + 1)), int(rng.integers(-w, g["H"] + 1))
                leaves = [(k, i + a, j + b) for a in range(w) for b in range(w)]
                bound = host.scores(h, [(k, i, j)])[0]
                assert bound >= host.scores(0, leaves).max(), (seed, h, k, i, j)


# ---- the caps ---------------------------------------------------------------------------------------------------------------
def test_caps_at_the_limit_and_one_below(rl):
    p = _cp(params(yaw_steps=1, num_levels=1))
    assert rl.rl_grid_limit(0, 0, (1 << 14) - 1, (1 << 14) - 1, C.byref(p)) == 0   # 2^28 cells
    assert rl.rl_grid_limit(0, 0, (1 << 14), (1 << 14) - 1, C.byref(p)) == 1
    p = _cp(params(yaw_steps=4096, num_levels=1))                                    # roots: 4096 * TW * TH <= 2^32
    assert rl.rl_grid_limit(0, 0, 1023, 1023, C.byref(p)) == 0 and rl.rl_grid_limit(0, 0, 1024, 1023, C.byref(p)) == 2
    p = _cp(params(yaw_steps=4096, num_levels=6))                                    # leaves: 4096 * W * H < 2^40
    assert rl.rl_grid_limit(0, 0, (1 << 14) - 1, (1 << 14) - 2, C.byref(p)) == 0
    assert rl.rl_grid_limit(0, 0, (1 << 14) - 1, (1 << 14) - 1, C.byref(p)) == 2
    p = _cp(params(yaw_steps=1, num_levels=16))                                      # the pyramid's bytes, margins included
    W = 1
    sizes = lambda W, H: sum((W + (1 << h) - 1) * (H + (1 << h) - 1) for h in range(16))
    A = sum(W + (1 << h) - 1 for h in range(16))
    H = ((1 << 32) - sizes(W, 0)) // A  # sizes is A * H + sizes(W, 0)
    assert sizes(W, H) <= 1 << 32 < sizes(W, H + 1)
    assert rl.rl_grid_limit(0, 0, W - 1, H - 1, C.byref(p)) == 0 and rl.rl_grid_limit(0, 0, W - 1, H, C.byref(p)) == 1
    assert rl.rl_points_limit((1 << 24) - 1, 4) == 0 and rl.rl_points_limit(1 << 24, 4) == 1     # m
    assert rl.rl_points_limit(1 << 18, 256) == 0 and rl.rl_points_limit((1 << 18) + 1, 256) == 1  # yaw_steps * m <= 2^26
    for bad in (dict(resolution=0.0), dict(resolution=math.inf), dict(z_min=1.0, z_max=1.0), dict(z_min=math.nan),
                dict(yaw_steps=0), dict(yaw_steps=4097), dict(num_levels=0), dict(num_levels=17), dict(min_score=-0.1),
                dict(min_score=1.5), dict(top_k=0), dict(top_k=65), dict(accept_fitness=0.0), dict(resolution=1e-320)):
        assert rl.rl_valid(C.byref(_cp(params(**bad)))) == 0, bad
    assert rl.rl_valid(C.byref(_cp(params(yaw_steps=4096, num_levels=16, top_k=64, min_score=1.0)))) == 1


def test_heading_limits_are_checked_by_every_search(rl):
    """A pyramid serves searches with any yaw_steps, so the limits that depend on the headings (roots, leaves) are checked
    by each search, not when the pyramid is built: one built for 8 headings refuses a search with 4096 over 2^32 roots."""
    m = np.array([[0.05, 0.05, 1.0, 0.0], [409.55, 102.35, 1.0, 0.0]], dtype=F32)  # 4096 x 1024 cells at 0.1 m
    s = np.array([[0.0, 0.0, 1.0, 0.0]], dtype=F32)
    host = Host(rl, m, params(resolution=0.1, yaw_steps=8, num_levels=1))
    assert not host.refused and host.grid["W"] * host.grid["H"] == 4096 * 1024
    host.set_scan(s, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    assert "error" not in host.search()
    rl.rl_set_yaw_steps(1024)  # 2^32 roots: at the limit
    host.set_scan(s, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    assert rl.rl_grid_limit(0, 0, 4095, 1023, C.byref(_cp(params(resolution=0.1, yaw_steps=1024, num_levels=1)))) == 0
    rl.rl_set_yaw_steps(1025)
    host.set_scan(s, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    assert "roots" in host.search()["error"]


def test_frontier_cap_is_reported_by_level(rl):
    # the frontier cap is a stated constant; a search far below it never reports one
    m, s, pos, quat, p = _random_case(7)
    host = Host(rl, m, p)
    host.set_scan(s, pos, quat)
    assert "error" not in host.search() and R.MAX_FRONTIER == 1 << 26


# ---- the mutations ----------------------------------------------------------------------------------------------------------
def _outcome(m, s, pos, quat, p, mut=()):
    g, levels, offs, mm = replay(m, s, pos, quat, p, mut)
    probes = None
    if g is not None and mm:
        probes = [R.scores(levels, g, offs, h, _probe_nodes(g, p["yaw_steps"], np.random.default_rng(1))) for h in range(p["num_levels"])]
    return g, [l.tobytes() for l in levels], offs.tobytes(), probes, R.search(levels, g, offs, mm, p, mut=mut)


def _same(a, b):
    return a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and a[4] == b[4] and (
        (a[3] is None and b[3] is None) or (a[3] is not None and b[3] is not None and all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))))


@pytest.mark.parametrize("mut", R.MUTATIONS)
def test_mutations_are_told_apart(rl, mut):
    told = False
    cases = [(c[1], c[2], c[3], _yaw_quat(c[4]), c[5]) for c in HAND] + [_random_case(s) for s in range(60)]
    for m, s, pos, quat, p in cases:
        good = _outcome(m, s, pos, quat, p)
        host = Host(rl, m, p)
        host.set_scan(s, pos, quat)
        assert good[4] == host.search()
        if not _same(good, _outcome(m, s, pos, quat, p, {mut})):
            told = True
            break
    assert told, mut
