"""The occupancy grid's definitions on the CPU: the product's header csrc/occupancy_grid.hpp compiled with g++
-ffp-contract=off and run serially (tests/hostmath/occupancy_host.cpp) against the exact Python replay tests/occupancyref.py,
cell for cell, on hand-built rays at every edge the header names; the replay told apart from its named mutations; the
serial pipeline under AddressSanitizer and UBSan; and, on the ray-cast canyon drive, a grid that agrees with the analytic
scene."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import occupancyref as R

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "occupancy_host.cpp")
F32 = np.float32
FIX = 2.0 ** -16  # one fixed-point unit at resolution 1


class Host:
    """tests/hostmath/occupancy_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
        lib.ogh_build.argtypes = [vp, vp, vp, vp, i]
        lib.ogh_info.argtypes = [vp, vp]
        lib.ogh_get.argtypes = [vp, vp, vp, vp]
        lib.ogh_save.argtypes = [C.c_char_p, C.c_char_p]
        lib.ogh_walk.argtypes = [ll, ll, ll, ll, vp, ll]
        lib.ogh_walk.restype = ll
        self.lib = lib

    def build(self, submaps, p=None):
        """Same arguments as occupancyref.build; the same dict keys (hits, frees, values (H, W), pgm bytes, counts), or the
        harness's negative return code."""
        p = R.params(**(p or {}))
        par = np.array([p["resolution"], p["z_min"], p["z_max"], p["max_range"], *p["sensor_origin"], p["occupied_thresh"],
                        p["free_thresh"]], dtype=np.float64)
        rows = [np.zeros((0, 4), dtype=F32)]
        offsets = [0]
        poses = []
        for pts, P in submaps:
            pts = np.asarray(pts, dtype=F32)
            q = np.zeros((len(pts), 4), dtype=F32)
            if len(pts):
                q[:, :3] = pts[:, :3]
            rows.append(q)
            offsets.append(offsets[-1] + len(pts))
            poses.append(np.asarray(P, dtype=np.float64).T.reshape(16))
        pts = np.ascontiguousarray(np.concatenate(rows))
        off = np.array(offsets, dtype=np.int64)
        P = np.ascontiguousarray(np.array(poses, dtype=np.float64).reshape(-1)) if poses else np.zeros(16)
        rc = self.lib.ogh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, len(submaps))
        if rc != 0:
            return rc
        info = np.zeros(7, dtype=np.uint64)
        org = np.zeros(2, dtype=np.float64)
        self.lib.ogh_info(info.ctypes.data, org.ctypes.data)
        W, H = int(info[0]), int(info[1])
        vals = np.zeros((H, W), dtype=np.int8)
        hits = np.zeros((H, W), dtype=np.uint32)
        frees = np.zeros((H, W), dtype=np.uint32)
        pgm = np.zeros(H * W, dtype=np.uint8)
        self.lib.ogh_get(vals.ctypes.data, hits.ctypes.data, frees.ctypes.data, pgm.ctypes.data)
        return dict(width=W, height=H, origin=(float(org[0]), float(org[1])), hits=hits, frees=frees, values=vals,
                    pgm=pgm.tobytes(), n_rays=int(info[2]), n_skipped=int(info[3]), n_occupied=int(info[4]),
                    n_free=int(info[5]), n_unknown=int(info[6]), p=p)

    def save(self, pgm_path, yaml_path):
        return self.lib.ogh_save(os.fsencode(pgm_path), os.fsencode(yaml_path))

    def walk(self, a, b):
        cap = abs((b[0] >> 16) - (a[0] >> 16)) + abs((b[1] >> 16) - (a[1] >> 16)) + 1
        out = np.zeros(2 * cap, dtype=np.int32)
        n = self.lib.ogh_walk(a[0], a[1], b[0], b[1], out.ctypes.data, cap)
        return [tuple(v) for v in out[:2 * min(n, cap)].reshape(-1, 2).tolist()], n


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("og"), "libocc_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    return Host(lib)


def T(x=0.0, y=0.0, z=0.0, yaw=0.0):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix((x, y, z), (0.0, 0.0, yaw))


def pts(*rows):
    return np.array(rows, dtype=F32).reshape(-1, 3)


UNIT = dict(resolution=1.0, z_min=0.5, z_max=1.5, max_range=50.0, sensor_origin=(0.0, 0.0, 1.0))


def same(a, b):
    assert isinstance(a, dict) and isinstance(b, dict), (a, b)
    for k in ("width", "height", "origin", "n_rays", "n_skipped", "n_occupied", "n_free", "n_unknown", "pgm"):
        assert a[k] == b[k], k
    for k in ("hits", "frees", "values"):
        assert np.array_equal(a[k], b[k]), k


# Every hand-built case: (name, submaps, params). Resolution 1 puts cell edges on integers and one fixed-point unit at 2^-16.
def cases():
    nan, inf = float("nan"), float("inf")
    c = []
    c.append(("axis_parallel", [(pts((5.5, 0.5, 1), (-4.5, 0.5, 1), (0.5, 7.5, 1), (0.5, -3.5, 1)), T(0.5, 0.5))], UNIT))
    c.append(("diagonal_corners", [(pts((5.5, 5.5, 1), (-3.5, -3.5, 1), (4.5, -3.5, 1), (-2.5, 2.5, 1)), T(0.5, 0.5))], UNIT))
    c.append(("diagonal_from_corner", [(pts((4, 4, 1), (-3, 3, 1), (3, -3, 1), (-2, -2, 1)), T())], UNIT))
    c.append(("along_edges", [(pts((6, 0, 1), (0, -5, 1), (-4, 0, 1), (0, 3, 1), (3, 2, 1)), T())], UNIT))
    c.append(("zero_length", [(pts((0.2, 0.1, 1), (0.0, 0.0, 1), (0.4, 0.45, 1), (-0.5, -0.5, 1)), T(0.5, 0.5))], UNIT))
    c.append(("negative", [(pts((-1.3, -2.7, 1), (2.2, -0.6, 1), (-0.25, 0.75, 1), (-5.5, -5.5, 1)), T(-10.3, -7.7))], UNIT))
    band = pts((3, 0.5, 0.5), (3, 1.5, 0.5 - FIX), (3, 2.5, 0.5 + FIX), (3, -1.5, 1.5), (3, -2.5, 1.5 + FIX), (3, -3.5, 1.5 - FIX))
    c.append(("band_edges", [(band, T())], UNIT))
    above = dict(UNIT, sensor_origin=(0.0, 0.0, 3.0))
    c.append(("origin_above_band", [(pts((6.5, 0.5, -3), (0.5, 8.5, -2.0), (-5.5, 0.5, -1.0), (2.5, -2.5, -2.9)), T())], above))
    below = dict(UNIT, sensor_origin=(0.0, 0.0, -1.0))
    c.append(("origin_below_band", [(pts((6.5, 0.5, 4), (0.5, -8.5, 2.0), (-3.5, 0.5, 1.5), (4.5, 4.5, 0.8)), T())], below))
    c.append(("entirely_above_or_below", [(pts((5, 1, 0.2), (-3, 2, 0.95), (4, -4, -3.0)), T()),
                                          (pts((5, 1, 0.0), (-3, 2, 1.0), (4, -4, 3.0)), T(0, 0, 1.5))],
              dict(UNIT, sensor_origin=(0.0, 0.0, 0.6), z_min=1.0, z_max=1.2)))
    c.append(("flat_ray_outside_band", [(pts((5, 1, 2.0), (-4, 2, 2.0)), T(0.25, 0.25))], dict(UNIT, sensor_origin=(0, 0, 2.0))))
    rng = dict(UNIT, max_range=5.0)
    c.append(("max_range_equality", [(pts((5, 0, 1), (5 + FIX, 0, 1), (0, -5, 1), (0, -5 - FIX, 1), (3, 4, 1), (3, 4 + FIX, 1),
                                          (-4, 3, 1), (-4 - FIX, -3, 1)), T())], rng))
    c.append(("nan_inf", [(pts((nan, 1, 1), (1, nan, 1), (1, 1, nan), (inf, 0, 1), (0, -inf, 1), (2, 2, inf), (3.5, 0.5, 1)),
                           T(0.5, 0.5))], UNIT))
    c.append(("empty_submap", [(np.zeros((0, 3), dtype=F32), T(4.5, 4.5)), (pts((2.5, 0.5, 1)), T())], UNIT))
    c.append(("hit_and_free_same_submap", [(pts((5.5, 0, 1), (2.5, 0, 1)), T(0.5, 0.5))], UNIT))
    c.append(("hit_and_free_different_submaps", [(pts((2.5, 0, 1)), T(0.5, 0.5)), (pts((5.5, 0, 1)), T(0.5, 0.5))], UNIT))
    # cell (3, 0) hit by one submap and freed by seven: 100 / 8 = 12.5 -> 13
    half = [(pts((3.5, 0, 1), (2.5, 0, 1)), T(0.5, 0.5))] + [(pts((3.5, 0, 1)), T(0.5, 0.5))] * 7
    c.append(("half_rounds_up", half, UNIT))
    for occ, fr in ((0.13, 0.12), (0.14, 0.13), (0.135, 0.125), (0.5, 0.0), (1.0, 0.99), (0.65, 0.25)):
        c.append((f"thresholds_{occ}_{fr}", half, dict(UNIT, occupied_thresh=occ, free_thresh=fr)))
    c.append(("rotated_pose", [(pts((7.3, 1.1, 0.2), (-2.2, 4.9, -0.3), (0.4, -6.6, 0.1)), T(1.7, -2.2, 0.9, 0.7))],
              dict(UNIT, resolution=0.25, sensor_origin=(0.3, -0.1, 0.2))))
    return c


@pytest.mark.parametrize("name,subs,p", cases(), ids=[c[0] for c in cases()])
def test_host_compile_equals_replay(host, name, subs, p):
    same(host.build(subs, p), R.build(subs, p))


def test_hand_built_outcomes(host):
    """What the hand-built cases must show, read off the replay (which the test above ties to the header)."""
    by = {n: R.build(s, p) for n, s, p in cases()}

    def cellv(g, key, x, y):
        x0, y0 = g["cells0"]
        return int(g[key][y - y0, x - x0])

    g = by["diagonal_corners"]
    # from (0.5, 0.5) to (5.5, 5.5): every corner crossing steps x first, so (1, 0) is freed and (0, 1) is not
    assert cellv(g, "frees", 1, 0) == 1 and cellv(g, "frees", 0, 1) == 0 and cellv(g, "frees", 2, 1) == 1
    # towards (-3.5, -3.5): again x first, (-1, 0) freed, (0, -1) not
    assert cellv(g, "frees", -1, 0) == 1 and cellv(g, "frees", 0, -1) == 0
    g = by["along_edges"]  # y = 0 exactly lies in row 0, x = 0 in column 0
    assert cellv(g, "frees", 3, 0) == 1 and cellv(g, "frees", 3, -1) == 0 and cellv(g, "frees", 0, -3) == 1
    assert cellv(g, "frees", -1, -3) == 0 and cellv(g, "hits", -4, 0) == 1
    g = by["zero_length"]
    assert g["width"] == 1 and g["height"] == 1 and int(g["hits"][0, 0]) == 1 and int(g["frees"][0, 0]) == 0
    g = by["negative"]  # floor: (-11.6, -10.4) is cell (-12, -11), not (-11, -10)
    assert cellv(g, "hits", -12, -11) == 1 and cellv(g, "hits", -11, -10) == 0
    g = by["band_edges"]
    assert [cellv(g, "hits", 3, y) for y in (0, 1, 2, -2, -3, -4)] == [1, 0, 1, 1, 0, 1]
    g = by["origin_above_band"]
    # the ground ray from z = 3 to (6.5, 0.5, -3) is in the band for x in [1.5, 2.5]: cells 1 and 2 only
    assert [cellv(g, "frees", x, 0) for x in range(0, 7)] == [0, 1, 1, 0, 0, 0, 0]
    g = by["origin_below_band"]
    assert [cellv(g, "frees", x, 0) for x in range(0, 7)] == [0, 1, 1, 1, 0, 0, 0]  # in the band for x in [1.95, 3.25]
    g = by["entirely_above_or_below"]
    assert int(g["frees"].sum()) == 0 and int(g["hits"].sum()) == 0 and g["n_rays"] == 6
    assert int(by["flat_ray_outside_band"]["frees"].sum()) == 0
    g = by["max_range_equality"]
    assert g["n_rays"] == 4 and g["n_skipped"] == 4
    g = by["nan_inf"]
    assert g["n_rays"] == 1 and g["n_skipped"] == 6
    g = by["empty_submap"]
    assert g["width"] == 5 and g["height"] == 5 and g["origin"] == (0.0, 0.0)
    g = by["hit_and_free_same_submap"]
    assert cellv(g, "hits", 3, 0) == 1 and cellv(g, "frees", 3, 0) == 0 and cellv(g, "values", 3, 0) == 100
    g = by["hit_and_free_different_submaps"]
    assert cellv(g, "hits", 3, 0) == 1 and cellv(g, "frees", 3, 0) == 1 and cellv(g, "values", 3, 0) == 50
    g = by["half_rounds_up"]
    assert cellv(g, "values", 3, 0) == 13 and cellv(g, "values", 4, 0) == 100 and cellv(g, "values", 1, 0) == 0
    px = {n: g2["pgm"][3 - g2["cells0"][0]] for n, g2 in by.items() if n.startswith("thr")}
    assert px == {"thresholds_0.13_0.12": 0, "thresholds_0.14_0.13": 254, "thresholds_0.135_0.125": 205,
                  "thresholds_0.5_0.0": 205, "thresholds_1.0_0.99": 254, "thresholds_0.65_0.25": 254}


def test_value_formula():
    from fractions import Fraction

    for n in range(1, 300):
        for h in range(0, n + 1):
            assert R.value(h, n - h) == math.floor(Fraction(100 * h, n) + Fraction(1, 2))  # round half up, exactly
    assert R.value(0, 0) == -1 and R.value(1, 7) == 13 and R.value(1, 1) == 50 and R.value(1, 199) == 1


def test_walks_equal_replay(host):
    """Random segments, many through exact corners and along edges: the host walk is the replay's cell for cell, 4-connected,
    from cell(A) to cell(B)."""
    rng = np.random.default_rng(5)
    for k in range(3000):
        scale = [1 << 16, 1 << 14, 1 << 20][k % 3]
        a = [int(v) for v in rng.integers(-40 * scale, 40 * scale, size=2)]
        if k % 4 == 0:  # a diagonal through lattice corners
            d = int(rng.integers(-30, 30)) << 16
            a = [(a[0] >> 16) << 16, (a[1] >> 16) << 16]
            b = [a[0] + d, a[1] + (d if k % 8 else -d)]
        elif k % 4 == 1:  # along an edge
            a = [(a[0] >> 16) << 16, a[1]]
            b = [a[0], a[1] + int(rng.integers(-40 << 16, 40 << 16))]
        else:
            b = [a[0] + int(rng.integers(-50 << 16, 50 << 16)), a[1] + int(rng.integers(-50 << 16, 50 << 16))]
        got, n = host.walk(a, b)
        want = R.walk(a, b)
        assert got == want and n == len(want), (a, b)
        assert all(abs(p[0] - q[0]) + abs(p[1] - q[1]) == 1 for p, q in zip(want[:-1], want[1:]))


def test_refusals_match(host):
    sub = [(pts((1, 1, 1)), T())]
    for p, code in ((dict(resolution=0.0), -1), (dict(resolution=float("nan")), -1), (dict(z_min=2.0, z_max=2.0), -1),
                    (dict(z_min=float("inf")), -1), (dict(max_range=0.0), -1), (dict(max_range=-1.0), -1),
                    (dict(max_range=16384.0 * 0.05 + 1e-9), -1), (dict(sensor_origin=(0, float("nan"), 0)), -1),
                    (dict(free_thresh=0.65), -1), (dict(occupied_thresh=1.01), -1), (dict(free_thresh=-0.01), -1)):
        assert host.build(sub, p) == code, p
        with pytest.raises(R.Refused) as e:
            R.build(sub, p)
        assert e.value.code == code
    assert host.build(sub, dict(max_range=16384.0 * 0.05)) != -1  # the range bound at equality
    assert host.build([], {}) == -4
    far = [(pts((1, 1, 1)), T(0, 0, 6000.0))]  # an origin 2^17 cells above the band
    assert host.build(far, dict(resolution=0.05)) == -2
    wide = [(pts((90, 0, 1)), T(0, 0, 1)), (pts((0, 0, 1)), T(2e4, 2e4, 1))]
    assert host.build(wide, dict(resolution=0.5)) == -3
    with pytest.raises(R.Refused) as e:
        R.build(wide, dict(resolution=0.5))
    assert e.value.code == -3


def test_files_equal_replay(host, tmp_path):
    import yaml

    subs, p = cases()[5][1], cases()[5][2]
    g = R.build(subs, dict(p, resolution=0.05, max_range=20.0))
    host.build(subs, dict(p, resolution=0.05, max_range=20.0))
    assert host.save(str(tmp_path / "map.pgm"), str(tmp_path / "map.yaml")) == 0
    assert (tmp_path / "map.pgm").read_bytes() == R.pgm_bytes(g)
    text = (tmp_path / "map.yaml").read_text()
    assert text == R.yaml_text(g, str(tmp_path / "map.pgm"))
    y = yaml.safe_load(text)
    assert y["image"] == "map.pgm" and y["mode"] == "trinary" and y["negate"] == 0
    assert float(y["resolution"]) == 0.05 and [float(v) for v in y["origin"][:2]] == list(g["origin"])
    assert y["occupied_thresh"] == 0.65 and y["free_thresh"] == 0.25
    for v in (1e-5, 2.5e-7, -3e20, 0.1, 1.0 / 3.0, -0.0, 12345678.9):
        s = R.number(v)
        assert float(yaml.safe_load(f"v: {s}")["v"]) == v, s


def test_mutations_change_an_outcome():
    by = {n: (s, p) for n, s, p in cases()}

    def differs(name, mut):
        s, p = by[name]
        a, b = R.build(s, p), R.build(s, p, mut={mut})
        return any(not np.array_equal(a[k], b[k]) for k in ("hits", "frees", "values")) or a["pgm"] != b["pgm"] or \
            a["width"] != b["width"]

    assert differs("diagonal_corners", "y_first")
    assert differs("origin_above_band", "no_clip")
    assert differs("negative", "trunc")
    assert differs("hit_and_free_same_submap", "free_wins")
    assert differs("origin_above_band", "no_flip")
    for mut in R.MUTATIONS:  # and no mutation is invisible on the whole set
        assert any(differs(n, mut) for n in by), mut


def test_serial_pipeline_under_sanitizers(tmp_path):
    """The executable form of the harness: grids from generated submaps (non-finite rows, negative coordinates, empty
    submaps) under -fsanitize=address,undefined, each equal to the grid of its submaps in reverse order."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = os.path.join(tmp_path, "occupancy_asan")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-DOG_HOST_MAIN", "-x", "c++", SRC, "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr or "ubsan" in build.stderr):
        pytest.skip("this toolchain has no sanitizer runtime")
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0 and "0 failures" in run.stdout, run.stdout + run.stderr


# ---------------------------------------------------------------- the ray-cast canyon drive against the analytic scene
DRIVE = dict(resolution=0.1, z_min=0.3, z_max=1.3, max_range=100.0)  # every obstacle of the scene spans the band


def _footprints(scene, x0, y0, W, H, res, grow):
    """Masks over the grid: cells whose square, widened by `grow` cells on every side, meets (any) or lies inside (all) a
    box or cylinder footprint of the scene, or the solid ground beyond the facades (|y| >= facade_y)."""
    xs = x0 + res * np.arange(W + 1)
    ys = y0 + res * np.arange(H + 1)
    meet = np.zeros((H, W), dtype=bool)
    inside = np.zeros((H, W), dtype=bool)
    lo_x, hi_x = xs[:-1] - grow * res, xs[1:] + grow * res
    lo_y, hi_y = ys[:-1] - grow * res, ys[1:] + grow * res
    meet |= (hi_y[:, None] > scene.facade_y) | (lo_y[:, None] < -scene.facade_y)
    for b in scene.boxes:
        cx = (hi_x > b[0]) & (lo_x < b[3])
        cy = (hi_y > b[1]) & (lo_y < b[4])
        meet |= cy[:, None] & cx[None, :]
        ix = (xs[:-1] >= b[0]) & (xs[1:] <= b[3])
        iy = (ys[:-1] >= b[1]) & (ys[1:] <= b[4])
        inside |= iy[:, None] & ix[None, :]
    for cxc, cyc, r, _ in scene.cylinders:
        dx = np.maximum(np.maximum(lo_x - cxc, cxc - hi_x), 0.0)
        dy = np.maximum(np.maximum(lo_y - cyc, cyc - hi_y), 0.0)
        meet |= dy[:, None] ** 2 + dx[None, :] ** 2 <= r * r
        fx = np.maximum(np.abs(xs[:-1] - cxc), np.abs(xs[1:] - cxc))
        fy = np.maximum(np.abs(ys[:-1] - cyc), np.abs(ys[1:] - cyc))
        inside |= fy[:, None] ** 2 + fx[None, :] ** 2 <= r * r
    return meet, inside


def test_canyon_drive_grid_agrees_with_the_scene(host):
    """The drive of tests/scancontextref.py (31 submaps, 16 x 450 rays each) at its true poses through the host compile,
    against synth.make_scene(): nothing beyond the solid facades is observed, obstacle footprints are not free, occupied
    cells lie at obstacles, and the street along the drive is free. Measured with this compile: 0 observed cells beyond
    |y| = 18.2 m; 3.8 % (36 of 944) of the observed cells wholly inside a footprint free; 0.0 % of the occupied cells more than one
    cell from every footprint; 99.6 % of the street cells (x in [-30, 30], |y| <= 15, more than 1 m from every footprint)
    free. The band [0.3, 1.3] m lies below the top of every obstacle, so a footprint cell is free only where range noise
    (0.02 m) carried an endpoint past a face."""
    from lidarslam_ros2_b200 import synth
    import scancontextref as SC

    scans, poses, _ = SC.drive()
    g = host.build(list(zip(scans, poses)), DRIVE)
    scene = synth.make_scene()
    res = DRIVE["resolution"]
    x0, y0 = g["origin"]
    W, H = g["width"], g["height"]
    observed = (g["hits"] + g["frees"]) > 0
    pix = np.frombuffer(g["pgm"], dtype=np.uint8).reshape(H, W)[::-1]  # back to row 0 = bottom
    free, occ = (pix == 254) & observed, pix == 0
    yl = y0 + res * np.arange(H)
    beyond = (yl >= 18.2) | (yl + res <= -18.2)
    assert int(observed[beyond].sum()) == 0
    near, inside = _footprints(scene, x0, y0, W, H, res, grow=1)
    far_from, _ = _footprints(scene, x0, y0, W, H, res, grow=10)
    free_on_footprint = (free & inside).sum() / max(1, (observed & inside).sum())
    stray_occupied = (occ & ~near).sum() / max(1, occ.sum())
    xl = x0 + res * np.arange(W)
    street = ((xl[None, :] >= -30) & (xl[None, :] + res <= 30)) & ((yl[:, None] >= -15) & (yl[:, None] + res <= 15)) & ~far_from
    street_free = (free & street).sum() / street.sum()
    print(f"free on footprints {free_on_footprint:.4f}, stray occupied {stray_occupied:.4f}, street free {street_free:.4f}, "
          f"observed inside {(observed & inside).sum()}, occupied {occ.sum()}, street {street.sum()}")
    assert (observed & inside).sum() > 500 and occ.sum() > 1000 and street.sum() > 100000
    assert free_on_footprint <= 0.05  # measured 0.038
    assert stray_occupied <= 0.001  # measured 0
    assert street_free >= 0.99  # measured 0.9963


@pytest.mark.parametrize("name", ["map: v2 #1.pgm", "&anchor.pgm", "- dash.pgm", 'q"uo\\te.pgm', "tab\there.pgm", "plain.pgm",
                                  "ünï.pgm", "'single'.pgm", "*star.pgm", "[br].pgm"])
def test_yaml_image_name_reads_back(host, tmp_path, name):
    """The image name is a double-quoted scalar: a name with ': ', '#', quotes, a backslash, a control byte or a leading
    YAML indicator reads back as itself, and the host compile writes the replay's text."""
    import yaml

    subs, p = cases()[0][1], cases()[0][2]
    g = R.build(subs, p)
    host.build(subs, p)
    pgm = str(tmp_path / name)
    assert host.save(pgm, str(tmp_path / "map.yaml")) == 0
    text = (tmp_path / "map.yaml").read_text(encoding="utf-8")
    assert text == R.yaml_text(g, pgm)
    assert yaml.safe_load(text)["image"] == name
    assert (tmp_path / name).read_bytes() == R.pgm_bytes(g)
