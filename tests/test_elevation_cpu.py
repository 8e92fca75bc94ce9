"""The elevation / traversability map's definitions on the CPU: the product's header csrc/elevation_map.hpp compiled with
g++ -ffp-contract=off and run serially (tests/hostmath/elevation_host.cpp) against the exact Python replay
tests/elevationref.py, cell for cell, on hand-built cases at every edge the header names; the replay told apart from its
named mutations; the serial pipeline under AddressSanitizer and UBSan; and, on the ray-cast terrain drive
(tests/terrainscene.py), a map that reads the ramps, the curb, the wall and the road under the bridge as the terrain is."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import elevationref as R
import terrainscene as TS

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "elevation_host.cpp")
F32 = np.float32
LAYERS = ("n", "h", "lo", "step", "tan_slope", "roughness", "value")
COUNTS = ("width", "height", "origin", "n_points", "n_skipped", "n_overhang", "n_observed", "n_lethal", "n_traversable",
          "n_unknown", "pgm")


def param_vector(p):
    return np.array([p["resolution"], p["max_range"], *p["sensor_origin"], p["clearance"], p["min_points"], p["window_cells"],
                     p["min_cells"], p["max_slope"], p["max_step"], p["max_roughness"], p["occupied_thresh"],
                     p["free_thresh"]], dtype=np.float64)


class Host:
    """tests/hostmath/elevation_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp, i = C.c_void_p, C.c_int
        lib.elh_build.argtypes = [vp, vp, vp, vp, i]
        lib.elh_info.argtypes = [vp, vp]
        lib.elh_get.argtypes = [vp] * 8
        lib.elh_save.argtypes = [C.c_char_p, C.c_char_p]
        lib.elh_const.argtypes = [vp, vp]
        self.lib = lib

    def build(self, submaps, p=None):
        """Same arguments as elevationref.build; the same dict keys, or the harness's negative return code."""
        p = R.params(**(p or {}))
        par = param_vector(p)
        rows = [np.zeros((0, 4), dtype=F32)]
        offsets = [0]
        poses = []
        for pts, P in submaps:
            pts = np.asarray(pts, dtype=F32).reshape(len(pts), -1) if len(pts) else np.zeros((0, 3), F32)
            q = np.zeros((len(pts), 4), dtype=F32)
            if len(pts):
                q[:, :3] = pts[:, :3]
            rows.append(q)
            offsets.append(offsets[-1] + len(pts))
            poses.append(np.asarray(P, dtype=np.float64).T.reshape(16))
        pts = np.ascontiguousarray(np.concatenate(rows))
        off = np.array(offsets, dtype=np.int64)
        P = np.ascontiguousarray(np.array(poses, dtype=np.float64).reshape(-1)) if poses else np.zeros(16)
        rc = self.lib.elh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, len(submaps))
        if rc != 0:
            return rc
        return self.last(p)

    def last(self, p):
        info = np.zeros(9, dtype=np.uint64)
        org = np.zeros(2, dtype=np.float64)
        self.lib.elh_info(info.ctypes.data, org.ctypes.data)
        W, H = int(info[0]), int(info[1])
        out = dict(n=np.zeros((H, W), np.uint32), h=np.zeros((H, W), np.int64), lo=np.zeros((H, W), np.int64),
                   step=np.zeros((H, W), F32), tan_slope=np.zeros((H, W), F32), roughness=np.zeros((H, W), F32),
                   value=np.zeros((H, W), np.int8))
        pgm = np.zeros(H * W, dtype=np.uint8)
        self.lib.elh_get(*[out[k].ctypes.data for k in LAYERS], pgm.ctypes.data)
        names = ("n_points", "n_skipped", "n_overhang", "n_observed", "n_lethal", "n_traversable", "n_unknown")
        return dict(width=W, height=H, origin=(float(org[0]), float(org[1])), pgm=pgm.tobytes(), p=p,
                    **{k: int(v) for k, v in zip(names, info[2:])}, **out)

    def const(self, p):
        out = np.zeros(6)
        rc = self.lib.elh_const(param_vector(R.params(**p)).ctypes.data, out.ctypes.data)
        return rc, out

    def save(self, pgm_path, yaml_path):
        return self.lib.elh_save(os.fsencode(pgm_path), os.fsencode(yaml_path))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("el"), "libelev_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    return Host(lib)


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def same(a, b):
    """Two maps bit for bit (float layers compared as bits, NaN included)."""
    assert isinstance(a, dict) and isinstance(b, dict), (a, b)
    for k in COUNTS:
        assert a[k] == b[k], k
    for k in LAYERS:
        assert np.array_equal(bits(a[k]), bits(b[k])), k


def T(x=0.0, y=0.0, z=0.0, yaw=0.0):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix((x, y, z), (0.0, 0.0, yaw))


def grid(nx, ny, f, x0=0, y0=0, per=1):
    """per points at the centre of every cell (x0 + i, y0 + j) at height f(i, j), resolution 1."""
    return np.array([(x0 + i + 0.5, y0 + j + 0.5, f(i, j)) for j in range(ny) for i in range(nx) for _ in range(per)], dtype=F32)


U = 2.0 ** -16  # one fixed-point unit at resolution 1
UNIT = dict(resolution=1.0, max_range=50.0, clearance=2.0, min_points=1, window_cells=1, min_cells=3, max_slope=20.0,
            max_step=0.15, max_roughness=0.05)
LOOSE = dict(UNIT, max_slope=80.0, max_step=10.0, max_roughness=10.0)


def _rough_case():
    """A 3 x 3 patch with a bump: its roughness, from the replay, as the limit (equality: not lethal) and one ulp below."""
    pts = grid(3, 3, lambda i, j: 0.25 if (i, j) == (1, 1) else 0.0)
    c = R.prepare(R.params(**LOOSE))
    detail = {}
    R.window(c, lambda u, v: 16384 if (u, v) == (0, 0) else 0, detail=detail)
    return pts, detail["roughness"]


def cases():
    nan, inf = float("nan"), float("inf")
    c = []
    c.append(("flat", [(grid(5, 5, lambda i, j: 0.0), T())], UNIT))
    c.append(("tilted", [(grid(6, 5, lambda i, j: 0.05 * i + 0.02 * j), T())], dict(UNIT, max_step=0.3)))
    c.append(("cell_edges_negative", [(np.array([(x, y, 0.01 * (x - y)) for x in (-3.0, -2.0, -1.0, 0.0, 1.0, -U, 1 - U)
                                                 for y in (-2.0, -1.0, 0.0, -U)], dtype=F32), T(-0.0, 0.0))], LOOSE))
    c.append(("negative_pose", [(grid(4, 4, lambda i, j: 0.1 * i), T(-10.25, -7.75, 0.5, 0.3))], LOOSE))
    # one cell's points at Z = lo + C exactly (surface) and one unit above (overhang)
    c.append(("clearance_edge", [(np.array([(0.5, 0.5, 0.0), (0.5, 0.5, 2.0), (1.5, 0.5, 0.0), (1.5, 0.5, 2.0 + U),
                                            (2.5, 0.5, 0.0), (0.5, 1.5, 0.0), (1.5, 1.5, 0.0)], dtype=F32), T())], LOOSE))
    # n at min_points - 1 and at min_points
    c.append(("min_points_edge", [(np.concatenate([grid(3, 3, lambda i, j: 0.0, per=2), grid(2, 1, lambda i, j: 0.05, x0=3)]),
                                   T())], dict(LOOSE, min_points=2)))
    # windows of min_cells - 1 and min_cells observed cells
    c.append(("min_cells_edge", [(np.array([(0.5, 0.5, 0), (1.5, 0.5, 0), (0.5, 1.5, 0), (4.5, 4.5, 0), (5.5, 4.5, 0.1),
                                            (4.5, 5.5, 0), (5.5, 5.5, 0)], dtype=F32), T())], dict(LOOSE, min_cells=4)))
    c.append(("border_windows", [(grid(2, 2, lambda i, j: 0.1 * i * j), T())], dict(LOOSE, window_cells=2, min_cells=3)))
    c.append(("collinear", [(np.concatenate([grid(6, 1, lambda i, j: 0.1 * i), grid(1, 1, lambda i, j: 0.0, x0=10, y0=10),
                                             np.array([(20.5 + k, 20.5 + k, 0.0) for k in range(4)], dtype=F32)]), T())],
              dict(LOOSE, window_cells=2)))
    # step at K and one unit past it (0.125 m = 8192 units at resolution 1)
    c.append(("step_equal", [(grid(3, 3, lambda i, j: 0.125 if i == 2 else 0.0), T())], dict(LOOSE, max_step=0.125)))
    c.append(("step_past", [(grid(3, 3, lambda i, j: 0.125 + U if i == 2 else 0.0), T())], dict(LOOSE, max_step=0.125)))
    # slope just under and just over the limit: a plane of tangent 0.25 (14.036 degrees)
    ang = math.degrees(math.atan(0.25))
    c.append(("slope_under", [(grid(3, 3, lambda i, j: 0.25 * i), T())], dict(LOOSE, max_slope=ang * (1 + 1e-9))))
    c.append(("slope_over", [(grid(3, 3, lambda i, j: 0.25 * i), T())], dict(LOOSE, max_slope=ang * (1 - 1e-9))))
    pts, rough = _rough_case()
    c.append(("roughness_equal", [(pts, T())], dict(LOOSE, max_roughness=rough)))
    c.append(("roughness_past", [(pts, T())], dict(LOOSE, max_roughness=math.nextafter(rough, 0.0))))
    # the range gate at exactly R: |dx| = R, dx^2 + dy^2 = R^2 (3-4-5) kept; one fixed-point unit farther skipped
    c.append(("range_gate", [(np.array([(5.0, 0.0, 0.0), (0.0, -5.0, 0.0), (3.0, 4.0, 0.0), (-4.0, 3.0, 0.0),
                                        (5.0 + U, 0.0, 0.0), (3.0, 4.0 + U, 0.0),
                                        (0.5, 0.5, 0.0), (1.5, 0.5, 0.0), (0.5, 1.5, 0.0)], dtype=F32), T())],
              dict(LOOSE, max_range=5.0)))
    c.append(("non_finite", [(np.array([(nan, 0.5, 0.0), (0.5, inf, 0.0), (0.5, 0.5, -inf), (0.5, 0.5, 0.0), (1.5, 0.5, 0.1),
                                        (0.5, 1.5, 0.0)], dtype=F32), T()), (np.zeros((0, 3), F32), T(1.0))], LOOSE))
    c.append(("sensor_origin", [(grid(5, 5, lambda i, j: 0.03 * j), T(1.0, 2.0)), (grid(4, 4, lambda i, j: 0.0, x0=2), T(-1.0))],
              dict(UNIT, sensor_origin=(0.5, -0.25, 1.0), max_range=3.5, min_points=1)))
    # the height extent just inside 2^40 units (2^24 - 1 cells)
    c.append(("height_extent_inside", [(np.array([(0.5, 0.5, 0.0), (1.5, 0.5, 16777215.0), (0.5, 1.5, 0.0)], dtype=F32), T())],
              LOOSE))
    return c


CASES = cases()


@pytest.mark.parametrize("name,subs,p", CASES, ids=[c[0] for c in CASES])
def test_host_equals_replay(host, name, subs, p):
    same(host.build(subs, p), R.build(subs, p))


def test_cases_reach_their_edges(host):
    got = {name: host.build(subs, p) for name, subs, p in CASES}
    assert got["clearance_edge"]["n_overhang"] == 1 and got["clearance_edge"]["h"][0, 0] == 2 * 65536
    mp = got["min_points_edge"]
    assert mp["n_observed"] == 9 and mp["n"][0, 3] == 1 and mp["value"][0, 3] == -1  # pairs observed, single points not
    mc = got["min_cells_edge"]["value"]
    assert mc[0, 0] == -1 and (mc[4:6, 4:6] >= 0).all()
    assert (got["collinear"]["value"] == -1).all()
    assert got["step_equal"]["value"][1, 1] == 99 and got["step_past"]["value"][1, 1] == 100
    assert got["slope_under"]["value"][1, 1] == 99 and got["slope_over"]["value"][1, 1] == 100
    assert got["roughness_equal"]["value"][1, 1] == 99 and got["roughness_past"]["value"][1, 1] == 100
    assert got["range_gate"]["n_points"] == 7 and got["range_gate"]["n_skipped"] == 2
    assert got["non_finite"]["n_skipped"] == 3
    border = got["border_windows"]
    assert (border["width"], border["height"]) == (2, 2) and (border["value"] >= 0).all()


def _refusals():
    ok = [(grid(3, 3, lambda i, j: 0.0), T())]
    bad = [dict(resolution=0.0), dict(resolution=float("nan")), dict(resolution=1e-320), dict(max_range=0.0),
           dict(max_range=1e6, resolution=0.1), dict(sensor_origin=(0, float("inf"), 0)), dict(clearance=-1e-9),
           dict(clearance=float("inf")), dict(min_points=0), dict(window_cells=0), dict(window_cells=9), dict(min_cells=2),
           dict(window_cells=1, min_cells=10), dict(max_slope=0.0), dict(max_slope=90.0), dict(max_slope=float("nan")),
           dict(max_step=0.0), dict(max_step=1e-7), dict(max_step=float("inf")), dict(max_roughness=0.0),
           dict(max_roughness=float("inf")), dict(occupied_thresh=0.2, free_thresh=0.25), dict(occupied_thresh=1.01)]
    out = [(f"param{k}", ok, dict(UNIT, **b), -1) for k, b in enumerate(bad)]
    out.append(("no_submaps", [], UNIT, -4))
    out.append(("only_empty", [(np.zeros((0, 3), F32), T())], UNIT, -5))
    out.append(("all_skipped", [(np.array([(100.0, 0.0, 0.0), (float("nan"), 0, 0)], F32), T())], UNIT, -5))
    out.append(("origin", [(grid(1, 1, lambda i, j: 0.0), T(2.0 ** 31))], UNIT, -2))
    out.append(("cells", [(grid(1, 1, lambda i, j: 0.0), T(20000.0)), (grid(1, 1, lambda i, j: 0.0), T(0.0, 20000.0))], UNIT, -3))
    out.append(("height_extent", [(np.array([(0.5, 0.5, 0.0), (1.5, 0.5, 16777216.0)], dtype=F32), T())], UNIT, -6))
    return out


@pytest.mark.parametrize("name,subs,p,code", _refusals(), ids=[r[0] for r in _refusals()])
def test_refusals(host, name, subs, p, code):
    with pytest.raises(R.Refused) as e:
        R.build(subs, p)
    assert e.value.code == code
    assert host.build(subs, p) == code


def test_refusal_keeps_the_last_map(host):
    name, subs, p = CASES[0]
    first = host.build(subs, p)
    assert host.build(subs, dict(p, window_cells=0)) == -1
    same(host.last(first["p"]), first)


def test_constants_match(host):
    for p in (UNIT, LOOSE, R.DEFAULTS, dict(R.DEFAULTS, resolution=0.05, max_slope=35.0, clearance=1.3)):
        rc, v = host.const(p)
        c = R.prepare(R.params(**p))
        assert rc == 0 and list(v) == [c["S"], float(c["R"]), float(c["C"]), float(c["K"]), c["G"], c["G2"]]


@pytest.mark.parametrize("mut", R.MUTATIONS)
def test_replay_tells_mutations_apart(mut):
    def differs(name, subs, p):
        a, b = R.build(subs, p), R.build(subs, p, mut=mut)
        try:
            same(a, b)
            return False
        except AssertionError:
            return True

    assert any(differs(*c) for c in CASES), mut


def test_sanitised_host_run(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "elevation_host_asan")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-DEL_HOST_MAIN", SRC, "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert out.returncode == 0 and "0 failures" in out.stdout, out.stdout + out.stderr


# ---- the terrain drive ----

@pytest.fixture(scope="module")
def terrain():
    subs, labels = TS.drive()
    return subs, labels


@pytest.fixture(scope="module")
def terrain_map(host, terrain):
    m = host.build(terrain[0])  # the defaults
    assert isinstance(m, dict), m
    return m


def _centres(m):
    res = m["p"]["resolution"]
    x = m["origin"][0] + (np.arange(m["width"]) + 0.5) * res
    y = m["origin"][1] + (np.arange(m["height"]) + 0.5) * res
    return np.meshgrid(x, y)


def test_terrain_ramp10_reads_10_degrees_and_is_traversable(terrain_map):
    m = terrain_map
    X, Y = _centres(m)
    inner = (X > 7) & (X < 23) & (Y > 4) & (Y < 8) & (m["value"] >= 0)
    assert inner.sum() > 500
    deg = np.degrees(np.arctan(m["tan_slope"][inner].astype(np.float64)))
    assert abs(np.median(deg) - 10.0) < 0.5, np.median(deg)
    assert (m["value"][inner] < 100).mean() > 0.97


def test_terrain_ramp30_is_lethal(terrain_map):
    m = terrain_map
    X, Y = _centres(m)
    inner = (X > 7) & (X < 23) & (Y > -8) & (Y < -4) & (m["value"] >= 0)
    assert inner.sum() > 200
    assert (m["value"][inner] == 100).mean() > 0.97


def test_terrain_curb_is_lethal_only_at_its_edge(terrain_map):
    m = terrain_map
    X, Y = _centres(m)
    r = m["p"]["window_cells"] * m["p"]["resolution"]
    span = (X > 37) & (X < 48) & (m["value"] >= 0)
    edge = span & (np.abs(Y - 3.0) < 0.1)
    away = span & (np.abs(Y - 3.0) > r + 0.2) & (Y > 1.0) & (Y < 6.0)
    assert edge.sum() > 50 and away.sum() > 200
    assert (m["value"][edge] == 100).mean() > 0.9
    assert (m["value"][away] < 100).mean() > 0.97


def test_terrain_road_under_the_bridge_is_traversable(terrain_map, terrain):
    m = terrain_map
    X, Y = _centres(m)
    under = (X > 28.5) & (X < 31.5) & (np.abs(Y) < 2.0) & (m["value"] >= 0)
    assert under.sum() > 300
    assert (m["value"][under] < 100).mean() > 0.97
    deck = sum(int((lab == TS.DECK).sum()) for lab in terrain[1])
    assert deck > 1000 and m["n_overhang"] >= deck // 2


def test_terrain_wall_is_lethal(terrain_map):
    m = terrain_map
    X, Y = _centres(m)
    wall = (X > 37) & (X < 53) & (np.abs(Y + 4.6) < 0.15) & (m["value"] >= 0)  # the face the road sees
    assert wall.sum() > 50
    assert (m["value"][wall] == 100).all()


def test_terrain_occupancy_grid_frees_the_curb_and_the_steep_ramp(terrain, terrain_map):
    """Why the elevation map exists. The occupancy grid's band is fixed in the map frame (defaults [0.2, 2.0] m): the 0.2 m
    curb lies below it, and rays to the upper part of a ramp cross its lower part inside it. On this drive the occupancy
    grid marks the curb's edge free and most of the 30 degree ramp free, where the elevation map marks both lethal."""
    import tempfile

    import occupancyref
    from test_occupancy_cpu import Host as OgHost

    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libocc.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++",
                               os.path.join(HERE, "hostmath", "occupancy_host.cpp"), "-o", so])
        g = OgHost(so).build(terrain[0])
    res = occupancyref.params()["resolution"]
    X, Y = np.meshgrid(g["origin"][0] + (np.arange(g["width"]) + 0.5) * res, g["origin"][1] + (np.arange(g["height"]) + 0.5) * res)
    curb = (X > 37) & (X < 48) & (np.abs(Y - 3.0) < 0.1)
    assert curb.sum() > 500 and (g["values"][curb] == 0).mean() > 0.9
    ramp = (X > 7) & (X < 23) & (Y > -8) & (Y < -4) & (g["values"] >= 0)
    assert ramp.sum() > 1000 and (g["values"][ramp] >= 65).mean() < 0.1
    m = terrain_map
    EX, EY = _centres(m)
    assert (m["value"][(EX > 37) & (EX < 48) & (np.abs(EY - 3.0) < 0.1) & (m["value"] >= 0)] == 100).mean() > 0.9
