"""The static map's definitions on the CPU: the product's header csrc/static_map.hpp compiled with g++ -ffp-contract=off
and run serially (tests/hostmath/static_map_host.cpp) against the exact Python replay tests/staticmapref.py, voxel for
voxel and point for point, on hand-built rays at every edge the header names; the replay told apart from its named
mutations; the serial pipeline under AddressSanitizer and UBSan; and, on the moving-object drive of tests/staticscene.py,
the cars removed and the static scene kept."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import staticmapref as R

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "static_map_host.cpp")
F32 = np.float32
FIX = 2.0 ** -16  # one fixed-point unit at resolution 1


class Host:
    """tests/hostmath/static_map_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
        lib.smh_build.argtypes = [vp, vp, vp, vp, i]
        lib.smh_info.argtypes = [vp]
        lib.smh_voxels.argtypes = [vp, vp, vp, vp, vp]
        lib.smh_static.argtypes = [vp, vp]
        lib.smh_walk.argtypes = [ll, ll, ll, ll, ll, ll, vp, ll]
        lib.smh_walk.restype = ll
        lib.smh_box.argtypes = [vp, vp, vp]
        self.lib = lib

    def build(self, submaps, p=None):
        """Same arguments as staticmapref.build; the same dict keys, or the harness's negative return code."""
        p = R.params(**(p or {}))
        par = np.array([p["resolution"], p["max_range"], *p["sensor_origin"], p["ray_fraction"], p["min_frees"],
                        p["dynamic_thresh"]], dtype=np.float64)
        rows = [np.zeros((0, 4), dtype=F32)]
        offsets = [0]
        poses = []
        for pts, P in submaps:
            pts = np.asarray(pts, dtype=F32)
            q = np.zeros((len(pts), 4), dtype=F32)
            if len(pts):
                q[:, :pts.shape[1]] = pts[:, :4]
            rows.append(q)
            offsets.append(offsets[-1] + len(pts))
            poses.append(np.asarray(P, dtype=np.float64).T.reshape(16))
        pts = np.ascontiguousarray(np.concatenate(rows))
        off = np.array(offsets, dtype=np.int64)
        P = np.ascontiguousarray(np.array(poses, dtype=np.float64).reshape(-1)) if poses else np.zeros(16)
        rc = self.lib.smh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, len(submaps))
        if rc != 0:
            return rc
        info = np.zeros(12, dtype=np.int64)
        self.lib.smh_info(info.ctypes.data)
        V, n = int(info[8]), int(info[10])
        ijk = np.zeros((V, 3), dtype=np.int32)
        hits = np.zeros(V, dtype=np.uint32)
        frees = np.zeros(V, dtype=np.uint32)
        dyn = np.zeros(V, dtype=np.uint8)
        keep = np.zeros(n, dtype=np.uint8)
        self.lib.smh_voxels(ijk.ctypes.data, hits.ctypes.data, frees.ctypes.data, dyn.ctypes.data, keep.ctypes.data)
        static = np.zeros((max(1, int(info[11])), 4), dtype=F32)
        offs = np.zeros(len(submaps) + 1, dtype=np.int64)
        self.lib.smh_static(static.ctypes.data, offs.ctypes.data)
        return dict(lo=tuple(int(v) for v in info[0:3]), dims=tuple(int(v) for v in info[3:6]), n_rays=int(info[6]),
                    n_skipped=int(info[7]), ijk=ijk, hits=hits, frees=frees, dynamic=dyn, keep=keep.astype(bool), offsets=offs,
                    n_voxels=V, n_dynamic=int(info[9]), n_points=n, n_static=int(info[11]), static=static[:int(info[11])], p=p)

    def walk(self, a, b):
        cap = sum(abs((b[k] >> 16) - (a[k] >> 16)) for k in range(3)) + 1
        out = np.zeros(3 * cap, dtype=np.int32)
        n = self.lib.smh_walk(*a, *b, out.ctypes.data, cap)
        return [tuple(v) for v in out[:3 * min(n, cap)].reshape(-1, 3).tolist()], n

    def box(self, lo, hi):
        lo, hi = np.array(lo, dtype=np.int32), np.array(hi, dtype=np.int32)
        cells = C.c_ulonglong(0)
        ok = self.lib.smh_box(lo.ctypes.data, hi.ctypes.data, C.byref(cells))
        return cells.value if ok else None


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("sm"), "libstatic_map_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    return Host(lib)


def T(x=0.0, y=0.0, z=0.0, yaw=0.0):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix((x, y, z), (0.0, 0.0, yaw))


def pts(*rows):
    a = np.array(rows, dtype=F32).reshape(-1, 3)
    out = np.zeros((len(a), 4), dtype=F32)
    out[:, :3] = a
    out[:, 3] = np.arange(len(a), dtype=F32)
    return out


# resolution 1 puts voxel edges on integers and one fixed-point unit at 2^-16; the full ray is freed unless a case says
UNIT = dict(resolution=1.0, max_range=50.0, ray_fraction=1.0, min_frees=1, dynamic_thresh=0.5)


def same(a, b):
    assert isinstance(a, dict) and isinstance(b, dict), (a, b)
    for k in ("lo", "dims", "n_rays", "n_skipped", "n_voxels", "n_dynamic", "n_points", "n_static"):
        assert a[k] == b[k], k
    for k in ("ijk", "hits", "frees", "dynamic", "keep", "offsets"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def _blocker(n, *rows):
    """n submaps whose only rays end at the given points: occupied voxels for the walks of the other submaps to cross."""
    return [(pts(*rows), T())] * n


# Every hand-built case: (name, submaps, params).
def cases():
    nan, inf = float("nan"), float("inf")
    c = []
    wall = [(6.5, 0.5, 0.5), (-4.5, 0.5, 0.5), (0.5, 7.5, 0.5), (0.5, -3.5, 0.5), (0.5, 0.5, 5.5), (0.5, 0.5, -3.5)]
    c.append(("axis_parallel", [(pts(*wall), T())] + _blocker(1, (3.5, 0.5, 0.5), (0.5, 3.5, 0.5), (0.5, 0.5, 3.5)), UNIT))
    diag = [(5, 5, 0), (-4, -4, 0), (0, 4, 4), (4, 0, 4), (4, 4, 4), (-4, -4, -4)]  # from (0.5, 0.5, 0.5): edges and corners
    occ = [(1.5, 0.5, 0.5), (0.5, 1.5, 0.5), (0.5, 0.5, 1.5), (-0.5, 0.5, 0.5), (0.5, -0.5, 0.5), (0.5, 0.5, -0.5),
           (1.5, 1.5, 0.5), (1.5, 0.5, 1.5), (0.5, 1.5, 1.5), (-0.5, -0.5, 0.5), (-0.5, 0.5, -0.5)]
    c.append(("diagonal_edges_corners", [(pts(*diag), T(0.5, 0.5, 0.5))] + _blocker(1, *occ), UNIT))
    c.append(("diagonal_from_corner", [(pts((4, 4, 4), (-3, 3, 0), (3, -3, 3), (-2, -2, -2)), T())] +
              _blocker(1, (0.5, 0.5, 0.5), (-0.5, 0.5, 0.5), (0.5, -0.5, 0.5), (0.5, 0.5, -0.5), (-0.5, -0.5, -0.5)), UNIT))
    c.append(("zero_length", [(pts((0.2, 0.1, 0.3), (0.0, 0.0, 0.0), (0.4, 0.45, 0.45), (-0.5, -0.5, -0.5)), T(0.5, 0.5, 0.5))], UNIT))
    c.append(("negative", [(pts((-1.3, -2.7, -0.4), (2.2, -0.6, -3.3), (-0.25, 0.75, -0.5), (-5.5, -5.5, -5.5)), T(-10.3, -7.7, -2.1))] +
              [(pts((-11.6, -10.4, -2.5)), T())], UNIT))
    c.append(("fraction_1", [(pts((6.5, 0.5, 0.5), (0.5, 6.5, 0.5)), T())] + _blocker(1, (5.5, 0.5, 0.5), (0.5, 5.5, 0.5)), UNIT))
    # ray_fraction 0.5, one ray per submap from the origin: to x = 6 + 2^-16 the freed segment ends at floor(3 + 2^-17) = 3
    # (voxel 3, on the boundary); to 6 - 2^-16 one unit below it (voxel 2); to -6 - 2^-16 at -3 - 2^-16 (voxel -4, where a
    # truncation would stop at -3 exactly, voxel -3); to -6 + 2^-16 at -3 (voxel -3)
    half = dict(UNIT, ray_fraction=0.5)
    c.append(("fraction_on_boundary", [(pts((6 + FIX, 0.5, 0.5)), T()), (pts((6 - FIX, 0.5, 0.5)), T()), (pts((-6 - FIX, 0.5, 0.5)), T()),
                                       (pts((-6 + FIX, 0.5, 0.5)), T())] + _blocker(1, (3.5, 0.5, 0.5), (-3.5, 0.5, 0.5)), half))
    rng = dict(UNIT, max_range=5.0)
    c.append(("max_range_equality", [(pts((5, 0, 0), (5 + FIX, 0, 0), (0, -5, 0), (0, -5 - FIX, 0), (0, 0, 5), (0, 0, 5 + FIX),
                                          (3, 4, 0), (3, 4 + FIX, 0), (0, 3, -4), (0, -3, -4 - FIX), (5 - FIX, 0, 0)), T())], rng))
    c.append(("nan_inf", [(pts((nan, 1, 1), (1, nan, 1), (1, 1, nan), (inf, 0, 1), (0, -inf, 1), (2, 2, inf), (3.5, 0.5, 0.5)),
                           T(0.5, 0.5, 0.5))] + [(pts((2.5, 0.5, 0.5)), T(4.5, 0.5, 0.5))], UNIT))
    c.append(("empty_submap", [(np.zeros((0, 4), dtype=F32), T(4.5, 4.5, 4.5)), (pts((2.5, 0.5, 0.5), (4.5, 0.5, 0.5)), T())] +
              _blocker(1, (1.5, 0.5, 0.5)), UNIT))
    # one submap hits voxel 3 and crosses it towards voxel 5: hit wins; another only crosses it
    c.append(("hit_and_free_same_submap", [(pts((5.5, 0.5, 0.5), (3.5, 0.5, 0.5)), T())], UNIT))
    c.append(("hit_and_free_different_submaps", [(pts((3.5, 0.5, 0.5)), T()), (pts((5.5, 0.5, 0.5)), T())], UNIT))
    # voxel 3 hit by one submap (twice) and crossed by three others (one of them twice): min_frees and the value at equality
    base = [(pts((3.5, 0.5, 0.5), (3.5, 0.6, 0.5)), T())] + [(pts((5.5, 0.5, 0.5), (5.5, 0.5, 0.6)), T())] + \
        [(pts((5.5, 0.5, 0.5)), T())] * 2
    for mf in (2, 3, 4):
        c.append((f"min_frees_{mf}", base, dict(UNIT, min_frees=mf, dynamic_thresh=0.25)))
    for th in (0.25, 0.24, 0.255, 0.245):  # value 100 * 1 / 4 = 25: dynamic for 25, not for 24; rint(25.5) = 26, rint(24.5) = 24
        c.append((f"thresh_{th}", base, dict(UNIT, min_frees=1, dynamic_thresh=th)))
    c.append(("rotated_pose", [(pts((7.3, 1.1, 0.2), (-2.2, 4.9, -0.3), (0.4, -6.6, 0.1)), T(1.7, -2.2, 0.9, 0.7)),
                               (pts((3.1, 0.2, -0.8), (-1.0, 2.0, 0.05)), T(0.3, -0.4, 0.7, 0.2))],
              dict(UNIT, resolution=0.25, sensor_origin=(0.3, -0.1, 0.2), ray_fraction=0.85)))
    return c


@pytest.mark.parametrize("name,subs,p", cases(), ids=[c[0] for c in cases()])
def test_host_compile_equals_replay(host, name, subs, p):
    a, b = host.build(subs, p), R.build(subs, p)
    same(a, b)
    assert np.array_equal(a["static"].view(np.uint32), b["points"][b["keep"]].view(np.uint32))


def _voxel(g, key, v):
    hit = np.flatnonzero((g["ijk"] == np.array(v, dtype=np.int32)).all(axis=1))
    return int(g[key][hit[0]]) if len(hit) else None


def test_hand_built_outcomes():
    """What the hand-built cases must show, read off the replay (which the test above ties to the header)."""
    by = {n: R.build(s, p) for n, s, p in cases()}
    g = by["axis_parallel"]
    assert [_voxel(g, "frees", v) for v in ((3, 0, 0), (0, 3, 0), (0, 0, 3))] == [1, 1, 1]
    g = by["diagonal_edges_corners"]
    # from (0.5, 0.5, 0.5) towards (5.5, 5.5, 0.5) through x-y edges: x first, so (1, 0, 0) is freed and (0, 1, 0) is not
    # by that ray; towards (0.5, 4.5, 4.5): y before z, (0, 1, 0) then (0, 1, 1); towards (4.5, 0.5, 4.5): x before z
    h = 1 << 15
    assert R.walk((h, h, h), (11 * h, 11 * h, h))[:3] == [(0, 0, 0), (1, 0, 0), (1, 1, 0)]
    assert R.walk((h, h, h), (h, 9 * h, 9 * h))[:3] == [(0, 0, 0), (0, 1, 0), (0, 1, 1)]
    assert R.walk((h, h, h), (9 * h, h, 9 * h))[:3] == [(0, 0, 0), (1, 0, 0), (1, 0, 1)]
    # through the corners: x, then y, then z
    assert R.walk((h, h, h), (9 * h, 9 * h, 9 * h))[:4] == [(0, 0, 0), (1, 0, 0), (1, 1, 0), (1, 1, 1)]
    assert R.walk((h, h, h), (-7 * h, -7 * h, -7 * h))[:4] == [(0, 0, 0), (-1, 0, 0), (-1, -1, 0), (-1, -1, -1)]
    assert _voxel(g, "frees", (1, 0, 0)) == 1 and _voxel(g, "frees", (1, 1, 0)) == 1 and _voxel(g, "frees", (-1, 0, 0)) == 1
    g = by["zero_length"]
    assert g["dims"] == (1, 1, 1) and int(g["hits"][0]) == 1 and int(g["frees"][0]) == 0
    g = by["negative"]  # floor: (-11.6, -10.4, -2.5) is voxel (-12, -11, -3), not (-11, -10, -2)
    assert _voxel(g, "hits", (-12, -11, -3)) == 2 and _voxel(g, "hits", (-11, -10, -2)) is None
    g = by["fraction_on_boundary"]
    assert _voxel(g, "frees", (3, 0, 0)) == 1 and _voxel(g, "frees", (-4, 0, 0)) == 1
    g = by["max_range_equality"]
    assert g["n_rays"] == 6 and g["n_skipped"] == 5 and g["n_static"] == g["n_points"]
    g = by["nan_inf"]
    assert g["n_rays"] == 2 and g["n_skipped"] == 6 and bool(g["keep"][:6].all())
    g = by["empty_submap"]
    assert g["offsets"].tolist()[:2] == [0, 0]
    g = by["hit_and_free_same_submap"]
    assert _voxel(g, "hits", (3, 0, 0)) == 1 and _voxel(g, "frees", (3, 0, 0)) == 0
    g = by["hit_and_free_different_submaps"]
    assert _voxel(g, "hits", (3, 0, 0)) == 1 and _voxel(g, "frees", (3, 0, 0)) == 1
    assert _voxel(by["min_frees_3"], "frees", (3, 0, 0)) == 3 and _voxel(by["min_frees_3"], "hits", (3, 0, 0)) == 1
    assert [_voxel(by[f"min_frees_{m}"], "dynamic", (3, 0, 0)) for m in (2, 3, 4)] == [1, 1, 0]
    assert [_voxel(by[f"thresh_{t}"], "dynamic", (3, 0, 0)) for t in (0.25, 0.24, 0.255, 0.245)] == [1, 0, 1, 0]
    assert by["thresh_0.25"]["keep"].tolist()[:2] == [False, False]  # both rays into the dynamic voxel are removed


def test_walks_equal_replay(host):
    """Random segments, many through exact edges and corners: the host walk is the replay's voxel for voxel,
    6-connected, from voxel(A) to voxel(B)."""
    rng = np.random.default_rng(7)
    for k in range(3000):
        scale = [1 << 16, 1 << 14, 1 << 20][k % 3]
        a = [int(v) for v in rng.integers(-30 * scale, 30 * scale, size=3)]
        if k % 4 == 0:  # a diagonal through lattice corners
            d = int(rng.integers(-20, 20)) << 16
            a = [(v >> 16) << 16 for v in a]
            b = [a[0] + d, a[1] + (d if k % 8 else -d), a[2] + (d if k % 3 else -d)]
        elif k % 4 == 1:  # along an edge of two axes
            a = [(a[0] >> 16) << 16, (a[1] >> 16) << 16, a[2]]
            b = [a[0], a[1], a[2] + int(rng.integers(-30 << 16, 30 << 16))]
        elif k % 4 == 2:  # a diagonal in one plane through edges
            d = int(rng.integers(-25, 25)) << 16
            a = [(a[0] >> 16) << 16, (a[1] >> 16) << 16, a[2]]
            b = [a[0] + d, a[1] - d, a[2] + int(rng.integers(-1 << 16, 1 << 16))]
        else:
            b = [a[j] + int(rng.integers(-40 << 16, 40 << 16)) for j in range(3)]
        got, n = host.walk(a, b)
        want = R.walk(a, b)
        assert got == want and n == len(want), (a, b)
        assert all(sum(abs(p[j] - q[j]) for j in range(3)) == 1 for p, q in zip(want[:-1], want[1:]))


def test_box_bound(host):
    """2^31 - 1 cells are accepted, 2^31 refused, on the host compile and in the replay."""
    for lo, hi, ok in (((0, 0, 0), (2 ** 31 - 2, 0, 0), True), ((0, 0, 0), (2 ** 31 - 1, 0, 0), False),
                       ((-5, 0, 0), (7, 7, 2 ** 31 // 8 // 13 - 1), True),
                       ((0, 0, 0), (2 ** 16 - 1, 2 ** 15 - 1, 0), False), ((0, 0, 0), (2 ** 16 - 1, 2 ** 15 - 2, 0), True),
                       ((-1, -1, -1), (1288, 1288, 1288), True), ((0, 0, 0), (1290, 1290, 1290), False)):
        cells = 1
        for a in range(3):
            cells *= hi[a] - lo[a] + 1
        want = cells if cells <= 2 ** 31 - 1 else None
        assert (want is not None) == ok, (lo, hi)
        assert host.box(lo, hi) == want and R.box_cells(lo, hi) == want, (lo, hi)
    # a whole build refused over the box: two rays 20 km apart at 0.01 m in x, y and z
    far = [(pts((1, 1, 1)), T()), (pts((1, 1, 1)), T(20000.0, 20000.0, 20000.0))]
    assert host.build(far, dict(resolution=0.01, max_range=100.0)) == -3


def test_refusals_match(host):
    sub = [(pts((1, 1, 1)), T())]
    for p, code in ((dict(resolution=0.0), -1), (dict(resolution=float("nan")), -1), (dict(max_range=0.0), -1),
                    (dict(max_range=-1.0), -1), (dict(max_range=16384.0 * 0.2 + 1e-9), -1),
                    (dict(sensor_origin=(0, float("nan"), 0)), -1), (dict(ray_fraction=0.0), -1), (dict(ray_fraction=1.01), -1),
                    (dict(ray_fraction=2.0 ** -18), -1), (dict(min_frees=0), -1), (dict(dynamic_thresh=-0.01), -1),
                    (dict(dynamic_thresh=1.01), -1)):
        assert host.build(sub, p) == code, p
        with pytest.raises(R.Refused) as e:
            R.build(sub, p)
        assert e.value.code == code
    assert isinstance(host.build(sub, dict(max_range=16384.0 * 0.2)), dict)  # the range bound at equality
    assert isinstance(host.build(sub, dict(ray_fraction=2.0 ** -16)), dict)
    assert host.build([], {}) == -4
    assert host.build([(pts((1, 1, 1)), T(0, 0, 2.0 ** 30 * 0.2 * 1.01))], {}) == -2  # an origin beyond 2^30 voxels


def test_mutations_change_an_outcome():
    by = {n: (s, p) for n, s, p in cases()}

    def differs(name, mut):
        s, p = by[name]
        a, b = R.build(s, p), R.build(s, p, mut={mut})
        return any(not np.array_equal(a[k], b[k]) for k in ("ijk", "hits", "frees", "dynamic", "keep", "offsets"))

    assert differs("diagonal_edges_corners", "y_first")
    assert differs("fraction_on_boundary", "trunc")
    assert differs("hit_and_free_same_submap", "free_wins")
    assert differs("min_frees_3", "count_rays")
    assert differs("nan_inf", "drop_skipped")
    for mut in R.MUTATIONS:  # and no mutation is invisible on the whole set
        assert any(differs(n, mut) for n in by), mut


def test_serial_pipeline_under_sanitizers(tmp_path):
    """The executable form of the harness: static maps from generated submaps (non-finite rows, negative coordinates, empty
    submaps) under -fsanitize=address,undefined, each equal to the build of its submaps in reverse order."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = os.path.join(tmp_path, "static_map_asan")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-DSM_HOST_MAIN", "-x", "c++", SRC, "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr or "ubsan" in build.stderr):
        pytest.skip("this toolchain has no sanitizer runtime")
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0 and "0 failures" in run.stdout, run.stdout + run.stderr


# ------------------------------------------------------------------ the moving-object drive (tests/staticscene.py)
@pytest.fixture(scope="module")
def moving_drive():
    import staticscene

    scans, poses, labels = staticscene.drive()
    return list(zip(scans, poses)), np.concatenate(labels)


def removal(g, labels):
    """Fractions of the car, static (ground included) and ground points the build removes."""
    import staticscene as S

    gone = ~g["keep"]
    return {k: float(gone[labels == v].mean()) if k != "static" else float(gone[labels != S.CAR].mean())
            for k, v in (("car", S.CAR), ("static", None), ("ground", S.GROUND))}


def test_moving_cars_removed_static_scene_kept(host, moving_drive):
    """30 submaps 1.5 m apart down the canyon at their true poses, an oncoming car in submaps 4-20 and a car parked for
    submaps 0-6 that then leaves, through the host compile with the defaults (0.2 m voxels, ray_fraction 0.85, min_frees 2,
    dynamic_thresh 0.4). Measured with this compile: 82.5 % of the 5 161 car points removed, 0.89 % of the static points
    and 0.00 % of the ground (more than half of the static points removed lie on the top of a 1.4 m box beside the
    street, grazed by rays from far away). Why the two defaults: with ray_fraction = 1.0, rays that graze the ground free
    the ground voxels just short of their ends, and 45.1 % of the ground (28.9 % of the static scene) is removed; with
    dynamic_thresh = 0.25 only 39.2 % of the car is removed, since a car voxel is crossed only by the rays whose ends lie
    beyond it."""
    subs, labels = moving_drive
    g = host.build(subs, {})
    r = removal(g, labels)
    print(f"defaults: {r}, voxels {g['n_voxels']}, dynamic {g['n_dynamic']}, rays {g['n_rays']}, skipped {g['n_skipped']}")
    assert g["n_points"] == len(labels) and g["n_rays"] + g["n_skipped"] == len(labels)
    assert r["car"] >= 0.80 and r["static"] <= 0.01
    whole = host.build(subs, dict(ray_fraction=1.0))
    rw = removal(whole, labels)
    print(f"ray_fraction 1.0: {rw}")
    assert rw["ground"] >= 0.10
    strict = removal(host.build(subs, dict(dynamic_thresh=0.25)), labels)
    print(f"dynamic_thresh 0.25: {strict}")
    assert strict["car"] < 0.80
