"""The OctoMap's definitions on the CPU: the product's header csrc/octomap.hpp compiled with g++ -ffp-contract=off and
run serially (tests/hostmath/octomap_host.cpp, a pointer-based octree as OctoMap builds it) against the exact Python
replay tests/octomapref.py (a level-by-level tree from dicts of keys) and its independent .bt decoder: the worked
examples byte for byte, hand-built scenes at the box's edges, every refusal, the replay told apart from its named
mutations, and the serial pipeline under AddressSanitizer and UBSan."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import octomapref as R
import staticmapref as SR

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "octomap_host.cpp")
F32 = np.float32


class Host:
    """tests/hostmath/octomap_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp, i = C.c_void_p, C.c_int
        lib.omh_build.argtypes = [vp, vp, vp, vp, i]
        lib.omh_info.argtypes = [vp]
        lib.omh_result.argtypes = [vp, vp]
        lib.omh_encode.argtypes = [vp, vp, vp, C.c_double, vp, C.c_longlong, vp]
        lib.omh_encode.restype = C.c_longlong
        lib.omh_box.argtypes = [vp, vp]
        lib.omh_resolution_exact.argtypes = [C.c_double]
        self.lib = lib

    def build(self, submaps, p=None):
        """Same arguments as octomapref.build; the same keys, or the harness's negative return code."""
        p = SR.params(**(p or {}))
        par = np.array([p["resolution"], p["max_range"], *p["sensor_origin"], p["ray_fraction"], p["min_frees"],
                        p["dynamic_thresh"]], dtype=np.float64)
        rows, offsets, poses = [np.zeros((0, 4), dtype=F32)], [0], []
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
        rc = self.lib.omh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, len(submaps))
        if rc != 0:
            return rc
        return self.result()

    def result(self):
        info = np.zeros(16, dtype=np.int64)
        self.lib.omh_info(info.ctypes.data)
        dims = tuple(int(v) for v in info[3:6])
        S = np.zeros(dims[::-1], dtype=np.uint8)
        data = np.zeros(int(info[15]), dtype=np.uint8)
        self.lib.omh_result(S.ctypes.data, data.ctypes.data)
        return dict(lo=tuple(int(v) for v in info[0:3]), dims=dims, n_rays=int(info[6]), n_skipped=int(info[7]),
                    n_occupied=int(info[8]), n_dynamic=int(info[9]), n_free=int(info[10]), inner=int(info[11]),
                    occupied_leaves=int(info[12]), free_leaves=int(info[13]), size=int(info[14]), states=S, bytes=data.tobytes())

    def encode(self, lo, S, res):
        S = np.ascontiguousarray(S, dtype=np.uint8)
        lo = np.array(lo, dtype=np.int32)
        dims = np.array(S.shape[::-1], dtype=np.uint32)
        info = np.zeros(4, dtype=np.int64)
        n = self.lib.omh_encode(lo.ctypes.data, dims.ctypes.data, S.ctypes.data, res, None, 0, info.ctypes.data)
        out = np.zeros(n, dtype=np.uint8)
        self.lib.omh_encode(lo.ctypes.data, dims.ctypes.data, S.ctypes.data, res, out.ctypes.data, n, info.ctypes.data)
        return out.tobytes(), dict(inner=int(info[0]), occupied_leaves=int(info[1]), free_leaves=int(info[2]), size=int(info[3]))

    def box(self, lo, hi):
        lo, hi = np.array(lo, dtype=np.int32), np.array(hi, dtype=np.int32)
        return self.lib.omh_box(lo.ctypes.data, hi.ctypes.data)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("om"), "liboctomap_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    return Host(lib)


def T(x=0.0, y=0.0, z=0.0, yaw=0.0):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix((x, y, z), (0.0, 0.0, yaw))


def pts(*rows):
    a = np.array(rows, dtype=F32).reshape(-1, 3)
    out = np.zeros((len(a), 4), dtype=F32)
    out[:, :3] = a
    return out


UNIT = dict(resolution=1.0, max_range=50.0, ray_fraction=1.0, min_frees=1, dynamic_thresh=0.5)
HEAD = (b"# Octomap OcTree binary file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
        b"id OcTree\n")


def one_voxel(lo, state, n=1):
    return lo, np.full((n, n, n), state, dtype=np.uint8)


# ------------------------------------------------------------------ the worked examples, byte for byte
WORKED = [
    ("occupied_at_0", one_voxel((0, 0, 0), R.OCCUPIED), 17, bytes([0x00, 0xC0]) + bytes([0x03, 0x00]) * 14 + bytes([0x02, 0x00])),
    ("occupied_at_minus_1", one_voxel((-1, -1, -1), R.OCCUPIED), 17,
     bytes([0x03, 0x00]) + bytes([0x00, 0xC0]) * 14 + bytes([0x00, 0x80])),
    ("free_block", one_voxel((0, 0, 0), R.FREE, 2), 16, bytes([0x00, 0xC0]) + bytes([0x03, 0x00]) * 13 + bytes([0x01, 0x00])),
]


@pytest.mark.parametrize("name,box,size,data", WORKED, ids=[w[0] for w in WORKED])
def test_worked_examples(host, name, box, size, data):
    lo, S = box
    want = HEAD + b"size %d\nres 0.2\ndata\n" % size + data
    assert R.encode(lo, S, 0.2)[0] == want
    assert host.encode(lo, S, 0.2)[0] == want
    res, n, leaves = R.decode(want)
    assert (res, n) == (0.2, size)
    assert np.array_equal(R.expand(leaves, lo, S.shape[::-1]), S)


# ------------------------------------------------------------------ hand-built scenes: host compile == replay
def cases():
    c = []
    ring = [(2.5, 1.5, 0.5), (-2.5, -1.5, -0.5), (0.5, -2.5, 1.5), (-1.5, 2.5, -1.5), (3.0, 0.0, 0.0)]
    c.append(("straddles_key_0x8000", [(pts(*ring), T(0.25, 0.25, 0.25))], UNIT))
    c.append(("odd_origin", [(pts(*ring), T(3.5, 5.5, 7.5))], UNIT))
    c.append(("even_origin", [(pts(*ring), T(4.5, 6.5, 8.5))], UNIT))
    # a car seen by one submap, driven through by the next two: its voxel is dynamic and FREE
    car = (4.5, 0.5, 0.5)
    c.append(("dynamic_turns_free", [(pts(car, (8.5, 0.5, 0.5)), T()), (pts((8.5, 0.5, 0.5)), T()), (pts((8.5, 0.5, 0.5)), T())],
              UNIT))
    c.append(("skipped_rows", [(pts((float("nan"), 0, 0), (1.5, 1.5, 1.5), (500, 0, 0)), T()), (pts(), T(2.0))], UNIT))
    c.append(("no_ray", [(pts((float("nan"), 0, 0)), T())], UNIT))
    c.append(("defaults_negative", [(pts((-1.3, -2.7, -0.4), (2.2, -0.6, -3.3), (-0.25, 0.75, -0.5)), T(-10.3, -7.7, -2.1, 0.4))],
              None))
    rng = np.random.default_rng(7)
    subs = [(rng.uniform(-6, 6, (150, 3)).astype(F32), T(*rng.uniform(-2, 2, 3), yaw=float(rng.uniform(0, 6)))) for _ in range(4)]
    c.append(("random", subs, dict(resolution=0.5, max_range=20.0, min_frees=1, dynamic_thresh=0.3)))
    return c


CASES = cases()


@pytest.mark.parametrize("name,subs,p", CASES, ids=[c[0] for c in CASES])
def test_host_compile_equals_replay(host, name, subs, p):
    h, r = host.build(subs, p), R.build(subs, p)
    assert isinstance(h, dict), h
    for k in ("lo", "dims", "n_rays", "n_skipped", "n_occupied", "n_dynamic", "n_free", "inner", "occupied_leaves", "free_leaves",
              "size"):
        assert h[k] == r[k], k
    assert np.array_equal(h["states"], r["states"])
    assert h["bytes"] == r["bytes"]
    res, size, leaves = R.decode(h["bytes"])
    assert size == h["size"] and size == h["inner"] + h["occupied_leaves"] + h["free_leaves"]
    assert np.array_equal(R.expand(leaves, h["lo"], h["dims"]), h["states"])


def test_hand_built_outcomes(host):
    by = {c[0]: host.build(c[1], c[2]) for c in CASES}
    g = by["straddles_key_0x8000"]
    assert g["lo"][0] < 0 <= g["lo"][0] + g["dims"][0] - 1  # keys on both sides of 0x8000: the root has two children
    assert g["bytes"].split(b"data\n", 1)[1][:2] not in (b"\x00\xC0", b"\x03\x00")
    assert by["odd_origin"]["lo"][0] % 2 == 1 and by["even_origin"]["lo"][0] % 2 == 0
    d = by["dynamic_turns_free"]
    car = d["states"][0 - d["lo"][2], 0 - d["lo"][1], 4 - d["lo"][0]]
    assert d["n_dynamic"] == 1 and car == R.FREE
    assert d["states"][0 - d["lo"][2], 0 - d["lo"][1], 8 - d["lo"][0]] == R.OCCUPIED
    assert by["no_ray"]["size"] == 0 and by["no_ray"]["bytes"].endswith(b"size 0\nres 1\ndata\n")
    assert by["skipped_rows"]["n_skipped"] == 2


def test_large_free_cube_collapses_near_the_root(host):
    """A FREE cube of 64^3 voxels aligned on key 0x8000: one level-6 leaf under a chain of 10 inner nodes."""
    S = np.full((64, 64, 64), R.FREE, dtype=np.uint8)
    data, counts = host.encode((0, 0, 0), S, 0.2)
    assert data == R.encode((0, 0, 0), S, 0.2)[0]
    assert counts == dict(inner=10, occupied_leaves=0, free_leaves=1, size=11)
    res, size, leaves = R.decode(data)
    assert leaves == [(6, R.KEY, R.KEY, R.KEY, R.FREE)]
    # one voxel OCCUPIED breaks the collapse along its branch only
    S[5, 9, 33] = R.OCCUPIED
    data, counts = host.encode((0, 0, 0), S, 0.2)
    assert data == R.encode((0, 0, 0), S, 0.2)[0]
    assert counts["inner"] == 16 and counts["occupied_leaves"] == 1 and counts["free_leaves"] == 6 * 7
    assert np.array_equal(R.expand(R.decode(data)[2], (0, 0, 0), (64, 64, 64)), S)


def test_refusals(host):
    far = dict(UNIT, max_range=100.0)
    cases = [
        (dict(UNIT, resolution=0.1000001), [(pts((1, 1, 1)), T())], -6),
        (UNIT, [(pts((1.5, 0, 0)), T(32767.5))], -5),  # the endpoint voxel 32769 is beyond key 65535
        (UNIT, [(pts((-1.5, 0, 0)), T(-32768.5))], -5),
        (far, [(pts((1, 1, 1)), T(-16000, -16000, -8000)), (pts((1, 1, 1)), T(16000, 16000, 8000))], -3),
        (dict(UNIT, resolution=-1.0), [(pts((1, 1, 1)), T())], -1),
        (UNIT, [], -4),
    ]
    for p, subs, code in cases:
        assert host.build(subs, p) == code, (p, code)
        with pytest.raises(R.Refused) as e:
            R.build(subs, p)
        assert e.value.code == code, (p, code, e.value.args)
    # the origin's voxel widens the box: an endpoint inside the key range seen from an origin beyond it is refused
    assert host.build([(pts((-3.5, 0, 0)), T(32768.5))], UNIT) == -5
    assert host.box((-32768, 0, 0), (32767, 0, 0)) == 0 and host.box((-32769, 0, 0), (0, 0, 0)) == -5
    assert host.box((0, 0, 0), (2047, 2047, 511)) == -3
    assert host.lib.omh_resolution_exact(0.05) == 1 and host.lib.omh_resolution_exact(0.1 + 0.2) == 0


def test_mutations_change_an_outcome(host):
    scene = CASES[[c[0] for c in CASES].index("random")]
    base = R.build(scene[1], scene[2])
    assert base["bytes"] == host.build(scene[1], scene[2])["bytes"]
    S = np.full((4, 4, 4), R.FREE, dtype=np.uint8)
    S[0, 0, 0] = R.OCCUPIED
    for mut in R.MUTATIONS:
        differs = R.build(scene[1], scene[2], mut=(mut,))["bytes"] != base["bytes"]
        differs = differs or R.encode((0, 0, 0), S, 1.0, mut=(mut,))[0] != host.encode((0, 0, 0), S, 1.0)[0]
        assert differs, mut
    # the independent decoder refuses what the size mutation writes
    with pytest.raises(ValueError):
        R.decode(R.encode((0, 0, 0), S, 1.0, mut=("size_no_leaves",))[0])


def test_serial_pipeline_under_sanitizers(tmp_path):
    """The executable form of the harness: OctoMaps from generated submaps (non-finite rows, negative coordinates, empty
    submaps) under -fsanitize=address,undefined, each equal to the build of its submaps in reverse order."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = os.path.join(tmp_path, "octomap_asan")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-DOM_HOST_MAIN", "-x", "c++", SRC, "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr or "ubsan" in build.stderr):
        pytest.skip("this toolchain has no sanitizer runtime")
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0 and "0 failures" in run.stdout, run.stdout + run.stderr
