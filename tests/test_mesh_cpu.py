"""The surface mesh's definitions on the CPU: the product's header csrc/mesh.hpp compiled with g++ -ffp-contract=off and
run serially (tests/hostmath/mesh_host.cpp) against the exact Python replay tests/meshref.py, voxel for voxel, vertex bit
for bit and face for face, on hand-built rays at every edge the header names; analytic shapes (a plane, a sphere) in the
replay; the replay told apart from its named mutations; the serial pipeline under AddressSanitizer and UBSan; and the
mesh of tests/staticscene.py's drive held to the quality figures DESIGN.md section 7b reports."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import meshref as R

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "mesh_host.cpp")
F32 = np.float32
SCALARS = ("lo", "dims", "n_points", "n_rays", "n_skipped", "n_walked", "n_band_voxels", "n_observed_voxels", "n_vertices",
           "n_faces")
ARRAYS = ("ijk", "sum", "weight", "faces")


class Host:
    """tests/hostmath/mesh_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp = C.c_void_p
        lib.msh_build.argtypes = [vp, vp, vp, vp, C.c_int]
        lib.msh_info.argtypes = [vp]
        lib.msh_arrays.argtypes = [vp] * 5
        lib.msh_extract.argtypes = [vp, vp, vp, vp, vp, C.c_longlong, C.c_double, C.c_uint]
        lib.msh_box.argtypes = [vp, vp, C.c_int, vp, vp]
        self.lib = lib

    def _result(self):
        info = np.zeros(14, dtype=np.int64)
        self.lib.msh_info(info.ctypes.data)
        B, V, Fc = int(info[10]), int(info[12]), int(info[13])
        out = dict(ijk=np.zeros((B, 3), dtype=np.int32), sum=np.zeros(B, dtype=np.int64), weight=np.zeros(B, dtype=np.uint32),
                   vertices=np.zeros((V, 3), dtype=F32), faces=np.zeros((Fc, 3), dtype=np.uint32))
        self.lib.msh_arrays(*[out[k].ctypes.data for k in ("ijk", "sum", "weight", "vertices", "faces")])
        out.update(lo=tuple(int(v) for v in info[0:3]), dims=tuple(int(v) for v in info[3:6]), n_points=int(info[6]),
                   n_rays=int(info[7]), n_skipped=int(info[8]), n_walked=int(info[9]), n_band_voxels=B,
                   n_observed_voxels=int(info[11]), n_vertices=V, n_faces=Fc)
        return out

    def build(self, submaps, p=None):
        """Same arguments as meshref.build; the same dict keys, or the harness's negative return code."""
        p = R.params(**(p or {}))
        par = np.array([p["resolution"], p["truncation"], p["max_range"], *p["sensor_origin"], p["min_weight"]], dtype=np.float64)
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
        rc = self.lib.msh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, len(submaps))
        return rc if rc != 0 else self._result()

    def extract(self, lo, dims, ijk, sums, weights, res, min_weight):
        lo = np.array(lo, dtype=np.int32)
        dims = np.array(dims, dtype=np.uint32)
        ijk = np.ascontiguousarray(np.array(ijk, dtype=np.int32).reshape(-1, 3))
        sums = np.ascontiguousarray(np.array(sums, dtype=np.int64))
        weights = np.ascontiguousarray(np.array(weights, dtype=np.uint32))
        assert self.lib.msh_extract(lo.ctypes.data, dims.ctypes.data, ijk.ctypes.data, sums.ctypes.data, weights.ctypes.data,
                                    len(sums), float(res), int(min_weight)) == 0
        return self._result()

    def box(self, lo, hi, r):
        lo, hi = np.array(lo, dtype=np.int32), np.array(hi, dtype=np.int32)
        blo, dims = np.zeros(3, dtype=np.int32), np.zeros(3, dtype=np.uint32)
        ok = self.lib.msh_box(lo.ctypes.data, hi.ctypes.data, int(r), blo.ctypes.data, dims.ctypes.data)
        return (tuple(int(v) for v in blo), tuple(int(v) for v in dims)) if ok else None


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("ms"), "libmesh_host.so")
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


def wall(x, y0=-1.0, y1=1.0, z0=-1.0, z1=1.0, step=0.1):
    """Points on the plane x = const, a grid over [y0, y1] x [z0, z1]."""
    ys = np.arange(y0, y1 + 1e-9, step)
    zs = np.arange(z0, z1 + 1e-9, step)
    Y, Z = np.meshgrid(ys, zs, indexing="ij")
    return pts(*np.stack([np.full(Y.size, x), Y.ravel(), Z.ravel()], axis=1))


def same(a, b):
    assert isinstance(a, dict) and isinstance(b, dict), (a, b)
    for k in SCALARS:
        assert a[k] == b[k], k
    for k in ARRAYS:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    assert np.array_equal(a["vertices"].view(np.uint32), b["vertices"].view(np.uint32))


# resolution 0.5, truncation 1.0 (two voxels), min_weight 2, two submaps at one pose unless a case says otherwise
P = dict(resolution=0.5, truncation=1.0, max_range=50.0, min_weight=2)
UNIT = dict(resolution=1.0, truncation=2.0, max_range=20.0, min_weight=1)
EMPTY = np.zeros((0, 4), dtype=F32)


def cases():
    nan = float("nan")
    c = []
    c.append(("wall", [(wall(3.3), T())] * 2, P))
    c.append(("wall_on_boundary", [(wall(3.0), T())] * 2, P))  # every endpoint exactly on a voxel boundary
    # |d| == T (A = O, the walk starts at the origin) and |d| < T, beside a wall
    c.append(("l_equal_and_below_t", [(np.vstack([wall(4.25), pts((2.0, 0.0, 0.0), (1.0, 0.3, 0.2))]), T())] * 2, UNIT))
    c.append(("zero_length", [(np.vstack([wall(3.3), pts((0.0, 0.0, 0.0))]), T())] * 2, P))
    # four rays ending at a voxel centre along x: s = T exactly at the centre 2 voxels in front, -T 2 behind, 0 at the centre
    c.append(("s_at_t_and_zero", [(pts((5.5, 0.0, 0.0), (5.5, 0.0, 0.0)), T(0.0, 0.5, 0.5))] * 2, UNIT))
    # the same four rays: every voxel of the walk has weight 4, observed at min_weight 4 and not at 5
    c.append(("weight_at_min", [(pts((5.5, 0.0, 0.0), (5.5, 0.0, 0.0)), T(0.0, 0.5, 0.5))] * 2, dict(UNIT, min_weight=4)))
    c.append(("weight_below_min", [(pts((5.5, 0.0, 0.0), (5.5, 0.0, 0.0)), T(0.0, 0.5, 0.5))] * 2, dict(UNIT, min_weight=5)))
    # a wall seen by both submaps over y in [-1, 1] and by one over (1, 2]: cells with one unobserved corner
    c.append(("one_unobserved_corner", [(wall(3.3, y1=2.0), T()), (wall(3.3), T())], dict(P, min_weight=5)))
    c.append(("negative_and_nonfinite", [(np.vstack([wall(-3.3), pts((nan, 0.0, 0.0), (0.0, float("inf"), 0.0))]), T(-7.1, -3.9, -2.2, 2.9))] * 2,
                                         P))
    c.append(("empty_submap", [(EMPTY, T(1, 1, 1)), (wall(3.3), T()), (EMPTY, T()), (wall(3.3), T())], P))
    # max_range 4: a ray of exactly 4 m is cast, one unit (2^-16 voxel) longer is not, one unit shorter is
    u = 2.0 ** -16
    c.append(("max_range_edges", [(np.vstack([wall(2.5), pts((4.0, 0.0, 0.0), (4.0 + u, 0.0, 0.0), (4.0 - u, 0.0, 0.0))]), T())] * 2,
                                  dict(UNIT, max_range=4.0)))
    c.append(("ratio_1", [(wall(3.3), T())] * 2, dict(P, truncation=0.5)))
    c.append(("ratio_16", [(wall(3.3), T())] * 2, dict(P, truncation=8.0)))
    c.append(("rotated_poses", [(wall(3.3, step=0.07), T(0.4, -0.2, 0.1, 0.3)), (wall(2.9, step=0.07), T(-0.1, 0.3, -0.2, -0.2))],
              dict(P, sensor_origin=(0.1, -0.05, 0.2))))
    return c


@pytest.mark.parametrize("name,subs,p", cases(), ids=[c[0] for c in cases()])
def test_host_compile_equals_replay(host, name, subs, p):
    same(host.build(subs, p), R.build(subs, p))


def _by():
    return {n: R.build(s, p) for n, s, p in cases()}


def test_hand_built_outcomes():
    """What the hand-built cases must show, read off the replay (which the test above ties to the header)."""
    by = _by()
    for n in ("wall", "wall_on_boundary", "ratio_1", "ratio_16", "rotated_poses", "negative_and_nonfinite", "empty_submap"):
        assert by[n]["n_faces"] > 0, n
    g = by["zero_length"]  # the zero-length ray is a ray that walks nothing
    assert g["n_rays"] == by["wall"]["n_rays"] + 2 and g["n_walked"] == by["wall"]["n_walked"]
    assert np.array_equal(g["sum"], by["wall"]["sum"])
    g = by["s_at_t_and_zero"]
    field = {tuple(v): (int(s), int(w)) for v, s, w in zip(g["ijk"].tolist(), g["sum"], g["weight"])}
    Tq = g["c"]["T"]
    assert Tq == 2 << 16 and field[(3, 0, 0)] == (4 * Tq, 4) and field[(7, 0, 0)] == (-4 * Tq, 4) and field[(5, 0, 0)] == (0, 4)
    g = by["l_equal_and_below_t"]  # both short rays start their walks at the origin's voxel
    assert (0, 0, 0) in {tuple(v) for v in g["ijk"].tolist()}
    assert by["weight_at_min"]["n_observed_voxels"] == by["weight_at_min"]["n_band_voxels"]
    assert by["weight_below_min"]["n_observed_voxels"] == 0 and by["weight_below_min"]["n_faces"] == 0
    g = by["max_range_edges"]
    assert g["n_skipped"] == 2 and g["n_rays"] == 2 * (len(wall(2.5)) + 2)
    g = by["negative_and_nonfinite"]
    assert g["n_skipped"] == 4 and min(g["lo"]) < 0
    g = by["empty_submap"]
    assert g["n_points"] == 2 * len(wall(3.3)) and g["n_faces"] == by["wall"]["n_faces"]
    # a cell with exactly one unobserved corner and signs that differ: no vertex, and no face refers to it
    g = by["one_unobserved_corner"]
    obs = {tuple(v) for v, w in zip(g["ijk"].tolist(), g["weight"]) if w >= 5}
    sign = {tuple(v): s < 0 for v, s in zip(g["ijk"].tolist(), g["sum"])}
    corners = [(a & 1, (a >> 1) & 1, (a >> 2) & 1) for a in range(8)]
    seven = 0
    for v in g["ijk"].tolist():
        cs = [tuple(v[k] + o[k] for k in range(3)) for o in corners]
        seen = [c for c in cs if c in obs]
        if len(seen) == 7 and len({sign[c] for c in seen}) == 2:
            seven += 1
    assert seven > 0
    assert g["n_faces"] > 0 and g["faces"].max() < g["n_vertices"]


def _checkerboard_field():
    """A 4 x 4 x 3 block of observed voxels (weight 3) whose sums fall with z, except the four voxels (1..2, 1..2, 1),
    which alternate in sign: a checkerboard cell face in the plane z = 1."""
    vox, sums = [], []
    for z in range(3):
        for y in range(4):
            for x in range(4):
                if z == 1 and x in (1, 2) and y in (1, 2):
                    s = -5000 if (x + y) % 2 else 7000
                else:
                    s = 9000 - 6000 * z + 100 * x - 50 * y
                vox.append((x, y, z))
                sums.append(s)
    return vox, np.array(sums, dtype=np.int64), np.full(len(vox), 3, dtype=np.uint32)


def test_checkerboard_face_and_extraction(host):
    """The extraction alone on a hand-made field with a checkerboard cell face: host and replay agree, and the dual edge
    across that face is shared by four quads (the non-manifold case the header names)."""
    vox, sums, w = _checkerboard_field()
    verts, faces = R.extract(vox, sums, w, 0.5, 2)
    g = host.extract((0, 0, 0), (4, 4, 3), vox, sums, w, 0.5, 2)
    assert np.array_equal(g["vertices"].view(np.uint32), verts.view(np.uint32)) and np.array_equal(g["faces"], faces)
    assert len(faces) > 0 and _non_manifold_edges(faces) > 0
    # min_weight above every weight: nothing is observed, no vertex
    assert len(R.extract(vox, sums, w, 0.5, 4)[0]) == 0


def _non_manifold_edges(faces):
    from collections import Counter

    f = np.asarray(faces, dtype=np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    cnt = Counter(map(tuple, e.tolist()))
    return sum(1 for v in cnt.values() if v > 2)


def test_parameter_and_box_refusals(host):
    w = [(wall(3.3), T())] * 2
    for bad in (dict(truncation=0.5 * 0.999), dict(truncation=8.0 * 1.001), dict(truncation=float("nan")), dict(min_weight=0),
                dict(resolution=0.0), dict(max_range=0.5 * 16385)):
        assert host.build(w, dict(P, **bad)) == -1, bad
        with pytest.raises(R.Refused) as e:
            R.build(w, dict(P, **bad))
        assert e.value.code == -1
    assert host.build([], P) == -4
    # the box check at its edge: 2^31 - 1 voxels accepted, 2^31 refused (a prime, so only r = 0 reaches it exactly);
    # with r = 1, 3 x 3 x 238609294 = 2^31 - 2 accepted and one more row refused
    for lo, hi, r, ok in (((0, 0, 0), ((1 << 31) - 2, 0, 0), 0, True), ((0, 0, 0), ((1 << 31) - 1, 0, 0), 0, False),
                          ((5, -7, 0), (5, -7, 238609291), 1, True), ((5, -7, 0), (5, -7, 238609292), 1, False)):
        got, want = host.box(lo, hi, r), R.box(lo, hi, r)
        assert (got is not None) == ok and got == want, (lo, hi, r)
    far = [(wall(3.3), T()), (wall(3.3), T(0.0, 0.0, 0.0)), (pts((0.0, 0.0, 0.0)), T(30000.0, 30000.0, 30000.0))]
    assert host.build(far, dict(P, resolution=0.02, truncation=0.04, max_range=100.0)) == -3


def test_mutations_change_an_outcome(host):
    by = {n: (s, p) for n, s, p in cases()}

    def differs(name, mut):
        s, p = by[name]
        a = R.build(s, p)
        b = R.build(s, p, mut={mut})
        return any(not np.array_equal(a[k], b[k]) for k in ARRAYS + ("vertices",))

    vox, sums, w = _checkerboard_field()
    sums[vox.index((3, 3, 1))] = 0  # a sum of exactly 0 is POS
    a, b = R.extract(vox, sums, w, 0.5, 2), R.extract(vox, sums, w, 0.5, 2, mut={"zero_neg"})
    assert not np.array_equal(a[0], b[0]) or not np.array_equal(a[1], b[1])
    assert differs("wall", "ceil_off")
    assert differs("wall", "centre_vertex")
    assert differs("rotated_poses", "flip_y")
    assert differs("one_unobserved_corner", "three_active")
    assert differs("zero_length", "weight_per_submap") or differs("wall", "weight_per_submap")
    vox, sums, w = _checkerboard_field()
    base = R.extract(vox, sums, w, 0.5, 2)
    assert any(not np.array_equal(base[1], R.extract(vox, sums, w, 0.5, 2, mut={m})[1]) for m in ("flip_y",))


# ------------------------------------------------------------------ analytic shapes in the replay
def _sphere(radius, n, seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return pts(*(radius * v))


def _normals(g):
    v = g["vertices"].astype(np.float64)
    f = g["faces"].astype(np.int64)
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    return v[f].mean(axis=1), n


def test_plane_seen_from_one_origin():
    """A wall at x = 3.3 seen from the origin: every vertex within 0.02 m (a tenth of a voxel) of the plane, every face
    normal pointing back to the sensor (-x)."""
    g = R.build([(wall(3.3, -1.5, 1.5, -1.5, 1.5, 0.05), T())] * 2, dict(resolution=0.2, truncation=0.6, max_range=50.0))
    assert g["n_vertices"] > 100
    x = g["vertices"][:, 0].astype(np.float64)
    print(f"plane: {g['n_vertices']} vertices, max |x - 3.3| {np.abs(x - 3.3).max():.4f} m")
    assert np.abs(x - 3.3).max() < 0.02
    _, n = _normals(g)
    assert (n[:, 0] < 0).all()


def test_sphere_seen_from_its_centre():
    """A sphere of radius 2 m seen from its centre: every vertex within resolution / 4 of the radius, every face normal
    pointing inwards, to the sensor."""
    g = R.build([(_sphere(2.0, 6000, k), T()) for k in range(2)], dict(resolution=0.2, truncation=0.6, max_range=50.0))
    rad = np.linalg.norm(g["vertices"].astype(np.float64), axis=1)
    print(f"sphere: {g['n_vertices']} vertices, radius error max {np.abs(rad - 2.0).max():.4f} m")
    assert g["n_vertices"] > 500 and np.abs(rad - 2.0).max() < 0.05
    c, n = _normals(g)
    assert ((c * n).sum(axis=1) < 0).all()


def test_serial_pipeline_under_sanitizers(tmp_path):
    """The executable form of the harness: meshes of generated submaps (non-finite rows, zero-length rays, empty submaps)
    under -fsanitize=address,undefined, each equal to the build of the submaps and points in reverse order."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = os.path.join(tmp_path, "mesh_asan")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-DMS_HOST_MAIN", "-x", "c++", SRC, "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr or "ubsan" in build.stderr):
        pytest.skip("this toolchain has no sanitizer runtime")
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0 and "0 failures" in run.stdout, run.stdout + run.stderr


# ------------------------------------------------------------------ the drive (tests/staticscene.py)
@pytest.fixture(scope="module")
def drive():
    import staticscene

    return staticscene.drive()


def true_distance(x):
    """Distance of points (n, 3) to synth.make_scene()'s surfaces: the ground z = 0, the facades, the boxes' faces and the
    cylinders' sides."""
    from lidarslam_ros2_b200 import synth

    sc = synth.make_scene()
    d = np.abs(x[:, 2])
    for ys in (sc.facade_y, -sc.facade_y):
        d = np.minimum(d, np.abs(x[:, 1] - ys))
    for b in sc.boxes:
        lo, hi = b[:3], b[3:]
        out = np.maximum(np.maximum(lo - x, x - hi), 0.0)
        outside = np.linalg.norm(out, axis=1)
        inside = np.minimum(x - lo, hi - x).min(axis=1)
        d = np.minimum(d, np.where(outside > 0, outside, np.abs(inside)))
    for cx, cy, r, h in sc.cylinders:
        rad = np.hypot(x[:, 0] - cx, x[:, 1] - cy)
        side = np.hypot(np.abs(rad - r), np.maximum(np.maximum(-x[:, 2], x[:, 2] - h), 0.0))
        d = np.minimum(d, side)
    return d


def car_distance(x, boxes):
    d = np.full(len(x), np.inf)
    for b in boxes:
        lo, hi = b[:3], b[3:]
        out = np.linalg.norm(np.maximum(np.maximum(lo - x, x - hi), 0.0), axis=1)
        inside = np.minimum(x - lo, hi - x).min(axis=1)
        d = np.minimum(d, np.where(out > 0, out, np.abs(inside)))
    return d


def quality(host, drive, p=None):
    import staticscene as S
    from scipy.spatial import cKDTree

    scans, poses, labels = drive
    g = host.build(list(zip(scans, poses)), p or {})
    res = R.params(**(p or {}))["resolution"]
    v = g["vertices"].astype(np.float64)
    cars = np.vstack([S.cars(k) for k in range(S.N_SUB)])
    parked = S.cars(0)  # the parked car alone (the oncoming one arrives at submap 4)
    dcar = car_distance(v, parked)
    on_car = dcar < res
    dist = true_distance(v)
    scene_v = ~on_car
    # completeness: noiseless static hits (the scene without cars, re-cast) within one resolution of a vertex or face centre
    f = g["faces"].astype(np.int64)
    centres = v[f].mean(axis=1)
    tree = cKDTree(np.vstack([v, centres]))
    hits = []
    from lidarslam_ros2_b200 import synth

    sc = synth.make_scene()
    for k in range(0, S.N_SUB, 3):
        P = S.pose(k)
        d = scans[k][:, :3].astype(np.float64)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        dw = d @ P[:3, :3].T
        r = synth._ray_cast(sc, P[:3, 3], dw, 100.0)
        ok = np.isfinite(r) & (labels[k] != S.CAR)
        hits.append(P[:3, 3] + r[ok, None] * dw[ok])
    hits = np.vstack(hits)
    near, _ = tree.query(hits, distance_upper_bound=res)
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    ground = (np.abs(centres[:, 2]) < res) & (car_distance(centres, cars) > res) & (true_distance(centres) >= np.abs(centres[:, 2]) - 1e-9)
    out = dict(n_vertices=g["n_vertices"], n_faces=g["n_faces"], n_band_voxels=g["n_band_voxels"],
               dist_median=float(np.median(dist[scene_v])), dist_p95=float(np.percentile(dist[scene_v], 95)),
               completeness=float(np.isfinite(near).mean()),
               ground_up=float((n[ground, 2] > 0).mean()),
               non_manifold=_non_manifold_edges(f) / max(1, len(f) * 3 // 2),
               car_vertices=int(on_car.sum()), car_dist_median=float(np.median(dcar[on_car])) if on_car.any() else None)
    return out


def test_drive_quality(host, drive):
    """30 submaps down the canyon at their true poses through the host compile at the shipped defaults (0.2 m voxels,
    truncation 0.6 m, min_weight 2). The figures this compile gives are in DESIGN.md section 7b; the bounds hold them."""
    q = quality(host, drive)
    print(f"drive quality: {q}")
    assert q["dist_median"] < 0.03 and q["dist_p95"] < 0.10
    assert q["completeness"] > 0.80
    assert q["ground_up"] > 0.99
    assert q["non_manifold"] < 0.01
    assert q["car_vertices"] > 0  # the parked car is meshed, as it should be
