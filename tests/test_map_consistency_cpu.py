"""The map consistency's definitions on the CPU: the product's header csrc/map_consistency.hpp compiled with g++
-ffp-contract=off and run serially (tests/hostmath/consistency_host.cpp) against the exact Python replay
tests/consistencyref.py, point for point, on hand-built cases at every edge the header names and on random maps; the
replay told apart from its named mutations; mc_log and the Jacobi sweeps against libm and LAPACK; the serial pipeline under
AddressSanitizer and UBSan; and, on the place-recognition drive, a metric that ranks the true, drifted, adjusted and
wrongly adjusted maps as a user would."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import consistencyref as R

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "consistency_host.cpp")
F32 = np.float32
ROW_KEYS = ("n_points", "n_queries", "n_valid", "n_neighbors", "sum_h_q", "sum_plane_q")
INFO_KEYS = ("box_origin", "box_dims", "n_points", "n_skipped", "n_cells", "n_candidates", "n_queries", "n_valid", "n_neighbors",
             "sum_h_q", "sum_plane_q")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Host:
    """tests/hostmath/consistency_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
        lib.mch_build.argtypes = [vp, vp, vp, vp, i]
        lib.mch_info.argtypes = [vp, vp, vp]
        lib.mch_get.argtypes = [vp, vp, vp]
        lib.mch_log.argtypes = [vp, vp, ll]
        lib.mch_lambda.argtypes = [vp, vp, ll]
        lib.mch_box.argtypes = [vp, vp, vp]
        lib.mch_const.argtypes = [vp, vp]
        self.lib = lib

    def build(self, submaps, p=None):
        """Same arguments as consistencyref.build; the same dict keys, or the harness's negative return code."""
        p = R.params(**(p or {}))
        par = np.array([p["radius"], p["min_neighbors"], p["query_stride"]], dtype=np.float64)
        rows, offsets, poses = [np.zeros((0, 4), F32)], [0], []
        for pts, P in submaps:
            pts = np.asarray(pts, dtype=F32).reshape(len(pts), -1) if len(pts) else np.zeros((0, 3), F32)
            q = np.zeros((len(pts), 4), dtype=F32)
            q[:, :3] = pts[:, :3]
            rows.append(q)
            offsets.append(offsets[-1] + len(pts))
            poses.append(np.asarray(P, dtype=np.float64).T.reshape(16))
        pts = np.ascontiguousarray(np.concatenate(rows))
        off = np.array(offsets, dtype=np.int64)
        P = np.ascontiguousarray(np.array(poses, dtype=np.float64).reshape(-1)) if poses else np.zeros(16)
        rc = self.lib.mch_build(_p(par), _p(pts), _p(off), _p(P), len(submaps))
        if rc != 0:
            return rc
        return self.last(len(submaps))

    def last(self, n_sub):
        info = np.zeros(10, dtype=np.int64)
        rows = np.zeros((max(n_sub, 1), 6), dtype=np.int64)
        means = np.zeros(2 * n_sub + 2)
        self.lib.mch_info(_p(info), _p(rows), _p(means))
        M = int(info[6])
        out = dict(n=np.zeros(M, np.uint32), h=np.zeros(M), plane_var=np.zeros(M))
        self.lib.mch_get(_p(out["n"]), _p(out["h"]), _p(out["plane_var"]))
        r = {k: rows[:n_sub, j].copy() for j, k in enumerate(ROW_KEYS)}
        r["mme"], r["mpv"] = means[0:2 * n_sub:2].copy(), means[1:2 * n_sub:2].copy()
        inf = dict(box_origin=tuple(int(v) for v in info[0:3]), box_dims=tuple(int(v) for v in info[3:6]), n_points=M,
                   n_skipped=int(info[7]), n_cells=int(info[8]), n_candidates=int(info[9]),
                   **{k: int(r[k].sum()) for k in ROW_KEYS[1:]}, mme=float(means[2 * n_sub]), mpv=float(means[2 * n_sub + 1]))
        return dict(out, rows=r, info=inf)

    def log(self, x):
        x = np.ascontiguousarray(x, dtype=np.float64)
        out = np.zeros_like(x)
        self.lib.mch_log(_p(x), _p(out), len(x))
        return out

    def lam(self, a6):
        a6 = np.ascontiguousarray(a6, dtype=np.float64)
        out = np.zeros(len(a6))
        self.lib.mch_lambda(_p(a6), _p(out), len(a6))
        return out


def compile_host(tmp):
    lib = os.path.join(tmp, "libconsistency_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    return Host(lib)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return compile_host(str(tmp_path_factory.mktemp("mc")))


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def same(a, b):
    """Two builds bit for bit (doubles compared as bits, NaN included)."""
    assert isinstance(a, dict) and isinstance(b, dict), (a, b)
    for k in ("n", "h", "plane_var"):
        assert np.array_equal(bits(a[k]), bits(b[k])), k
    for k in ROW_KEYS + ("mme", "mpv"):
        assert np.array_equal(bits(np.asarray(a["rows"][k], dtype=b["rows"][k].dtype)), bits(b["rows"][k])), k
    for k in INFO_KEYS:
        assert a["info"][k] == b["info"][k], k
    for k in ("mme", "mpv"):
        assert bits(np.float64(a["info"][k])) == bits(np.float64(b["info"][k])), k


def T(x=0.0, y=0.0, z=0.0, yaw=0.0):
    from lidarslam_ros2_b200 import synth

    return synth.pose_matrix((x, y, z), (0.0, 0.0, yaw))


def replay(submaps, p=None, mut=None):
    try:
        return R.build(submaps, p, mut)
    except R.Refused as e:
        return e.code


def plane(n, rng, z=0.0, extent=1.0, noise=0.0):
    xy = rng.uniform(-extent, extent, size=(n, 2))
    zz = z + noise * rng.standard_normal(n)
    return np.column_stack([xy, zz]).astype(F32)


# radius 1: S = 2^16, so a coordinate v is exactly v * 2^16 in fixed point for dyadic v
U = 1.0 / 65536.0


def hand_cases():
    rng = np.random.default_rng(7)
    I = np.eye(4)
    blob = rng.normal(0, 0.3, size=(40, 3)).astype(F32)
    cases = {
        # a neighbour at exactly D^2 = 2^32 (1 radius on x) and one unit beyond it on the other side
        "radius_edge": ([(np.array([[0.5, 0.5, 0.5], [1.5, 0.5, 0.5], [-0.5 - U, 0.5, 0.5]] + [[0.5 + 0.01 * i, 0.5 + 0.013 * j,
                                                                                            0.5 + 0.011 * (i * j % 3)]
                                                                                           for i in range(3) for j in range(3)],
                                  dtype=F32), I)], dict(radius=1.0, min_neighbors=4)),
        # points on cell faces and corners, at negative coordinates
        "faces_corners": ([(np.array([[x, y, z] for x in (-1.0, 0.0, 1.0, -0.5) for y in (-1.0, 0.0, 0.25) for z in (-2.0, 0.0, 0.5)],
                                     dtype=F32), I)], dict(radius=1.0, min_neighbors=4)),
        # a query alone in its cell, far from the rest
        "alone": ([(np.vstack([blob, [[40.0, 40.0, 40.0]]]).astype(F32), I)], dict(radius=1.0, min_neighbors=4)),
        # n at min_neighbors and one below: a tetrahedron plus neighbours, min_neighbors 5 vs 6
        "min_at": ([(np.array([[0, 0, 0], [0.3, 0, 0], [0, 0.3, 0], [0, 0, 0.3], [0.2, 0.2, 0.2]], dtype=F32), I)],
                   dict(radius=1.0, min_neighbors=5)),
        "min_below": ([(np.array([[0, 0, 0], [0.3, 0, 0], [0, 0.3, 0], [0, 0, 0.3], [0.2, 0.2, 0.2]], dtype=F32), I)],
                      dict(radius=1.0, min_neighbors=6)),
        # exactly coplanar and collinear neighbourhoods: det < 1, invalid
        "coplanar": ([(np.array([[0.1 * i, 0.07 * j, 0.0] for i in range(5) for j in range(5)], dtype=F32), I)],
                     dict(radius=1.0, min_neighbors=4)),
        "collinear": ([(np.array([[0.05 * i, 0.0, 0.25] for i in range(12)], dtype=F32), I)], dict(radius=1.0, min_neighbors=4)),
        # non-finite rows and an empty submap
        "nonfinite_empty": ([(np.vstack([blob, [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]]]).astype(F32), T(1, 2, 0, 0.3)),
                             (np.zeros((0, 3), F32), T(5, 0, 0)), (blob[::-1].copy(), T(1.1, 2, 0.05, 0.31))],
                            dict(radius=0.5, min_neighbors=4)),
        # query_stride larger than the map
        "stride_big": ([(blob, I)], dict(radius=0.5, min_neighbors=4, query_stride=1000)),
        "stride_3": ([(blob, I), (blob, T(0.2, 0, 0))], dict(radius=0.5, min_neighbors=4, query_stride=3)),
        # caller poses, negative coordinates
        "poses": ([(plane(300, rng, extent=2.0, noise=0.01), T(-3.0, -4.0, -1.0, 1.0)),
                   (plane(300, rng, extent=2.0, noise=0.01), T(-3.2, -4.1, -1.02, 1.05))], dict(radius=0.3, min_neighbors=10)),
        "every_point_skipped": ([(np.array([[np.nan, 0, 0]], dtype=F32), I)], {}),
    }
    return cases


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_host_matches_replay_on_hand_cases(host, name):
    submaps, p = hand_cases()[name]
    a, b = host.build(submaps, p), replay(submaps, p)
    same(a, b)
    info = b["info"]
    if name == "radius_edge":
        # the query at x = 0.5 counts the point at exactly one radius and not the one a unit beyond it
        assert b["n"][0] == 1 + 1 + 9 and b["n"][2] >= 1
    if name == "alone":
        assert b["n"][-1] == 1 and np.isnan(b["h"][-1])
    if name == "min_at":
        assert info["n_valid"] >= 1 and b["n"][0] == 5
    if name == "min_below":
        assert info["n_valid"] == 0 and math.isnan(info["mme"])
    if name in ("coplanar", "collinear"):
        assert info["n_valid"] == 0 and info["n_queries"] == info["n_points"]
    if name == "nonfinite_empty":
        assert info["n_skipped"] == 3 and b["rows"]["n_queries"][1] == 0 and math.isnan(b["rows"]["mme"][1])
    if name == "stride_big":
        assert info["n_queries"] == 1
    if name == "every_point_skipped":
        assert info["n_skipped"] == 1 and info["box_dims"] == (0, 0, 0) and info["n_queries"] == 0


def random_map(rng, n_total, n_sub):
    cuts = np.sort(rng.integers(0, n_total + 1, size=n_sub - 1))
    sizes = np.diff(np.concatenate([[0], cuts, [n_total]]))
    subs = []
    for k, m in enumerate(sizes):
        kind = rng.integers(3)
        if kind == 0:
            pts = rng.uniform(-2, 2, size=(m, 3))
        elif kind == 1:
            pts = np.column_stack([rng.uniform(-3, 3, size=(m, 2)), 0.01 * rng.standard_normal(m)])
        else:
            pts = rng.normal(0, 0.4, size=(m, 3))
        subs.append((pts.astype(F32), T(*rng.uniform(-1, 1, 3), yaw=rng.uniform(-3, 3))))
    return subs


@pytest.mark.parametrize("seed,n_total,n_sub", [(1, 0, 1), (2, 1, 1), (3, 700, 3), (4, 5000, 4), (5, 1 << 16, 6)])
def test_host_matches_replay_on_random_maps_and_order_free(host, seed, n_total, n_sub):
    rng = np.random.default_rng(seed)
    subs = random_map(rng, n_total, n_sub)
    p = dict(radius=0.25, min_neighbors=6, query_stride=1 + seed % 2)
    a, b = host.build(subs, p), replay(subs, p)
    same(a, b)
    if n_total == 0:
        return
    # shuffling each submap's points permutes the per-point values and changes no aggregate (stride 1: every point a query)
    p1 = dict(p, query_stride=1)
    base = host.build(subs, p1)
    perms = [rng.permutation(len(s[0])) for s in subs]
    shuf = host.build([(s[0][q], s[1]) for s, q in zip(subs, perms)], p1)
    off = np.concatenate([[0], np.cumsum([len(s[0]) for s in subs])])
    idx = np.concatenate([off[k] + q for k, q in enumerate(perms)])
    for k in ("n", "h", "plane_var"):
        assert np.array_equal(bits(shuf[k]), bits(base[k][idx])), k
    for k in INFO_KEYS:
        assert shuf["info"][k] == base["info"][k], k
    for k in ROW_KEYS:
        assert np.array_equal(shuf["rows"][k], base["rows"][k]), k


@pytest.mark.parametrize("mut", R.MUTATIONS)
def test_replay_tells_each_mutation_apart(mut):
    rng = np.random.default_rng(11)
    subs = [(np.vstack([plane(400, rng, extent=1.0, noise=0.02), rng.uniform(-1, 1, size=(200, 3))]).astype(F32), np.eye(4))]
    # lattice points a whole radius apart on x (D^2 = 2^32 exactly) and a point with a negative coordinate off the lattice
    lat = np.array([[i * 0.5, j * 0.25, k * 0.25] for i in range(-2, 3) for j in range(3) for k in range(3)], dtype=F32)
    subs.append((np.vstack([lat, [[-0.3, 0.1, 0.1]]]).astype(F32), np.eye(4)))
    p = dict(radius=0.5, min_neighbors=4)
    good, bad = R.build(subs, p), R.build(subs, p, mut)
    differs = any(not np.array_equal(bits(good[k]), bits(bad[k])) for k in ("n", "h", "plane_var"))
    assert differs, mut


def test_log_within_2ulp_of_libm(host):
    rng = np.random.default_rng(3)
    x = np.concatenate([np.exp2(rng.uniform(0, 100, 10 ** 6 - 6)), [1.0, 2.0, math.sqrt(2.0), 1.0 + 2 ** -52, 2.0 ** 100,
                                                                      R.TWO_PI_E]])
    got = R.mc_log(x)
    ref = np.log(x)  # glibc's log: correctly rounded or within one ulp
    ulp = np.spacing(np.abs(ref))
    ulp = np.where(ref == 0.0, np.spacing(0.0), ulp)
    assert np.max(np.abs(got - ref) / ulp) <= 2.0
    assert np.array_equal(bits(host.log(x[:20000])), bits(got[:20000]))
    assert all(math.isclose(float(a), math.log(float(v)), rel_tol=3e-16, abs_tol=1e-300) for a, v in zip(got[-6:], x[-6:]))


def test_jacobi_lambda_min_against_eigvalsh(host):
    rng = np.random.default_rng(5)
    n = 10 ** 5
    Q, _ = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    ev = rng.uniform(0, 1, size=(n, 3)) * np.exp2(rng.uniform(-20, 32, size=(n, 1)))
    ev[: n // 4, 1] = ev[: n // 4, 0]                    # a repeated eigenvalue
    ev[n // 4: n // 2, 2] = ev[n // 4: n // 2, 0]        # a repeated smallest or largest
    ev[n // 2: n // 2 + 1000] = ev[n // 2: n // 2 + 1000, :1]  # all three equal
    A = np.einsum("nij,nj,nkj->nik", Q, ev, Q)
    A = 0.5 * (A + A.transpose(0, 2, 1))
    a6 = np.column_stack([A[:, 0, 0], A[:, 0, 1], A[:, 0, 2], A[:, 1, 1], A[:, 1, 2], A[:, 2, 2]])
    got = R.lambda_min(*a6.T)
    w = np.linalg.eigvalsh(A)
    assert np.all(np.abs(got - w[:, 0]) <= 1e-12 * np.abs(w[:, 2]))
    assert np.array_equal(bits(host.lam(a6[:20000])), bits(got[:20000]))
    # diagonal input: no rotation happens at all
    assert R.lambda_min(3.0, 0.0, 0.0, 1.0, 0.0, 2.0) == 1.0


def test_constants_and_box_limit(host):
    for r in (0.01, 0.3, 0.5, 100.0):
        out = np.zeros(4)
        assert host.lib.mch_const(_p(np.array([r, 10, 1.0])), _p(out)) == 0
        c = R.prepare(R.params(radius=r))
        assert np.array_equal(bits(out), bits(np.array([c["S"], c["S2"], c["r2"], c["c0"]])))
    for bad in (dict(radius=0.00999), dict(radius=100.01), dict(radius=float("nan")), dict(min_neighbors=3), dict(query_stride=0)):
        sub = [(np.zeros((5, 3), F32), np.eye(4))]
        assert host.build(sub, bad) == -1 and replay(sub, bad) == -1
    # the box: 2^31 - 1 cells accepted, 2^31 refused, by the host's sm_box and the replay alike
    dims = np.zeros(3, dtype=np.uint32)
    for lo, hi, ok in [((-(1 << 30), 0, 0), ((1 << 30) - 2, 0, 0), True), ((0, 0, 0), ((1 << 16) - 1, (1 << 15) - 1, 0), False),
                       ((0, 0, 0), (46339, 46339, 0), True), ((0, 0, 5), (0, 0, 4), False)]:
        rc = host.lib.mch_box(_p(np.array(lo, np.int32)), _p(np.array(hi, np.int32)), _p(dims))
        assert (rc == 0) == ok and (R.box(lo, hi) is not None) == ok
        if ok:
            assert list(dims) == R.box(lo, hi)


def test_refusals_keep_the_last_build(host):
    rng = np.random.default_rng(2)
    subs = [(plane(500, rng, noise=0.01), np.eye(4))]
    first = host.build(subs, dict(radius=0.3))
    # a coordinate of 2^46 fixed-point units or more (2^30 radii), a box beyond 2^31 - 1 cells, a parameter, no submaps
    far = [(np.array([[0, 0, 0], [float(2 ** 30) * 0.3 * 1.01, 0, 0]], dtype=F32), np.eye(4))]
    wide = [(np.array([[0, 0, 0], [2.0 ** 16 * 100, 2.0 ** 15 * 100, 0]], dtype=F32), np.eye(4))]
    for s, p, code in [(far, dict(radius=0.3), -3), (wide, dict(radius=100.0), -4), (subs, dict(radius=0.0), -1), ([], {}, -2)]:
        assert host.build(s, p) == code and replay(s, p) == code
        same(host.last(1), first)


def test_sanitised_host_pipeline(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "mc_asan")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=undefined", "-DMC_HOST_MAIN", "-x", "c++", SRC, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 failures" in r.stdout


# ---- quality on the place-recognition drive, fixed on the CPU -----------------------------------------------------------

def drive_maps():
    import scancontextref as SC

    scans, gt, (back, back_match, rev, rev_match) = SC.drive()
    idx = list(range(rev + 1))
    drifted, _ = SC.session(gt, idx)
    return scans, [gt[i] for i in idx], drifted, (rev, rev_match)


def adjust(pg, drifted, loop):
    n = len(drifted)
    P = np.ascontiguousarray(np.asarray(drifted, dtype=np.float64).reshape(n, 16))
    f, t, Z = loop
    ids = np.array([f, t], dtype=np.int32)
    rel = np.ascontiguousarray(np.asarray(Z, dtype=np.float64).reshape(16))
    out, res, tr, nt = np.zeros((n, 16)), np.zeros(4), np.zeros(4 * 1000), C.c_int(0)
    pg.pg_adjust(n, _p(P), 5, 1, _p(ids), _p(rel), 10, _p(out), _p(res), 1000, _p(tr), C.byref(nt))
    return list(out.reshape(n, 4, 4))


@pytest.fixture(scope="module")
def pg(tmp_path_factory):
    src = os.path.join(HERE, "hostmath", "posegraph_host.cpp")
    lib = os.path.join(str(tmp_path_factory.mktemp("pg")), "libposegraph_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    return C.CDLL(lib)


def test_quality_on_the_drive(host, pg):
    scans, gt, drifted, (rev, match) = drive_maps()
    Z = np.linalg.inv(gt[match]) @ gt[rev]
    Zbad = Z @ T(7.0)  # the revisit one pilaster (7 m) along the canyon
    maps = dict(true=gt, drifted=drifted, adjusted=adjust(pg, drifted, (match, rev, Z)),
                wrong=adjust(pg, drifted, (match, rev, Zbad)))
    res = {k: host.build(list(zip(scans, P))) for k, P in maps.items()}
    mme = {k: r["info"]["mme"] for k, r in res.items()}
    mpv = {k: r["info"]["mpv"] for k, r in res.items()}
    print("MME", mme, "MPV", mpv)
    # at the defaults (radius 0.5 m, min_neighbors 10): the true map is the crispest by both means, and the edge one
    # pilaster off makes the adjusted map worse. Two expectations do not hold on this fixture and are reported in DESIGN.md
    # section 7b with their numbers: one loop edge moves the drifted map's MME by less than the drift's own spread
    # (adjusted -3.0712 against drifted -3.0754), and the worst submap is the canyon's end, where the way out and the way
    # back first overlap, rather than one under the revisit.
    assert mme["true"] < mme["drifted"] and mpv["true"] < mpv["drifted"]
    assert mme["true"] < mme["adjusted"] and mpv["true"] < mpv["adjusted"]
    assert mme["wrong"] > mme["adjusted"]
    worst = int(np.nanargmax(res["drifted"]["rows"]["mme"]))
    print("worst submap", worst, res["drifted"]["rows"]["mme"])
    assert 0 <= worst < len(gt)
