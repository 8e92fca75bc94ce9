"""The map changes' definitions on the CPU: the product's header csrc/map_changes.hpp compiled with g++ -ffp-contract=off
and run serially (tests/hostmath/map_changes_host.cpp) against the exact Python replay tests/changeref.py, voxel for voxel
and point for point, on hand-built rays at every edge the header names; the replay told apart from its named mutations;
each epoch's counts equal to the static map of that epoch alone; the serial pipeline under AddressSanitizer and UBSan;
and, on the two-day drive of tests/changescene.py, the vanished car and the new container found and the static scene
left alone."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import changeref as R
from test_static_map_cpu import host as sm_host  # noqa: F401 (fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "map_changes_host.cpp")
F32 = np.float32
COUNTS = ("hits_before", "frees_before", "hits_after", "frees_after")
SCALARS = ("lo", "dims", "split", "n_rays", "n_skipped", "n_voxels", "n_appeared_voxels", "n_vanished_voxels", "n_points",
           "n_appeared_points", "n_vanished_points", "n_updated_points")
ARRAYS = ("ijk",) + COUNTS + ("label", "point_label", "offsets")


class Host:
    """tests/hostmath/map_changes_host.cpp through ctypes."""

    def __init__(self, path):
        lib = C.CDLL(path)
        vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
        lib.chh_build.argtypes = [vp, ll, ll, vp, vp, vp, i]
        lib.chh_info.argtypes = [vp]
        lib.chh_voxels.argtypes = [vp] * 7
        lib.chh_updated.argtypes = [vp, vp]
        self.lib = lib

    def build(self, submaps, split_submap, p=None, last_segment_first=0):
        """Same arguments as changeref.build; the same dict keys (and `updated`, the updated map), or the harness's negative
        return code."""
        p = R.params(**(p or {}))
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
        rc = self.lib.chh_build(par.ctypes.data, int(split_submap), int(last_segment_first), pts.ctypes.data, off.ctypes.data,
                                P.ctypes.data, len(submaps))
        if rc != 0:
            return rc
        info = np.zeros(16, dtype=np.int64)
        self.lib.chh_info(info.ctypes.data)
        V, n, kept = int(info[9]), int(info[12]), int(info[15])
        out = dict(ijk=np.zeros((V, 3), dtype=np.int32), label=np.zeros(V, dtype=np.uint8), point_label=np.zeros(n, dtype=np.uint8))
        for k in COUNTS:
            out[k] = np.zeros(V, dtype=np.uint32)
        self.lib.chh_voxels(*[out[k].ctypes.data for k in ("ijk",) + COUNTS + ("label", "point_label")])
        upd = np.zeros((max(1, kept), 4), dtype=F32)
        offs = np.zeros(len(submaps) + 1, dtype=np.int64)
        self.lib.chh_updated(upd.ctypes.data, offs.ctypes.data)
        out.update(lo=tuple(int(v) for v in info[0:3]), dims=tuple(int(v) for v in info[3:6]), split=int(info[6]),
                   n_rays=int(info[7]), n_skipped=int(info[8]), n_voxels=V, n_appeared_voxels=int(info[10]),
                   n_vanished_voxels=int(info[11]), n_points=n, n_appeared_points=int(info[13]), n_vanished_points=int(info[14]),
                   n_updated_points=kept, offsets=offs, updated=upd[:kept], p=p)
        return out


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("ch"), "libmap_changes_host.so")
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


def same(a, b):
    assert isinstance(a, dict) and isinstance(b, dict), (a, b)
    for k in SCALARS:
        assert a[k] == b[k], k
    for k in ARRAYS:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


# resolution 1 puts voxel edges on integers; the full ray is freed. Voxel (3, 0, 0) is the one the cases watch: a "wall"
# submap hits it, a "through" submap's ray crosses it to end at (5.5, 0.5, 0.5).
UNIT = dict(resolution=1.0, max_range=50.0, ray_fraction=1.0, min_frees=1, dynamic_thresh=0.5)
EMPTY = np.zeros((0, 4), dtype=F32)


def wall(n=1):
    return [(pts((3.5, 0.5, 0.5), (3.5, 0.6, 0.5)), T())] * n


def through(n=1):
    return [(pts((5.5, 0.5, 0.5)), T())] * n


# Every hand-built case: (name, submaps, split_submap, params, last_segment_first).
def cases():
    nan = float("nan")
    c = []
    c.append(("appeared", through(2) + wall(2), 2, UNIT, 0))
    c.append(("vanished", wall(2) + through(2), 2, UNIT, 0))
    c.append(("hit_in_both", wall(1) + through(1) + wall(1) + through(1), 2, UNIT, 0))
    for mf in (2, 3):  # frees_e of min_frees - 1 and of exactly min_frees, in each epoch
        c.append((f"min_frees_{mf}_before", through(2) + wall(1), 2, dict(UNIT, min_frees=mf), 0))
        c.append((f"min_frees_{mf}_after", wall(1) + through(2), 1, dict(UNIT, min_frees=mf), 0))
    # og_value exactly at dyn_value: one hit and three frees in an epoch is 25; dynamic_thresh 0.25 makes it free, 0.24 not
    for th in (0.25, 0.24):
        c.append((f"value_at_dyn_{th}_before", wall(1) + through(3) + wall(2), 4, dict(UNIT, dynamic_thresh=th), 0))
        c.append((f"value_at_dyn_{th}_after", wall(2) + wall(1) + through(3), 2, dict(UNIT, dynamic_thresh=th), 0))
    # a BEFORE point in an APPEARED voxel: one BEFORE submap hits voxel 3 and three free it; an AFTER point in a VANISHED one
    c.append(("before_point_in_appeared", wall(1) + through(3) + wall(2), 4, dict(UNIT, dynamic_thresh=0.3), 0))
    c.append(("after_point_in_vanished", wall(2) + wall(1) + through(3), 2, dict(UNIT, dynamic_thresh=0.3), 0))
    c.append(("empty_submaps_both_sides", [(EMPTY, T(4.5, 4.5, 4.5))] + through(2) + [(EMPTY, T())] + wall(2) + [(EMPTY, T(1, 1, 1))],
              3, UNIT, 0))
    c.append(("empty_submap_at_split", through(2) + [(EMPTY, T())] + wall(2), 2, UNIT, 0))
    c.append(("all_skipped_before", [(pts((nan, 0.5, 0.5), (90.0, 0.5, 0.5)), T())] * 2 + wall(2), 2, UNIT, 0))
    c.append(("all_skipped_after", wall(2) + [(pts((0.5, nan, 0.5), (0.5, 0.5, 70.0)), T())] * 2, 2, UNIT, 0))
    c.append(("split_at_1", through(1) + wall(3), 1, UNIT, 0))
    c.append(("split_at_n_minus_1", wall(3) + through(1), 3, UNIT, 0))
    c.append(("split_last_segment", through(2) + wall(2), -1, UNIT, 2))
    c.append(("rotated_pose", [(pts((7.3, 1.1, 0.2), (-2.2, 4.9, -0.3), (0.4, -6.6, 0.1)), T(1.7, -2.2, 0.9, 0.7)),
                               (pts((3.1, 0.2, -0.8), (-1.0, 2.0, 0.05)), T(0.3, -0.4, 0.7, 0.2)),
                               (pts((6.3, 1.0, 0.2), (-1.2, 4.0, -0.3)), T(1.2, -2.0, 0.9, 0.6))],
              2, dict(UNIT, resolution=0.25, sensor_origin=(0.3, -0.1, 0.2), ray_fraction=0.85), 0))
    return c


@pytest.mark.parametrize("name,subs,split,p,last", cases(), ids=[c[0] for c in cases()])
def test_host_compile_equals_replay(host, name, subs, split, p, last):
    a, b = host.build(subs, split, p, last), R.build(subs, split, p, last)
    same(a, b)
    keep = b["point_label"] != R.VANISHED
    assert np.array_equal(a["updated"].view(np.uint32), b["points"][keep].view(np.uint32))


def _voxel(g, key, v=(3, 0, 0)):
    hit = np.flatnonzero((g["ijk"] == np.array(v, dtype=np.int32)).all(axis=1))
    return int(g[key][hit[0]]) if len(hit) else None


def test_hand_built_outcomes():
    """What the hand-built cases must show, read off the replay (which the test above ties to the header)."""
    by = {n: R.build(s, sp, p, last) for n, s, sp, p, last in cases()}
    assert _voxel(by["appeared"], "label") == R.APPEARED and by["appeared"]["n_appeared_points"] == 4
    assert _voxel(by["vanished"], "label") == R.VANISHED and by["vanished"]["n_vanished_points"] == 4
    g = by["vanished"]
    assert g["n_updated_points"] == g["n_points"] - 4 and g["offsets"].tolist() == [0, 0, 0, 1, 2]
    g = by["hit_in_both"]
    assert [_voxel(g, k) for k in COUNTS] == [1, 1, 1, 1] and _voxel(g, "label") == R.UNCHANGED
    # min_frees 2: two frees suffice; min_frees 3: two are one short, and the voxel is not free in that epoch
    assert _voxel(by["min_frees_2_before"], "label") == R.APPEARED and _voxel(by["min_frees_3_before"], "label") == R.UNCHANGED
    assert _voxel(by["min_frees_2_after"], "label") == R.VANISHED and _voxel(by["min_frees_3_after"], "label") == R.UNCHANGED
    assert _voxel(by["value_at_dyn_0.25_before"], "label") == R.APPEARED
    assert _voxel(by["value_at_dyn_0.24_before"], "label") == R.UNCHANGED
    assert _voxel(by["value_at_dyn_0.25_after"], "label") == R.VANISHED
    assert _voxel(by["value_at_dyn_0.24_after"], "label") == R.UNCHANGED
    g = by["before_point_in_appeared"]  # the BEFORE wall's two points stay UNCHANGED, the AFTER wall's four are APPEARED
    assert _voxel(g, "label") == R.APPEARED and g["point_label"][:2].tolist() == [0, 0] and g["n_appeared_points"] == 4
    g = by["after_point_in_vanished"]  # the BEFORE walls' four points vanish, the AFTER wall's two are kept UNCHANGED
    assert _voxel(g, "label") == R.VANISHED and g["point_label"][4:6].tolist() == [0, 0] and g["n_vanished_points"] == 4
    g = by["empty_submaps_both_sides"]
    assert _voxel(g, "label") == R.APPEARED and g["offsets"].tolist() == [0, 0, 1, 2, 2, 4, 6, 6]
    g = by["empty_submap_at_split"]  # the first AFTER submap is empty
    assert _voxel(g, "label") == R.APPEARED and g["offsets"].tolist() == [0, 1, 2, 2, 4, 6]
    for n in ("all_skipped_before", "all_skipped_after"):
        g = by[n]
        assert g["n_skipped"] == 4 and g["n_appeared_points"] + g["n_vanished_points"] == 0 and g["n_updated_points"] == g["n_points"]
    assert by["split_at_1"]["split"] == 1 and _voxel(by["split_at_1"], "label") == R.APPEARED
    assert by["split_at_n_minus_1"]["split"] == 3 and _voxel(by["split_at_n_minus_1"], "label") == R.VANISHED
    assert by["split_last_segment"]["split"] == 2 and _voxel(by["split_last_segment"], "label") == R.APPEARED


def test_split_refusals(host):
    subs = through(2) + wall(2)
    for split, last in ((-1, 0), (0, 0), (0, 2), (-2, 2), (4, 0), (5, 2), (1 << 40, 0)):
        assert host.build(subs, split, UNIT, last) == -5, (split, last)
        with pytest.raises(R.Refused) as e:
            R.build(subs, split, UNIT, last)
        assert e.value.code == -5
    assert host.build(subs, 3, UNIT, 0)["split"] == 3 and host.build(subs, -1, UNIT, 1)["split"] == 1
    assert host.build(subs, 1, dict(UNIT, min_frees=0)) == -1 and host.build([], 1, UNIT) == -4


def test_mutations_change_an_outcome():
    by = {n: (s, sp, p, last) for n, s, sp, p, last in cases()}

    def differs(name, mut):
        s, sp, p, last = by[name]
        a = R.build(s, sp, p, last)
        try:
            b = R.build(s, sp, p, last, mut={mut})
        except (IndexError, R.Refused):
            return True
        return any(not np.array_equal(a[k], b[k]) for k in ARRAYS)

    assert differs("appeared", "split_late")
    assert differs("before_point_in_appeared", "epoch_blind")
    assert differs("value_at_dyn_0.25_before", "strict_dyn")
    assert differs("min_frees_3_before", "no_min_frees")
    assert differs("vanished", "pooled_before")
    for mut in R.MUTATIONS:  # and no mutation is invisible on the whole set
        assert any(differs(n, mut) for n in by), mut


def test_epoch_counts_equal_static_map_of_the_epoch(host, sm_host):  # noqa: F811
    """Each epoch's counts equal the static map of that epoch's submaps alone, for every voxel that build has; and an
    APPEARED or VANISHED point is one that static map keeps."""
    from lidarslam_ros2_b200 import synth

    rng = np.random.default_rng(5)
    subs = []
    for k in range(8):
        q = rng.uniform(-12, 12, size=(400, 3)).astype(F32)
        q[:, 2] = rng.uniform(-2, 3, size=400)
        q[::7, :] *= 0.4
        subs.append((q, synth.pose_matrix((rng.uniform(-2, 2), rng.uniform(-2, 2), 1.0), (0.0, 0.0, rng.uniform(0, 6.28)))))
    p = dict(resolution=0.5, max_range=30.0, min_frees=1, dynamic_thresh=0.5)
    for split in (1, 3, 7):
        g = host.build(subs, split, p)
        for e, part in ((0, subs[:split]), (1, subs[split:])):
            s = sm_host.build(part, p)
            idx = {tuple(v): r for r, v in enumerate(g["ijk"].tolist())}
            rows = np.array([idx[tuple(v)] for v in s["ijk"].tolist()], dtype=np.int64)
            assert np.array_equal(g[COUNTS[2 * e]][rows], s["hits"]) and np.array_equal(g[COUNTS[2 * e + 1]][rows], s["frees"])
            # every voxel the epoch's static map lacks has no hit in that epoch
            others = np.setdiff1d(np.arange(g["n_voxels"]), rows)
            assert not g[COUNTS[2 * e]][others].any()
            n0 = sum(len(q) for q, _ in subs[:split])
            mine = g["point_label"][:n0] if e == 0 else g["point_label"][n0:]
            changed = mine == (R.VANISHED if e == 0 else R.APPEARED)
            assert s["keep"][changed].all()
        assert g["n_appeared_points"] + g["n_vanished_points"] > 0


def test_serial_pipeline_under_sanitizers(tmp_path):
    """The executable form of the harness: changes of generated submaps (non-finite rows, negative coordinates, empty
    submaps) under -fsanitize=address,undefined, each equal to the build of each epoch's submaps in reverse order."""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = os.path.join(tmp_path, "map_changes_asan")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-DCH_HOST_MAIN", "-x", "c++", SRC, "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr or "ubsan" in build.stderr):
        pytest.skip("this toolchain has no sanitizer runtime")
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0 and "0 failures" in run.stdout, run.stdout + run.stderr


# ------------------------------------------------------------------ the two-day drive (tests/changescene.py)
@pytest.fixture(scope="module")
def two_days():
    import changescene

    d1, d2 = changescene.day(1), changescene.day(2)
    subs = list(zip(d1[0], d1[1])) + list(zip(d2[0], d2[1]))
    return subs, np.concatenate(d1[2]), np.concatenate(d2[2])


def shares(g, l1, l2):
    import changescene as S

    lab = g["point_label"]
    a, b = lab[:len(l1)], lab[len(l1):]
    still = (S.STATIC, S.GROUND)
    return dict(car_vanished=float((a[l1 == S.VANISHED_CAR] == R.VANISHED).mean()),
                container_appeared=float((b[l2 == S.CONTAINER] == R.APPEARED).mean()),
                transient_appeared=float((b[l2 == S.TRANSIENT] == R.APPEARED).mean()),
                static_labelled_day1=float((a[np.isin(l1, still)] != R.UNCHANGED).mean()),
                static_labelled_day2=float((b[np.isin(l2, still)] != R.UNCHANGED).mean()))


def test_two_day_drive_changes(host, two_days):
    import changescene

    """30 submaps per day down the canyon at their true poses, split at day 2's first submap, through the host compile
    with the static map's defaults (0.2 m voxels, ray_fraction 0.85, min_frees 2, dynamic_thresh 0.4). The figures this
    compile gives are in DESIGN.md section 7b."""
    subs, l1, l2 = two_days
    g = host.build(subs, changescene.N_SUB, {})
    s = shares(g, l1, l2)
    print(f"defaults: {s}, voxels {g['n_voxels']}, appeared {g['n_appeared_voxels']}, vanished {g['n_vanished_voxels']}")
    assert g["n_points"] == len(l1) + len(l2)
    assert s["car_vanished"] >= 0.75 and s["container_appeared"] >= 0.75
    assert s["static_labelled_day1"] <= 0.01 and s["static_labelled_day2"] <= 0.01
    # the updated map keeps every day-2 point, and drops only day-1 points labelled VANISHED
    assert g["offsets"][30] == len(l1) - g["n_vanished_points"] and g["n_updated_points"] == g["offsets"][30] + len(l2)
    assert not (g["point_label"][len(l1):] == R.VANISHED).any()
