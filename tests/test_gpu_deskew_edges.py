"""The IMU de-skew kernels (K9: deskew_orient -> deskew_time -> deskew_scan -> deskew_apply) point by point against the
replay of tests/deskewref.py, on the scenes that reach their edges: the deskew_scan partition (1024 chunks of
ceil(n / 1024) points) with lower-bound steps on the chunk edges, fix points of 1, 2 and >= 3 passes, the IMU ring
window crossing 199 -> 0, span 0 and 199, imu_ptr_last_ == 0 after a wrap, ties between stamps and point times,
duplicate stamps, a point exactly scan_period from its sample, the IMU clock stepping back, every azimuth layout, NaN
rays and infinite coordinates.

Per scan: the trace (rel_time, t, front, skip, k_first) equals the replay exactly and the pass count its Jacobi count;
the carried pointers are exact; x, y, z equal the float32 replay bit for bit (NaN patterns first) with every other field
untouched; |kernel - float64 reference| is within the per-point bound of deskewref (largest ratio printed); and the
literal oracle (oracle/deskew.py, with the kernel's double-then-round trigonometry) has the same pointers and leaves the
same points untouched."""
import numpy as np
import pytest

import deskewref as DR
from oracle import deskew
from test_deskewref_cpu import ORACLE_MAX_N, _DoubleTrig

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


@pytest.fixture
def double_trig(monkeypatch):
    monkeypatch.setattr(deskew, "np", _DoubleTrig())


def _bitwise_xyz(got, want):
    g, w = got[:, :3], want[:, :3]
    assert np.array_equal(np.isnan(g), np.isnan(w))
    m = ~np.isnan(w)
    assert np.array_equal(g[m].view(np.uint32), w[m].view(np.uint32)), np.flatnonzero((g != w).any(axis=1))[:10]


def _check_trace(tr, r):
    if not r["ran"]:
        assert tr["n"] == 0
        return
    assert tr["n"] == r["n"]
    nan = np.isnan(r["rel"])  # NaN rays: the device's canonical NaN and numpy's differ in sign / payload
    assert np.array_equal(np.isnan(tr["rel_time"]), nan)
    assert np.array_equal(tr["rel_time"][~nan].view(np.uint32), r["rel"][~nan].view(np.uint32))
    assert np.array_equal(tr["t"], r["t"], equal_nan=True)
    assert np.array_equal(tr["front"], r["front"]), np.flatnonzero(tr["front"] != r["front"])[:10]
    assert np.array_equal(tr["skip"], r["skip"])
    assert tr["k_first"] == r["k_first"] and tr["rounds"] == r["rounds"], (tr["k_first"], tr["rounds"], r["k_first"], r["rounds"])


def _ratio(out, r):
    fin = np.isfinite(out[:, :3]) & np.isfinite(r["ref64"]) & (r["bound"] > 0)
    assert np.array_equal(np.isfinite(out[:, :3]), np.isfinite(r["out"][:, :3]))
    if not fin.any():
        return 0.0
    return float((np.abs(out[:, :3].astype(np.float64) - r["ref64"])[fin] / r["bound"][fin]).max())


SCENES = DR.all_scenes()


@pytest.mark.parametrize("sc", SCENES, ids=[s.name for s in SCENES])
def test_deskew_edges(sm, sc, double_trig):
    g = sm.LidarUndistortion(scan_period=sc.scan_period)
    o = deskew.LidarUndistortion(scan_period=sc.scan_period)
    worst = 0.0
    for step in sc.steps:
        if step[0] == "imu":
            DR.feed([g, o], step[1])
            continue
        _, cloud, st, claim = step
        ring = DR.Ring.from_device(g, sc.scan_period)
        assert ring.ptr_last_iter == o.ptr_last_iter and ring.ptr_front == o.ptr_front
        r = DR.replay(cloud, ring, st)
        assert not r["ambiguous"].any()
        out = g.adjustDistortion(cloud, st)
        tr = g.trace()
        claim(tr, ring)  # the property the scan exists for, on the device's own trace
        _check_trace(tr, r)
        pf, pl, pli = g.pointers()
        assert (pf, pli) == (r["ptr_front"], r["ptr_last_iter"])
        assert np.array_equal(out[:, 3].view(np.uint32), cloud[:, 3].view(np.uint32))
        _bitwise_xyz(out, r["out"])
        worst = max(worst, _ratio(out, r))
        if len(cloud) <= ORACLE_MAX_N:
            a = o.adjust_distortion(cloud, st)
            assert (o.ptr_front, o.ptr_last_iter) == (pf, pli)
            untouched = np.all((out[:, :3] == cloud[:, :3]) | np.isnan(cloud[:, :3]), axis=1)
            assert np.array_equal(a[untouched], cloud[untouched], equal_nan=True)
            assert np.array_equal(np.isnan(a), np.isnan(out))
        else:
            o.ptr_front, o.ptr_last_iter = pf, pli
    print(f"\n{sc.name}: largest |kernel - float64| / bound = {worst:.3f}")
    assert worst <= 1.0


def test_nan_rays_through_the_frontend_frame(sm):
    """An organised scan with NaN rays, de-skewed inside the frame (deskewNextScan + setScan) with and without the range
    filter: the frame's trace and carried pointers equal the replay; with the sensor transform on, the NaN rays still walk
    to the newest sample and are not skipped."""
    T, sp = 10.0, 0.1
    msgs = DR.imu_messages(T - 0.3 + 0.01 * np.arange(60), seed=41)
    cloud = DR.sweep_scan(8000, seed=42)
    rows = [0 + 17, 2500, 2501, 7999]
    cloud[rows, :3] = np.nan
    for use_filter, tf in ((False, False), (True, False), (True, True)):
        s = sm.ScanMatcher(device=0, ndt_resolution=2.0, vg_size_for_input=0.1, use_min_max_filter=use_filter,
                           scan_min_range=1.0, scan_max_range=200.0)
        imu = sm.LidarUndistortion(session=s._h, scan_period=sp)
        DR.feed([imu], msgs)
        if tf:
            s.setSensorTransform([0.1, -0.2, 0.3], [0.0, 0.0, np.sin(0.05), np.cos(0.05)])
        ring = DR.Ring.from_device(imu, sp)
        s.deskewNextScan(T + 0.2)
        s.setScan(cloud)
        tr = imu.trace()
        assert tr["n"] == len(cloud)
        assert (tr["front"][rows] == ring.ptr_last).all() and not tr["skip"][rows].any()
        if not tf:
            r = DR.replay(cloud, ring, T + 0.2)
            _check_trace(tr, r)
            assert imu.pointers()[0] == r["ptr_front"] and imu.pointers()[2] == r["ptr_last_iter"]


def test_adjust_distortion_on_32_byte_records(sm):
    """b200sm_imu_adjust_distortion on PointXYZI-like records (32 bytes, intensity at offset 16): x, y, z equal the
    replay bit for bit, every other word of the record is untouched."""
    import ctypes as C

    T, sp = 70.0, 0.1
    g = sm.LidarUndistortion(scan_period=sp)
    DR.feed([g], DR.imu_messages(T - 0.3 + 0.01 * np.arange(60), seed=51))
    c = DR.sweep_scan(5000, seed=52)
    c[1234, :3] = np.nan
    rec = np.random.default_rng(53).random((len(c), 8)).astype(np.float32)
    rec[:, :3] = c[:, :3]
    rec[:, 4] = c[:, 3]
    before = rec.copy()
    ring = DR.Ring.from_device(g, sp)
    r = DR.replay(c, ring, T + 0.2)
    rc = g._lib.b200sm_imu_adjust_distortion(g._s, rec.ctypes.data, len(rec), 32, 16, C.c_double(T + 0.2))
    assert rc == 0
    _bitwise_xyz(rec, r["out"])
    assert np.array_equal(rec[:, 3:].view(np.uint32), before[:, 3:].view(np.uint32))
    _check_trace(g.trace(), r)


def test_ring_entries_bitwise_after_getImu(sm):
    """getImu's ring (roll, pitch, yaw, shift, velo) against deskewref.glibc_ring, which calls glibc's atan2f / asinf,
    bit for bit, through a wrap of the ring and a gap longer than scan_period."""
    sp = 0.1
    g = sm.LidarUndistortion(scan_period=sp)
    msgs = DR.imu_messages(50.0 + 0.01 * np.arange(230), seed=61) + DR.imu_messages([52.5, 52.7], seed=62)
    DR.feed([g], msgs)
    want = DR.glibc_ring(msgs, sp)
    got = DR.Ring.from_device(g, sp)
    assert (got.ptr_front, got.ptr_last) == (want.ptr_front, want.ptr_last)
    assert np.array_equal(got.time, want.time)
    for name in ("rpy", "shift", "velo"):
        assert np.array_equal(getattr(got, name).view(np.uint32), getattr(want, name).view(np.uint32)), name
