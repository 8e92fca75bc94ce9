"""Every C-ABI call that takes a caller's cloud as host records, at the record layouts real callers send, against the same
call on the same points packed as (N, 4) float32 (stride 16, intensity at 12; the session's default 0 when the records
carry no intensity). The rest of the suite anchors the packed path to float64 and host-compiled references, so bitwise
equality with it carries those references over to every layout. The write-back paths (b200reg_voxelgrid's output
records, b200sm_imu_adjust_distortion's in-place x, y, z) are checked byte for byte against a numpy model.

Layouts (tests/test_record_layouts_cpu.py builds them): strides 12, 16, 20, 24 (a PointCloud2 point_step of 22 rounded up
to whole floats), 32 (PCL's PointXYZI), 48 and 64; intensity offsets -1, 12, 16 and stride - 4, where each fits. Every
byte of a record that the call must not read holds a different NaN payload, +-inf or +-FLT_MAX in each row, so a stray
read changes the result instead of hiding in zeros.

Determinism: every fixture coordinate lies on the 2^-12 m lattice within +-128 m and every intensity is an integer. Then
all partial sums are exact in float64 — VoxelGrid's coordinate sums, and the NDT voxel map's sums of products (38 bits
each, up to 2^15 points per voxel) — so the order of the device's float64 atomics cannot change them, and bitwise
comparison is sound for VoxelGrid's outputs and every pose computed downstream of them. Two kinds of case leave the
lattice: the +-3e38 rows (the grid overflows and the input comes back unchanged, compared bitwise) and points moved by a
sensor transform, which are held to the float64 VoxelGrid reference within the bound of tests/test_gpu_grid_edges.py.
getFitnessScore and calculateScore add per-warp float64 partials of non-lattice values with atomics; they are compared
within 1e-12 relative.

Also here: refused layouts (an intensity float that would end past the record, or an offset that is not a multiple of 4)
leave every session unchanged; the upload at the unpack kernels' block edges, either side of the four-thread staging
threshold and from pinned memory; and the scan bounds the upload pass measures against VoxelGrid's own bounds pass. Run on
an H100 with -m gpu."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import frontendref as fr
import gridref as R
import test_gpu_localize as TL
from test_deskew_oracle import _spinning_scan
from test_gpu_deskew import _feed
from test_gpu_grid_edges import _check_voxelgrid
from test_gpu_sensor_frame import MOUNT_POS, MOUNT_QUAT, _assert_same_state
from test_record_layouts_cpu import LAYOUTS, STRIDES, bad_offsets, lattice, packed, records, voxelgrid_writeback

pytestmark = pytest.mark.gpu

F32 = np.float32
LEAF = 0.5
KW = dict(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3, trans_for_mapupdate=1.0)
FOUR_THREAD_BYTES = 8 << 20  # staged_h2d stages a pageable source of this size or more with four host threads
PIECE_BYTES = 2 << 20  # ... in pieces of this size


@pytest.fixture(scope="module")
def sm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


@pytest.fixture(scope="module")
def lib(sm):
    from lidarslam_ros2_b200 import _capi

    return _capi.lib()


def _in_box(c, r=120.0):
    c = np.asarray(c)
    return c[(np.abs(c[:, :3]) < r).all(axis=1)]


@pytest.fixture(scope="module")
def frames():
    """4 drive frames on the lattice, integer intensities."""
    from lidarslam_ros2_b200 import synth

    rng = np.random.default_rng(52)
    return [lattice(np.c_[_in_box(s), rng.integers(0, 256, len(_in_box(s)))])
            for s, _ in synth.drive_stream(4, rings=16, azimuths=400, step=0.8)]


@pytest.fixture(scope="module")
def world():
    """The canyon prior map and three drive frames, on the lattice."""
    return lattice(_in_box(TL.canyon_map(40_000))), [(lattice(s), T) for s, T in TL.drive(3)]


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _same(a, b, what=""):
    assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), what


class _RecordsLib:
    """The library as a wrapper method of ScanMatcher sees it, with records in place of its packed array: the call's
    (packed pointer, n, 16, 12) arguments become (records, n, stride, offset). `dummy` is the array to hand the wrapper."""

    def __init__(self, lib, recs, stride, offset):
        self._lib, self._recs, self._stride, self._offset = lib, recs, stride, offset
        self.dummy = np.zeros((len(recs), 4), dtype=F32)
        self.swapped = 0

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            args = list(args)
            for i, a in enumerate(args):
                if isinstance(a, C.c_void_p) and a.value == self.dummy.ctypes.data:
                    assert args[i + 1:i + 4] == [len(self._recs), 16, 12], (name, args)
                    args[i:i + 4] = [_ptr(self._recs), len(self._recs), self._stride, self._offset]
                    self.swapped += 1
                    break
            return fn(*args)

        return call


@contextlib.contextmanager
def _records_for(obj, recs, stride, offset):
    lib = obj._lib
    proxy = _RecordsLib(lib, recs, stride, offset)
    obj._lib = proxy
    try:
        yield proxy.dummy
        assert proxy.swapped == 1
    finally:
        obj._lib = lib


def _call(obj, method, recs, stride, offset, *args, **kw):
    """obj.method(records, *args, **kw) through the wrapper, the records passed with their own stride and offset."""
    with _records_for(obj, recs, stride, offset) as d:
        return getattr(obj, method)(d, *args, **kw)


# ---- b200reg_voxelgrid: the output records against the write-back model -------------------------------------------------
@pytest.mark.parametrize("stride,offset", LAYOUTS)
def test_voxelgrid_records(lib, frames, stride, offset):
    """x, y, z and the intensity hold the packed call's result, the padding float is 1.0 only where bytes 12-15 are not the
    intensity (stride 32 with the intensity at 12 keeps its intensity), every other output byte keeps its sentinel, and
    a capacity below the result writes that many records and nothing past them."""
    from lidarslam_ros2_b200 import voxel_grid_filter

    cloud = frames[0]
    n = len(cloud)
    want = voxel_grid_filter(packed(cloud, offset), LEAF)
    assert 100 < len(want) < n
    r = records(cloud, stride, offset, seed=stride + offset)
    r0 = r.copy()
    sentinel = np.random.default_rng(100 * stride + offset).integers(0, 256, (n, stride), dtype=np.uint8)
    for cap in (n, len(want) // 2):
        out = sentinel.copy()
        m = C.c_size_t(0)
        assert lib.b200reg_voxelgrid(0, _ptr(r), n, stride, offset, LEAF, _ptr(out), cap, C.byref(m)) == 0
        assert m.value == len(want)
        assert np.array_equal(out, voxelgrid_writeback(sentinel, want[:cap], stride, offset)), cap
    assert np.array_equal(r, r0)
    if offset >= 0:
        assert len(np.unique(want[:, 3])) > 10  # the intensities are really there to lose


@pytest.mark.parametrize("stride,offset", [(16, 12), (24, -1), (32, 16), (64, 60)])
def test_voxelgrid_overflow_returns_the_records(lib, frames, stride, offset):
    """+-3e38 rows: the grid overflows int32 and PCL returns the input; the output records are the input records, every
    byte of them."""
    cloud = frames[1][:1000].copy()
    cloud[10, 0], cloud[500, 1], cloud[999, 2] = 3e38, -3e38, 3e38
    assert R.leaf_geometry(cloud, LEAF)["overflow"]
    r = records(cloud, stride, offset, seed=5)
    out = np.zeros_like(r)
    m = C.c_size_t(0)
    assert lib.b200reg_voxelgrid(0, _ptr(r), len(r), stride, offset, LEAF, _ptr(out), len(r), C.byref(m)) == 0
    assert m.value == len(r) and np.array_equal(out, r)


# ---- b200reg_encode_pcd_ascii ------------------------------------------------------------------------------------------
def _encode(lib, buf, stride, offset):
    nb = C.c_size_t(0)
    assert lib.b200reg_encode_pcd_ascii(0, _ptr(buf), len(buf), stride, offset, None, 0, C.byref(nb)) == 0
    out = np.zeros(nb.value, dtype=np.uint8)
    assert lib.b200reg_encode_pcd_ascii(0, _ptr(buf), len(buf), stride, offset, _ptr(out), out.size, C.byref(nb)) == 0
    return out.tobytes()


@pytest.mark.parametrize("stride,offset", [(s, o) for s, o in LAYOUTS if o >= 0])
def test_encode_pcd_records(lib, frames, stride, offset):
    cloud = frames[1]
    want = _encode(lib, packed(cloud, offset), 16, 12)
    assert b"POINTS %d\n" % len(cloud) in want
    assert _encode(lib, records(cloud, stride, offset, seed=offset), stride, offset) == want


# ---- b200sm_import_submap ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stride,offset", LAYOUTS)
def test_import_submap_records(sm, frames, stride, offset):
    from lidarslam_ros2_b200 import synth

    a, b = sm.ScanMatcher(), sm.ScanMatcher()
    for k in range(2):
        M = synth.pose_matrix((1.5 * k, 0.5, 0.0), (0.0, 0.0, 0.1 * k))
        _call(a, "importSubmap", records(frames[k], stride, offset, seed=k), stride, offset, M, 1.5 * k)
        b.importSubmap(packed(frames[k], offset), M, 1.5 * k)
    for k in range(2):
        (ca, Ma, da), (cb, Mb, db) = a.submap(k), b.submap(k)
        _same(ca, packed(frames[k], offset), k)
        _same(ca, cb, k)
        assert np.array_equal(Ma, Mb) and da == db
    (ma, oa), (mb, ob) = a.assembleMap(), b.assembleMap()
    _same(ma, mb)
    assert np.array_equal(oa, ob)


# ---- b200sm_set_scan, b200sm_receive_cloud --------------------------------------------------------------------------------
@pytest.mark.parametrize("stride,offset", LAYOUTS)
def test_frontend_records(sm, frames, stride, offset):
    a, b = sm.ScanMatcher(**KW), sm.ScanMatcher(**KW)
    recs = [records(c, stride, offset, seed=k) for k, c in enumerate(frames)]
    n = _call(a, "setScan", recs[0], stride, offset)
    assert n == b.setScan(packed(frames[0], offset)) > 0
    f = a.filteredScan()
    _same(f, b.filteredScan())
    assert (f[:, 3] != 0).any() if offset >= 0 else (f[:, 3] == 0).all()  # intensities averaged by VoxelGrid
    for k, c in enumerate(frames):
        pa, Ta, ua = _call(a, "receiveCloud", recs[k], stride, offset)
        pb, Tb, ub = b.receiveCloud(packed(c, offset))
        assert np.array_equal(pa, pb) and np.array_equal(_bits(Ta), _bits(Tb)) and ua == ub, k
        _same(a.filteredScan(), b.filteredScan(), k)
    assert a.numSubmaps() >= 2
    _assert_same_state(a, b)


# ---- b200sm_imu_adjust_distortion: x, y, z written back in place, nothing else -------------------------------------------
@pytest.mark.parametrize("stride,offset", LAYOUTS)
def test_deskew_records_in_place(sm, lib, stride, offset):
    s = _spinning_scan(n=2400, rings=4)
    s[:, 3] *= 255.0
    cloud = lattice(s)
    ua, ub = sm.LidarUndistortion(scan_period=0.1), sm.LidarUndistortion(scan_period=0.1)
    _feed([ua, ub], t0=100.0, n=100)
    r = records(cloud, stride, offset, seed=offset)
    r0 = r.copy()
    assert lib.b200sm_imu_adjust_distortion(ua._s, _ptr(r), len(r), stride, offset, 100.2) == 0
    want = ub.adjustDistortion(packed(cloud, offset), 100.2)
    w, w0 = r.view(np.uint32), r0.view(np.uint32)
    assert np.array_equal(w[:, :3], _bits(want[:, :3]))
    assert not np.array_equal(w[:, :3], w0[:, :3])  # the de-skew moved the points
    assert np.array_equal(w[:, 3:], w0[:, 3:])  # every other byte of every record unchanged
    assert ua.pointers() == ub.pointers()


# ---- localisation: b200sm_set_prior_map, _localize_cloud, _localize_init, _localize_global, _relocalize ---------------------
def _close(a, b):
    """getFitnessScore and calculateScore add per-warp float64 partials with atomics: equal up to their summation order."""
    return abs(a - b) <= 1e-12 * max(abs(a), abs(b))


def _rows_equal(ra, rb):
    assert len(ra) == len(rb)
    for x, y in zip(ra, rb):
        assert x.keys() == y.keys()
        for k in x:
            if isinstance(x[k], np.ndarray):
                assert np.array_equal(_bits(x[k]), _bits(y[k])), k
            elif k == "fitness":
                assert _close(x[k], y[k]), (x[k], y[k])
            else:
                assert x[k] == y[k], k


@pytest.mark.parametrize("stride,offset", LAYOUTS)
def test_localize_records(sm, world, stride, offset):
    prior, drive = world
    a, b = TL._session(sm, None), TL._session(sm, None)
    assert _call(a, "setPriorMap", records(prior, stride, offset, seed=1), stride, offset) == len(prior)
    b.setPriorMap(packed(prior, offset))
    recs = [records(s, stride, offset, seed=k) for k, (s, _) in enumerate(drive)]
    pk = [packed(s, offset) for s, _ in drive]
    for k in range(2):
        pa, Ta, ca = _call(a, "localizeCloud", recs[k], stride, offset)
        pb, Tb, cb = b.localizeCloud(pk[k])
        assert np.array_equal(pa, pb) and np.array_equal(_bits(Ta), _bits(Tb)) and ca == cb, k
        _same(a.cutCloud(), b.cutCloud(), k)
        _same(a.filteredScan(), b.filteredScan(), k)
    cut = a.cutCloud()
    assert len(cut) > 1000 and ((cut[:, 3] != 0).any() if offset >= 0 else (cut[:, 3] == 0).all())
    G = TL.hypotheses(drive[2][1])
    ia, ib = _call(a, "localizeInit", recs[2], stride, offset, G), b.localizeInit(pk[2], G)
    assert ia[0] == ib[0]
    _rows_equal(ia[1], ib[1])
    ga, gb = _call(a, "localizeGlobal", recs[2], stride, offset, 1.0, 1.0, 4, 2), b.localizeGlobal(pk[2], 1.0, 1.0, 4, 2)
    assert ga[0] == gb[0] and np.array_equal(ga[1], gb[1])
    _rows_equal(ga[2], gb[2])
    assert {k: v for k, v in ga[3].items() if k != "score_ms"} == {k: v for k, v in gb[3].items() if k != "score_ms"}
    p = dict(yaw_steps=64, num_levels=4, top_k=2)
    ra, rb = _call(a, "relocalize", recs[2], stride, offset, **p), b.relocalize(pk[2], **p)
    assert ra[0] == rb[0]
    _rows_equal(ra[1], rb[1])
    assert {k: v for k, v in ra[2].items() if k != "search_ms"} == {k: v for k, v in rb[2].items() if k != "search_ms"}
    assert ra[2]["width"] > 0
    for h in range(p["num_levels"]):
        assert np.array_equal(a.relocalizeGrid(h), b.relocalizeGrid(h)), h


# ---- b200reg_set_input_target / _source, _ndt_calculate_score, _nn1: stride only ---------------------------------------
@pytest.mark.parametrize("method", ["NDT", "GICP"])
@pytest.mark.parametrize("stride", STRIDES)
def test_registration_records(frames, method, stride):
    """The records are handed to the wrapper as (n, stride / 4) float32 rows: it passes their row stride as is."""
    import lidarslam_ros2_b200 as m

    def run(rows):
        g = m.NormalDistributionsTransform() if method == "NDT" else m.GeneralizedIterativeClosestPoint()
        if method == "NDT":
            g.setResolution(2.0)
        g.setInputTarget(rows(0))
        g.setInputSource(rows(1))
        out = dict(T=_bits(g.align()), converged=g.hasConverged(), fitness=g.getFitnessScore(), nn=g.nearest(rows(2)))
        if method == "NDT":
            out.update(score=g.calculateScore(rows(2)), p=g.getTransformationProbability(), it=g.getFinalNumIteration())
        return out

    got = run(lambda k: records(frames[k], stride, -1, seed=k).view(F32))
    want = run(lambda k: packed(frames[k], -1))
    for k in want:
        if k == "nn":
            assert np.array_equal(got[k][0], want[k][0]) and np.array_equal(_bits(got[k][1]), _bits(want[k][1]))
        elif k in ("fitness", "score"):
            assert _close(got[k], want[k]), (k, got[k], want[k])
        else:
            assert np.array_equal(got[k], want[k]), k


# ---- refusals: an intensity float past the record, or a misaligned one, leaves every session as it was ---------------------
@pytest.mark.parametrize("stride", [16, 24, 32])
def test_refused_layouts_leave_the_sessions_unchanged(sm, lib, frames, world, stride):
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    def refused(obj, method, recs, offset, *args, **kw):
        with pytest.raises(B200RegError) as e:
            _call(obj, method, recs, stride, offset, *args, **kw)
        assert e.value.code == _capi.ERR_ARG, (method, offset)

    # a mapping session with a scan, submaps (received and imported) and a target, and its twin
    a, b = sm.ScanMatcher(**KW), sm.ScanMatcher(**KW)
    for g in (a, b):
        for c in frames[:3]:
            g.receiveCloud(c)
        g.importSubmap(frames[3], np.eye(4), 9.0)
        g.setScan(frames[1])
    n_sub, stats = a.numSubmaps(), a.stats()
    recs = records(frames[2], stride, -1, seed=stride)
    for offset in bad_offsets(stride):
        refused(a, "setScan", recs, offset)
        refused(a, "receiveCloud", recs, offset)
        refused(a, "importSubmap", recs, offset, np.eye(4), 10.0)
        r = recs.copy()
        assert lib.b200sm_imu_adjust_distortion(a._h, _ptr(r), len(r), stride, offset, 0.0) == _capi.ERR_ARG
        assert np.array_equal(r, recs)
    assert a.numSubmaps() == n_sub and a.stats() == stats
    _same(a.filteredScan(), b.filteredScan())
    _assert_same_state(a, b)
    ra, rb = a.receiveCloud(frames[0]), b.receiveCloud(frames[0])  # the pose too
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(_bits(ra[1]), _bits(rb[1])) and ra[2] == rb[2]

    # a localising session with a prior map, a cut and a relocalisation pyramid, and its twin
    prior, drive = world
    c, d = TL._session(sm, prior), TL._session(sm, prior)
    for g in (c, d):
        g.localizeCloud(drive[0][0])
        g.relocalize(drive[1][0], yaw_steps=64, num_levels=4, top_k=2)
    cut, lstats = c.cutCloud(), c.localizeStats()
    recs = records(drive[1][0], stride, -1, seed=stride)
    G = TL.hypotheses(drive[1][1])
    for offset in bad_offsets(stride):
        refused(c, "setPriorMap", records(prior[:5000], stride, -1), offset)
        refused(c, "localizeCloud", recs, offset)
        refused(c, "localizeInit", recs, offset, G)
        refused(c, "localizeGlobal", recs, offset, 1.0, 1.0, 4, 2)
        refused(c, "relocalize", recs, offset, yaw_steps=64, num_levels=4, top_k=2)
    _same(c.cutCloud(), cut)
    assert c.localizeStats() == lstats
    for h in range(4):
        assert np.array_equal(c.relocalizeGrid(h), d.relocalizeGrid(h)), h
    for k in (1, 2):  # the prior map and the pose: the next frames are the twin's
        rc, rd = c.localizeCloud(drive[k][0]), d.localizeCloud(drive[k][0])
        assert np.array_equal(rc[0], rd[0]) and np.array_equal(_bits(rc[1]), _bits(rd[1])) and rc[2] == rd[2], k
        _same(c.cutCloud(), d.cutCloud(), k)


# ---- the upload: unpack block edges, the staging threshold, pinned sources -----------------------------------------------
def _upload_sizes(stride):
    """n = 1 and the 256-thread block edges; pageable sources of 8 MB - stride, 8 MB and 8 MB + stride bytes (either side
    of the four-thread staging threshold); one that does not end on a 2 MB staging piece."""
    sizes = [1, 255, 256, 257] + [(FOUR_THREAD_BYTES + d) // stride for d in (-stride, 0, stride)]
    odd = (5 * PIECE_BYTES // 2 + 3 * stride) // stride
    assert (odd * stride) % PIECE_BYTES != 0
    return sizes + [odd]


@pytest.fixture(scope="module")
def big():
    rng = np.random.default_rng(77)
    n = (FOUR_THREAD_BYTES + 16) // 16
    return lattice(np.c_[rng.uniform(-60, 60, (n, 2)), rng.uniform(-5, 5, n), rng.integers(0, 256, n)])


@pytest.mark.parametrize("stride,offset", [(16, 12), (32, 16)])
def test_upload_edges(sm, big, stride, offset):
    a, b = sm.ScanMatcher(**KW), sm.ScanMatcher(**KW)
    imported = 0
    for n in _upload_sizes(stride):
        cloud = big[:n]
        for pinned in (False, True) if n in (257, FOUR_THREAD_BYTES // stride) else (False,):
            r = records(cloud, stride, offset, seed=n, pinned=pinned)
            assert _call(a, "setScan", r, stride, offset) == b.setScan(packed(cloud, offset)), (n, pinned)
            _same(a.filteredScan(), b.filteredScan(), (n, pinned))
            _call(a, "importSubmap", r, stride, offset, np.eye(4), float(n))
            sub, _, dist = a.submap(imported)
            imported += 1
            assert dist == float(n)
            _same(sub, packed(cloud, offset), (n, pinned))


# ---- the bounds of the upload pass against VoxelGrid's own bounds pass ------------------------------------------------------
def _bounds_cases():
    """name -> (N, 4) cloud. The base cloud has all coordinates >= 0, so that a signed zero is the minimum."""
    rng = np.random.default_rng(90)
    base = lattice(np.c_[rng.uniform(0, 20, (1000, 3)), rng.integers(0, 256, 1000)])
    cases = {}
    for axis in range(3):
        for v in (np.nan, np.inf, -np.inf):
            c = base.copy()
            c[[0, 255, 256, len(c) - 1], axis] = v  # first row, both sides of a block edge, last row
            cases[f"{'xyz'[axis]}={v}"] = c
    c = base.copy()
    c[0:8, :3], c[8:16, :3] = F32(-0.0), F32(0.0)
    c[16:24:2, 0], c[17:24:2, 0] = F32(-0.0), F32(0.0)
    cases["signed zeros"] = c
    c = np.full((257, 4), np.nan, dtype=F32)
    c[::3, 0], c[1::3, 1] = np.inf, -np.inf
    c[256] = base[7]  # the one finite row, alone in its block
    cases["one finite row"] = c
    cases["all non-finite"] = np.full((300, 4), np.nan, dtype=F32)
    c = base.copy()
    c[3, :3], c[300, :3], c[600, :3] = (3e38, 0, 0), (0, -3e38, 0), (0, 0, 3e38)
    cases["+-3e38"] = c
    return cases


BOUNDS_CASES = _bounds_cases()


@pytest.mark.parametrize("transform", [False, True])
@pytest.mark.parametrize("case", list(BOUNDS_CASES))
def test_upload_bounds_equal_voxelgrid_bounds(sm, case, transform):
    """The session's filteredScan() against voxel_grid_filter of the same points (moved on the host by the float32 replay of
    the device transform, when one is set) at vg_size_for_input."""
    from lidarslam_ros2_b200 import _capi, voxel_grid_filter
    from lidarslam_ros2_b200.registration import B200RegError

    pts = BOUNDS_CASES[case]
    leaf = KW["vg_size_for_input"]
    g = sm.ScanMatcher(**KW)
    moved = pts
    if transform:
        g.setSensorTransform(MOUNT_POS, MOUNT_QUAT)
        moved = fr.transform_cloud(pts, fr.sensor_matrix(MOUNT_POS, MOUNT_QUAT))
    want = voxel_grid_filter(moved, leaf)
    if case == "all non-finite":
        with pytest.raises(B200RegError) as e:
            g.setScan(pts)
        assert e.value.code == _capi.ERR_ARG
        assert len(g.filteredScan()) == 0 and len(want) == 0
        return
    g.setScan(pts)
    got = g.filteredScan()
    ref, err = R.voxelgrid_ref(moved, leaf)
    if err is None:  # the grid overflows: both return the (moved) input
        _same(got, moved)
        _same(want, moved)
    elif not transform:  # on the lattice: bit for bit
        _same(got, want)
    else:
        assert got.shape == want.shape
        _check_voxelgrid(got, moved, leaf, case)
        _check_voxelgrid(want, moved, leaf, case)
    assert len(got) == 1 if case == "one finite row" else len(got) > 100
