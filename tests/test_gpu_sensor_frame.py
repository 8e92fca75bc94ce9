"""The cloud callback's sensor-to-robot transform and use_odom guess on the frontend session (b200sm_set_sensor_transform,
b200sm_odom_next_scan): the transform made in the upload pass against the float32 restatement (tests/frontendref.py) bit
for bit; a session given LiDAR-frame points and the transform against one given the same points moved on the host, bit
for bit (the solver is deterministic run to run), with and without the range filter and with the de-skew armed; the
odometry guess against the restated frontend within 1e-3 m / 1e-3 rad."""
import numpy as np
import pytest

import frontendref as fr
import oracle
import oracle.scanmatcher as osm
from lidarslam_ros2_b200 import synth

pytestmark = pytest.mark.gpu

MOUNT_POS = (1.2, 0.0, 2.0)  # mapping_car.launch.py:27-28, plus a rotation
MOUNT_QUAT = osm.quat_from_matrix(synth.rpy_matrix(0.02, -0.04, 0.35))
KW = dict(ndt_resolution=2.0, vg_size_for_input=0.4, vg_size_for_map=0.3, num_targeted_cloud=3, scan_min_range=2.0,
          scan_max_range=60.0)


@pytest.fixture(scope="module")
def sm():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher


@pytest.fixture(scope="module")
def frames():
    """10 drive frames in the LiDAR frame, with an intensity column."""
    rng = np.random.default_rng(41)
    out = []
    for scan, T_gt in synth.drive_stream(10, rings=16, azimuths=400, step=0.6):
        c = np.concatenate([scan, rng.uniform(0, 255, size=(len(scan), 1)).astype(np.float32)], axis=1)
        out.append((c, T_gt))
    return out


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _sorted(c):
    c = np.asarray(c)
    return c[np.lexsort((c[:, 3], c[:, 2], c[:, 1], c[:, 0]))]


def _state(g):
    subs = [g.submap(i) for i in range(g.numSubmaps())]
    return subs, g.targetedCloud()


def _assert_same_state(a, b):
    sa, ta = _state(a)
    sb, tb = _state(b)
    assert len(sa) == len(sb)
    for (ca, Ma, da), (cb, Mb, db) in zip(sa, sb):
        assert np.array_equal(_bits(ca), _bits(cb)) and np.array_equal(Ma, Mb) and da == db
    assert np.array_equal(_bits(ta), _bits(tb))


@pytest.mark.parametrize("quat_scale", [1.0, 1.01])
def test_upload_transform_bitwise(sm, frames, quat_scale):
    """With a leaf so small that the grid overflows, PCL's VoxelGrid returns its input: the filtered scan IS the scan as the
    unpack pass stored it, and equals the float32 restatement bit for bit, intensity included (the quaternion is used as
    given, so 1.01 scales the points)."""
    cloud = frames[3][0]
    q = quat_scale * np.asarray(MOUNT_QUAT)
    g = sm.ScanMatcher(ndt_resolution=2.0, vg_size_for_input=1e-3)
    g.setSensorTransform(MOUNT_POS, q)
    n = g.setScan(cloud)
    got = g.filteredScan()
    want = fr.transform_cloud(cloud, fr.sensor_matrix(MOUNT_POS, q))
    assert n == len(cloud) == len(got)
    assert np.array_equal(_bits(_sorted(got)), _bits(_sorted(want)))
    assert np.abs(got[:, :3] - cloud[:, :3]).max() > 1.0  # the points really moved


def test_voxelgrid_on_the_transformed_scan(sm, frames):
    """Both VoxelGrids of a frame are sized from the bounds the unpack pass measures: they must be the transformed points'."""
    import oracle as oracle_pkg

    cloud = frames[5][0]
    g = sm.ScanMatcher(ndt_resolution=2.0, vg_size_for_input=0.4)
    g.setSensorTransform(MOUNT_POS, MOUNT_QUAT)
    g.setScan(cloud)
    got = g.filteredScan()
    want = oracle_pkg.voxelgrid(fr.transform_cloud(cloud, fr.sensor_matrix(MOUNT_POS, MOUNT_QUAT)), 0.4)
    assert len(got) == len(want)
    assert np.abs(_sorted(got)[:, :3] - _sorted(want)[:, :3]).max() < 1e-4


def _drive_pair(sm, frames, use_filter, deskew=False):
    """Session a: LiDAR-frame records + setSensorTransform; session b: records moved on the host by the float32 restatement."""
    a, b = sm.ScanMatcher(use_min_max_filter=use_filter, **KW), sm.ScanMatcher(use_min_max_filter=use_filter, **KW)
    a.setSensorTransform(MOUNT_POS, MOUNT_QUAT)
    E = fr.sensor_matrix(MOUNT_POS, MOUNT_QUAT)
    imus = []
    if deskew:
        from test_gpu_deskew import _feed

        imus = [sm.LidarUndistortion(session=a._h), sm.LidarUndistortion(session=b._h)]
        _feed(imus, t0=100.0, n=110)
    n_upd = 0
    for k, (cloud, _) in enumerate(frames):
        if deskew:
            a.deskewNextScan(100.0 + 0.1 * k)
            b.deskewNextScan(100.0 + 0.1 * k)
        pa, Ta, ua = a.receiveCloud(cloud)
        pb, Tb, ub = b.receiveCloud(fr.transform_cloud(cloud, E))
        assert ua == ub and np.array_equal(pa, pb) and np.array_equal(_bits(Ta), _bits(Tb)), k
        assert np.array_equal(_bits(_sorted(a.filteredScan())), _bits(_sorted(b.filteredScan()))), k
        n_upd += int(ua)
    assert n_upd >= 2
    _assert_same_state(a, b)
    if deskew:
        assert imus[0].pointers() == imus[1].pointers() and imus[0].pointers()[1] > 0


@pytest.mark.parametrize("use_filter", [False, True])
def test_transform_on_device_equals_transform_on_host(sm, frames, use_filter):
    _drive_pair(sm, frames, use_filter)


def test_deskew_sees_the_robot_frame_points(sm, frames):
    """cloud_callback's order: doTransform, then adjustDistortion, then the range filter. The de-skew's first / last
    azimuths must come from the transformed records for the two sessions to agree bit for bit."""
    _drive_pair(sm, frames, use_filter=True, deskew=True)


def _odom(k, R_gt):
    M = R_gt @ synth.pose_matrix((0.02 * k, -0.01 * k, 0.0), (0.0, 0.0, 0.001 * k))  # ground truth with a growing drift
    return M[:3, 3], osm.quat_from_matrix(M[:3, :3])


def test_odometry_guess_parity(sm, frames):
    """use_odom on the GPU against the restated frontend, odometry armed on every frame except frame 6: same update
    decisions, poses within 1e-3 m / 1e-3 rad."""
    E = osm.pose_matrix(MOUNT_POS, MOUNT_QUAT)
    Einv = np.linalg.inv(E)
    g = sm.ScanMatcher(**KW)
    o = fr.ScanMatcher(num_threads=oracle.max_threads(), **KW)
    for s in (g, o):
        (s.setSensorTransform if hasattr(s, "setSensorTransform") else s.set_sensor_transform)(MOUNT_POS, MOUNT_QUAT)
    n_upd = 0
    for k, (cloud, T_gt) in enumerate(frames):
        odom = None if k == 6 else _odom(k, E @ T_gt @ Einv)
        if odom is not None:
            g.odomNextScan(*odom)
        pg, Tg, ug = g.receiveCloud(cloud)
        po, To, uo = o.receive_cloud(cloud, odom=odom)
        assert ug == uo, k
        n_upd += int(ug)
        dt, dr = synth.pose_error(Tg, To)
        assert dt < 1e-3 and dr < 1e-3, (k, dt, dr)
        dt, dr = synth.pose_error(Tg, E @ T_gt @ Einv)
        assert dt < 0.5 and dr < 0.02, (k, dt, dr)
    assert n_upd >= 2 and g.numSubmaps() == len(o.submaps)


def test_odometry_first_frame_and_unarmed_frames(sm, frames):
    """The first armed frame only stores the odometry (previous_odom_mat_ is Identity), and un-armed frames keep today's
    guess: odometry armed on frame 0 alone gives the bitwise result of a session that never had one. Armed on every frame,
    the guess does change the result."""
    plain, first, every = (sm.ScanMatcher(**KW) for _ in range(3))
    E = osm.pose_matrix(MOUNT_POS, MOUNT_QUAT)
    Einv = np.linalg.inv(E)
    differs = False
    for k, (cloud, T_gt) in enumerate(frames[:6]):
        odom = _odom(k, E @ T_gt @ Einv)
        if k == 0:
            first.odomNextScan(*odom)
        every.odomNextScan(*odom)
        rp, rf, re = plain.receiveCloud(cloud), first.receiveCloud(cloud), every.receiveCloud(cloud)
        assert np.array_equal(rp[0], rf[0]) and np.array_equal(_bits(rp[1]), _bits(rf[1])) and rp[2] == rf[2], k
        if k == 0:
            assert np.array_equal(_bits(rp[1]), _bits(re[1]))
        differs = differs or not np.array_equal(_bits(rp[1]), _bits(re[1]))
    _assert_same_state(plain, first)
    assert differs


def test_sensor_transform_off_means_off(sm, frames):
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    a, b = sm.ScanMatcher(**KW), sm.ScanMatcher(**KW)
    a.setSensorTransform(MOUNT_POS, MOUNT_QUAT)
    a.setScan(frames[0][0])
    b.setScan(frames[0][0])
    assert not np.array_equal(_bits(_sorted(a.filteredScan())), _bits(_sorted(b.filteredScan())))
    a.setSensorTransform(None, None)
    for k, (cloud, _) in enumerate(frames[:5]):
        ra, rb = a.receiveCloud(cloud), b.receiveCloud(cloud)
        assert np.array_equal(ra[0], rb[0]) and np.array_equal(_bits(ra[1]), _bits(rb[1])) and ra[2] == rb[2], k
    _assert_same_state(a, b)
    # argument validation: non-finite translation or quaternion, zero quaternion, one of the two missing
    bad = [((np.nan, 0, 0), (0, 0, 0, 1)), ((0, np.inf, 0), (0, 0, 0, 1)), ((0, 0, 0), (0, np.nan, 0, 1)),
           ((0, 0, 0), (0, 0, -np.inf, 1)), ((0, 0, 0), (0, 0, 0, 0))]
    for fn in (a.setSensorTransform, a.odomNextScan):
        for t, q in bad:
            with pytest.raises(B200RegError) as e:
                fn(t, q)
            assert e.value.code == _capi.ERR_ARG, (fn, t, q)
    L = a._lib
    q = np.array([0, 0, 0, 1.0])
    assert L.b200sm_set_sensor_transform(a._h, None, q.ctypes.data) == _capi.ERR_ARG
    assert L.b200sm_odom_next_scan(a._h, None, None) == _capi.ERR_ARG
    # a rejected call leaves the session as it was: still off, still bitwise equal to b
    cloud = frames[5][0]
    ra, rb = a.receiveCloud(cloud), b.receiveCloud(cloud)
    assert np.array_equal(_bits(ra[1]), _bits(rb[1]))
