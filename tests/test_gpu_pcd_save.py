"""savePCDFileASCII on the device (b200reg_encode_pcd_ascii, b200sm_save_map_pcd_ascii): every byte against the restated
PCL writer (tests/hostmath/pcd_writer_ref.hpp), on special values, random bit patterns, the golden target, a synthetic
map, and saved session maps whose sizes straddle the encoder's chunk of PCD_CHUNK_POINTS points."""
import ctypes as C

import numpy as np
import pytest

import lidarslam_ros2_b200 as m
from lidarslam_ros2_b200 import _capi, synth
from lidarslam_ros2_b200.registration import B200RegError
from test_pcd_format_cpu import build_pcd_host, f32, reference_pcd_bytes

pytestmark = pytest.mark.gpu
CHUNK = 1 << 22  # PCD_CHUNK_POINTS (csrc/engine.hpp)


@pytest.fixture(scope="module")
def ph(tmp_path_factory):
    return build_pcd_host(str(tmp_path_factory.mktemp("pcd_host")))


def _with_intensity(xyz, rng):
    return np.concatenate([xyz, rng.uniform(0, 255, size=(len(xyz), 1))], axis=1).astype(np.float32)


def test_special_values(ph):
    nans = [0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fbfffff, 0xffffffff, 0x7fc12345, 0xffd00bad]
    other = [0x00000000, 0x80000000, 0x7f800000, 0xff800000, 0x7f7fffff, 0xff7fffff, 0x00000001, 0x80000001,
             0x00800000, 0x007fffff]
    ties = [np.float32(v).view(np.uint32) for v in (1234567.25, 1234567.75, -1234567.25, 1e-5, 1e8, 1e-4, 9.9999999e-5)]
    bits = nans + other + [int(b) for b in ties]
    cloud = f32(bits + [0] * (-len(bits) % 4)).reshape(-1, 4)
    got = m.encode_pcd_ascii(cloud)
    assert got == reference_pcd_bytes(ph, cloud)
    assert got.split(b"DATA ascii\n")[1].startswith(b"nan nan nan nan\nnan nan nan nan\n0 -0 inf -inf\n")


def test_ten_million_random_finite_patterns(ph):
    rng = np.random.default_rng(11)
    bits = rng.integers(0, 1 << 32, size=10_000_000, dtype=np.uint64).astype(np.uint32)
    bits = bits[(bits & 0x7f800000) != 0x7f800000]
    cloud = f32(bits[: len(bits) // 4 * 4]).reshape(-1, 4)
    assert m.encode_pcd_ascii(cloud) == reference_pcd_bytes(ph, cloud)


def test_golden_target_and_a_synthetic_map(ph, golden_dir):
    import os

    rng = np.random.default_rng(12)
    tgt = _with_intensity(np.load(os.path.join(golden_dir, "pcd_target_ds.npy")), rng)
    assert m.encode_pcd_ascii(tgt) == reference_pcd_bytes(ph, tgt)
    mp = _with_intensity(synth.sample_map(synth.make_scene(1), 300_000, stream=5), rng)
    assert m.encode_pcd_ascii(mp) == reference_pcd_bytes(ph, mp)
    # PointXYZI records as PCL lays them out (32 bytes, intensity at byte 16)
    rec = np.zeros((len(mp), 8), dtype=np.float32)
    rec[:, :3], rec[:, 4] = mp[:, :3], mp[:, 3]
    L = _capi.lib()
    n = C.c_size_t(0)
    assert L.b200reg_encode_pcd_ascii(0, rec.ctypes.data, len(rec), 32, 16, None, 0, C.byref(n)) == 0
    buf = C.create_string_buffer(n.value)
    assert L.b200reg_encode_pcd_ascii(0, rec.ctypes.data, len(rec), 32, 16, buf, n.value, C.byref(n)) == 0
    assert buf.raw == reference_pcd_bytes(ph, mp)


def test_size_query_and_short_capacity(ph):
    rng = np.random.default_rng(13)
    cloud = rng.normal(size=(CHUNK + 1000, 4)).astype(np.float32) * np.float32(50)
    want = reference_pcd_bytes(ph, cloud)
    L = _capi.lib()
    n = C.c_size_t(0)
    assert L.b200reg_encode_pcd_ascii(0, cloud.ctypes.data, len(cloud), 16, 12, None, 0, C.byref(n)) == 0
    assert n.value == len(want)
    for cap in (1, 100, 317, len(want) // 2, len(want) - 1):  # inside the header, the first chunk, the second chunk
        buf = np.full(cap + 64, 0xAB, dtype=np.uint8)
        n = C.c_size_t(0)
        assert L.b200reg_encode_pcd_ascii(0, cloud.ctypes.data, len(cloud), 16, 12, buf.ctypes.data, cap, C.byref(n)) == 0
        assert n.value == len(want)
        assert buf[:cap].tobytes() == want[:cap] and (buf[cap:] == 0xAB).all()


def test_encode_argument_errors():
    L = _capi.lib()
    cloud = np.ones((10, 8), dtype=np.float32)
    n = C.c_size_t(0)
    for stride, ioff, count in ((32, 16, 0), (32, -1, 10), (32, 14, 10), (30, 16, 10), (18, 12, 10), (16, 16, 10)):
        assert L.b200reg_encode_pcd_ascii(0, cloud.ctypes.data, count, stride, ioff, None, 0, C.byref(n)) == _capi.ERR_ARG
    with pytest.raises(ValueError):
        m.encode_pcd_ascii(cloud[:, :3])


def _session(sizes, rng):
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher()
    for i, k in enumerate(sizes):
        c = _with_intensity(rng.uniform(-60, 60, size=(k, 3)), rng)
        g.importSubmap(c, synth.pose_matrix(rng.normal(size=3) * 50.0, rng.uniform(-np.pi, np.pi, size=3)), 2.0 * i)
    return g


@pytest.mark.parametrize("sizes", [[1], [CHUNK // 2, CHUNK // 4, CHUNK // 4], [CHUNK, 1], [CHUNK + 7, CHUNK, CHUNK // 2 - 7]],
                         ids=["1", "chunk", "chunk+1", "2.5chunks"])
def test_save_map_after_pose_adjust_and_with_the_session_poses(ph, tmp_path, sizes):
    rng = np.random.default_rng(len(sizes) * 1000 + sum(sizes) % 997)
    g = _session(sizes, rng)
    n = g.numSubmaps()
    loops = [(0, n - 1, synth.pose_matrix((1.0, 0.5, 0.0), (0.0, 0.0, 0.1)))] if n > 1 else []
    poses, _ = g.poseAdjust(loops)
    for P, name in ((poses, "adjusted.pcd"), (None, "session.pcd")):
        path = tmp_path / name
        points, size = g.saveMapPCDASCII(str(path), P)
        cloud, _ = g.assembleMap(P)
        want = reference_pcd_bytes(ph, cloud)
        assert points == sum(sizes) == len(cloud) and size == len(want)
        assert path.read_bytes() == want
    path.write_bytes(b"x" * (len(want) + 10))  # an existing file is replaced, not appended to or left longer
    g.saveMapPCDASCII(str(path))
    assert path.read_bytes() == want


def test_save_twenty_million_points(ph, tmp_path):
    rng = np.random.default_rng(5)
    g = _session([20_000] * 1000, rng)  # the sizes of test_gpu_pose_adjust's one-launch assembly
    adjusted = np.array([synth.pose_matrix(rng.normal(size=3) * 100.0, rng.uniform(-np.pi, np.pi, size=3)) for _ in range(1000)])
    path = tmp_path / "map.pcd"
    points, size = g.saveMapPCDASCII(str(path), adjusted)
    cloud, _ = g.assembleMap(adjusted)
    want = reference_pcd_bytes(ph, cloud)
    assert points == 20_000_000 and size == len(want) and path.stat().st_size == len(want)
    assert path.read_bytes() == want


def test_save_errors(tmp_path):
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher()
    path = tmp_path / "map.pcd"
    with pytest.raises(B200RegError) as e:
        g.saveMapPCDASCII(str(path))
    assert e.value.code == _capi.ERR_ARG and not path.exists()
    g.importSubmap(np.zeros((0, 4), dtype=np.float32), np.eye(4), 0.0)  # a map of empty submaps is empty too
    with pytest.raises(B200RegError) as e:
        g.saveMapPCDASCII(str(path))
    assert e.value.code == _capi.ERR_ARG and not path.exists()
    g = _session([100], np.random.default_rng(1))
    with pytest.raises(B200RegError) as e:
        g.saveMapPCDASCII(str(tmp_path / "missing" / "map.pcd"))
    assert e.value.code == _capi.ERR_IO and not (tmp_path / "missing").exists()
    assert g.saveMapPCDASCII(str(path))[0] == 100
