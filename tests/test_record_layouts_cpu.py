"""Host record layouts of the C-ABI's cloud inputs, the part that needs no GPU: the fixture builders shared with
tests/test_gpu_record_layouts.py, and the argument check of the two stand-alone calls that take an intensity offset,
b200reg_voxelgrid and b200reg_encode_pcd_ascii, which refuse a bad layout before they touch CUDA.

A layout (stride_bytes, intensity_offset_bytes) is valid when the stride is >= 12 and a multiple of 4 and the intensity
offset is negative (no intensity) or a multiple of 4 with offset + 4 <= stride (include/b200reg.h, "Conventions"). The
offsets from stride - 3 to stride + 4 and those that are not a multiple of 4 are refused with ERR_ARG, and the caller's
output buffer and count are left as they were.

The layouts are those real callers send: packed rows (stride 12 or 16), PCL's PointXYZI (stride 32, intensity at 16) and
sensor_msgs/PointCloud2 records (point_step 20-64, intensity at 12, 16 or the last float; a point_step of 22 is 24 here,
rounded up to whole floats)."""
import ctypes as C

import numpy as np
import pytest

F32 = np.float32
STRIDES = (12, 16, 20, 24, 32, 48, 64)
LATTICE = 2.0**-12  # metres: every fixture coordinate is a multiple of it
EXTENT = 128.0  # ... and within +-EXTENT metres
FLT_MAX_BITS = 0x7F7FFFFF


def intensity_offsets(stride):
    """-1 (no intensity), 12, 16 and the last float of the record, where each fits after x, y, z."""
    return sorted({o for o in (-1, 12, 16, stride - 4) if o < 0 or 12 <= o <= stride - 4})


LAYOUTS = [(s, o) for s in STRIDES for o in intensity_offsets(s)]


def bad_offsets(stride):
    """Offsets a record of `stride` bytes cannot hold an intensity float at: stride - 3 ... stride + 4 (the float would end
    past the record), offsets inside it that are not a multiple of 4, and one far past it."""
    return sorted(set(range(stride - 3, stride + 5)) | {13, 14, 15, stride - 5, 1 << 31} - {stride - 4})


def valid_layout(stride, offset):
    return stride >= 12 and stride % 4 == 0 and (offset < 0 or (offset % 4 == 0 and offset + 4 <= stride))


def lattice(cloud):
    """x, y, z rounded to the 2^-12 m lattice and intensity to an integer. The coordinates must lie within +-128 m. Then a
    coordinate has at most 19 significant bits and a product of two at most 38: VoxelGrid's float64 sums and the NDT voxel
    map's sums of products are exact for up to 2^15 points per voxel, whatever order the device's atomics add them in."""
    c = np.array(cloud, dtype=np.float64)
    c[:, :3] = np.round(c[:, :3] / LATTICE) * LATTICE
    assert np.all(np.abs(c[:, :3]) < EXTENT), np.abs(c[:, :3]).max()
    if c.shape[1] > 3:
        c[:, 3] = np.round(c[:, 3])
    return np.ascontiguousarray(c, dtype=F32)


def packed(cloud, offset):
    """The packed (N, 4) rows of the same points: intensity in column 3, or the sessions' default 0 when offset < 0."""
    c = np.asarray(cloud, dtype=F32)
    out = np.zeros((len(c), 4), dtype=F32)
    out[:, :3] = c[:, :3]
    if offset >= 0:
        out[:, 3] = c[:, 3]
    return out


def poison_words(n, w, seed=0):
    """(n, w) uint32 float bit patterns a call must never read: NaN with a payload that differs per row and column (both
    signs), +-inf and +-FLT_MAX, the kind rotating with row and column."""
    seed %= 65521
    i = np.arange(n, dtype=np.uint64)[:, None]
    j = np.arange(w, dtype=np.uint64)[None, :]
    payload = ((i * 2654435761 + j * 40503 + seed * 977) % 0x3FFFFF + 1).astype(np.uint32)
    kinds = np.stack(np.broadcast_arrays(
        np.uint32(0x7FC00000) | payload, np.uint32(0x7F800000) | payload, np.uint32(0xFFC00000) | payload,
        np.full((n, w), 0x7F800000, np.uint32), np.full((n, w), 0xFF800000, np.uint32),
        np.full((n, w), FLT_MAX_BITS, np.uint32), np.full((n, w), 0x80000000 | FLT_MAX_BITS, np.uint32)))
    k = ((i + 3 * j + seed) % len(kinds)).astype(np.intp)
    return np.take_along_axis(kinds, k[None], axis=0)[0]


def records(cloud, stride, offset, seed=0, pinned=False):
    """(n, stride) uint8 host records of `cloud`: x, y, z at bytes 0, 4, 8, the intensity at `offset` (when >= 0), and
    poison_words in every other 4 bytes. pinned: page-locked memory from torch."""
    c = np.asarray(cloud, dtype=F32)
    n, w = len(c), stride // 4
    assert stride % 4 == 0 and w >= 3
    if pinned:
        import torch

        out = torch.empty((n, stride), dtype=torch.uint8, pin_memory=True).numpy()
    else:
        out = np.empty((n, stride), dtype=np.uint8)
    words = out.view(np.uint32)
    words[:] = poison_words(n, w, seed)
    words[:, :3] = c[:, :3].view(np.uint32)
    if offset >= 0:
        words[:, offset // 4] = c[:, 3].view(np.uint32)
    return out


def unread_words(stride, offset):
    """Word indices of a record that hold neither x, y, z nor the intensity."""
    return [j for j in range(3, stride // 4) if j != offset // 4 or offset < 0]


def voxelgrid_writeback(sentinel, rows, stride, offset):
    """What b200reg_voxelgrid leaves in an output buffer that held `sentinel` ((cap, stride) uint8) when the filter returns
    `rows` ((m, 4) float32): x, y, z and the intensity of each row, PointXYZ's padding float data[3] = 1.0 when the stride
    has one and bytes 12-15 are not the intensity, and every other byte as it was."""
    out = np.array(sentinel, dtype=np.uint8)
    words = out.view(np.uint32)
    m = len(rows)
    r = np.ascontiguousarray(rows, dtype=F32).view(np.uint32)
    words[:m, :3] = r[:, :3]
    if stride >= 16 and offset != 12:
        words[:m, 3] = np.float32(1.0).view(np.uint32)
    if offset >= 0:
        words[:m, offset // 4] = r[:, 3]
    return out


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def lib():
    from lidarslam_ros2_b200 import _capi

    return _capi.lib()


@pytest.fixture(scope="module")
def cloud():
    rng = np.random.default_rng(3)
    return lattice(np.c_[rng.uniform(-20, 20, (700, 3)), rng.integers(0, 256, 700)])


# ---- the builders ---------------------------------------------------------------------------------------------------
def test_layout_matrix():
    assert all(valid_layout(s, o) for s, o in LAYOUTS)
    assert (32, 12) in LAYOUTS and (32, 16) in LAYOUTS and (24, 20) in LAYOUTS and (64, 60) in LAYOUTS
    assert {s for s, _ in LAYOUTS} == set(STRIDES) and len(LAYOUTS) == 22
    for s in STRIDES:
        assert not any(valid_layout(s, o) for o in bad_offsets(s))
        assert valid_layout(s, s - 4) and len([o for o in bad_offsets(s) if s - 3 <= o <= s + 4]) == 8


def test_lattice_sums_are_exact(cloud):
    """Every coordinate is k * 2^-12 with |k| < 2^19: a float64 sum of 2^15 of them, or of their pairwise products, is exact."""
    k = cloud[:, :3].astype(np.float64) / LATTICE
    assert np.array_equal(k, np.round(k)) and np.abs(k).max() < 2**19
    assert np.array_equal(cloud[:, 3], np.round(cloud[:, 3]))


@pytest.mark.parametrize("stride,offset", LAYOUTS)
def test_records_hold_the_points_and_poison_elsewhere(cloud, stride, offset):
    r = records(cloud, stride, offset, seed=stride)
    words = r.view(np.uint32)
    f = r.view(F32)
    assert np.array_equal(f[:, :3].view(np.uint32), cloud[:, :3].view(np.uint32))
    if offset >= 0:
        assert np.array_equal(f[:, offset // 4], cloud[:, 3])
    rest = unread_words(stride, offset)
    if rest:
        v = f[:, rest]
        assert np.all(~np.isfinite(v) | (np.abs(v) == np.finfo(F32).max))
        assert np.isnan(v).any() and np.isinf(v).any()
        assert (words[1:, rest] != words[:-1, rest]).all()  # differs from one row to the next


# ---- refusals of the stand-alone calls --------------------------------------------------------------------------------
@pytest.mark.parametrize("stride", STRIDES)
def test_voxelgrid_refuses_an_intensity_outside_the_record(lib, cloud, stride):
    from lidarslam_ros2_b200 import _capi

    n = len(cloud)
    sentinel = np.random.default_rng(stride).integers(0, 256, (n, stride), dtype=np.uint8)
    for offset in bad_offsets(stride):
        r = records(cloud, stride, 12 if stride >= 16 else -1)
        out = sentinel.copy()
        m = C.c_size_t(777)
        rc = lib.b200reg_voxelgrid(0, _ptr(r), n, stride, offset, 0.5, _ptr(out), n, C.byref(m))
        assert rc == _capi.ERR_ARG, (stride, offset, rc)
        assert m.value == 777 and np.array_equal(out, sentinel), (stride, offset)
    # strides that are not whole floats or too short for x, y, z
    for bad_stride in (0, 4, 8, stride + 2, stride + 1):
        out = sentinel.copy()
        m = C.c_size_t(777)
        assert lib.b200reg_voxelgrid(0, _ptr(r), n, bad_stride, -1, 0.5, _ptr(out), n, C.byref(m)) == _capi.ERR_ARG
        assert m.value == 777 and np.array_equal(out, sentinel)


@pytest.mark.parametrize("stride", STRIDES)
def test_voxelgrid_accepts_every_valid_layout(lib, cloud, stride):
    """Past the argument check: no device gives ERR_CUDA, a device a result; never ERR_ARG."""
    from lidarslam_ros2_b200 import _capi

    n = len(cloud)
    for offset in intensity_offsets(stride):
        r = records(cloud, stride, offset)
        out = np.zeros((n, stride), dtype=np.uint8)
        m = C.c_size_t(0)
        rc = lib.b200reg_voxelgrid(0, _ptr(r), n, stride, offset, 0.5, _ptr(out), n, C.byref(m))
        assert rc in (_capi.OK, _capi.ERR_CUDA), (stride, offset, rc)


@pytest.mark.parametrize("stride", STRIDES)
def test_encode_pcd_refuses_an_intensity_outside_the_record(lib, cloud, stride):
    """The encoder's own extra rule: the file always has an intensity column, so a negative offset is refused too."""
    from lidarslam_ros2_b200 import _capi

    n = len(cloud)
    r = records(cloud, stride, -1)
    for offset in bad_offsets(stride) + [-1, -4]:
        out = np.full(4096, 0xA5, dtype=np.uint8)
        nb = C.c_size_t(777)
        rc = lib.b200reg_encode_pcd_ascii(0, _ptr(r), n, stride, offset, _ptr(out), out.size, C.byref(nb))
        assert rc == _capi.ERR_ARG, (stride, offset, rc)
        assert nb.value == 777 and (out == 0xA5).all(), (stride, offset)
    for offset in intensity_offsets(stride):
        if offset >= 0:
            nb = C.c_size_t(0)
            rc = lib.b200reg_encode_pcd_ascii(0, _ptr(records(cloud, stride, offset)), n, stride, offset, None, 0, C.byref(nb))
            assert rc in (_capi.OK, _capi.ERR_CUDA), (stride, offset, rc)
