"""loadPCDFile on the device (b200reg_load_pcd, b200reg_set_input_target_pcd): every point against the restated PCL 1.12
reader (tests/hostmath/pcd_reader_ref.hpp), bit for bit, NaN bits included: saved maps, random bit patterns, files whose
newlines sit at the reader's piece edges, other layouts, binary files against a numpy view, the error codes (with the
previous target kept), and NDT / GICP targets set from a file against the same cloud set from the host."""
import ctypes as C
import os

import numpy as np
import pytest

import lidarslam_ros2_b200 as m
from lidarslam_ros2_b200 import _capi, synth
from lidarslam_ros2_b200.registration import B200RegError
from test_pcd_parse_cpu import build_pcd_parse_host, hdr, reference_read

pytestmark = pytest.mark.gpu
PIECE = _capi.PCD_LOAD_PIECE_BYTES


@pytest.fixture(scope="module")
def pp(tmp_path_factory):
    return build_pcd_parse_host(str(tmp_path_factory.mktemp("pcd_parse_host")))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same_as_reference(pp, path):
    rc, want, _ = reference_read(pp, path)
    assert rc == 0
    got = m.read_pcd(str(path))
    assert got.shape == want.shape and np.array_equal(bits(got), bits(want))
    return got


def g9_body(cloud):
    return "".join(" ".join("%.9g" % v for v in row) + "\n" for row in cloud.astype(np.float64)).encode()


@pytest.mark.parametrize("sizes", [[1], [1000, 37], [20_000] * 1000], ids=["1", "small", "20M"])
def test_saved_map_round_trip(pp, tmp_path, sizes):
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    rng = np.random.default_rng(len(sizes))
    g = ScanMatcher()
    for i, k in enumerate(sizes):
        c = np.concatenate([rng.uniform(-60, 60, size=(k, 3)), rng.uniform(0, 255, size=(k, 1))], axis=1).astype(np.float32)
        g.importSubmap(c, synth.pose_matrix(rng.normal(size=3) * 50.0, rng.uniform(-np.pi, np.pi, size=3)), 2.0 * i)
    path = tmp_path / "map.pcd"
    points, _ = g.saveMapPCDASCII(str(path))
    got = same_as_reference(pp, path)
    assert len(got) == points == sum(sizes)
    cloud, _ = g.assembleMap(None)
    assert np.allclose(got, cloud, rtol=1e-7, atol=0)  # %.8g keeps about eight digits


def test_random_bit_patterns_and_g9_exactness(pp, tmp_path):
    rng = np.random.default_rng(9)
    pat = rng.integers(0, 1 << 32, size=(500_000, 4), dtype=np.uint64).astype(np.uint32)
    pat[:2] = np.array([0x7fc00000, 0xffc00001, 0x7f800000, 0xff800000, 0x00000001, 0x807fffff, 0x80000000, 0x7f7fffff],
                       dtype=np.uint32).reshape(2, 4)
    cloud = pat.view(np.float32)
    path = tmp_path / "bits.pcd"
    path.write_bytes(m.encode_pcd_ascii(cloud))
    got = same_as_reference(pp, path)
    assert bits(got[0]).tolist() == [0x7fc00000, 0x7fc00000, 0x7f800000, 0xff800000]  # every NaN is written as "nan"
    finite = cloud[~np.isnan(cloud).any(axis=1)]
    path.write_bytes(hdr(w=len(finite), n=len(finite)) + g9_body(finite))
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(finite))  # %.9g reads back exactly


def _cloud(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(n, 4)) * 100).astype(np.float32)


def _newline_at(lines, target, pad_line=0):
    """lines (bytes, each ending in '\\n'): pads line pad_line with spaces so that a newline falls at body offset target"""
    ends = np.cumsum([len(l) for l in lines]) - 1
    k = int(np.searchsorted(ends, target, side="right")) - 1
    assert k > pad_line
    extra = target - int(ends[k])
    lines = list(lines)
    lines[pad_line] = lines[pad_line].replace(b" ", b" " * (1 + extra), 1)
    return lines


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_newlines_at_the_piece_edge(pp, tmp_path, delta):
    cloud = _cloud(PIECE // 40, 20 + delta)
    lines = [l + b"\n" for l in g9_body(cloud).split(b"\n")[:-1]]
    lines = _newline_at(lines, PIECE - 1 + delta)  # '\n' the last byte of the first piece, one before, one after
    body = b"".join(lines)
    assert body[PIECE - 1 + delta:PIECE + delta] == b"\n"
    path = tmp_path / "edge.pcd"
    path.write_bytes(hdr(w=len(cloud), n=len(cloud)) + body)
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(cloud))


def test_straddling_long_line_and_a_last_line_without_newline(pp, tmp_path):
    cloud = _cloud(PIECE // 30, 33)
    lines = [l + b"\n" for l in g9_body(cloud).split(b"\n")[:-1]]
    k = int(np.searchsorted(np.cumsum([len(l) for l in lines]), PIECE)) - 3
    lines[k] = lines[k].replace(b" ", b" " * 20000, 1)  # longer than a tile and its spill, across the piece edge
    lines[-1] = lines[-1][:-1]
    path = tmp_path / "long.pcd"
    path.write_bytes(hdr(w=len(cloud), n=len(cloud)) + b"".join(lines))
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(cloud))


def test_ascii_layouts(pp, tmp_path):
    c = _cloud(300, 4)
    path = tmp_path / "l.pcd"
    # extra fields: COUNT 3, unsigned and 2-byte fields, skipped whatever their text
    rows = "".join(f"{i} {x!r} 0.1 0.2 0.3 {y!r} {z!r} {w!r} {i % 64}\n" for i, (x, y, z, w) in enumerate(c.tolist()))
    path.write_bytes(hdr(f="rgb x normal y z intensity ring", s="4 4 4 4 4 4 2", t="U F F F F F U", c="1 1 3 1 1 1 1", w=300, n=300)
                     + rows.encode())
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(c))
    # x y z only: intensity 0
    path.write_bytes(hdr(f="x y z", s="4 4 4", t="F F F", c="1 1 1", w=300, n=300) + g9_body(c[:, :3]))
    got = same_as_reference(pp, path)
    assert np.array_equal(bits(got[:, :3]), bits(c[:, :3])) and (bits(got[:, 3]) == 0).all()
    # another order
    path.write_bytes(hdr(f="intensity z x y", w=300, n=300) + g9_body(c[:, [3, 2, 0, 1]]))
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(c))
    # tabs, CRLF, blank lines, padded columns
    body = g9_body(c).replace(b"\n", b"\r\n").replace(b" ", b"\t  ")
    body = body.replace(b"\r\n", b"\r\n\n", 50)
    path.write_bytes(hdr(w=300, n=300) + body)
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(c))
    # more lines than POINTS (even malformed ones) are not read
    path.write_bytes(hdr(w=200, n=200) + g9_body(c) + b"not a point\n")
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(c[:200]))
    # HEIGHT > 1 comes out flat
    path.write_bytes(hdr(w=60, h=5, n=300) + g9_body(c))
    assert np.array_equal(bits(same_as_reference(pp, path)), bits(c))


@pytest.mark.parametrize("layout", ["16", "32", "20", "24"])
def test_binary_layouts(tmp_path, layout):
    c = _cloud(100_003, 7)
    n = len(c)
    if layout == "16":
        head, rec = hdr(w=n, n=n, d="binary"), c.copy()
    elif layout == "32":  # pcl::PointXYZI as PCL writes it: padding fields "_"
        head = hdr(f="x y z _ intensity _", s="4 4 4 1 4 1", t="F F F U F U", c="1 1 1 4 1 12", w=n, n=n, d="binary")
        rec = np.zeros((n, 8), dtype=np.float32)
        rec[:, :3], rec[:, 4] = c[:, :3], c[:, 3]
    elif layout == "20":  # a field before x
        head = hdr(f="t x y z intensity", s="4 4 4 4 4", t="F F F F F", c="1 1 1 1 1", w=n, n=n, d="binary")
        rec = np.concatenate([np.full((n, 1), 7.0, np.float32), c], axis=1)
    else:  # no intensity, two 2-byte fields after z
        head = hdr(f="x y z ring flags t", s="4 4 4 2 2 4", t="F F F U U F", c="1 1 1 1 1 2", w=n, n=n, d="binary")
        rec = np.concatenate([c[:, :3], np.full((n, 3), 3.0, np.float32)], axis=1)
        c = c.copy()
        c[:, 3] = 0
    path = tmp_path / "b.pcd"
    path.write_bytes(head + np.ascontiguousarray(rec).tobytes())
    got = m.read_pcd(str(path))
    assert np.array_equal(bits(got), bits(c))


def _ndt(tgt=None):
    g = m.NormalDistributionsTransform(device=0)
    g.setResolution(2.0)
    g.setTransformationEpsilon(0.01)
    if tgt is not None:
        g.setInputTarget(tgt)
    return g


BAD = {
    "binary_compressed": (hdr(w=1, n=1, d="binary_compressed") + b"\0" * 64, _capi.ERR_FORMAT),
    # bodies long enough for POINTS by size, so that the device's line checks decide
    "token_count": (hdr(w=2, n=2) + b"1 2 3 4\n1 2 3        \n", _capi.ERR_FORMAT),
    "too_few_lines": (hdr(w=3, n=3) + b"1 2 3 4\n\n1 2 3 4\n" + b"\n" * 10, _capi.ERR_FORMAT),
    "truncated_binary": (hdr(w=3, n=3, d="binary") + b"\0" * 47, _capi.ERR_FORMAT),
    "missing_x": (hdr(f="y z intensity", s="4 4 4", t="F F F", c="1 1 1", w=1, n=1) + b"1 2 3\n", _capi.ERR_FORMAT),
    "x_f8": (hdr(s="8 4 4 4", w=1, n=1) + b"1 2 3 4\n", _capi.ERR_FORMAT),
    "malformed_token": (hdr(w=2, n=2) + b"1 2 3 4\n1 2.5abc 3 4\n", _capi.ERR_FORMAT),
    "missing_file": (None, _capi.ERR_IO),
}


@pytest.mark.parametrize("case", list(BAD))
def test_errors_keep_the_previous_target(tmp_path, case):
    src, tgt, _ = synth.registration_pair("tiny", 2.0)
    good = tmp_path / "good.pcd"
    xyzi = np.concatenate([tgt[:, :3], np.zeros((len(tgt), 1))], axis=1).astype(np.float32)
    good.write_bytes(m.encode_pcd_ascii(xyzi))
    g = _ndt()
    assert g.setInputTargetPCD(str(good)) == len(tgt)
    g.setInputSource(src)
    T0, v0 = g.align(), g.voxels()
    content, code = BAD[case]
    path = tmp_path / "bad.pcd"
    if content is not None:
        path.write_bytes(content)
    with pytest.raises(B200RegError) as e:
        m.read_pcd(str(path))
    assert e.value.code == code
    with pytest.raises(B200RegError) as e:
        g.setInputTargetPCD(str(path))
    assert e.value.code == code
    msg = _capi.lib().b200reg_last_error(g._h).decode()
    assert "setInputTargetPCD" in msg and (case not in ("token_count", "malformed_token") or "line 12" in msg), msg
    assert case != "too_few_lines" or "2 data lines, POINTS says 3" in msg, msg
    v1 = g.voxels()
    assert all(np.array_equal(v0[k], v1[k]) for k in v0)
    assert np.array_equal(g.align(), T0)


@pytest.mark.parametrize("kind", ["ndt", "gicp"])
def test_target_from_file_equals_target_from_host(pp, tmp_path, kind):
    src, tgt, _ = synth.registration_pair("tiny", 2.0)
    rng = np.random.default_rng(2)
    xyzi = np.concatenate([tgt[:, :3], rng.uniform(0, 255, size=(len(tgt), 1))], axis=1).astype(np.float32)
    path = tmp_path / "map.pcd"
    path.write_bytes(m.encode_pcd_ascii(xyzi))
    rc, ref_cloud, _ = reference_read(pp, path)
    assert rc == 0
    make = _ndt if kind == "ndt" else (lambda: m.GeneralizedIterativeClosestPoint(device=0))
    a, b = make(), make()
    a.setInputTarget(ref_cloud)
    assert b.setInputTargetPCD(str(path)) == len(ref_cloud)
    for g in (a, b):
        g.setInputSource(src)
    Ta, Tb = a.align(), b.align()
    fa, fb = a.getFitnessScore(), b.getFitnessScore()
    if kind == "gicp":
        assert np.array_equal(Ta, Tb) and fa == fb
    else:
        # the same voxels; their sums are accumulated with double atomics, so two builds of one cloud agree to rounding
        # only, and so do the solves on them
        assert np.allclose(Ta, Tb, rtol=0, atol=1e-5) and abs(fa - fb) <= 1e-6 * abs(fa)
        va, vb = a.voxels(), b.voxels()
        assert np.array_equal(va["idx"], vb["idx"]) and np.array_equal(va["npts"], vb["npts"])
        assert all(np.allclose(va[k], vb[k], rtol=1e-9, atol=1e-12) for k in ("mean", "icov"))
        assert np.allclose(va["centroid"], vb["centroid"], rtol=1e-6, atol=1e-6)


def test_points_beyond_the_body_and_data_past_points(tmp_path):
    path = tmp_path / "p.pcd"
    for d in ("ascii", "binary"):  # refused from the file size, before anything is allocated for POINTS
        path.write_bytes(hdr(w=999999999999, n=999999999999, d=d) + b"1 2 3 4\n" * 12)
        for call in (lambda: m.read_pcd(str(path)), lambda: _ndt().setInputTargetPCD(str(path))):
            with pytest.raises(B200RegError) as e:
                call()
            assert e.value.code == _capi.ERR_FORMAT
    # after POINTS lines reading stops: a trailing line longer than a piece is not an error
    path.write_bytes(hdr(w=2, n=2) + b"1 2 3 4\n5 6 7 8\n" + b"x" * (PIECE + 100) + b"\n")
    assert m.read_pcd(str(path)).tolist() == [[1, 2, 3, 4], [5, 6, 7, 8]]
    path.write_bytes(hdr(w=3, n=3) + b"1 2 3 4\n5 6 7 8\n" + b"x" * (PIECE + 100) + b"\n")
    with pytest.raises(B200RegError) as e:
        m.read_pcd(str(path))
    assert e.value.code == _capi.ERR_FORMAT


def test_grid_overflow_keeps_the_previous_target(tmp_path):
    src, tgt, _ = synth.registration_pair("tiny", 2.0)
    g = _ndt(tgt)
    g.setInputSource(src)
    T0, v0 = g.align(), g.voxels()
    far = np.array([[0, 0, 0, 0], [1e6, 1e6, 1e6, 0]] * 4, dtype=np.float32)  # 500 000^3 voxels at resolution 2
    path = tmp_path / "far.pcd"
    path.write_bytes(m.encode_pcd_ascii(far))
    with pytest.raises(B200RegError) as e:
        g.setInputTargetPCD(str(path))
    assert e.value.code == _capi.ERR_GRID
    v1 = g.voxels()
    assert all(np.array_equal(v0[k], v1[k]) for k in v0) and np.array_equal(g.align(), T0)
