"""CPU tests of the ASCII PCD formatter (csrc/pcd_format.cuh built for the host by tests/hostmath/pcd_host.cpp) against
glibc's snprintf("%.8g", (double)f) — what libstdc++'s `ostream << float` at precision 8 prints, and so what PCL's
writeASCII writes — and of the restated PCL writer (tests/hostmath/pcd_writer_ref.hpp) against the same bytes assembled
in Python from '%.8g'. The exhaustive sweep of all 2^32 patterns is tests/diag/sweep_pcd_format.py."""
import ctypes as C
import ctypes.util
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "pcd_host.cpp")

HEADER = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\n"
          "COUNT 1 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA ascii\n")


def build_pcd_host(out_dir):
    """Compiles the host shim (OpenMP for the bulk comparisons) into out_dir and loads it."""
    lib = os.path.join(out_dir, "libpcd_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    L = C.CDLL(lib)
    L.ph_format.argtypes = [C.c_float, C.c_char_p]
    L.ph_format_line.argtypes = [C.c_void_p, C.c_char_p]
    L.ph_check_range.restype = C.c_longlong
    L.ph_check_range.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p]
    L.ph_check_list.restype = C.c_longlong
    L.ph_check_list.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    L.ph_write_pcd_ascii_mem.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.ph_save_pcd_ascii.argtypes = [C.c_char_p, C.c_void_p, C.c_size_t]
    return L


def reference_pcd_bytes(L, xyzi):
    """The restated savePCDFileASCII bytes of an (N, 4) float32 cloud."""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32)
    n = C.c_size_t(0)
    assert L.ph_write_pcd_ascii_mem(xyzi.ctypes.data, len(xyzi), None, 0, C.byref(n)) == 0
    buf = C.create_string_buffer(n.value)
    assert L.ph_write_pcd_ascii_mem(xyzi.ctypes.data, len(xyzi), buf, n.value, C.byref(n)) == 0
    return buf.raw[:n.value]


def python_pcd_bytes(xyzi):
    lines = [" ".join("nan" if np.isnan(v) else "%.8g" % float(v) for v in row) for row in np.asarray(xyzi, dtype=np.float32)]
    return (HEADER.format(n=len(lines)) + "".join(l + "\n" for l in lines)).encode()


def f32(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


@pytest.fixture(scope="module")
def ph(tmp_path_factory):
    return build_pcd_host(str(tmp_path_factory.mktemp("pcd_host")))


@pytest.fixture(scope="module")
def libc_g8():
    libc = C.CDLL(ctypes.util.find_library("c"))
    buf = C.create_string_buffer(64)

    def g8(f):
        n = libc.snprintf(buf, 64, b"%.8g", C.c_double(float(f)))
        return buf.raw[:n]
    return g8


def _ours(ph, f):
    buf = C.create_string_buffer(32)
    n = ph.ph_format(float(f), buf)
    return buf.raw[:n]


def _check_list(ph, bits):
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    first = C.c_uint32(0)
    bad = ph.ph_check_list(bits.ctypes.data, len(bits), C.byref(first))
    assert bad == 0, f"{bad} mismatches, first 0x{first.value:08x}"


def test_special_values_and_ties_match_glibc(ph, libc_g8):
    specials = [0x00000000, 0x80000000, 0x7f800000, 0xff800000, 0x7f7fffff, 0xff7fffff, 0x00000001, 0x80000001,
                0x00800000, 0x007fffff]
    for b in specials:
        f = f32(b)
        assert _ours(ph, f) == libc_g8(f), hex(b)
    assert [_ours(ph, f32(b)) for b in specials[:4]] == [b"0", b"-0", b"inf", b"-inf"]
    cases = {1234567.25: b"1234567.2", 1234567.75: b"1234567.8", 1e-5: b"9.9999997e-06", 1e8: b"1e+08",
             3.4028234663852886e38: b"3.4028235e+38", 1.401298464324817e-45: b"1.4012985e-45"}
    for v, want in cases.items():
        assert _ours(ph, np.float32(v)) == want == libc_g8(np.float32(v)), v
    for b in (0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fbfffff, 0xffffffff, 0x7fc12345):
        assert _ours(ph, f32(b)) == b"nan", hex(b)  # writeASCII prints every NaN as "nan"
    # exact ties: t / 2^j whose decimal expansion t * 5^j has exactly nine digits (so it ends in 5), t odd, t < 2^24
    rng = np.random.default_rng(7)
    parity = {0: 0, 1: 0}
    for j in range(1, 13):
        lo, hi = -(-10 ** 8 // 5 ** j), min(1 << 24, 10 ** 9 // 5 ** j)
        if lo >= hi:  # j = 1: nine digits need t > 2^24
            continue
        for t in set(int(v) | 1 for v in rng.integers(lo, hi, size=200)) | {lo | 1}:
            if not (lo <= t < hi):
                continue
            v = np.float32(t / 2.0 ** j)
            assert float(v) == t / 2.0 ** j
            digits = str(t * 5 ** j)
            assert len(digits) == 9 and digits[-1] == "5"
            parity[int(digits[7]) % 2] += 1
            for s in (v, -v):
                assert _ours(ph, s) == libc_g8(s), (t, j)
    assert parity[0] > 100 and parity[1] > 100  # ties that stay (even) and ties that round up (odd)


def test_powers_of_ten_plus_minus_64_ulps(ph, libc_g8):
    bits = []
    for k in range(-45, 39):
        b = int(np.float32(10.0 ** k).view(np.uint32))
        if b == 0:
            continue
        bits += [v for v in range(b - 64, b + 65) if 0 < v < 0x7f800000]
    bits = np.unique(np.array(bits, dtype=np.uint32))
    bits = np.concatenate([bits, bits | np.uint32(0x80000000)])
    for b in bits[::37]:  # a sample straight through ctypes, all of them through the shim's snprintf loop
        f = f32(b)
        assert _ours(ph, f) == libc_g8(f), hex(int(b))
    _check_list(ph, bits)


@pytest.mark.parametrize("v", [1e-5, 1e-4, 1.0, 1e7, 1e8])
def test_every_mantissa_of_the_binades_at_the_style_switches(ph, v):
    b = int(np.float32(v).view(np.uint32)) & 0x7f800000
    first = C.c_uint32(0)
    for lo in (b - 0x800000, b):  # the binade holding v and the one below it
        bad = ph.ph_check_range(lo, lo + 0x7fffff, C.byref(first))
        assert bad == 0, f"{bad} mismatches in binade 0x{lo:08x}, first 0x{first.value:08x}"


def test_every_subnormal_and_the_smallest_normal_binade(ph):
    first = C.c_uint32(0)
    for lo, hi in ((0x00000000, 0x00ffffff), (0x80000000, 0x807fffff)):
        bad = ph.ph_check_range(lo, hi, C.byref(first))
        assert bad == 0, f"{bad} mismatches, first 0x{first.value:08x}"


def test_twenty_million_random_bit_patterns(ph):
    rng = np.random.default_rng(20)
    _check_list(ph, rng.integers(0, 1 << 32, size=20_000_000, dtype=np.uint64).astype(np.uint32))


def test_reference_writer_equals_python_assembly(ph, tmp_path):
    rng = np.random.default_rng(3)
    special = f32([0x7fc00000, 0xffc00001, 0x80000000, 0x00000000, 0x7f800000, 0xff800000, 0x7f7fffff, 0x00000001])
    cloud = np.concatenate([rng.normal(size=(500, 4)).astype(np.float32) * np.float32(100),
                            f32(rng.integers(0, 1 << 32, size=(500, 4), dtype=np.uint64).astype(np.uint32)),
                            special.reshape(2, 4)], axis=0)
    want = python_pcd_bytes(cloud)
    assert reference_pcd_bytes(ph, cloud) == want
    assert reference_pcd_bytes(ph, cloud[:1]) == python_pcd_bytes(cloud[:1])
    path = tmp_path / "map.pcd"
    assert ph.ph_save_pcd_ascii(str(path).encode(), np.ascontiguousarray(cloud).ctypes.data, len(cloud)) == 0
    assert path.read_bytes() == want
    empty = np.zeros((0, 4), dtype=np.float32)
    n = C.c_size_t(0)
    assert ph.ph_write_pcd_ascii_mem(empty.ctypes.data, 0, None, 0, C.byref(n)) == -1
    assert ph.ph_save_pcd_ascii(str(tmp_path / "empty.pcd").encode(), empty.ctypes.data, 0) == -1
    assert not (tmp_path / "empty.pcd").exists()
    # the product's host line formatter gives the same lines
    body = want.split(b"DATA ascii\n", 1)[1]
    buf = C.create_string_buffer(64)
    lines = []
    for row in np.ascontiguousarray(cloud):
        n_line = ph.ph_format_line(row.ctypes.data, buf)
        assert n_line <= 60
        lines.append(buf.raw[:n_line])
    assert b"".join(lines) == body
