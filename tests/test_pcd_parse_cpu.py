"""CPU tests of the ASCII PCD reader's token parser and header parser (csrc/pcd_parse.cuh built for the host by
tests/hostmath/pcd_parse_host.cpp) against glibc's strtof and the restated PCL 1.12 reader
(tests/hostmath/pcd_reader_ref.hpp: getline, split, `istringstream >> float` in the classic locale, iequals("nan"), atof).
The exhaustive sweep of all 2^32 patterns through %.8g and %.9g is tests/diag/sweep_pcd_parse.py."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "pcd_parse_host.cpp")


def build_pcd_parse_host(out_dir):
    """Compiles the host shim (OpenMP for the bulk comparisons) into out_dir and loads it."""
    lib = os.path.join(out_dir, "libpcd_parse_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    L = C.CDLL(lib)
    L.pp_parse.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_uint32)]
    L.pp_ref_value.argtypes = [C.c_char_p, C.POINTER(C.c_uint32)]
    L.pp_strtof.argtypes = [C.c_char_p, C.POINTER(C.c_uint32)]
    for name in ("pp_check_range", "pp_check_list", "pp_check_strings"):
        getattr(L, name).restype = C.c_longlong
    L.pp_check_range.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.c_void_p]
    L.pp_check_list.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    L.pp_check_strings.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    L.pp_parse_line.argtypes = [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
    L.pp_parse_header.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.pp_read_ascii_ref.argtypes = [C.c_char_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    return L


def reference_read(L, path):
    """The restated PCL reader on a DATA ascii file: (status, (N, 4) float32 x y z intensity, bad line)."""
    n, bad = C.c_size_t(0), C.c_size_t(0)
    p = os.fsencode(str(path))
    rc = L.pp_read_ascii_ref(p, None, 0, C.byref(n), C.byref(bad))
    out = np.zeros((n.value, 4), dtype=np.float32)
    if n.value:
        L.pp_read_ascii_ref(p, out.ctypes.data, n.value, C.byref(n), C.byref(bad))
    return rc, out, bad.value


@pytest.fixture(scope="module")
def pp(tmp_path_factory):
    return build_pcd_parse_host(str(tmp_path_factory.mktemp("pcd_parse_host")))


def ours(pp, s):
    b = C.c_uint32(0)
    ok = pp.pp_parse(s, len(s), C.byref(b))
    return b.value if ok else None


def ref(pp, s):
    b = C.c_uint32(0)
    pp.pp_ref_value(s, C.byref(b))
    return b.value


def strtof(pp, s):
    b = C.c_uint32(0)
    n = pp.pp_strtof(s, C.byref(b))
    assert n == len(s), s
    return b.value


def check_strings(pp, strings):
    buf = b"\0".join(strings) + b"\0"
    first = C.c_uint64(0)
    bad = pp.pp_check_strings(buf, len(strings), C.byref(first))
    assert bad == 0, f"{bad} mismatches, first {strings[first.value][:80]!r}"


def check_list(pp, bits, prec):
    bits = np.ascontiguousarray(bits, dtype=np.uint32)
    first = C.c_uint32(0)
    bad = pp.pp_check_list(bits.ctypes.data, len(bits), prec, C.byref(first))
    assert bad == 0, f"%.{prec}g: {bad} mismatches, first 0x{first.value:08x}"


def f32_halfway(b):
    """The exact value halfway between the positive float with bits b and the next one up."""
    lo = Fraction(float(np.uint32(b).view(np.float32)))
    hi = Fraction(float(np.uint32(b + 1).view(np.float32))) if b + 1 < 0x7f800000 else Fraction(2) ** 128
    return (lo + hi) / 2


def decimal_digits(q, n):
    """(digits, exponent) with q = 0.digits * 10^exponent, digits exact when len <= n (q a dyadic rational)"""
    e = 0
    while q >= 1:
        q /= 10
        e += 1
    while q < Fraction(1, 10):
        q *= 10
        e -= 1
    d = []
    for _ in range(n):
        q *= 10
        k = int(q)
        d.append(k)
        q -= k
        if q == 0:
            break
    return d, e, q == 0


def test_bit_patterns_through_g8_and_g9(pp):
    rng = np.random.default_rng(31)
    rand = rng.integers(0, 1 << 32, size=4_000_000, dtype=np.uint64).astype(np.uint32)
    strided = (np.arange(1 << 22, dtype=np.uint64) * 1021 + 7).astype(np.uint32)
    for prec in (8, 9):
        check_list(pp, rand, prec)
        check_list(pp, strided, prec)


@pytest.mark.parametrize("lo", [0x00000000, 0x00800000, 0x7f000000, 0x80000000, 0x80800000, 0xff000000])
def test_whole_binades_at_the_subnormal_boundary_and_flt_max(pp, lo):
    first = C.c_uint32(0)
    for prec in (8, 9):
        bad = pp.pp_check_range(lo, lo + 0x7fffff, prec, C.byref(first))
        assert bad == 0, f"%.{prec}g: {bad} mismatches in binade 0x{lo:08x}, first 0x{first.value:08x}"


def test_overflow_threshold(pp):
    T = Fraction(2) ** 128 - Fraction(2) ** 103  # FLT_MAX + half an ulp
    d, e, exact = decimal_digits(T, 60)
    assert exact
    s = "0." + "".join(map(str, d)) + f"e{e}"
    near = [s.encode(), b"3.4028235e38", b"3.40282357e38", b"3.4028236e38", b"1e39", b"-1e39", b"9.99e38", b"340282356779733661637539395458142568448",
            b"340282356779733661637539395458142568447", b"340282356779733661637539395458142568447.99999999999999"]
    check_strings(pp, near)
    assert ours(pp, near[0]) == 0x7f800000 and ours(pp, near[-1]) == 0x7f7fffff


def halfway_strings(b, ndig):
    """digit strings of the halfway point above the float with bits b, exact and moved by +-1 in digit `ndig`"""
    d, e, exact = decimal_digits(f32_halfway(b), 200)
    assert exact
    d = d + [0] * (ndig - len(d))
    out = []
    base = int("".join(map(str, d[:ndig])))
    for delta in (-1, 0, 1):
        digs = str(base + delta).rjust(ndig, "0")
        out.append(f"0.{digs}e{e}".encode())
    return out


@pytest.mark.parametrize("ndig", [40, 800])
def test_exact_halfway_points_decided_by_a_late_digit(pp, ndig):
    rng = np.random.default_rng(ndig)
    bits = list(rng.integers(1, 0x7f7fffff, size=300, dtype=np.uint64)) + [0, 1, 2, 0x007ffffe, 0x007fffff, 0x00800000, 0x3f800000,
                                                                            0x3f800001, 0x4b7fffff, 0x7f7ffffe]
    strings = []
    for b in bits:
        b = int(b)
        if len(decimal_digits(f32_halfway(b), 200)[0]) > ndig:
            continue
        strings += halfway_strings(b, ndig)
    assert len(strings) > 100
    check_strings(pp, strings)
    strings += [b"-" + s for s in strings]
    check_strings(pp, strings)
    # the exact tie goes to the even neighbour, one below goes down, one above goes up
    lo, tie, hi = halfway_strings(0x3f800001, ndig)  # 1 + 2^-23 is odd: the tie rounds up
    assert (ours(pp, lo), ours(pp, tie), ours(pp, hi)) == (0x3f800001, 0x3f800002, 0x3f800002)
    lo, tie, hi = halfway_strings(0x3f800000, ndig)  # 1.0 is even: the tie stays
    assert (ours(pp, lo), ours(pp, tie), ours(pp, hi)) == (0x3f800000, 0x3f800000, 0x3f800001)


def test_long_mantissas_leading_zeros_and_long_exponents(pp):
    rng = np.random.default_rng(5)
    strings = []
    for n in (50, 100, 200, 400, 800):
        for _ in range(40):
            digits = "".join(map(str, rng.integers(0, 10, size=n)))
            point = int(rng.integers(0, n))
            e = int(rng.integers(-60, 40))
            strings.append(f"{digits[:point]}.{digits[point:]}e{e}".encode())
            strings.append(f"-{digits}e{e - n}".encode())
    strings += [b"0." + b"0" * k + b"1e" + b"%+d" % (k + 1 + s) for k in (10, 49, 300, 5000) for s in (-50, 0, 38)]
    strings += [b"0.000000000000000000000000000000000000000000000000001e+50", b"1e0000000000000000000000001",
                b"1e-0000000000000000000000045", b"1e+0000000000000000000000039", b"123e-9999999999999999999999999",
                b"123e+9999999999999999999999999", b"0e9999999999999999999999999", b"000000000000000000000000000000001.5",
                b"7.006492321624085354618647916449580656401309709382578858785341419448955413429303e-46",
                b"7.006492321624085354618647916449580656401309709382578858785341419448955413429304e-46",
                b"1.4012984643e-45", b"1.17549435e-38", b"1.1754942e-38"]
    check_strings(pp, strings)
    assert ours(pp, b"0.000000000000000000000000000000000000000000000000001e+50") == 0x3dcccccd  # 0.1f


def test_signs_zero_nan_and_inf_spellings_match_pcl(pp):
    ok = [b"-0", b"+0", b"0", b"-0.0e5", b"+1.5", b"-.5", b".5", b"5.", b"1E3", b"1e+3", b"1e-3", b"00.00100"]
    for s in ok:
        assert ours(pp, s) == ref(pp, s) == strtof(pp, s), s
    assert ours(pp, b"-0") == 0x80000000
    spellings = [b"nan", b"NaN", b"NAN", b"nAn", b"+nan", b"-nan", b"-NaN", b"+NAN", b"inf", b"INF", b"-inf", b"+Inf", b"infinity",
                 b"-Infinity", b"+INFINITY"]
    for s in spellings:
        assert ours(pp, s) == ref(pp, s), (s, hex(ours(pp, s)), hex(ref(pp, s)))
    assert ours(pp, b"nan") == 0x7fc00000 and ours(pp, b"-nan") == 0xffc00000 and ours(pp, b"-inf") == 0xff800000


def test_tokens_outside_the_grammar_are_refused(pp):
    for s in (b"", b"+", b"-", b".", b"e5", b"1e", b"1e+", b"1.5abc", b"0x1p3", b"1..2", b"1.2.3", b"--1", b"nan(1)", b"infin",
              b"1,5", b"1 ", b" 1", b"inff", b"1e5.0"):
        assert ours(pp, s) is None, s


def _line(pp, text, layout):
    lay = np.array(layout, dtype=np.int32)
    out = np.zeros(4, dtype=np.float32)
    used = C.c_int(0)
    st = pp.pp_parse_line(text, len(text), lay.ctypes.data, out.ctypes.data, C.byref(used))
    return st, out, used.value


def test_line_tokenizer(pp):
    st, v, used = _line(pp, b"1 2 3 4\nrest", [4, 0, 1, 2, 3])
    assert st == 0 and used == 7 and list(v) == [1, 2, 3, 4]
    st, v, _ = _line(pp, b"  \t1\t\t2 \r 3   4 \r", [4, 0, 1, 2, 3])
    assert st == 0 and list(v) == [1, 2, 3, 4]
    st, v, _ = _line(pp, b"9 8 7 6 5 4", [6, 5, 3, 1, -1])  # x = token 5, y = 3, z = 1, no intensity
    assert st == 0 and list(v) == [4, 6, 8, 0]
    assert _line(pp, b"1 2 3", [4, 0, 1, 2, 3])[0] == 1
    assert _line(pp, b"1 2 3 4 5", [4, 0, 1, 2, 3])[0] == 1
    assert _line(pp, b"   ", [4, 0, 1, 2, 3])[0] == 1
    assert _line(pp, b"1 2 x 4", [4, 0, 1, 2, 3])[0] == 2
    assert _line(pp, b"1 2 3 4 junk", [5, 0, 1, 2, 3])[0] == 0  # a skipped field is only counted
    assert _line(pp, b"1 2 x", [4, 0, 1, 2, 3])[0] == 1  # the count is checked first


HDR = "VERSION 0.7\nFIELDS {f}\nSIZE {s}\nTYPE {t}\nCOUNT {c}\nWIDTH {w}\nHEIGHT {h}\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA {d}\n"


def _header(pp, text):
    out = np.zeros(13, dtype=np.int64)
    err = C.create_string_buffer(256)
    ok = pp.pp_parse_header(text, len(text), out.ctypes.data, err, 256)
    return (out, None) if ok else (None, err.value.decode())


def hdr(f="x y z intensity", s="4 4 4 4", t="F F F F", c="1 1 1 1", w=10, h=1, n=10, d="ascii"):
    return HDR.format(f=f, s=s, t=t, c=c, w=w, h=h, n=n, d=d).encode()


def test_header_accepts(pp):
    v, _ = _header(pp, b"# .PCD v0.7 - Point Cloud Data file format\n" + hdr())
    assert list(v[:12]) == [10, 0, 4, 0, 1, 2, 3, 16, 0, 4, 8, 12]
    v, _ = _header(pp, hdr(f="rgb x normal y z intensity ring", s="4 4 4 4 4 4 2", t="U F F F F F U", c="1 1 3 1 1 1 1", d="binary"))
    assert list(v[:12]) == [10, 1, 9, 1, 5, 6, 7, 34, 4, 20, 24, 28]
    v, _ = _header(pp, hdr(f="x y z", s="4 4 4", t="F F F", c="1 1 1", w=5, h=4, n=20))
    assert list(v[:7]) == [20, 0, 3, 0, 1, 2, -1]
    v, _ = _header(pp, b"FIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nPOINTS 3\n\nDATA ascii\n")  # COUNT and WIDTH absent
    assert list(v[:3]) == [3, 0, 3]
    v, _ = _header(pp, hdr(d="binary_compressed"))
    assert v[1] == 2  # recognised; the loader refuses it


@pytest.mark.parametrize("kw,why", [
    (dict(f="y z intensity", s="4 4 4", t="F F F", c="1 1 1"), "no field 'x'"),
    (dict(s="8 4 4 4"), "'x' must be"),
    (dict(t="F F F U"), "'intensity' must be"),
    (dict(c="1 2 1 1"), "'y' must be"),
    (dict(s="4 4 4"), "differ in length"),
    (dict(w=10, h=2, n=10), "WIDTH * HEIGHT"),
    (dict(d="xml"), "unknown storage"),
    (dict(s="4 4 3 4"), "bad SIZE"),
    (dict(n="-1"), "not an integer"),
    (dict(w=999999999999999999, h=999999999999999999, n=1), "WIDTH * HEIGHT"),
])
def test_header_refuses(pp, kw, why):
    v, err = _header(pp, hdr(**kw))
    assert v is None and why in err, err
    assert _header(pp, b"FIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nPOINTS 3\n")[1] == "no DATA line"


def test_reference_reader(pp, tmp_path):
    body = b"1 2 3 4\n\n5\t6\t7\t8\r\n 9 10 11 nan\n-inf 1e-45 -0 NaN\nextra line past POINTS\n"
    path = tmp_path / "a.pcd"
    path.write_bytes(hdr(w=4, n=4) + body)
    rc, cloud, _ = reference_read(pp, path)
    assert rc == 0 and cloud.shape == (4, 4)
    assert cloud.view(np.uint32)[3].tolist() == [0xff800000, 1, 0x80000000, 0x7fc00000]
    path.write_bytes(hdr(w=5, n=5) + body[:-len(b"extra line past POINTS\n")])
    assert reference_read(pp, path)[0] == -3
    path.write_bytes(hdr(w=2, n=2) + b"1 2 3 4\n1 2 3\n")
    rc, _, line = reference_read(pp, path)
    assert rc == -2 and line == 12
