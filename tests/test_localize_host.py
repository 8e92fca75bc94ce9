"""The prior-map cut on the CPU: the product's header csrc/map_cut.hpp (predicate, tile layout, rank of a kept row) compiled
with g++ and run as the two serial passes of tests/hostmath/map_cut_host.cpp, against map[mask] of the float64 replay
tests/localizeref.py bit for bit, on the fixtures the GPU tests use; and the same two passes under AddressSanitizer and
UBSan with an output buffer of exactly `total` rows."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import localizeref as L
import test_gpu_localize as G

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "map_cut_host.cpp")
HDR = os.path.join(HERE, "..", "lidarslam_ros2_b200", "csrc", "map_cut.hpp")
F32 = np.float32


@pytest.fixture(scope="module")
def mc():
    lib = os.path.join(HERE, "hostmath", "libmap_cut_host.so")
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in (SRC, HDR)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    lib = C.CDLL(lib)
    lib.mc_cut.restype = C.c_size_t
    lib.mc_cut.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_double, C.c_double, C.POINTER(C.POINTER(C.c_float)),
                           C.POINTER(C.c_int)]
    lib.mc_free.argtypes = [C.POINTER(C.c_float)]
    lib.mc_keep.argtypes = [C.c_size_t, C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_void_p]
    return lib


def _cut(mc, prior, cx, cy, r) -> np.ndarray:
    prior = np.ascontiguousarray(prior, dtype=F32).reshape(-1, 4)
    out, tripped = C.POINTER(C.c_float)(), C.c_int(0)
    total = mc.mc_cut(prior.ctypes.data, len(prior), cx, cy, r, C.byref(out), C.byref(tripped))
    assert tripped.value == 0
    got = np.ctypeslib.as_array(out, shape=(total, 4)).copy() if total else np.zeros((0, 4), dtype=F32)
    mc.mc_free(out)
    return got


def _check(mc, prior, cx, cy, r):
    want = prior[L.cut_mask(prior, cx, cy, r)]
    got = _cut(mc, prior, cx, cy, r)
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    return len(want)


def test_tile_size(mc):
    assert mc.mc_tile() == G.TILE


@pytest.mark.parametrize("n", (0,) + G.EDGE_SIZES)
def test_two_passes_equal_map_mask(mc, n):
    for pattern in G.PATTERNS:
        prior = G.edge_map(n, pattern) if n else np.zeros((0, 4), dtype=F32)
        kept = _check(mc, prior, *G.CENTRE, G.RADIUS)
        if n:
            assert kept == {"all": n, "none": 0, "last": 1}.get(pattern, kept)
            if pattern == "alternate":
                assert kept == (n + 1) // 2
            if pattern == "mixed" and n >= 31:
                assert 0 < kept < n


def test_at_the_radius(mc):
    prior = G.edge_map(G.TILE + 1, "mixed")
    for r in (G.RADIUS, math.nextafter(G.RADIUS, 0.0), math.nextafter(G.RADIUS, 10.0)):
        _check(mc, prior, *G.CENTRE, r)
        keep, xy = np.zeros(len(prior), dtype=np.uint8), np.ascontiguousarray(prior[:, :2])
        mc.mc_keep(len(prior), xy.ctypes.data, *G.CENTRE, r, keep.ctypes.data)
        assert np.array_equal(keep.astype(bool), L.cut_mask(prior, *G.CENTRE, r))
        assert bool(keep[3]) == bool(keep[5]) == (r >= G.RADIUS) and not keep[7] and keep[9]
        assert not keep[[11, 13, 17, 19]].any() and keep[15] == keep[21] == 1  # NaN / inf in x, y fail; in z they do not matter
    cx, cy, r = G.fused_case()
    _check(mc, prior, cx, cy, r)
    assert _cut(mc, prior, cx, cy, r)[:, 3].tolist().count(23.0) == 1  # the origin row is kept: the sum is not fused


def test_canyon_cut(mc):
    prior = G.canyon_map(40_000)
    kept = _check(mc, prior, G.X_START, 0.0, G.CROP)
    assert 0 < kept < len(prior)


def test_two_passes_under_sanitizers(tmp_path):
    """The executable form of the harness: every edge size and keep pattern with an output of exactly `total` rows, under
    -fsanitize=address,undefined."""
    exe = os.path.join(tmp_path, "map_cut_asan")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-DMAP_CUT_MAIN", "-x", "c++", SRC, "-o", exe]
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    build = subprocess.run(cmd, capture_output=True, text=True)
    if build.returncode != 0 and ("asan" in build.stderr or "ubsan" in build.stderr):
        pytest.skip("this toolchain has no sanitizer runtime")
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    assert run.returncode == 0 and "0 failures" in run.stdout, run.stdout + run.stderr
