"""Every one of the 2^32 float bit patterns printed with "%.8g" and with "%.9g" of the widened float, then read back by
the host build of csrc/pcd_parse.cuh and by glibc's strtof: the bits must agree (NaN patterns print as "nan" / "-nan").
CPU only; compiled with OpenMP.

    python tests/diag/sweep_pcd_parse.py [--blocks 256]

Prints the mismatch count per precision (expected 0), the first mismatching pattern if any, and the wall time.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "..", "hostmath", "pcd_parse_host.cpp")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--blocks", type=int, default=256, help="progress lines: the 2^32 patterns in this many blocks")
    args = ap.parse_args()
    bad_any = 0
    with tempfile.TemporaryDirectory() as tmp:
        lib = os.path.join(tmp, "libpcd_parse_omp.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
        L = C.CDLL(lib)
        L.pp_check_range.restype = C.c_longlong
        L.pp_check_range.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.c_void_p]
        step = (1 << 32) // args.blocks
        t_all = time.perf_counter()
        for prec in (8, 9):
            total, first = 0, None
            t0 = time.perf_counter()
            for b in range(args.blocks):
                f = C.c_uint32(0)
                bad = L.pp_check_range(b * step, (b + 1) * step - 1, prec, C.byref(f))
                if bad and first is None:
                    first = f.value
                total += bad
                if (b + 1) % max(1, args.blocks // 8) == 0:
                    print(f"  %.{prec}g: {b + 1}/{args.blocks} blocks, {total} mismatches, {time.perf_counter() - t0:.0f} s",
                          flush=True)
            print(f"%.{prec}g patterns 4294967296 mismatches {total} first {None if first is None else hex(first)} "
                  f"wall_s {time.perf_counter() - t0:.1f}", flush=True)
            bad_any += total
        print(f"total wall_s {time.perf_counter() - t_all:.1f} threads {os.environ.get('OMP_NUM_THREADS', os.cpu_count())}")
    sys.exit(1 if bad_any else 0)


if __name__ == "__main__":
    main()
