"""Every one of the 2^32 float bit patterns through the host build of csrc/pcd_format.cuh against glibc's
snprintf("%.8g", (double)f) ("nan" for every NaN, as PCL's writeASCII prints it). CPU only; compiled with OpenMP.

    python tests/diag/sweep_pcd_format.py [--blocks 256]

Prints the mismatch count (expected 0), the first mismatching pattern if any, and the wall time.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "..", "hostmath", "pcd_host.cpp")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--blocks", type=int, default=256, help="progress lines: the 2^32 patterns in this many blocks")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        lib = os.path.join(tmp, "libpcd_host_omp.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
        L = C.CDLL(lib)
        L.ph_check_range.restype = C.c_longlong
        L.ph_check_range.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p]
        total, first = 0, None
        step = (1 << 32) // args.blocks
        t0 = time.perf_counter()
        for b in range(args.blocks):
            f = C.c_uint32(0)
            bad = L.ph_check_range(b * step, (b + 1) * step - 1, C.byref(f))
            if bad and first is None:
                first = f.value
            total += bad
            if (b + 1) % max(1, args.blocks // 16) == 0:
                print(f"  {b + 1}/{args.blocks} blocks, {total} mismatches, {time.perf_counter() - t0:.0f} s", flush=True)
        wall = time.perf_counter() - t0
    print(f"patterns 4294967296 mismatches {total} first {None if first is None else hex(first)} "
          f"wall_s {wall:.1f} threads {os.environ.get('OMP_NUM_THREADS', os.cpu_count())}")
    sys.exit(1 if total else 0)


if __name__ == "__main__":
    main()
