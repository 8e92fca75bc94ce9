"""Measures the OctoMap of the scan-matcher session (b200sm_build_octomap): the static map's front half (K15a-K15e), the
freed walks into a box-wide bitmap (K22a), the state pyramid (K22b, K22c per level), the pre-order offsets (K22d per
level) and the .bt bytes (K22e), and the save of the file, on imported synthetic submaps.

    python tools/bench_octomap.py --out DIR [--submaps 100 1000] [--points 32768] [--resolution 0.2] [--repeats 5]
                                  [--host-submaps 10]

For each submap count: the device time of each kernel from torch.profiler in a run of its own; then, with the profiler
off, the wall time of the build and of the save (host clock around calls that end synchronised; median of --repeats).
The CPU comparison is the serial host compile of the same header (tests/hostmath/octomap_host.cpp, a pointer-based octree
as OctoMap builds one, g++ -O2 -ffp-contract=off, built into a temporary directory) on the first --host-submaps submaps
only (its tree of one node per known voxel does not fit in memory at the full sizes), against the device build of the
same submaps, with the states and bytes checked equal. The card's name, power limit and maximum SM clock, and the SM
clock after the timed loop, are read in the same run. Writes one JSON line per case to DIR/bench_octomap.jsonl (and
prints it). Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_localize import sm_clock_now, summary  # noqa: E402
from bench_occupancy import base_clouds, poses_on_ring  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("sm_bounds_kernel", "sm_mark_kernel", "sm_walk_kernel", "sm_fold_kernel", "sm_classify_kernel", "om_free_kernel",
           "om_leaf_kernel", "om_reduce_kernel", "om_offset_kernel", "om_write_kernel")


def kernel_ms(prof):
    """Device time per kernel name (ms, summed over the launches in the profile) and launch counts."""
    ms, count = {k: 0.0 for k in KERNELS}, {k: 0 for k in KERNELS}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k in KERNELS:
            if k in e.name:
                ms[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                count[k] += 1
    return ms, count


def host_compile(tmp):
    src = os.path.join(ROOT, "tests", "hostmath", "octomap_host.cpp")
    lib = os.path.join(tmp, "liboctomap_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.omh_build.argtypes = [vp, vp, vp, vp, C.c_int]
    L.omh_info.argtypes = [vp]
    L.omh_result.argtypes = [vp, vp]
    return L


def session(subs, poses):
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher()
    for k, (c, P) in enumerate(zip(subs, poses)):
        g.importSubmap(c, P, float(k))
    return g


def run(n_sub, args, clouds):
    import torch
    from torch.profiler import ProfilerActivity, profile

    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = session(subs, poses)
    prm = dict(resolution=args.resolution, max_range=100.0)
    line = {"submaps": n_sub, "points_per_submap": args.points, **prm, "ray_fraction": 0.85, "min_frees": 2, "dynamic_thresh": 0.4}
    info = g.buildOctoMap(**prm)  # warm-up: allocations, module load
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildOctoMap(**prm)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    for k in KERNELS:
        line[f"{k}_ms"] = ms[k]
        line[f"{k}_launches"] = cnt[k]
    line["kernels_ms"] = sum(ms.values())
    line.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in info.items()})
    build, save = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.buildOctoMap(**prm)
            build.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            g.saveOctoMapBt(os.path.join(tmp, "map.bt"))
            save.append(1e3 * (time.perf_counter() - t0))
        line["bt_bytes"] = os.path.getsize(os.path.join(tmp, "map.bt"))
    line["wall_ms_build"] = summary(build)
    line["wall_ms_save"] = summary(save)
    return line


def run_host(args, clouds, host):
    """The serial host compile and the device build of the first --host-submaps submaps."""
    import torch

    n_sub = args.host_submaps
    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = session(subs, poses)
    prm = dict(resolution=args.resolution, max_range=100.0)
    g.buildOctoMap(**prm)
    dev = []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        info = g.buildOctoMap(**prm)
        dev.append(1e3 * (time.perf_counter() - t0))
    pts = np.ascontiguousarray(np.concatenate(subs).astype(np.float32))
    off = np.arange(n_sub + 1, dtype=np.int64) * args.points
    P = np.ascontiguousarray(np.array([M.T.reshape(16) for M in poses]))
    par = np.array([args.resolution, prm["max_range"], 0, 0, 0, 0.85, 2, 0.4], dtype=np.float64)
    t0 = time.perf_counter()
    rc = host.omh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, n_sub)
    host_ms = 1e3 * (time.perf_counter() - t0)
    hinfo = np.zeros(16, dtype=np.int64)
    host.omh_info(hinfo.ctypes.data)
    states = np.zeros(int(np.prod(hinfo[3:6])), dtype=np.uint8)
    data = np.zeros(int(hinfo[15]), dtype=np.uint8)
    host.omh_result(states.ctypes.data, data.ctypes.data)
    equal = rc == 0 and np.array_equal(states, g.octoMapStates()["states"].reshape(-1)) and data.tobytes() == g.octoMapBytes()
    return {"host_submaps": n_sub, "host_compile_serial_ms": host_ms, "device_wall_ms_build_same_submaps": summary(dev),
            "host_tree_size": int(hinfo[14]), "device_tree_size": info["tree_size"], "host_compile_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_octomap.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--resolution", type=float, default=0.2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--host-submaps", type=int, default=10, help="submaps of the host compile comparison; 0 skips it")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_octomap needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(16, args.points)
    os.makedirs(args.out, exist_ok=True)

    def emit(line):
        text = json.dumps({"tool": "bench_octomap", **gpu_info(), **line, "sm_clock_after_loop": sm_clock_now()})
        with open(os.path.join(args.out, "bench_octomap.jsonl"), "a") as f:
            f.write(text + "\n")
        print(text, flush=True)

    for n_sub in args.submaps:
        emit(run(n_sub, args, clouds))
    if args.host_submaps > 0:
        with tempfile.TemporaryDirectory() as tmp:
            emit(run_host(args, clouds, host_compile(tmp)))


if __name__ == "__main__":
    main()
