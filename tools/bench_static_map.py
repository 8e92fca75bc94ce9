"""Measures the static map of the scan-matcher session (b200sm_build_static_map): a 3D free-space ray-cast from every
submap's sensor origin on the device (K15a bounds, K15b rank index, K15c walks, K15d fold, K15e classify, K15f / K15g
compaction) and the PCD save of the result, on imported synthetic submaps.

    python tools/bench_static_map.py --out DIR [--submaps 100 1000] [--points 32768] [--resolution 0.2] [--repeats 5]

For each submap count: the device time of each K15 kernel from torch.profiler in a run of its own; then, with the
profiler off, the wall time of the build and of the save (host clock around calls that end synchronised; median of
--repeats), and the voxels the walks visit (a float64 estimate from the shortened segments' 6-connected lengths) per
second of build. The CPU comparison is the serial host compile of the same header (tests/hostmath/static_map_host.cpp,
g++ -O2 -ffp-contract=off, built into a temporary directory) on the same submaps — a stand-in for a CPU remover, not
Peopleremover's code — run at the smaller submap count only, with its static map checked equal. The card's name, power
limit and maximum SM clock, and the SM clock after the timed loop, are read in the same run. Writes one JSON line per case
to DIR/bench_static_map.jsonl (and prints it). Needs a CUDA device; there is no CPU fallback.
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

KERNELS = ("sm_bounds_kernel", "sm_mark_kernel", "sm_walk_kernel", "sm_fold_kernel", "sm_classify_kernel", "sm_compact_kernel")


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
    src = os.path.join(ROOT, "tests", "hostmath", "static_map_host.cpp")
    lib = os.path.join(tmp, "libstatic_map_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.smh_build.argtypes = [vp, vp, vp, vp, C.c_int]
    L.smh_info.argtypes = [vp]
    L.smh_static.argtypes = [vp, vp]
    return L


def walked_voxels(clouds, poses, resolution, fraction):
    """Voxels the walks visit: the 6-connected length of each shortened segment, plus one."""
    total = 0.0
    for c, P in zip(clouds, poses):
        e = c[:, :3].astype(np.float64) @ P[:3, :3].T + P[:3, 3]
        d = np.abs(e - P[:3, 3]) * fraction / resolution
        total += float(d.sum() + len(d))
    return total


def run(n_sub, args, clouds, host):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = ScanMatcher()
    for k in range(n_sub):
        g.importSubmap(subs[k], poses[k], float(k))
    prm = dict(resolution=args.resolution, max_range=100.0)
    line = {"submaps": n_sub, "points_per_submap": args.points, **prm, "ray_fraction": 0.85, "min_frees": 2, "dynamic_thresh": 0.4}
    info = g.buildStaticMap(**prm)  # warm-up: allocations, module load
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildStaticMap(**prm)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    for k in KERNELS:
        line[f"{k}_ms"] = ms[k]
        line[f"{k}_launches"] = cnt[k]
    line["kernels_ms"] = sum(ms.values())
    line.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in info.items()})
    visits = walked_voxels(subs, poses, args.resolution, 0.85)
    line["walked_voxels_estimate"] = visits
    build, save = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.buildStaticMap(**prm)
            build.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            g.saveStaticMapPcd(os.path.join(tmp, "static.pcd"))
            save.append(1e3 * (time.perf_counter() - t0))
        line["pcd_bytes"] = os.path.getsize(os.path.join(tmp, "static.pcd"))
    line["wall_ms_build"] = summary(build)
    line["wall_ms_save"] = summary(save)
    line["walked_voxels_per_s"] = visits / (line["wall_ms_build"]["median"] / 1e3) if isinstance(line["wall_ms_build"], dict) else None
    if ms["sm_walk_kernel"] > 0:
        line["walked_voxels_per_s_walk_kernel"] = visits / (ms["sm_walk_kernel"] / 1e3)
    if host is not None and n_sub == min(args.submaps):
        pts = np.zeros((n_sub * args.points, 4), dtype=np.float32)
        for k in range(n_sub):
            pts[k * args.points:(k + 1) * args.points] = subs[k]
        off = np.arange(n_sub + 1, dtype=np.int64) * args.points
        P = np.ascontiguousarray(np.array([M.T.reshape(16) for M in poses]))
        par = np.array([args.resolution, prm["max_range"], 0, 0, 0, 0.85, 2, 0.4], dtype=np.float64)
        t0 = time.perf_counter()
        rc = host.smh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, n_sub)
        line["host_compile_serial_ms"] = 1e3 * (time.perf_counter() - t0)
        hinfo = np.zeros(12, dtype=np.int64)
        host.smh_info(hinfo.ctypes.data)
        hs = np.zeros((max(1, int(hinfo[11])), 4), dtype=np.float32)
        host.smh_static(hs.ctypes.data, None)
        got, _ = g.staticMap()
        line["host_compile_equal"] = bool(rc == 0 and np.array_equal(hs[:int(hinfo[11])].view(np.uint32), got.view(np.uint32)))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_static_map.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--resolution", type=float, default=0.2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the serial host compile")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_static_map needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(16, args.points)
    os.makedirs(args.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        host = None if args.no_host else host_compile(tmp)
        for n_sub in args.submaps:
            line = {"tool": "bench_static_map", **gpu_info(), **run(n_sub, args, clouds, host), "sm_clock_after_loop": sm_clock_now()}
            text = json.dumps(line)
            with open(os.path.join(args.out, "bench_static_map.jsonl"), "a") as f:
                f.write(text + "\n")
            print(text, flush=True)


if __name__ == "__main__":
    main()
