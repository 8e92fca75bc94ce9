"""Measures the occupancy grid of the scan-matcher session (b200sm_build_occupancy_grid): free space ray-cast from every
submap's sensor origin on the device (K14a bounds, K14b walks, K14c fold, K14d classify) and the map_server pair written
by b200sm_save_occupancy_map, on imported synthetic submaps.

    python tools/bench_occupancy.py --out DIR [--submaps 100 1000] [--points 32768] [--resolutions 0.1 0.05] [--repeats 5]

For each (submap count, resolution): the device time of each K14 kernel from torch.profiler in a run of its own (kernels
og_bounds_kernel, og_walk_kernel, og_fold_kernel, og_classify_kernel); then, with the profiler off, the wall time of the
build and of the save (host clock around calls that end synchronised; median of --repeats), and the algorithmic counts:
points read (twice: bounds and walks), cells visited by the walks, bitmap and count traffic. The CPU comparison is the
serial host compile of the same header (tests/hostmath/occupancy_host.cpp, g++ -O2 -ffp-contract=off, built into a
temporary directory) on the same submaps — a stand-in for a CPU ray caster, not OctoMap — run at the smaller submap count
only, with its grid checked equal. The card's name, power limit and maximum SM clock, and the SM clock after the timed
loop, are read in the same run. Writes one JSON line per case to DIR/bench_occupancy.jsonl (and prints it). Needs a CUDA
device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
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
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("og_bounds_kernel", "og_walk_kernel", "og_fold_kernel", "og_classify_kernel")
SENSOR_HEIGHT = 1.9
RING_RADIUS = 100.0


def base_clouds(n_base, n_points, seed=11):
    """Structured synthetic submaps (sensor frame): ground 1.9 m below the sensor, walls and boxes out to 90 m."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_base):
        p = np.empty((n_points, 4), dtype=np.float32)
        r = rng.uniform(1.0, 90.0, size=n_points)
        a = rng.uniform(0, 2 * np.pi, size=n_points)
        p[:, 0], p[:, 1] = r * np.cos(a), r * np.sin(a)
        wall = np.abs(p[:, 1]) > rng.uniform(10, 20)
        p[:, 2] = np.where(wall, rng.uniform(-SENSOR_HEIGHT, 8.0, size=n_points), -SENSOR_HEIGHT + rng.normal(0, 0.02, n_points))
        p[:, 3] = rng.uniform(0, 255, size=n_points)
        out.append(p)
    return out


def poses_on_ring(n_sub):
    """Submaps evenly spaced on a 100 m circle, heading along it, sensor 1.9 m above the map's ground."""
    out = []
    for k in range(n_sub):
        th = 2 * math.pi * k / n_sub
        M = np.eye(4)
        M[:2, :2] = [[-math.sin(th), -math.cos(th)], [math.cos(th), -math.sin(th)]]
        M[:3, 3] = (RING_RADIUS * math.cos(th), RING_RADIUS * math.sin(th), SENSOR_HEIGHT)
        out.append(M)
    return out


def kernel_ms(prof):
    """Device time per kernel name (ms, summed over the launches in the profile) and launch counts."""
    ms, count = {k: 0.0 for k in KERNELS}, {k: 0 for k in KERNELS}
    for e in prof.events():
        for k in KERNELS:
            if e.name.endswith(k) or (k + "(") in e.name or e.name.split("(")[0].endswith("::" + k):
                if e.device_type.name == "CUDA":
                    ms[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                    count[k] += 1
    return ms, count


def host_compile(tmp):
    src = os.path.join(ROOT, "tests", "hostmath", "occupancy_host.cpp")
    lib = os.path.join(tmp, "libocc_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.ogh_build.argtypes = [vp, vp, vp, vp, C.c_int]
    L.ogh_info.argtypes = [vp, vp]
    L.ogh_get.argtypes = [vp, vp, vp, vp]
    return L


def walked_cells(clouds, poses, resolution, z_min, z_max):
    """Cells the walks visit (a float64 estimate from the clipped segments' 4-connected lengths, for the byte count)."""
    total = 0.0
    for c, P in zip(clouds, poses):
        e = c[:, :3].astype(np.float64) @ P[:3, :3].T + P[:3, 3]
        o = P[:3, 3]
        dz = e[:, 2] - o[2]
        with np.errstate(divide="ignore", invalid="ignore"):
            t_lo = np.where(dz != 0, (z_min - o[2]) / dz, -np.inf)
            t_hi = np.where(dz != 0, (z_max - o[2]) / dz, np.inf)
        t0 = np.clip(np.minimum(t_lo, t_hi), 0, 1)
        t1 = np.clip(np.maximum(t_lo, t_hi), 0, 1)
        span = np.where(t1 > t0, t1 - t0, 0.0)
        total += float(((np.abs(e[:, 0] - o[0]) + np.abs(e[:, 1] - o[1])) * span / resolution + 1).sum())
    return total


def run(n_sub, resolution, args, clouds, host):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = ScanMatcher()
    for k in range(n_sub):
        g.importSubmap(subs[k], poses[k], float(k))
    prm = dict(resolution=resolution, z_min=0.2, z_max=2.0, max_range=100.0)
    line = {"submaps": n_sub, "points_per_submap": args.points, **prm}
    info = g.buildOccupancyGrid(**prm)  # warm-up: allocations, module load
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildOccupancyGrid(**prm)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    for k in KERNELS:
        line[f"{k}_ms"] = ms[k]
        line[f"{k}_launches"] = cnt[k]
    line["kernels_ms"] = sum(ms.values())
    line.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in info.items()})
    cells = info["width"] * info["height"]
    visits = walked_cells(subs, poses, resolution, prm["z_min"], prm["z_max"])
    line["walked_cells_estimate"] = visits
    # algorithmic bytes: points read by K14a and K14b (16 B each, twice), bitmaps zeroed + folded (2 bits per window cell
    # written by memset and read by K14c), grid counts zeroed, folded (atomics) and read by K14d, values and image written
    line["algorithmic_bytes"] = 2 * 16 * n_sub * args.points + 10 * cells
    build, save = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.buildOccupancyGrid(**prm)
            build.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            g.saveOccupancyMap(os.path.join(tmp, "map.pgm"), os.path.join(tmp, "map.yaml"))
            save.append(1e3 * (time.perf_counter() - t0))
        line["pgm_bytes"] = os.path.getsize(os.path.join(tmp, "map.pgm"))
    line["wall_ms_build"] = summary(build)
    line["wall_ms_save"] = summary(save)
    if host is not None and n_sub == min(args.submaps):
        pts = np.zeros((n_sub * args.points, 4), dtype=np.float32)
        for k in range(n_sub):
            pts[k * args.points:(k + 1) * args.points] = subs[k]
        off = np.arange(n_sub + 1, dtype=np.int64) * args.points
        P = np.ascontiguousarray(np.array([M.T.reshape(16) for M in poses]))
        par = np.array([resolution, prm["z_min"], prm["z_max"], prm["max_range"], 0, 0, 0, 0.65, 0.25], dtype=np.float64)
        t0 = time.perf_counter()
        rc = host.ogh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, n_sub)
        line["host_compile_serial_ms"] = 1e3 * (time.perf_counter() - t0)
        hits = np.zeros(cells, dtype=np.uint32)
        frees = np.zeros(cells, dtype=np.uint32)
        host.ogh_get(None, hits.ctypes.data, frees.ctypes.data, None)
        got = g.occupancyGrid()
        line["host_compile_equal"] = bool(rc == 0 and np.array_equal(hits, got["hits"].reshape(-1)) and
                                          np.array_equal(frees, got["frees"].reshape(-1)))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_occupancy.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--resolutions", type=float, nargs="+", default=[0.1, 0.05])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the serial host compile")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_occupancy needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(16, args.points)
    os.makedirs(args.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        host = None if args.no_host else host_compile(tmp)
        for n_sub in args.submaps:
            for res in args.resolutions:
                line = {"tool": "bench_occupancy", **gpu_info(), **run(n_sub, res, args, clouds, host), "sm_clock_after_loop": sm_clock_now()}
                text = json.dumps(line)
                with open(os.path.join(args.out, "bench_occupancy.jsonl"), "a") as f:
                    f.write(text + "\n")
                print(text, flush=True)


if __name__ == "__main__":
    main()
