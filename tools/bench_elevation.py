"""Measures the elevation / traversability map of the scan-matcher session (b200sm_build_elevation_map): occupancy's K14a
bounds, then K18a lowest points, K18b surface heights and K18c windows on the device, and the map_server pair written by
b200sm_save_traversability_map, on imported synthetic submaps (tools/bench_occupancy.py's submaps on its 100 m ring).

    python tools/bench_elevation.py --out DIR [--submaps 100 1000] [--points 32768] [--resolutions 0.2 0.1]
                                    [--windows 3 8] [--repeats 5]

For each (submap count, resolution, window_cells): the device time of each kernel from torch.profiler in a run of its own;
then, with the profiler off, the wall time of the build and of the save (host clock around calls that end synchronised;
median of --repeats), and the algorithmic counts: points read per pass (three passes), window cells visited by K18c and
bytes per cell kept. The CPU comparison is the serial host compile of the same header (tests/hostmath/elevation_host.cpp,
g++ -O2 -ffp-contract=off, built into a temporary directory) on the same submaps, run at the smaller submap count only,
with every layer checked equal. The card's name, power limit and maximum SM clock, and the SM clock after the timed loop,
are read in the same run. Writes one JSON line per case to DIR/bench_elevation.jsonl (and prints it). Needs a CUDA device;
there is no CPU fallback.
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

KERNELS = ("og_bounds_kernel", "el_lowest_kernel", "el_top_kernel", "el_window_kernel")
BYTES_PER_CELL = 34


def kernel_ms(prof):
    ms, count = {k: 0.0 for k in KERNELS}, {k: 0 for k in KERNELS}
    for e in prof.events():
        for k in KERNELS:
            if e.name.endswith(k) or (k + "(") in e.name or e.name.split("(")[0].endswith("::" + k):
                if e.device_type.name == "CUDA":
                    ms[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                    count[k] += 1
    return ms, count


def host_compile(tmp):
    src = os.path.join(ROOT, "tests", "hostmath", "elevation_host.cpp")
    lib = os.path.join(tmp, "libelev_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.elh_build.argtypes = [vp, vp, vp, vp, C.c_int]
    L.elh_get.argtypes = [vp] * 8
    return L


def run(n_sub, resolution, window, args, clouds, host):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = ScanMatcher()
    for k in range(n_sub):
        g.importSubmap(subs[k], poses[k], float(k))
    prm = dict(resolution=resolution, window_cells=window, min_cells=6)
    line = {"submaps": n_sub, "points_per_submap": args.points, **prm}
    info = g.buildElevationMap(**prm)  # warm-up: allocations, module load
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildElevationMap(**prm)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    for k in KERNELS:
        line[f"{k}_ms"] = ms[k]
        line[f"{k}_launches"] = cnt[k]
    line["kernels_ms"] = sum(ms.values())
    line.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in info.items()})
    cells = info["width"] * info["height"]
    line["points_read_per_pass"] = n_sub * args.points
    line["point_passes"] = 3
    line["window_cells_visited"] = 2 * (2 * window + 1) ** 2 * info["n_observed"]  # two passes per observed cell
    line["bytes_per_cell"] = BYTES_PER_CELL
    line["map_bytes"] = BYTES_PER_CELL * cells
    build, save = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.buildElevationMap(**prm)
            build.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            g.saveTraversabilityMap(os.path.join(tmp, "t.pgm"), os.path.join(tmp, "t.yaml"))
            save.append(1e3 * (time.perf_counter() - t0))
        line["pgm_bytes"] = os.path.getsize(os.path.join(tmp, "t.pgm"))
    line["wall_ms_build"] = summary(build)
    line["wall_ms_save"] = summary(save)
    if host is not None and n_sub == min(args.submaps):
        pts = np.zeros((n_sub * args.points, 4), dtype=np.float32)
        for k in range(n_sub):
            pts[k * args.points:(k + 1) * args.points] = subs[k]
        off = np.arange(n_sub + 1, dtype=np.int64) * args.points
        P = np.ascontiguousarray(np.array([M.T.reshape(16) for M in poses]))
        par = np.array([resolution, 100.0, 0, 0, 0, 2.0, 2, window, 6, 20.0, 0.15, 0.05, 0.65, 0.25], dtype=np.float64)
        t0 = time.perf_counter()
        rc = host.elh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, n_sub)
        line["host_compile_serial_ms"] = 1e3 * (time.perf_counter() - t0)
        got = g.elevationMap()
        want = {k: np.zeros(cells, dtype=got[k].dtype) for k in ("n", "h", "lo", "step", "tan_slope", "roughness", "value")}
        host.elh_get(*[want[k].ctypes.data for k in ("n", "h", "lo", "step", "tan_slope", "roughness", "value")], None)
        line["host_compile_equal"] = bool(rc == 0 and all(
            np.array_equal(want[k].view(np.uint8), np.ascontiguousarray(got[k]).reshape(-1).view(np.uint8)) for k in want))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_elevation.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--resolutions", type=float, nargs="+", default=[0.2, 0.1])
    ap.add_argument("--windows", type=int, nargs="+", default=[3, 8])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the serial host compile")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_elevation needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(16, args.points)
    os.makedirs(args.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        host = None if args.no_host else host_compile(tmp)
        for n_sub in args.submaps:
            for res in args.resolutions:
                for w in args.windows:
                    line = {"tool": "bench_elevation", **gpu_info(), **run(n_sub, res, w, args, clouds, host),
                            "sm_clock_after_loop": sm_clock_now()}
                    text = json.dumps(line)
                    with open(os.path.join(args.out, "bench_elevation.jsonl"), "a") as f:
                        f.write(text + "\n")
                    print(text, flush=True)


if __name__ == "__main__":
    main()
