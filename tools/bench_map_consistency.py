"""Measures the map consistency of the scan-matcher session (b200sm_build_map_consistency): K19a bounds, the K19b cell
passes and the K19c neighbourhood kernel on the device, and the entropy heat map written by
b200sm_save_map_consistency_pcd_ascii, on imported synthetic submaps (tools/bench_occupancy.py's submaps on its 100 m ring).

    python tools/bench_map_consistency.py --out DIR [--submaps 100 1000] [--points 32768] [--radii 0.3 0.5] [--repeats 5]

For each (submap count, radius): the device time of each kernel from torch.profiler in a run of its own; then, with the
profiler off, the wall time of the build and of the save (host clock around calls that end synchronised; median of
--repeats), and the neighbour candidates tested and neighbours accepted per second of build wall time, from the counts the
build returns. The CPU comparison is the serial host compile of the same header (tests/hostmath/consistency_host.cpp,
g++ -O2 -ffp-contract=off, built into a temporary directory) on the same submaps, run at the smaller submap count only,
with every layer and the info checked equal. The card's name, power limit and maximum SM clock, and the SM clock after
the timed loop, are read in the same run. Writes one JSON line per case to DIR/bench_map_consistency.jsonl (and prints
it). Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_localize import sm_clock_now, summary  # noqa: E402
from bench_occupancy import base_clouds, poses_on_ring  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("mc_bounds_kernel", "mc_cells_kernel", "mc_chunks_kernel", "mc_neighbour_kernel", "sm_voxel_list_kernel")


def kernel_ms(prof):
    ms, count = {k: 0.0 for k in KERNELS}, {k: 0 for k in KERNELS}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k in KERNELS:
            if k in e.name:
                ms[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                count[k] += 1
    return ms, count


def run(n_sub, radius, args, clouds, host):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = ScanMatcher()
    for k in range(n_sub):
        g.importSubmap(subs[k], poses[k], float(k))
    prm = dict(radius=radius)
    line = {"submaps": n_sub, "points_per_submap": args.points, **prm}
    info = g.buildMapConsistency(**prm)  # warm-up: allocations, module load
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildMapConsistency(**prm)
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
            g.buildMapConsistency(**prm)
            build.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            g.saveMapConsistencyPcd(os.path.join(tmp, "h.pcd"))
            save.append(1e3 * (time.perf_counter() - t0))
        line["pcd_bytes"] = os.path.getsize(os.path.join(tmp, "h.pcd"))
    line["wall_ms_build"] = summary(build)
    line["wall_ms_save"] = summary(save)
    med = float(np.median(build)) / 1e3
    line["candidates_per_s_build_wall"] = info["n_candidates"] / med
    line["neighbors_per_s_build_wall"] = info["n_neighbors"] / med
    kn = ms["mc_neighbour_kernel"] / 1e3
    if kn > 0:
        line["candidates_per_s_k19c"] = info["n_candidates"] / kn
    if host is not None and n_sub == min(args.submaps):
        t0 = time.perf_counter()
        want = host.build(list(zip(subs, poses)), prm)
        line["host_compile_serial_ms"] = 1e3 * (time.perf_counter() - t0)
        got = g.mapConsistency()
        line["host_compile_equal"] = bool(isinstance(want, dict) and all(
            np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)) for k in ("n", "h", "plane_var"))
            and all(want["info"][k] == (tuple(info[k]) if k.startswith("box") else info[k])
                    for k in ("box_origin", "box_dims", "n_candidates", "n_neighbors", "n_valid", "sum_h_q", "sum_plane_q")))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_map_consistency.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--radii", type=float, nargs="+", default=[0.3, 0.5])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the serial host compile")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_consistency needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(16, args.points)
    os.makedirs(args.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        host = None
        if not args.no_host:
            from test_map_consistency_cpu import compile_host

            host = compile_host(tmp)
        for n_sub in args.submaps:
            for r in args.radii:
                line = {"tool": "bench_map_consistency", **gpu_info(), **run(n_sub, r, args, clouds, host),
                        "sm_clock_after_loop": sm_clock_now()}
                text = json.dumps(line)
                with open(os.path.join(args.out, "bench_map_consistency.jsonl"), "a") as f:
                    f.write(text + "\n")
                print(text, flush=True)


if __name__ == "__main__":
    main()
