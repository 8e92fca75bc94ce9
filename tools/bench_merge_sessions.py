"""Measures merging a second session into the scan-matcher session (b200sm_merge_session): the cross-session Scan Context
scores of every pair (K16, merge_scores_kernel), the per-row candidate selection (merge_select_kernel), and whole merges,
on imported synthetic submaps (tools/bench_place_recognition.py's clouds) at 20 x 60 bins.

    python tools/bench_merge_sessions.py --out DIR [--submaps 1000 5000] [--points 8000] [--repeats 3]

For each n_A = n_B: the K16 and selection kernel times from torch.profiler in a run of its own, set against n_B launches of
K13b (scan_context_search_kernel) over the same n_A candidates (one K13b launch is profiled, averaged over the repeats and
multiplied by n_B: the place search scores one query per launch); the achieved double-precision operation rate of K16
from a count computed from the shapes (a multiply and an add per pair, shift, column and ring; the per-column quotients and
square roots are not counted); and, with the profiler off, the wall time of whole merges (host clock around a call that
ends synchronised, into a freshly loaded dst each time) with max_verifications 16 and 64. The card's name, power limit and
maximum SM clock, and the SM clock after the timed loop, are read in the same run. Writes one JSON line per size to
DIR/bench_merge_sessions.jsonl (and prints it). Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_localize import sm_clock_now, summary  # noqa: E402
from bench_place_recognition import base_clouds, import_submaps  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("merge_scores_kernel", "merge_select_kernel", "scan_context_search_kernel")
R_, S_ = 20, 60


def kernel_ms(prof):
    ms, count = {k: 0.0 for k in KERNELS}, {k: 0 for k in KERNELS}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k in KERNELS:
            if k in e.name:
                ms[k] += (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
                count[k] += 1
    return ms, count


def sessions(n, clouds):
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    a, b = ScanMatcher(), ScanMatcher()
    import_submaps(a, clouds, n)
    import_submaps(b, clouds, n, start=7)  # the same clouds in another order, at other poses
    a.scanContext(0)  # descriptors built before anything is timed
    b.scanContext(0)
    return a, b


def run(n, args, clouds):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher, backend_registration

    reg = backend_registration("NDT", ndt_resolution=2.0)
    line = {"n_a": n, "n_b": n, "points_per_submap": args.points, "descriptor_bins": [R_, S_]}
    a, b = sessions(n, clouds)
    # the kernels, profiled: a merge with no candidate runs K16 and the selection only
    a.mergeSession(b, reg, sc_threshold=-1.0)  # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.repeats):
            _, _, res = a.mergeSession(b, reg, sc_threshold=-1.0)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    line["query_tile"] = res["query_tile"]
    line["k16_ms"] = ms["merge_scores_kernel"] / max(cnt["merge_scores_kernel"], 1)
    line["select_ms"] = ms["merge_select_kernel"] / max(cnt["merge_select_kernel"], 1)
    flop = 2.0 * n * n * S_ * S_ * R_
    line["k16_flop"] = flop
    line["k16_flop_per_s"] = flop / (line["k16_ms"] * 1e-3) if line["k16_ms"] > 0 else None
    # K13b over the same n_A candidates, one query per launch
    p = ScanMatcher()
    import_submaps(p, clouds, n)
    import_submaps(p, clouds, 1, start=n)  # the query, newest: every submap behind it is a candidate
    place = dict(voxel_leaf_size=0.5, distance_loop_closure=-1.0, sc_threshold=-1.0, top_k=1, capacity=0)
    p.searchLoopPlace(reg, **place)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.repeats):
            p.searchLoopPlace(reg, **place)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    k13b = ms["scan_context_search_kernel"] / max(cnt["scan_context_search_kernel"], 1)
    assert cnt["scan_context_search_kernel"] == args.repeats
    line["k13b_candidates"] = n
    line["k13b_one_launch_ms"] = k13b
    line["k13b_n_b_launches_ms"] = k13b * n
    # whole merges, profiler off, each into a freshly loaded dst (a successful merge appends src to it)
    for maxv in (16, 64):
        walls, last = [], None
        for _ in range(args.repeats):
            a, b = sessions(n, clouds)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows, _, last = a.mergeSession(b, reg, max_verifications=maxv)
            walls.append(1e3 * (time.perf_counter() - t0))
        line[f"merge_wall_ms_max_verifications_{maxv}"] = summary(walls)
        line[f"verified_{maxv}"] = last["verified"]
        line[f"merged_{maxv}"] = bool(last["merged"])
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_merge_sessions.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[1000, 5000])
    ap.add_argument("--points", type=int, default=8000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_merge_sessions needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(64, args.points)
    os.makedirs(args.out, exist_ok=True)
    for n in args.submaps:
        line = {"tool": "bench_merge_sessions", **gpu_info(), **run(n, args, clouds), "sm_clock_after_loop": sm_clock_now()}
        text = json.dumps(line)
        with open(os.path.join(args.out, "bench_merge_sessions.jsonl"), "a") as f:
            f.write(text + "\n")
        print(text, flush=True)


if __name__ == "__main__":
    main()
