"""Measures savePCDFileASCII on the device (b200sm_save_map_pcd_ascii) for a pose-adjusted map of imported synthetic
submaps: the encode kernels' device time and output rate, the device-to-host copies of the text, and the wall time of
the whole call writing a local temporary file (deleted afterwards).

    python tools/bench_pcd_save.py --out DIR [--configs 100x32768,1000x32768]

Writes one JSON line to DIR/bench_pcd_save.jsonl (and prints it). Device times are the durations torch.profiler records
for the kernels and copies of one call; the wall time is a host clock around calls that return after the file is
closed. The CPU comparison (the restated PCL writer on the same map) is tests/diag/diag_pcd_save.py. The card's name and
power limit are read in the same run. Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_pose_adjust import drive, gpu_info  # noqa: E402

ENCODE_KERNELS = ("pcd_measure_kernel", "pcd_encode_kernel", "scan_local_kernel", "scan_tile_sums_kernel", "scan_apply_kernel")


def build_session(n_sub, n_pts, seed=2024):
    """Imported submaps along bench_pose_adjust's drifted drive and the adjusted poses of its loop edges."""
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    rng = np.random.default_rng(seed)
    g = ScanMatcher()
    poses, loops = drive(n_sub, rng)
    for i in range(n_sub):
        c = np.concatenate([rng.uniform(-60, 60, size=(n_pts, 3)), rng.uniform(0, 255, size=(n_pts, 1))], axis=1).astype(np.float32)
        g.importSubmap(c, poses[i], 2.0 * i)
    adjusted, _ = g.poseAdjust(loops, num_adjacent_pose_cnstraints=5, max_iterations=10)
    return g, adjusted


def run_config(n_sub, n_pts, reps, tmp):
    from torch.profiler import ProfilerActivity, profile

    g, adjusted = build_session(n_sub, n_pts)
    path = os.path.join(tmp, "map.pcd")
    points, size = g.saveMapPCDASCII(path, adjusted)  # warm-up: map, text and pinned staging buffers allocated
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        g.saveMapPCDASCII(path, adjusted)
        wall.append(time.perf_counter() - t0)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        g.saveMapPCDASCII(path, adjusted)
    trace = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f).get("traceEvents", [])
    os.remove(trace)
    os.remove(path)
    kern = {k: sum(e["dur"] for e in events if e.get("cat") == "kernel" and k in e.get("name", "")) for k in ENCODE_KERNELS}
    assemble = sum(e["dur"] for e in events if e.get("cat") == "kernel" and "assemble_map_kernel" in e.get("name", ""))
    d2h = [e for e in events if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]
    d2h_text = [e["dur"] for e in d2h if e.get("args", {}).get("bytes", 0) > (1 << 20)]
    encode_us = sum(kern.values())
    del g
    return {
        "submaps": n_sub, "points_per_submap": n_pts, "points": points, "file_bytes": size,
        "encode_kernels_us": encode_us, "encode_kernels_us_by_name": kern,
        "encode_output_bytes_per_s": size / (encode_us * 1e-6) if encode_us else None,
        "assemble_kernel_us": assemble,
        "d2h_text_us": sum(d2h_text), "d2h_text_copies": len(d2h_text),
        "d2h_text_bytes_per_s": size / (sum(d2h_text) * 1e-6) if d2h_text else None,
        "save_wall_ms_median": 1e3 * statistics.median(wall), "save_wall_ms_min": 1e3 * min(wall), "save_wall_samples": len(wall),
        "file_bytes_per_s_wall": size / statistics.median(wall),
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_pcd_save.jsonl")
    ap.add_argument("--configs", default="100x32768,1000x32768", help="comma-separated SUBMAPSxPOINTS")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_pcd_save needs a CUDA device (there is no CPU fallback)")
    line = {"tool": "bench_pcd_save", **gpu_info(), "configs": []}
    with tempfile.TemporaryDirectory() as tmp:
        for cfg in args.configs.split(","):
            n_sub, n_pts = (int(v) for v in cfg.lower().split("x"))
            line["configs"].append(run_config(n_sub, n_pts, args.reps, tmp))
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_pcd_save.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
