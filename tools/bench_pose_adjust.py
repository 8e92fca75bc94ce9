"""Measures the backend pose adjustment of the session: the map-assembly kernel (b200sm_assemble_map), its read-back to
pinned and pageable host memory, and the host pose-graph solve (b200sm_pose_adjust), on synthetic imported submaps.

    python tools/bench_pose_adjust.py --out DIR [--configs 1000x32768,100x32768]

Writes one JSON line to DIR/bench_pose_adjust.jsonl (and prints it). Kernel and copy times are the device durations
torch.profiler records for the assembly kernel and the device-to-host copies; host times are wall clock around calls that
end in a synchronisation. The CPU comparison is numpy (a per-submap float transform + concatenate), not PCL.
The card's name and power limit are read in the same run. Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12  # H100 SXM data sheet, HBM3 bytes/s
BYTES_PER_POINT = 32  # one float4 read, one float4 written


def transform_f32_numpy(cloud, T):
    """((m0 x + m1 y) + m2 z) + m3 in float32, intensity copied: the association of pcl::transformPointCloud(Matrix4f)."""
    T = T.astype(np.float32)
    out = cloud.copy()
    x, y, z = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    for r in range(3):
        out[:, r] = ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
    return out


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in q.split(","))
        return {"gpu": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:  # the numbers below still stand, but without their card they are not reported as measured
        return {"gpu": None, "power_limit": None, "error": str(e)}


def drive(n, rng):
    """Submap poses along a winding drive with drift, and 20 loop edges (true relative pose) between submaps > 50 apart."""
    from lidarslam_ros2_b200 import synth

    gt, dr = [np.eye(4)], [np.eye(4)]
    for i in range(n - 1):
        M = synth.pose_matrix((2.0, 0, 0), (0, 0, 0.3 * np.sin(i / 20)))
        gt.append(gt[-1] @ M)
        dr.append(dr[-1] @ M @ synth.pose_matrix((0.01, 0.02, 0.002), (0.0005, -0.0005, 0.003)))
    loops = [(0, n - 1)]
    while len(loops) < 20:
        a, b = sorted(int(v) for v in rng.integers(0, n, size=2))
        if b - a > min(50, n // 3):
            loops.append((a, b))
    return dr, [(a, b, np.linalg.inv(gt[a]) @ gt[b]) for a, b in loops]


def run_config(n_sub, n_pts, reps, rng):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher()
    poses, loops = drive(n_sub, rng)
    clouds = []
    for i in range(n_sub):
        c = np.concatenate([rng.uniform(-60, 60, size=(n_pts, 3)), rng.uniform(0, 255, size=(n_pts, 1))], axis=1).astype(np.float32)
        g.importSubmap(c, poses[i], 2.0 * i)
        clouds.append(c)
    total = n_sub * n_pts

    t_adjust = []
    for _ in range(3):
        t0 = time.perf_counter()
        adjusted, res = g.poseAdjust(loops, num_adjacent_pose_cnstraints=5, max_iterations=10)
        t_adjust.append(time.perf_counter() - t0)

    L, h = g._lib, g._h
    import ctypes as C

    Pc = np.ascontiguousarray(adjusted.transpose(0, 2, 1))
    pinned = torch.empty((total, 4), dtype=torch.float32, pin_memory=True)
    pageable = np.empty((total, 4), dtype=np.float32)
    n = C.c_size_t(0)

    def call(ptr):
        rc = L.b200sm_assemble_map(h, Pc.ctypes.data, ptr, total, C.byref(n), None)
        if rc != 0:
            raise RuntimeError(f"b200sm_assemble_map: {rc}")

    for _ in range(3):  # warm-up: table and map buffers allocated, pages of the host buffers touched
        call(pinned.data_ptr())
        call(pageable.ctypes.data)
    wall = {"pinned": [], "pageable": []}
    for _ in range(reps):
        for name, ptr in (("pinned", pinned.data_ptr()), ("pageable", pageable.ctypes.data)):
            t0 = time.perf_counter()
            call(ptr)
            wall[name].append(time.perf_counter() - t0)

    with tempfile.TemporaryDirectory() as tmp:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call(pinned.data_ptr())
                call(pageable.ctypes.data)
        trace = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            events = json.load(f).get("traceEvents", [])
    kern = [e["dur"] for e in events if e.get("cat") == "kernel" and "assemble_map_kernel" in e.get("name", "")]
    d2h_pinned = [e["dur"] for e in events if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "") and "Pinned" in e.get("name", "")]
    d2h_pageable = [e["dur"] for e in events if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "") and "Pageable" in e.get("name", "")]

    t0 = time.perf_counter()
    ref = np.concatenate([transform_f32_numpy(clouds[i], adjusted[i]) for i in range(n_sub)], axis=0)
    t_numpy = time.perf_counter() - t0
    bitwise = bool(np.array_equal(pinned.numpy().view(np.uint32), ref.view(np.uint32)) and
                   np.array_equal(pageable.view(np.uint32), ref.view(np.uint32)))

    med = lambda v: statistics.median(v) if v else None  # noqa: E731
    k_us = med(kern)
    bytes_ = BYTES_PER_POINT * total
    out = {
        "submaps": n_sub, "points_per_submap": n_pts, "points": total, "bitwise_equal_numpy": bitwise,
        "assemble_kernel_us_median": k_us, "assemble_kernel_us_min": min(kern) if kern else None, "kernel_samples": len(kern),
        "assemble_bytes": bytes_,
        "assemble_bytes_per_s": bytes_ / (k_us * 1e-6) if k_us else None,
        "assemble_share_of_datasheet_hbm": bytes_ / (k_us * 1e-6) / HBM_PEAK if k_us else None,
        "d2h_pinned_us_median": med(d2h_pinned), "d2h_pageable_us_median": med(d2h_pageable),
        "call_wall_ms_pinned_median": 1e3 * med(wall["pinned"]), "call_wall_ms_pageable_median": 1e3 * med(wall["pageable"]),
        "pose_adjust_host_ms_median": 1e3 * med(t_adjust), "pose_adjust_vertices": res["n_vertices"],
        "pose_adjust_edges": res["n_edges"], "pose_adjust_iterations": res["iterations"], "pose_adjust_trials": res["trials"],
        "pose_adjust_chi2": [res["chi2_initial"], res["chi2_final"]],
        "numpy_transform_concat_ms": 1e3 * t_numpy,
    }
    del g
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_pose_adjust.jsonl")
    ap.add_argument("--configs", default="1000x32768,100x32768", help="comma-separated SUBMAPSxPOINTS")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_pose_adjust needs a CUDA device (there is no CPU fallback)")
    rng = np.random.default_rng(2024)
    line = {"tool": "bench_pose_adjust", **gpu_info(), "hbm_datasheet_bytes_per_s": HBM_PEAK, "configs": []}
    for cfg in args.configs.split(","):
        n_sub, n_pts = (int(v) for v in cfg.lower().split("x"))
        line["configs"].append(run_config(n_sub, n_pts, args.reps, rng))
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_pose_adjust.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
