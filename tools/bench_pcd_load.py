"""Measures loadPCDFile on the device (b200reg_load_pcd, b200reg_set_input_target_pcd) on the map.pcd that
b200sm_save_map_pcd_ascii writes for bench_pcd_save's pose-adjusted maps, in a local temporary directory (deleted
afterwards): the parse kernels' device time and the host-to-device copies of the text, the wall time of both calls
(median of --reps with a warm page cache), and the restated single-threaded PCL reader (tests/hostmath/pcd_reader_ref.hpp)
on the same file, whose cloud must equal the device's bit for bit.

    python tools/bench_pcd_load.py --out DIR [--configs 100x32768,1000x32768]

Writes one JSON line to DIR/bench_pcd_load.jsonl (and prints it). Device times are the durations torch.profiler records
for the kernels and copies of --profiled b200reg_load_pcd calls, per call. The kernel time is null unless the trace holds
one of each kernel per piece (pieces counted by pcd_advance_kernel launches); the trace can drop a copy record, so the
copy time of the whole text is its size at the rate of the copies recorded, with both counts reported. The reference reader is timed over one pass into a buffer sized from the header. The
card's name and power limit are read in the same run. Needs a CUDA device; there is no CPU fallback.
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
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
sys.path.insert(0, HERE)

from bench_pcd_save import build_session  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

PIECE = 64 << 20  # B200REG_PCD_LOAD_PIECE_BYTES

PARSE_KERNELS = ("pcd_line_count_kernel", "pcd_parse_kernel", "pcd_advance_kernel", "scan_local_kernel",
                 "scan_tile_sums_kernel", "scan_apply_kernel")


def run_config(n_sub, n_pts, reps, profiled, tmp, pp):
    import ctypes as C

    import lidarslam_ros2_b200 as m
    from torch.profiler import ProfilerActivity, profile

    g, adjusted = build_session(n_sub, n_pts)
    path = os.path.join(tmp, "map.pcd")
    points, size = g.saveMapPCDASCII(path, adjusted)
    del g
    cloud = m.read_pcd(path)  # warm-up: page cache, pinned pieces and device buffers
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        m.read_pcd(path)
        wall.append(time.perf_counter() - t0)
    ndt = m.NormalDistributionsTransform(device=0)
    ndt.setResolution(2.0)
    ndt.setInputTargetPCD(path)
    wall_target = []
    for _ in range(reps):
        t0 = time.perf_counter()
        ndt.setInputTargetPCD(path)
        wall_target.append(time.perf_counter() - t0)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(profiled):
            m.read_pcd(path)
    trace = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f).get("traceEvents", [])
    os.remove(trace)
    kern_ev = {k: [e["dur"] for e in events if e.get("cat") == "kernel" and k in e.get("name", "")] for k in PARSE_KERNELS}
    pieces = len(kern_ev["pcd_advance_kernel"]) // profiled
    h2d_ev = [e for e in events if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", "")
              and e.get("args", {}).get("bytes", 0) > 64]  # the pieces, not the 16-byte counter reset
    complete = (pieces >= (size - 400) // PIECE
                and all(len(kern_ev[k]) == pieces * profiled for k in ("pcd_line_count_kernel", "pcd_parse_kernel", "pcd_advance_kernel")))
    kern = {k: sum(v) / profiled for k, v in kern_ev.items()}
    parse_us = sum(kern.values()) if complete else None
    # the trace can drop a copy record: the copy time of the whole text is taken at the rate of the copies it recorded
    h2d_bytes, h2d_dur = sum(e["args"]["bytes"] for e in h2d_ev), sum(e["dur"] for e in h2d_ev)
    h2d_rate = h2d_bytes / (h2d_dur * 1e-6) if h2d_dur else None
    h2d_us = size / h2d_rate * 1e6 if h2d_rate else None
    ref_cloud = np.zeros((points, 4), dtype=np.float32)
    n_ref, bad = C.c_size_t(0), C.c_size_t(0)
    t0 = time.perf_counter()  # one pass of the restated reader, into a buffer sized from the header
    rc = pp.pp_read_ascii_ref(os.fsencode(path), ref_cloud.ctypes.data, points, C.byref(n_ref), C.byref(bad))
    ref_s = time.perf_counter() - t0
    equal = rc == 0 and n_ref.value == points and np.array_equal(cloud.view(np.uint32), ref_cloud.view(np.uint32))
    os.remove(path)
    return {
        "submaps": n_sub, "points_per_submap": n_pts, "points": points, "file_bytes": size,
        "pieces": pieces, "profiled_calls": profiled, "trace_complete": bool(complete),
        "parse_kernels_us": parse_us, "parse_kernels_us_by_name": kern if complete else None,
        "parse_input_bytes_per_s": size / (parse_us * 1e-6) if parse_us else None,
        "h2d_text_us": h2d_us, "h2d_copies_recorded": len(h2d_ev), "h2d_copies_issued": pieces * profiled,
        "h2d_text_bytes_per_s": h2d_rate,
        "load_wall_ms_median": 1e3 * statistics.median(wall), "load_wall_ms_min": 1e3 * min(wall), "load_wall_samples": len(wall),
        "file_bytes_per_s_wall": size / statistics.median(wall),
        "set_input_target_pcd_wall_ms_median": 1e3 * statistics.median(wall_target),
        "reference_reader_s": ref_s, "reference_reader_status": rc, "bitwise_equal_to_reference": bool(equal),
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_pcd_load.jsonl")
    ap.add_argument("--configs", default="100x32768,1000x32768", help="comma-separated SUBMAPSxPOINTS")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profiled", type=int, default=3, help="calls traced by torch.profiler for the device times")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_pcd_load needs a CUDA device (there is no CPU fallback)")
    from test_pcd_parse_cpu import build_pcd_parse_host

    line = {"tool": "bench_pcd_load", **gpu_info(), "configs": []}
    with tempfile.TemporaryDirectory() as tmp:
        pp = build_pcd_parse_host(tmp)
        for cfg in args.configs.split(","):
            n_sub, n_pts = (int(v) for v in cfg.lower().split("x"))
            line["configs"].append(run_config(n_sub, n_pts, args.reps, args.profiled, tmp, pp))
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_pcd_load.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
