"""Measures the frontend frame (b200sm_receive_cloud) at the BASELINE frame size (32 x 1875 rays, the node's parameters)
with the sensor-to-robot transform off and on, and the device time of the upload's unpack pass both ways.

    python tools/bench_frontend_frame.py --out DIR [--frames 40] [--warmup 6]

Two sessions follow the same drive, one frame each in turn: one is given the LiDAR-frame scans as they are, the other the
same scans with the mapping_car mount (1.2 m forward, 2.0 m up, plus a rotation) set by setSensorTransform. Frame times
are wall clock around receiveCloud, which ends in a synchronisation (the pose comes back to the host). The unpack kernel
times are the device durations torch.profiler records, in a separate profiled pass. The host comparison is the same
transform in numpy float32 on one frame: a stand-in for tf2::doTransform, which is not available here, not a measurement
of it. Writes one JSON line to DIR/bench_frontend_frame.jsonl (and prints it); the card's name and power limit are read in
the same run. Needs a CUDA device; there is no CPU fallback.
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

NODE = dict(ndt_resolution=5.0, vg_size_for_input=0.2, vg_size_for_map=0.1, trans_for_mapupdate=1.5, num_targeted_cloud=10)
MOUNT_POS = (1.2, 0.0, 2.0)  # scanmatcher/launch/mapping_car.launch.py:27-28


def spread(v):
    v = sorted(v)
    q = lambda f: v[min(len(v) - 1, int(f * (len(v) - 1) + 0.5))]  # noqa: E731
    return {"median": statistics.median(v), "p10": q(0.1), "p90": q(0.9), "min": v[0], "max": v[-1], "n": len(v)}


def transform_f32_numpy(cloud, T):
    out = cloud.copy()
    x, y, z = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    for r in range(3):
        out[:, r] = ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_frontend_frame.jsonl")
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=6, help="leading frames left out of the frame-time statistics")
    ap.add_argument("--profiled", type=int, default=10, help="frames per session in the profiled pass")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("bench_frontend_frame needs a CUDA device (there is no CPU fallback)")
    from bench_pose_adjust import gpu_info

    from lidarslam_ros2_b200 import synth
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    mount_quat = np.array([0.009, -0.02, 0.174, 0.9845])
    mount_quat /= np.linalg.norm(mount_quat)
    workers = max(1, min(32, (os.cpu_count() or 1)))
    n_total = args.frames + args.profiled
    frames = [np.ascontiguousarray(s) for s, _ in synth.drive_stream(n_total, rings=32, azimuths=1875, step=0.5, workers=workers)]
    off, on = ScanMatcher(**NODE), ScanMatcher(**NODE)
    on.setSensorTransform(MOUNT_POS, mount_quat)

    t = {"off": [], "on": []}
    for k in range(args.frames):
        for name, s in (("off", off), ("on", on)) if k % 2 == 0 else (("on", on), ("off", off)):
            t0 = time.perf_counter()
            s.receiveCloud(frames[k])
            dt = time.perf_counter() - t0
            if k >= args.warmup:
                t[name].append(1e3 * dt)

    with tempfile.TemporaryDirectory() as tmp:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for k in range(args.frames, n_total):
                off.receiveCloud(frames[k])
                on.receiveCloud(frames[k])
        trace = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            events = json.load(f).get("traceEvents", [])
    unpack = [e for e in events if e.get("cat") == "kernel" and "unpack_points_bounds_kernel" in e.get("name", "")]
    k_off = [e["dur"] for e in unpack if "<false>" in e["name"]]
    k_on = [e["dur"] for e in unpack if "<true>" in e["name"]]

    x, y, z, w = mount_quat
    T = np.eye(4)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    T[:3, 3] = MOUNT_POS
    T = T.astype(np.float32)
    host = []
    for _ in range(50):
        t0 = time.perf_counter()
        transform_f32_numpy(frames[0], T)
        host.append(1e3 * (time.perf_counter() - t0))

    n_pts = [len(f) for f in frames]
    bytes_per_point = frames[0].strides[0] + 16  # the raw record read, one float4 written
    med_pts = statistics.median(n_pts)
    kern = {}
    for name, v in (("off", k_off), ("on", k_on)):
        us = statistics.median(v) if v else None
        kern[name] = {"us_median": us, "us_min": min(v) if v else None, "samples": len(v),
                      "bytes_per_s_at_median_frame": bytes_per_point * med_pts / (us * 1e-6) if us else None}
    line = {
        "tool": "bench_frontend_frame", **gpu_info(), "rays": [32, 1875], "points_per_frame_median": med_pts,
        "node_params": NODE, "mount": {"position": list(MOUNT_POS), "quat_xyzw": mount_quat.tolist()},
        "frames_timed_per_side": len(t["off"]),
        "receive_cloud_ms": {"transform_off": spread(t["off"]), "transform_on": spread(t["on"])},
        "unpack_kernel": {"transform_off": kern["off"], "transform_on": kern["on"], "algorithmic_bytes_per_point": bytes_per_point},
        "host_numpy_f32_transform_ms": spread(host),
        "host_note": "numpy float32 on one frame, a stand-in for tf2::doTransform (not measured here)",
    }
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_frontend_frame.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
