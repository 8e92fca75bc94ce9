"""Measures the map changes of the scan-matcher session (b200sm_build_map_changes): the static map's front half with the
counts kept per epoch (K15a bounds, K15b rank index, K15c walks, K15d fold), then K20a classify, K20b label and count and
K20c write, on imported synthetic submaps.

    python tools/bench_map_changes.py --out DIR [--submaps 500] [--points 32768] [--resolution 0.2] [--repeats 5]

Two segments of --submaps submaps each: the first is bench_static_map's workload (bench_occupancy's clouds on its ring of
poses); the second is a perturbed copy (poses moved by a few centimetres and milliradians, a box of points cut out of
every cloud and a new box's surface added elsewhere), split with split_submap. The device time of each kernel comes from
torch.profiler in a run of its own; then, with the profiler off, the wall time of the build (host clock around a call that
ends synchronised; median of --repeats) and, as the baseline, of buildStaticMap on the same session in the same run. The
card's name, power limit and maximum SM clock, and the SM clock after the timed loop, are read in the same run. Writes
one JSON line to DIR/bench_map_changes.jsonl (and prints it). Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_localize import sm_clock_now, summary  # noqa: E402
from bench_occupancy import base_clouds, poses_on_ring  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("sm_bounds_kernel", "sm_mark_kernel", "sm_walk_kernel", "sm_fold_kernel", "ch_classify_kernel", "ch_label_kernel",
           "ch_write_kernel")


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


def day2(cloud, k, rng):
    """A perturbed copy of a day-1 cloud: the points inside one box removed, and as many on the faces of a new box."""
    c = cloud.copy()
    lo = np.array([4.0 + (k % 5), -3.0 - (k % 3), -1.0])
    gone = np.all((c[:, :3] >= lo) & (c[:, :3] <= lo + 2.0), axis=1)
    n_new = max(int(gone.sum()), 256)
    keep = c[~gone]
    centre = np.array([-6.0 - (k % 4), 5.0 + (k % 2), 0.0])
    f = rng.integers(0, 3, size=n_new)
    u = rng.uniform(-1.0, 1.0, size=(n_new, 3))
    u[np.arange(n_new), f] = np.where(rng.uniform(size=n_new) < 0.5, -1.0, 1.0)  # on a face of the 2 m box
    new = np.zeros((n_new, 4), dtype=np.float32)
    new[:, :3] = centre + u
    new[:, 3] = 100.0
    out = np.concatenate([keep, new])[:len(cloud)]
    if len(out) < len(cloud):
        out = np.concatenate([out, keep[:len(cloud) - len(out)]])
    return np.ascontiguousarray(out, dtype=np.float32)


def run(args):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200 import synth
    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    n = args.submaps
    clouds = base_clouds(16, args.points)
    rng = np.random.default_rng(11)
    poses = poses_on_ring(n)
    g = ScanMatcher()
    for k in range(n):
        g.importSubmap(clouds[k % len(clouds)], poses[k], float(k))
    for k in range(n):
        d = synth.pose_matrix(tuple(rng.normal(0.0, 0.03, size=3)), tuple(rng.normal(0.0, 0.002, size=3)))
        g.importSubmap(day2(clouds[k % len(clouds)], k, rng), poses[k] @ d, float(n + k))
    prm = dict(resolution=args.resolution, max_range=100.0)
    line = {"submaps": 2 * n, "split_submap": n, "points_per_submap": args.points, **prm, "ray_fraction": 0.85, "min_frees": 2,
            "dynamic_thresh": 0.4}
    info = g.buildMapChanges(split_submap=n, **prm)  # warm-up: allocations, module load
    g.buildStaticMap(**prm)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildMapChanges(split_submap=n, **prm)
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    for k in KERNELS:
        line[f"{k}_ms"] = ms[k]
        line[f"{k}_launches"] = cnt[k]
    line["kernels_ms"] = sum(ms.values())
    line.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in info.items()})
    changes, static = [], []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g.buildMapChanges(split_submap=n, **prm)
        changes.append(1e3 * (time.perf_counter() - t0))
        t0 = time.perf_counter()
        g.buildStaticMap(**prm)
        static.append(1e3 * (time.perf_counter() - t0))
    line["wall_ms_build_map_changes"] = summary(changes)
    line["wall_ms_build_static_map"] = summary(static)
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_map_changes.jsonl")
    ap.add_argument("--submaps", type=int, default=500, help="submaps per segment")
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--resolution", type=float, default=0.2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_changes needs a CUDA device (there is no CPU fallback)")
    os.makedirs(args.out, exist_ok=True)
    line = {"tool": "bench_map_changes", **gpu_info(), **run(args), "sm_clock_after_loop": sm_clock_now()}
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_map_changes.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text, flush=True)


if __name__ == "__main__":
    main()
