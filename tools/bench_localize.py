"""Measures localisation in a prior map (b200sm_localize_cloud) against the alternative it replaces, the whole map as the
registration target (b200reg_set_input_target_pcd + set_input_source + align), NDT, on a synthetic canyon map saved and
loaded through the PCD path, over a drive down the canyon.

    python tools/bench_localize.py --out DIR [--map-points 8000000] [--frames 48] [--resolutions 2.0,1.0]

Per resolution the two arms are alternated frame by frame in one run, both given the same filtered scan and the same guess
(the session's pose before the frame): (a) one b200sm_localize_cloud call, whose target is the cut around the pose;
(b) set_input_source + align on a handle whose target is the whole map. Reported per arm: wall time per frame (host clock
around calls that end synchronised), the solver kernel's device time solve_ms, index_in_smem and n_voxels (b200reg_stats),
as median and p10 / p90 over the frames after --warmup. The two cut kernels' device times come from a separate torch.profiler
pass over a session that re-cuts after every frame; their rate is (32 n_map + 16 n_cut) bytes over the sum of both. The map
(16 bytes per point) is larger than the H100's 50 MB L2 at the default size, so each cut streams it from HBM; nothing is
flushed between frames, so the solver meets its target as warm in L2 as a running localiser would. The card's name, power
limit and maximum SM clock, and the SM clock right after the timed loop, are read in the same run.
Writes one JSON line to DIR/bench_localize.jsonl (and prints it). Needs a CUDA device; there is no CPU fallback.
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

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_pose_adjust import gpu_info  # noqa: E402

X_START = -100.0
CUT_KERNELS = ("cut_count_kernel", "cut_write_kernel")
SCAN_KERNELS = ("scan_local_kernel", "scan_tile_sums_kernel", "scan_apply_kernel")
KW = dict(vg_size_for_input=0.4, use_min_max_filter=True, scan_min_range=1.0, scan_max_range=40.0)
CROP, RECROP = 60.0, 20.0  # crop_radius = scan_max_range + recrop_distance


def summary(v):
    v = sorted(float(x) for x in v)
    if not v:
        return None
    q = lambda p: v[min(len(v) - 1, int(round(p * (len(v) - 1))))]  # noqa: E731
    return {"median": statistics.median(v), "p10": q(0.1), "p90": q(0.9), "n": len(v)}


def sm_clock_now():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0].strip()
    except Exception:
        return None


def make_world(map_points, frames, step, workers, tmp):
    """The canyon map written through the session's PCD writer, and the drive's scans with the sensor's pose in the map."""
    from lidarslam_ros2_b200 import scanmatcher, synth

    scene = synth.make_scene()
    pts = synth.sample_map(scene, map_points, stream=9501)
    cloud = np.concatenate([pts, np.zeros((len(pts), 1), dtype=np.float32)], axis=1)
    g = scanmatcher.ScanMatcher(**KW)
    g.importSubmap(cloud, np.eye(4), 0.0)
    path = os.path.join(tmp, "map.pcd")
    n, size = g.saveMapPCDASCII(path)
    del g, cloud, pts
    M0 = synth.pose_matrix((X_START, 0.0, 0.0), (0.0, 0.0, 0.0))
    drive = [(scan, M0 @ T) for scan, T in synth.drive_stream(frames, rings=32, azimuths=938, step=step, x_start=X_START,
                                                               workers=workers)]
    return path, n, size, drive


def run_resolution(res, path, drive, warmup):
    import oracle.scanmatcher as osm
    from lidarslam_ros2_b200 import scanmatcher, synth

    a = scanmatcher.ScanMatcher(ndt_resolution=res, **KW)
    n_map = a.setPriorMapPCD(path)
    a.setLocalizationParams(CROP, RECROP)
    a.setInitialPose((X_START, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    whole = scanmatcher.ScanMatcher(ndt_resolution=res, **KW).registration
    t0 = time.perf_counter()
    whole.setInputTargetPCD(path)
    whole_build_s = time.perf_counter() - t0
    pose = np.array([X_START, 0, 0, 0, 0, 0, 1.0])
    rows = {"cut": [], "whole": []}
    err = {"cut": [], "whole": []}
    recuts = 0
    for k, (scan, T_gt) in enumerate(drive):
        guess = osm.pose_matrix(pose[:3], pose[3:]).astype(np.float32)
        t0 = time.perf_counter()
        pose, final, recut = a.localizeCloud(scan)
        wall_a = time.perf_counter() - t0
        sa, la = a.registration.stats(), a.localizeStats()
        src = a.filteredScan()
        t0 = time.perf_counter()
        whole.setInputSource(src)
        final_w = whole.align(guess)
        wall_w = time.perf_counter() - t0
        sw = whole.stats()
        recuts += int(recut)
        if k >= warmup:
            rows["cut"].append(dict(wall_ms=1e3 * wall_a, solve_ms=sa["solve_ms"], index_in_smem=sa["index_in_smem"], n_voxels=sa["n_voxels"],
                                    n_target=la["n_target"], iterations=sa["iterations"], recut=int(recut)))
            rows["whole"].append(dict(wall_ms=1e3 * wall_w, solve_ms=sw["solve_ms"], index_in_smem=sw["index_in_smem"],
                                      n_voxels=sw["n_voxels"], n_target=sw["n_target"], iterations=sw["iterations"]))
            err["cut"].append(synth.pose_error(final, T_gt)[0])
            err["whole"].append(synth.pose_error(final_w, T_gt)[0])
    clock = sm_clock_now()
    out = {"resolution": res, "n_map": n_map, "frames_timed": len(rows["cut"]), "recuts": recuts, "sm_clock_after_loop": clock,
           "whole_map_set_input_target_pcd_s": whole_build_s}
    for arm in ("cut", "whole"):
        r = rows[arm]
        out[arm] = {"wall_ms": summary(x["wall_ms"] for x in r), "solve_ms": summary(x["solve_ms"] for x in r),
                    "index_in_smem": sorted({int(x["index_in_smem"]) for x in r}), "n_voxels": summary(x["n_voxels"] for x in r),
                    "n_target": summary(x["n_target"] for x in r), "iterations": summary(x["iterations"] for x in r),
                    "translation_error_m_max": max(err[arm])}
    c = [x for x in rows["cut"]]
    out["cut"]["wall_ms_frames_with_recut"] = summary(x["wall_ms"] for x in c if x["recut"])
    out["cut"]["wall_ms_frames_without_recut"] = summary(x["wall_ms"] for x in c if not x["recut"])
    return out


def profile_cuts(path, drive, frames, tmp):
    """Device time of the cut's kernels: a session that re-cuts after every frame, traced by torch.profiler."""
    from lidarslam_ros2_b200 import scanmatcher
    from torch.profiler import ProfilerActivity, profile

    g = scanmatcher.ScanMatcher(ndt_resolution=2.0, **KW)
    n_map = g.setPriorMapPCD(path)
    g.setLocalizationParams(CROP, 0.0)
    g.setInitialPose((X_START, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0))
    g.localizeCloud(drive[0][0])  # warm-up: module load, buffers
    n_cut = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], acc_events=True) as prof:
        for scan, _ in drive[1:1 + frames]:
            g.localizeCloud(scan)
            n_cut.append(g.localizeStats()["n_cut"])
    trace = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f).get("traceEvents", [])
    os.remove(trace)
    dur = {k: [e["dur"] for e in events if e.get("cat") == "kernel" and k in e.get("name", "")] for k in CUT_KERNELS + SCAN_KERNELS}
    complete = all(len(dur[k]) == len(n_cut) for k in CUT_KERNELS)
    out = {"n_map": n_map, "cuts_profiled": len(n_cut), "trace_complete": bool(complete), "n_cut": summary(n_cut),
           "kernel_us": {k: summary(v) for k, v in dur.items()}}
    if complete:
        both = [a + b for a, b in zip(dur["cut_count_kernel"], dur["cut_write_kernel"])]
        bytes_ = [32 * n_map + 16 * c for c in n_cut]
        out["cut_kernels_us"] = summary(both)
        out["algorithmic_bytes"] = summary(bytes_)
        out["algorithmic_bytes_per_s"] = summary(b / (t * 1e-6) for b, t in zip(bytes_, both))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_localize.jsonl")
    ap.add_argument("--map-points", type=int, default=8_000_000)
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=4, help="frames of the drive run but not reported")
    ap.add_argument("--step", type=float, default=1.5, help="metres driven per frame")
    ap.add_argument("--resolutions", default="2.0,1.0")
    ap.add_argument("--profiled", type=int, default=12, help="cuts traced by torch.profiler")
    ap.add_argument("--workers", type=int, default=8, help="processes ray-casting the drive's scans")
    args = ap.parse_args()
    if args.frames - args.warmup < 40:
        raise SystemExit("bench_localize reports at least 40 frames: raise --frames")
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_localize needs a CUDA device (there is no CPU fallback)")
    line = {"tool": "bench_localize", **gpu_info(), "crop_radius": CROP, "recrop_distance": RECROP, "session": KW,
            "l2_state": "not flushed: the solver's target is as warm as in a running localiser; the map exceeds L2 when map_bytes > 50 MB",
            "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        path, n, size, drive = make_world(args.map_points, args.frames, args.step, args.workers, tmp)
        line.update(map_points=n, map_bytes=16 * n, pcd_file_bytes=size, scan_points=summary(len(s) for s, _ in drive))
        for res in (float(v) for v in args.resolutions.split(",")):
            line["runs"].append(run_resolution(res, path, drive, args.warmup))
        line["cut"] = profile_cuts(path, drive, args.profiled, tmp)
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_localize.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
