"""Measures relocalisation anywhere in the prior map (b200sm_relocalize: the branch-and-bound (x, y, yaw) search of K17 on
the device, the best tiles refined with NDT) on two maps: the canyon of bench_localize.py (--map-points rows), and a larger
map of --tiles canyons (synth.make_scene(stream) for streams 1, 2, ...) side by side, 40 m apart across the street, which
b200sm_localize_global cannot cover within its 2^24-hypothesis cap at 1 m and 360 headings.

    python tools/bench_relocalize.py --out DIR [--map-points 4000000] [--tiles 4] [--trials 8]

Each trial takes one frame of a drive down the first canyon and starts the session from one fixed far-away pose (the
canyon's centre, heading 2 rad). Per map and trial, alternated in the same run: the default search (num_levels 6), the
exhaustive search (num_levels 1: every leaf scored), and on the canyon b200sm_localize_global with a radius covering the
canyon from the start (150 m, step 1 m, 72 headings, top_k 8; crop radius 200 m so its cut is the whole map). Reported:
the search's device time (CUDA events), nodes scored per level, T0 / T, the whole call's wall time (host clock around a
call that ends synchronised), and how often the adopted pose is within 0.3 m / 0.02 rad of the truth. Per-kernel device
times come from torch.profiler in a run of their own (two default searches on the canyon). The card's name, power limit
and maximum SM clock, and the SM clock after the timed loop, are read in the same run. Writes one JSON line to
DIR/bench_relocalize.jsonl (and prints it). Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_localize import X_START, summary, sm_clock_now  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

KW = dict(ndt_resolution=2.0, vg_size_for_input=0.4, use_min_max_filter=True, scan_min_range=1.0, scan_max_range=40.0)
CROP = 60.0
START = ((0.0, 0.0, 0.0), 2.0)  # the canyon's centre, a heading far from the drive's
GLOBAL = dict(radius=150.0, step=1.0, yaw_steps=72, top_k=8)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_relocalize.jsonl")
    ap.add_argument("--map-points", type=int, default=4_000_000)
    ap.add_argument("--tiles", type=int, default=4)
    ap.add_argument("--trials", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workers", type=int, default=8)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_relocalize needs a CUDA device (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher, synth

    def as_prior(pts):
        return np.concatenate([pts, np.zeros((len(pts), 1), dtype=np.float32)], axis=1)

    canyon = as_prior(synth.sample_map(synth.make_scene(), args.map_points, stream=9501))
    parts = [canyon]
    for t in range(1, args.tiles):
        p = synth.sample_map(synth.make_scene(1 + t), args.map_points, stream=9501 + t)
        p[:, 1] += 40.0 * t
        parts.append(as_prior(p))
    tiled = np.concatenate(parts)
    M0 = synth.pose_matrix((X_START, 0.0, 0.0), (0.0, 0.0, 0.0))
    drive = [(scan, M0 @ T) for scan, T in synth.drive_stream(args.warmup + args.trials, rings=32, azimuths=938, step=6.0,
                                                               x_start=X_START, workers=args.workers)]
    pos, yaw = START
    quat = (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))

    def session(prior, crop=CROP):
        g = scanmatcher.ScanMatcher(**KW)
        g.setPriorMap(prior)
        g.setLocalizationParams(crop, 1e9)
        return g

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        return out, 1e3 * (time.perf_counter() - t0)

    def verdict(final, T_true):
        dt, dr = synth.pose_error(final, T_true)
        return bool(dt < 0.3 and dr < 0.02), float(dt), float(dr)

    result = {"tool": "bench_relocalize", **gpu_info(), "session": KW, "start": dict(position=pos, yaw=yaw)}
    for name, prior in (("canyon", canyon), ("tiled", tiled)):
        g, g1 = session(prior), session(prior)
        gg = session(prior, 200.0) if name == "canyon" else None
        rows = []
        for k, (scan, T_true) in enumerate(drive):
            rec = dict(trial=k)
            for label, s_, kw in (("default", g, {}), ("exhaustive", g1, dict(num_levels=1))):
                s_.setInitialPose(pos, quat)
                (best, res, info), wall = timed(lambda: s_.relocalize(scan, **kw))
                ok = verdict(res[best]["final"], T_true) if best >= 0 else (False, None, None)
                rec[label] = dict(wall_ms=wall, search_ms=info["search_ms"], nodes=info["nodes"][:6], m=info["m"], t0=info["t0"],
                                  t=info["t"], leaves=info["leaves"], grid=(info["width"], info["height"]), best=best,
                                  success=ok[0], dt=ok[1], dr=ok[2], candidates=[(r["yaw_index"], *r["cell"], r["score"]) for r in res])
            rec["same_first_candidate"] = rec["default"]["candidates"][:1] == rec["exhaustive"]["candidates"][:1]
            if gg is not None:
                gg.setInitialPose(pos, quat)
                (best, cand, res, info), wall = timed(lambda: gg.localizeGlobal(scan, **GLOBAL))
                ok = verdict(res[best]["final"], T_true) if best >= 0 else (False, None, None)
                rec["localize_global"] = dict(wall_ms=wall, score_ms=info["score_ms"], hypotheses=info["n_hypotheses"], best=best,
                                              success=ok[0], dt=ok[1], dr=ok[2])
            if k >= args.warmup:
                rows.append(rec)
        m = {"map_points": len(prior), "trials": len(rows)}
        for label in ("default", "exhaustive", "localize_global"):
            if label not in rows[0]:
                continue
            r = [x[label] for x in rows]
            m[label] = {"wall_ms": summary(v["wall_ms"] for v in r),
                        "success_rate": sum(v["success"] for v in r) / len(r)}
            if label != "localize_global":
                m[label].update(search_ms=summary(v["search_ms"] for v in r), grid=r[0]["grid"], leaves=r[0]["leaves"],
                                m=summary(v["m"] for v in r), nodes_first_trial=r[0]["nodes"], t0_t_first_trial=(r[0]["t0"], r[0]["t"]))
            else:
                m[label].update(score_ms=summary(v["score_ms"] for v in r), hypotheses=r[0]["hypotheses"], spec=GLOBAL)
        m["same_first_candidate_rate"] = sum(x["same_first_candidate"] for x in rows) / len(rows)
        m["rows"] = rows
        result[name] = m
    result["sm_clock_after_loop"] = sm_clock_now()
    # per-kernel device times in a run of their own
    from torch.profiler import ProfilerActivity, profile

    g = session(canyon)
    scan = drive[-1][0]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            g.setInitialPose(pos, quat)
            g.relocalize(scan)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.key.find("rl_") >= 0 or e.key.find("counter_scan") >= 0:
            dev = getattr(e, "device_time_total", None)
            if dev is None:
                dev = getattr(e, "cuda_time_total", 0.0)
            kern[e.key[:120]] = dict(calls=int(e.count), device_us_total=float(dev))
    result["profiler_kernels_two_searches"] = kern
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(result)
    with open(os.path.join(args.out, "bench_relocalize.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
