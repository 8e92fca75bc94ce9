"""Measures global localisation in a prior map (b200sm_localize_global: an (x, y, yaw) grid scored on the device in one
launch, the top-k refined in one batch launch) against the alternative users have without it: the same grid passed to
b200sm_localize_init, which runs a full Newton solve per hypothesis. NDT, DIRECT7, on the canyon map of bench_localize.py.

    python tools/bench_localize_global.py --out DIR [--map-points 4000000] [--trials 8] [--init-trials 2]

Each trial takes one frame of a drive down the canyon and starts the session from a position offset 3 to 7 m from the
truth in a random direction with a random heading; radius 10 m, step 1 m, 72 yaw steps, top_k 8. Reported: the scoring
kernel's device time (CUDA events, b200sm_global_result.score_ms), hypotheses/s and point evaluations/s (H x N_filtered
over that time), its algorithmic bytes (into the SMs, mostly L1 hits: H (N 16 / 8 + N 7 8) + 48 hits, see csrc/ndt_score.cu) and their share
of the 3.35 TB/s data-sheet HBM bandwidth, the whole call's wall time (host clock around a call that ends synchronised),
and how often the adopted pose is within 0.3 m / 0.02 rad of the truth. The first --init-trials trials also run the same
grid through localize_init on a second session in the same run (alternating with the global call): its wall time and
whether its chosen pose is within the same bounds. The card's name, power limit and maximum SM clock, and the SM clock
right after the timed loop, are read in the same run. Writes one JSON line to DIR/bench_localize_global.jsonl (and prints
it). Needs a CUDA device; there is no CPU fallback.
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
CROP = 60.0  # >= radius + scan_max_range
HBM_BYTES_PER_S = 3.35e12


def start_pose(T, rng):
    d, a = rng.uniform(3.0, 7.0), rng.uniform(0.0, 2.0 * math.pi)
    yaw = rng.uniform(-math.pi, math.pi)
    pos = (float(T[0, 3]) + d * math.cos(a), float(T[1, 3]) + d * math.sin(a), float(T[2, 3]))
    return pos, (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_localize_global.jsonl")
    ap.add_argument("--map-points", type=int, default=4_000_000)
    ap.add_argument("--trials", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=1, help="trials run but not reported")
    ap.add_argument("--init-trials", type=int, default=2, help="trials that also run the grid through localize_init")
    ap.add_argument("--radius", type=float, default=10.0)
    ap.add_argument("--step", type=float, default=1.0)
    ap.add_argument("--yaw-steps", type=int, default=72)
    ap.add_argument("--top-k", type=int, default=8)
    ap.add_argument("--workers", type=int, default=8)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_localize_global needs a CUDA device (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher, synth

    pts = synth.sample_map(synth.make_scene(), args.map_points, stream=9501)
    prior = np.concatenate([pts, np.zeros((len(pts), 1), dtype=np.float32)], axis=1)
    M0 = synth.pose_matrix((X_START, 0.0, 0.0), (0.0, 0.0, 0.0))
    n_frames = args.warmup + args.trials
    drive = [(scan, M0 @ T) for scan, T in synth.drive_stream(n_frames, rings=32, azimuths=938, step=6.0, x_start=X_START,
                                                               workers=args.workers)]
    rng = np.random.default_rng(2024)

    def session():
        g = scanmatcher.ScanMatcher(**KW)
        g.setPriorMap(prior)
        g.setLocalizationParams(CROP, 1e9)
        return g

    g, gi = session(), session()
    rows, init_rows = [], []
    for k, (scan, T_true) in enumerate(drive):
        pos, quat = start_pose(T_true, rng)
        g.setInitialPose(pos, quat)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        best, cand, res, info = g.localizeGlobal(scan, args.radius, args.step, args.yaw_steps, args.top_k)
        wall = time.perf_counter() - t0
        n_f = g.stats()["n_filtered"]
        ok = False
        dt = dr = None
        if best >= 0:
            dt, dr = synth.pose_error(res[best]["final"], T_true)
            ok = dt < 0.3 and dr < 0.02
        H = info["n_hypotheses"]
        rec = dict(trial=k, start_offset_m=float(np.hypot(pos[0] - T_true[0, 3], pos[1] - T_true[1, 3])), hypotheses=H,
                   n_filtered=n_f, score_ms=info["score_ms"], wall_ms=1e3 * wall, best=best, success=bool(ok), dt=dt, dr=dr,
                   hits_total=info["hits_total"],
                   bytes=H * (n_f * 16 / 8 + n_f * 7 * 8) + 48 * info["hits_total"])
        if k >= args.warmup and len(init_rows) < args.init_trials:
            poses, _, _ = g.globalSearch()
            gi.setInitialPose(pos, quat)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            bi, ri = gi.localizeInit(scan, poses)
            wall_i = time.perf_counter() - t0
            oki = False
            if bi >= 0:
                dti, dri = synth.pose_error(ri[bi]["final"], T_true)
                oki = dti < 0.3 and dri < 0.02
            init_rows.append(dict(trial=k, hypotheses=len(poses), wall_ms=1e3 * wall_i, best=bi, success=bool(oki)))
        if k >= args.warmup:
            rows.append(rec)
    clock = sm_clock_now()
    score_s = [r["score_ms"] * 1e-3 for r in rows]
    line = {"tool": "bench_localize_global", **gpu_info(), "sm_clock_after_loop": clock, "session": KW, "crop_radius": CROP,
            "search": dict(radius=args.radius, step=args.step, yaw_steps=args.yaw_steps, top_k=args.top_k),
            "map_points": len(prior), "trials": len(rows),
            "hypotheses": summary(r["hypotheses"] for r in rows), "n_filtered": summary(r["n_filtered"] for r in rows),
            "score_ms": summary(r["score_ms"] for r in rows),
            "hypotheses_per_s": summary(r["hypotheses"] / s for r, s in zip(rows, score_s)),
            "point_evaluations_per_s": summary(r["hypotheses"] * r["n_filtered"] / s for r, s in zip(rows, score_s)),
            "algorithmic_bytes": summary(r["bytes"] for r in rows),
            "algorithmic_bytes_per_s": summary(r["bytes"] / s for r, s in zip(rows, score_s)),
            "share_of_hbm_datasheet": summary(r["bytes"] / s / HBM_BYTES_PER_S for r, s in zip(rows, score_s)),
            "wall_ms": summary(r["wall_ms"] for r in rows),
            "success_rate": sum(r["success"] for r in rows) / max(len(rows), 1),
            "localize_init_same_grid": {"wall_ms": summary(r["wall_ms"] for r in init_rows),
                                        "success_rate": (sum(r["success"] for r in init_rows) / len(init_rows)) if init_rows else None,
                                        "rows": init_rows},
            "rows": rows}
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_localize_global.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
