"""Measures the place search of the scan-matcher session (b200sm_search_loop_place): Scan Context descriptors built on the
device (K13a) and the newest one scored against every older one at every column shift (K13b), on imported synthetic
submaps of ~30 k points each.

    python tools/bench_place_recognition.py --out DIR [--submaps 1000 10000] [--points 30000] [--repeats 5]

For each submap count: the K13a time for all submaps cold (the first search after the import) and for one new submap (the
search after one more import), and the K13b time, all from torch.profiler in a run of its own (kernels
scan_context_kernel, scan_context_finish_kernel, scan_context_search_kernel); then, with the profiler off, the wall time of
a whole call (host clock around a call that ends synchronised) with top_k = 1 and 3, which includes the verifications.
The CPU comparison is a numpy exhaustive search on the host over the same descriptors (every shift of every candidate,
vectorised over the candidates): it is a stand-in written for this benchmark, not the paper's code. The card's name, power
limit and maximum SM clock, and the SM clock after the timed loop, are read in the same run. Writes one JSON line per
submap count to DIR/bench_place_recognition.jsonl (and prints it). Needs a CUDA device; there is no CPU fallback.
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
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("scan_context_kernel", "scan_context_finish_kernel", "scan_context_search_kernel")
ARGS = dict(voxel_leaf_size=0.5, threshold_loop_closure_score=1.0, distance_loop_closure=-1.0, search_submap_num=1,
            sc_threshold=2.0)


def base_clouds(n_base, n_points, seed=7):
    """Structured synthetic submaps: ground, two facades and random boxes of points around the sensor."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_base):
        p = np.empty((n_points, 4), dtype=np.float32)
        r = rng.uniform(1.0, 90.0, size=n_points)
        a = rng.uniform(0, 2 * np.pi, size=n_points)
        p[:, 0], p[:, 1] = r * np.cos(a), r * np.sin(a)
        p[:, 2] = np.where(np.abs(p[:, 1]) > rng.uniform(10, 20), rng.uniform(-1.9, 12.0, size=n_points), -1.9)
        p[:, 3] = rng.uniform(0, 255, size=n_points)
        out.append(p)
    return out


def import_submaps(g, clouds, n_sub, start=0):
    for k in range(start, start + n_sub):
        c = clouds[k % len(clouds)]
        th = 0.37 * k
        M = np.eye(4)
        M[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
        M[:2, 3] = (2.0 * k, 0.1 * k)
        g.importSubmap(c, M, 2.0 * k)


def kernel_ms(prof):
    """Device time per kernel name (ms, summed over the launches in the profile) and launch counts."""
    ms, count = {k: 0.0 for k in KERNELS}, {k: 0 for k in KERNELS}
    for e in prof.events():
        for k in KERNELS:
            if e.name.endswith(k) or (k + "(") in e.name or e.name.split("(")[0].endswith("::" + k):
                if e.device_type.name == "CUDA":
                    ms[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                    count[k] += 1
    return ms, count


def numpy_search(desc, q_index, eligible):
    """The host comparison: D and s* of descriptor q_index against descriptors `eligible` (float64, vectorised)."""
    Q = desc[q_index].astype(np.float64)
    C = desc[eligible].astype(np.float64)
    S = Q.shape[1]
    nQ = np.sqrt((Q * Q).sum(axis=0))
    nC = np.sqrt((C * C).sum(axis=1))
    j = np.arange(S)
    best = np.full(len(eligible), np.inf)
    shift = np.zeros(len(eligible), dtype=np.int64)
    for s in range(S):
        c = (j + s) % S
        dots = np.einsum("rj,nrj->nj", Q, C[:, :, c])
        den = nQ[None, :] * nC[:, c]
        use = (nQ[None, :] > 0) & (nC[:, c] > 0)
        cos = np.where(use, dots / np.where(use, den, 1.0), 0.0)
        m = use.sum(axis=1)
        d = np.where(m > 0, 1.0 - cos.sum(axis=1) / np.maximum(m, 1), 1.0)
        better = d < best
        best[better], shift[better] = d[better], s
    return best, shift


def run(n_sub, args, clouds):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher, backend_registration

    reg = backend_registration("NDT", ndt_resolution=2.0)
    line = {"submaps": n_sub, "points_per_submap": args.points, "descriptor_bins": [20, 60]}
    # profiled run: cold build of every descriptor, then one new submap, then the search alone
    g = ScanMatcher()
    import_submaps(g, clouds, n_sub)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.searchLoopPlace(reg, top_k=1, capacity=0, **ARGS)
        torch.cuda.synchronize()
    cold, _ = kernel_ms(prof)
    import_submaps(g, clouds, 1, start=n_sub)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.searchLoopPlace(reg, top_k=1, capacity=0, **ARGS)
        torch.cuda.synchronize()
    one, _ = kernel_ms(prof)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.repeats):
            g.searchLoopPlace(reg, top_k=1, capacity=0, **ARGS)
        torch.cuda.synchronize()
    search, cnt = kernel_ms(prof)
    line["k13a_cold_ms"] = cold["scan_context_kernel"] + cold["scan_context_finish_kernel"]
    line["k13a_cold_bin_ms"] = cold["scan_context_kernel"]
    line["k13a_one_new_ms"] = one["scan_context_kernel"] + one["scan_context_finish_kernel"]
    line["k13b_ms"] = search["scan_context_search_kernel"] / max(cnt["scan_context_search_kernel"], 1)
    line["k13b_flop"] = 2.0 * n_sub * 60 * 60 * 20  # one multiply and one add per (candidate, shift, column, ring)
    line["k13b_flop_per_s"] = line["k13b_flop"] / (line["k13b_ms"] * 1e-3) if line["k13b_ms"] > 0 else None
    # wall time of whole calls, profiler off
    for top_k in (1, 3):
        walls = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows, scored = g.searchLoopPlace(reg, top_k=top_k, **ARGS)
            walls.append(1e3 * (time.perf_counter() - t0))
        line[f"wall_ms_top_k_{top_k}"] = summary(walls)
        line[f"verified_top_k_{top_k}"] = len(rows)
    # the host comparison on the same descriptors
    n = g.numSubmaps()
    desc = np.stack([g.scanContext(k) for k in range(n)])
    D_dev, S_dev = g.placeScores()
    t0 = time.perf_counter()
    D, S = numpy_search(desc, n - 1, np.arange(n - 1))
    line["numpy_host_search_ms"] = 1e3 * (time.perf_counter() - t0)
    line["numpy_max_abs_diff_D"] = float(np.abs(D - D_dev[:n - 1]).max())
    line["numpy_shift_agreement"] = float((S == S_dev[:n - 1]).mean())
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_place_recognition.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[1000, 10000])
    ap.add_argument("--points", type=int, default=30000)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_place_recognition needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(64, args.points)
    os.makedirs(args.out, exist_ok=True)
    for n_sub in args.submaps:
        line = {"tool": "bench_place_recognition", **gpu_info(), **run(n_sub, args, clouds), "sm_clock_after_loop": sm_clock_now()}
        text = json.dumps(line)
        with open(os.path.join(args.out, "bench_place_recognition.jsonl"), "a") as f:
            f.write(text + "\n")
        print(text, flush=True)


if __name__ == "__main__":
    main()
