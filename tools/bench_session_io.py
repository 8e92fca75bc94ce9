"""Benchmark of saving a mapping session to disk and loading it back (b200sm_save_session / b200sm_load_session) on
synthetic imported submaps (tools/bench_pose_adjust.py's: uniform points with intensity, poses along a drifted drive, 20
loop edges), against what a caller does without them: b200sm_get_submap + ndarray.tofile per submap to save,
np.fromfile + b200sm_import_submap per submap to load.

Writes one JSON line to DIR/bench_session_io.jsonl (and prints it). Wall times are the host clock around calls that end
synchronised, median of --reps, files in a local temporary directory with the page cache warm (one save and one load run
before the timed ones). The copy times are the device durations torch.profiler records for the device-to-host,
host-to-device and device-to-device copies of one save and one load, in a run of their own. The card's name, power limit
and SM clocks are read in the same run. Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_pose_adjust import drive  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock, clock_max = (v.strip() for v in q.split(","))
        return {"gpu": name, "power_limit": power, "sm_clock": clock, "sm_clock_max": clock_max}
    except Exception as e:  # the numbers below still stand, but without their card they are not reported as measured
        return {"gpu": None, "power_limit": None, "error": str(e)}


def _tree_bytes(d):
    return sum(os.path.getsize(os.path.join(r, f)) for r, _, fs in os.walk(d) for f in fs)


def run_config(n_sub, n_pts, reps, rng, tmp):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    g = ScanMatcher()
    poses, loops = drive(n_sub, rng)
    for i in range(n_sub):
        c = np.concatenate([rng.uniform(-60, 60, size=(n_pts, 3)), rng.uniform(0, 255, size=(n_pts, 1))], axis=1).astype(np.float32)
        g.importSubmap(c, poses[i], 2.0 * i)
    adjusted, _ = g.poseAdjust(loops)
    d = os.path.join(tmp, "session")
    base = os.path.join(tmp, "caller")
    os.makedirs(base, exist_ok=True)

    def save():
        return g.saveSession(d, loops, 5, adjusted)

    def load():
        h = ScanMatcher()
        info = h.loadSession(d)[3]
        return h, info

    def caller_save():  # b200sm_get_submap + tofile per submap (the manifest left out: it is small)
        for i in range(n_sub):
            cloud, _, _ = g.submap(i)
            cloud.tofile(os.path.join(base, "%06d.bin" % i))

    def caller_load():  # np.fromfile + b200sm_import_submap per submap
        h = ScanMatcher()
        for i in range(n_sub):
            h.importSubmap(np.fromfile(os.path.join(base, "%06d.bin" % i), dtype=np.float32).reshape(-1, 4), poses[i], 2.0 * i)
        return h

    info = save()  # warm: the page cache holds the files, the staging buffers are allocated
    h, info_load = load()
    del h
    caller_save()
    caller_load()
    wall = {"save": [], "load": [], "caller_save": [], "caller_load": []}
    for _ in range(reps):
        for name, fn in (("save", save), ("load", load), ("caller_save", caller_save), ("caller_load", caller_load)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            wall[name].append(time.perf_counter() - t0)
            del out
    h, _ = load()
    same = all(np.array_equal(h.submap(i)[0].view(np.uint32), g.submap(i)[0].view(np.uint32)) for i in range(0, n_sub, max(1, n_sub // 50)))
    del h

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        save()
        h, _ = load()
        torch.cuda.synchronize()
    del h
    trace = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f).get("traceEvents", [])
    os.remove(trace)
    copies = {k: [e["dur"] for e in events if e.get("cat") == "gpu_memcpy" and k in e.get("name", "")] for k in ("DtoH", "HtoD", "DtoD")}
    kernels = [e["dur"] for e in events if e.get("cat") == "kernel"]

    med = lambda v: statistics.median(v)  # noqa: E731
    bytes_saved, bytes_loaded = int(info["n_bytes"]), int(info_load["n_bytes"])
    out = {
        "submaps": n_sub, "points_per_submap": n_pts, "points": n_sub * n_pts, "loop_edges": len(loops),
        "bytes_saved": bytes_saved, "bytes_loaded": bytes_loaded, "bytes_on_disk": _tree_bytes(d), "bitwise_round_trip": bool(same),
        "save_ms_median": 1e3 * med(wall["save"]), "load_ms_median": 1e3 * med(wall["load"]),
        "save_gb_per_s": bytes_saved / med(wall["save"]) / 1e9, "load_gb_per_s": bytes_loaded / med(wall["load"]) / 1e9,
        "caller_save_ms_median": 1e3 * med(wall["caller_save"]), "caller_load_ms_median": 1e3 * med(wall["caller_load"]),
        "save_ms_all": [1e3 * v for v in wall["save"]], "load_ms_all": [1e3 * v for v in wall["load"]],
        "profiled_save_and_load": {
            "d2h_copies": len(copies["DtoH"]), "d2h_us_total": sum(copies["DtoH"]),
            "h2d_copies": len(copies["HtoD"]), "h2d_us_total": sum(copies["HtoD"]),
            "d2d_copies": len(copies["DtoD"]), "d2d_us_total": sum(copies["DtoD"]),
            "kernels": len(kernels), "kernel_us_total": sum(kernels),
        },
    }
    shutil.rmtree(d, ignore_errors=True)
    shutil.rmtree(base, ignore_errors=True)
    del g
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_session_io.jsonl")
    ap.add_argument("--configs", default="100x32768,1000x32768", help="comma-separated SUBMAPSxPOINTS")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_session_io needs a CUDA device (there is no CPU fallback)")
    rng = np.random.default_rng(2024)
    line = {"tool": "bench_session_io", **gpu_info(), "configs": []}
    with tempfile.TemporaryDirectory() as tmp:
        line["tmp_filesystem"] = subprocess.run(["df", "-T", tmp], capture_output=True, text=True).stdout.strip().splitlines()[-1]
        for cfg in args.configs.split(","):
            n_sub, n_pts = (int(v) for v in cfg.lower().split("x"))
            line["configs"].append(run_config(n_sub, n_pts, args.reps, rng, tmp))
    line.update({"power_limit_after": gpu_info().get("power_limit")})
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "bench_session_io.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
