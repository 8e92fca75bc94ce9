"""Measures the surface mesh of the scan-matcher session (b200sm_build_mesh): the static map's endpoint bounds (K15a), then
the band walks into the rank index (K21a), the fusion (K21b), the voxel list, the ACTIVE cells (K21c), the vertices and face
counts (K21d) and the faces (K21e), and the PLY save of the result, on imported synthetic submaps at the default
parameters (0.2 m voxels, truncation 0.6 m, max_range 100 m, min_weight 2).

    python tools/bench_mesh.py --out DIR [--submaps 100 1000] [--points 32768] [--repeats 5]

For each submap count: the device time of each kernel from torch.profiler in a run of its own; then, with the profiler
off, the wall time of the build, of the save and of buildStaticMap on the same session (host clock around calls that end
synchronised; median of --repeats). The CPU comparison is the serial host compile of the same header
(tests/hostmath/mesh_host.cpp, g++ -O2 -ffp-contract=off, built into a temporary directory) on the same submaps, run at the
smaller submap count only, with its mesh checked equal. The card's name, power limit and maximum SM clock, and the SM
clock after the timed loop, are read in the same run. Writes one JSON line per case to DIR/bench_mesh.jsonl (and prints
it). Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_localize import sm_clock_now, summary  # noqa: E402
from bench_occupancy import base_clouds, poses_on_ring  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402

KERNELS = ("sm_bounds_kernel", "ms_mark_kernel", "ms_fuse_kernel", "sm_voxel_list_kernel", "ms_active_kernel", "ms_vertex_kernel",
           "ms_face_kernel")


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


def host_compile(tmp):
    src = os.path.join(ROOT, "tests", "hostmath", "mesh_host.cpp")
    lib = os.path.join(tmp, "libmesh_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", lib])
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.msh_build.argtypes = [vp, vp, vp, vp, C.c_int]
    L.msh_info.argtypes = [vp]
    L.msh_arrays.argtypes = [vp] * 5
    return L


def run(n_sub, args, clouds, host):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from lidarslam_ros2_b200.scanmatcher import ScanMatcher

    poses = poses_on_ring(n_sub)
    subs = [clouds[k % len(clouds)] for k in range(n_sub)]
    g = ScanMatcher()
    for k in range(n_sub):
        g.importSubmap(subs[k], poses[k], float(k))
    line = {"submaps": n_sub, "points_per_submap": args.points, "resolution": 0.2, "truncation": 0.6, "max_range": 100.0,
            "min_weight": 2}
    info = g.buildMesh()  # warm-up: allocations, module load
    g.buildStaticMap()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.buildMesh()
        torch.cuda.synchronize()
    ms, cnt = kernel_ms(prof)
    for k in KERNELS:
        line[f"{k}_ms"] = ms[k]
        line[f"{k}_launches"] = cnt[k]
    line["kernels_ms"] = sum(ms.values())
    line.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in info.items()})
    build, save, static = [], [], []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.buildMesh()
            build.append(1e3 * (time.perf_counter() - t0))
            t0 = time.perf_counter()
            line["ply_bytes"] = g.saveMeshPly(os.path.join(tmp, "mesh.ply"))
            save.append(1e3 * (time.perf_counter() - t0))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.buildStaticMap()
            static.append(1e3 * (time.perf_counter() - t0))
    line["wall_ms_build"] = summary(build)
    line["wall_ms_save"] = summary(save)
    line["wall_ms_build_static_map"] = summary(static)
    if ms["ms_fuse_kernel"] > 0:
        line["walked_voxels_per_s_fuse_kernel"] = info["n_walked"] / (ms["ms_fuse_kernel"] / 1e3)
    if host is not None and n_sub == min(args.submaps):
        pts = np.zeros((n_sub * args.points, 4), dtype=np.float32)
        for k in range(n_sub):
            pts[k * args.points:(k + 1) * args.points] = subs[k]
        off = np.arange(n_sub + 1, dtype=np.int64) * args.points
        P = np.ascontiguousarray(np.array([M.T.reshape(16) for M in poses]))
        par = np.array([0.2, 0.6, 100.0, 0, 0, 0, 2], dtype=np.float64)
        t0 = time.perf_counter()
        rc = host.msh_build(par.ctypes.data, pts.ctypes.data, off.ctypes.data, P.ctypes.data, n_sub)
        line["host_compile_serial_ms"] = 1e3 * (time.perf_counter() - t0)
        hinfo = np.zeros(14, dtype=np.int64)
        host.msh_info(hinfo.ctypes.data)
        hv = np.zeros((max(1, int(hinfo[12])), 3), dtype=np.float32)
        hf = np.zeros((max(1, int(hinfo[13])), 3), dtype=np.uint32)
        host.msh_arrays(None, None, None, hv.ctypes.data, hf.ctypes.data)
        v, f = g.mesh()
        line["host_compile_equal"] = bool(rc == 0 and np.array_equal(hv[:len(v)].view(np.uint32), v.view(np.uint32)) and
                                          len(v) == int(hinfo[12]) and len(f) == int(hinfo[13]) and np.array_equal(hf[:len(f)], f))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for bench_mesh.jsonl")
    ap.add_argument("--submaps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--points", type=int, default=32768)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the serial host compile")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh needs a CUDA device (there is no CPU fallback)")
    clouds = base_clouds(16, args.points)
    os.makedirs(args.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        host = None if args.no_host else host_compile(tmp)
        for n_sub in args.submaps:
            line = {"tool": "bench_mesh", **gpu_info(), **run(n_sub, args, clouds, host), "sm_clock_after_loop": sm_clock_now()}
            text = json.dumps(line)
            with open(os.path.join(args.out, "bench_mesh.jsonl"), "a") as f:
                f.write(text + "\n")
            print(text, flush=True)


if __name__ == "__main__":
    main()
