"""The CPU side of tools/bench_pcd_save.py: the restated PCL writer (tests/hostmath/pcd_writer_ref.hpp, std::ostringstream
at precision 8, single-threaded like pcl::io::savePCDFileASCII) timed on the same pose-adjusted map, and its file
compared byte for byte with the one b200sm_save_map_pcd_ascii writes. Run on a GPU node:

    python tests/diag/diag_pcd_save.py --out DIR [--configs 100x32768,1000x32768]

Appends one JSON line to DIR/diag_pcd_save.jsonl (and prints it).
"""
import argparse
import filecmp
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench_pcd_save import build_session  # noqa: E402
from bench_pose_adjust import gpu_info  # noqa: E402
from test_pcd_format_cpu import build_pcd_host  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--configs", default="100x32768,1000x32768")
    args = ap.parse_args()
    line = {"tool": "diag_pcd_save", **gpu_info(), "host_cpus": os.cpu_count(), "configs": []}
    with tempfile.TemporaryDirectory() as tmp:
        ph = build_pcd_host(tmp)
        for cfg in args.configs.split(","):
            n_sub, n_pts = (int(v) for v in cfg.lower().split("x"))
            g, adjusted = build_session(n_sub, n_pts)
            gpu_path, cpu_path = os.path.join(tmp, "gpu.pcd"), os.path.join(tmp, "cpu.pcd")
            t0 = time.perf_counter()
            points, size = g.saveMapPCDASCII(gpu_path, adjusted)
            t_gpu = time.perf_counter() - t0
            cloud = np.ascontiguousarray(g.assembleMap(adjusted)[0])
            t0 = time.perf_counter()
            rc = ph.ph_save_pcd_ascii(cpu_path.encode(), cloud.ctypes.data, len(cloud))
            t_cpu = time.perf_counter() - t0
            same = rc == 0 and filecmp.cmp(gpu_path, cpu_path, shallow=False)
            line["configs"].append({"submaps": n_sub, "points_per_submap": n_pts, "points": points, "file_bytes": size,
                                    "reference_writer_s": t_cpu, "device_save_s_first_call": t_gpu, "bytes_equal": same})
            os.remove(gpu_path)
            os.remove(cpu_path)
            del g
    os.makedirs(args.out, exist_ok=True)
    text = json.dumps(line)
    with open(os.path.join(args.out, "diag_pcd_save.jsonl"), "a") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
