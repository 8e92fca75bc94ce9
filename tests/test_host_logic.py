"""CPU tests of the host-side logic: C-ABI surface, synthetic generator determinism, and the multi-GPU sharding /
all-gather of the loop-closure sweep on a world_size-2 gloo group."""
import os
import re
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cabi_library_exports_every_declared_symbol():
    """include/b200reg.h is the drop-in boundary: every function it declares must be exported by the in-tree library
    (no compute calls here — there is no GPU in this container)."""
    import ctypes as C

    from lidarslam_ros2_b200 import _capi

    header = open(os.path.join(ROOT, "include", "b200reg.h")).read() + open(os.path.join(ROOT, "include", "b200comm.h")).read()
    declared = set(re.findall(r"\b(b200(?:reg|sm|comm)_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert os.path.exists(_capi.LIB_PATH), "build the library first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = C.CDLL(_capi.LIB_PATH)
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    assert declared == set(_capi.SYMBOLS), declared ^ set(_capi.SYMBOLS)


def test_no_cpu_fallback_without_device():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import lidarslam_ros2_b200 as m

    with pytest.raises(m.B200RegError):
        m.NormalDistributionsTransform()
    with pytest.raises(m.B200RegError):
        m.voxel_grid_filter(np.zeros((10, 3), dtype=np.float32), 0.5)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "lidarslam_ros2_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(import oracle|from oracle)", text, re.M), f
                assert not re.search(r"#\s*include\s*[\"<][^\n]*oracle", text), f
                assert "liboracle" not in text, f


def test_synth_is_deterministic():
    from lidarslam_ros2_b200 import synth

    a = synth.registration_pair("tiny", 2.0)
    b = synth.registration_pair("tiny", 2.0)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    # counter-based RNG: value k of a stream does not depend on how the stream is consumed
    r1, r2 = synth.Rng(7), synth.Rng(7)
    x = r1.uniform(100)
    y = np.concatenate([r2.uniform(40), r2.uniform(60)])
    assert np.array_equal(x, y)
    # pairs of the loop-closure workload are reproducible one by one
    p3 = next(iter(synth.loop_closure_pairs(8, n_tgt=2000, rings=4, azimuths=90, first=3, count=1)))
    allp = list(synth.loop_closure_pairs(8, n_tgt=2000, rings=4, azimuths=90))
    assert p3[0] == 3 and np.array_equal(p3[1], allp[3][1]) and np.array_equal(p3[2], allp[3][2])


def test_pose_error_metric():
    from lidarslam_ros2_b200 import synth

    A = synth.pose_matrix((0.4, -0.2, 0.06), (0.007, -0.005, 0.026))
    assert synth.pose_error(A.astype(np.float32), A) [1] < 1e-7  # float32 quantisation must not look like rotation
    B = synth.pose_matrix((0.4, -0.2, 0.06), (0.007, -0.005, 0.0265))
    assert abs(synth.pose_error(A, B)[1] - 5e-4) < 1e-6


def test_shard_pairs_partition():
    from lidarslam_ros2_b200 import batch

    for n, w in ((64, 1), (64, 2), (64, 8), (10, 4), (3, 8)):
        got = sorted(i for r in range(w) for i in batch.shard_pairs(n, r, w))
        assert got == list(range(n))
        sizes = [len(batch.shard_pairs(n, r, w)) for r in range(w)]
        assert max(sizes) - min(sizes) <= 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, n_pairs, q):
    import torch.distributed as dist

    from lidarslam_ros2_b200 import batch

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rows = []
    for i in batch.shard_pairs(n_pairs, rank, world):
        T = np.eye(4, dtype=np.float32)
        T[0, 3] = i  # recognisable per pair
        rows.append(batch.pack_row(i, T, 0.1 * i, i % 2 == 0, 5 + i))
    res = batch.gather_rows(np.array(rows), n_pairs, rank, world)
    q.put((rank, res["index"].tolist(), res["pose"][:, 0, 3].tolist(), res["fitness"].tolist(), res["iterations"].tolist()))
    dist.destroy_process_group()


def test_gather_rows_world2_gloo():
    import torch.multiprocessing as mp

    n_pairs, world = 7, 2  # ragged: ranks own 4 and 3 pairs
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, n_pairs, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, idx, tx, fit, it in out:  # every rank sees every pair, ordered by pair index
        assert idx == list(range(n_pairs))
        assert tx == [float(i) for i in range(n_pairs)]
        np.testing.assert_allclose(fit, [0.1 * i for i in range(n_pairs)], rtol=1e-6)
        assert it == [5 + i for i in range(n_pairs)]


def _build_adapter(out_dir):
    """Builds the adapter program into out_dir (a temporary directory: the tree may be read-only)."""
    import subprocess

    exe = os.path.join(out_dir, "adapter_smoke")
    src = os.path.join(ROOT, "tests", "cpp", "adapter_smoke.cpp")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L" + os.path.join(ROOT, "lidarslam_ros2_b200", "csrc"), "-lb200reg",
                           "-Wl,-rpath," + os.path.join(ROOT, "lidarslam_ros2_b200", "csrc")])
    return exe


def test_cpp_adapter_compiles_and_fails_loudly_without_gpu():
    """include/b200reg_pcl.hpp (the C++ host side of the boundary) builds against the C-ABI; without a GPU the
    engine refuses to construct (exit code 3) instead of falling back to a CPU path."""
    import subprocess
    import tempfile

    import torch

    with tempfile.TemporaryDirectory() as tmp:
        exe = _build_adapter(tmp)
        rc = subprocess.run([exe], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert rc.returncode == 0, rc.stdout
    else:
        assert rc.returncode == 3 and "no CUDA device" in rc.stdout, rc.stdout


def test_bench_reference_arm_contract():
    """bench.py --impl reference: rank 0 prints ONE JSON line with "impl": "reference" (the CPU restatement timed on the host
    cores), every other rank exits 0 without work or output."""
    import json
    import subprocess

    env = dict(os.environ, RANK="1", LOCAL_RANK="1", WORLD_SIZE="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1",
                        "--warmup", "1", "--workload", "c1"], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == ""
    env = dict(os.environ, RANK="0", LOCAL_RANK="0", WORLD_SIZE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1",
                        "--workload", "c1"], capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["value"] > 0 and line["unit"] == "registrations/s"
    assert line["cpu_baseline"]["kind"] == "port" and line["e2e"]["value"] == line["value"]
    assert line["steps"] == 2 and line["higher_is_better"] is True


def test_abi_header_is_plain_c():
    """include/b200reg.h must be consumable by a C compiler (cgo / JNI / ctypes-style bindings): C99, no C++ constructs."""
    import subprocess
    import tempfile

    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "hdr.c")
        with open(src, "w") as f:
            f.write('#include "b200reg.h"\n#include "b200comm.h"\nint main(void){b200reg_stats s; b200sm_stats t; b200sm_loop_result r; '
                    'b200reg_batch_result b; b200reg_sweep_result w; b200comm_t c = 0; (void)s; (void)t; (void)r; (void)b; (void)w; (void)c; return 0;}\n')
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I" + os.path.join(ROOT, "include"),
                               "-fsyntax-only", src])


def test_ndt_trace_record_layout_matches_numpy():
    """NormalDistributionsTransform.trace() reads b200reg_ndt_trace_record through a numpy dtype: its size and every field
    offset must be what a C compiler lays out for include/b200reg.h."""
    import subprocess
    import tempfile

    from lidarslam_ros2_b200.registration import NormalDistributionsTransform as NDT

    dt = NDT.TRACE_DTYPE
    body = "".join(f'printf("{k} %zu\\n", offsetof(b200reg_ndt_trace_record, {k}));' for k in dt.names)
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(src, "w") as f:
            f.write('#include <stddef.h>\n#include <stdio.h>\n#include "b200reg.h"\nint main(void){'
                    'printf("sizeof %zu\\n", sizeof(b200reg_ndt_trace_record));' + body + "return 0;}\n")
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), src, "-o", exe])
        got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    assert int(got.pop("sizeof")) == dt.itemsize
    assert {k: int(v) for k, v in got.items()} == {k: dt.fields[k][1] for k in dt.names}


def test_cpp_adapter_pcl_mode_type_checks():
    """include/b200reg_pcl.hpp compiled with -DB200REG_WITH_PCL against a PCL-1.12-shaped stub (tests/cpp/fake_pcl): the
    classes must derive from pcl::Registration, override its virtuals and be assignable to the nodes' `registration_` pointer
    (INTEGRATION.md section 2). Without a GPU the engine refuses to construct (exit code 3)."""
    import subprocess

    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:  # the program is built outside the tree, which may be read-only
        exe = os.path.join(tmp, "adapter_pcl_mode")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-DB200REG_WITH_PCL",
                               "-I" + os.path.join(ROOT, "tests", "cpp", "fake_pcl"), "-I" + os.path.join(ROOT, "include"),
                               os.path.join(ROOT, "tests", "cpp", "adapter_pcl_mode.cpp"), "-o", exe,
                               "-L" + os.path.join(ROOT, "lidarslam_ros2_b200", "csrc"), "-lb200reg",
                               "-Wl,-rpath," + os.path.join(ROOT, "lidarslam_ros2_b200", "csrc")])
        rc = subprocess.run([exe], capture_output=True, text=True)
    assert rc.returncode == 3 and "no CUDA device" in rc.stdout, rc.stdout


def test_recorded_round2_bench_line_follows_the_contract():
    """profiles/h100_bench_lines.jsonl, first line = `python bench.py --steps 20 --warmup 5` on an H100: every key of the bench
    contract, a roofline fraction consistent with its own fields, an e2e leg that moved bytes, one solver launch for the K
    steps, and the loop-closure sweep object."""
    import json

    with open(os.path.join(ROOT, "profiles", "h100_bench_lines.jsonl")) as f:
        line = json.loads(f.readline())
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert key in line, key
    assert line["higher_is_better"] is True and line["vs_baseline"] is None and line["n_gpus"] == 1
    assert abs(line["value"] - line["n_gpus"] * 1e3 / line["ms_per_step"]) < 1e-6 * line["value"]
    r = line["roofline"]
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(r["achieved"] - r["alg_bytes_per_launch"] / (r["launch_ms"] * 1e-3) / 1e9) < 1e-6 * r["achieved"]
    assert r["frac"] >= 0.40  # north_star: the fused derivative kernel at >= 40 % of the HBM roofline
    assert line["gpu_launches"] == 1 and line["details"]["batch_bitwise_equals_single_align"] is True
    e = line["e2e"]
    assert e["h2d_bytes_per_step"] > 1_000_000 and e["d2h_bytes_per_step"] > 0 and e["value"] > 0 and e["pageable"]["value"] > 0
    assert set(line["config"]) >= {"workload", "n_source", "n_target", "l2"}
    assert not set(line["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    c = line["cpu_baseline"]
    assert c["kind"] == "port" and c["value"] > 0 and line["e2e"]["value"] / c["value"] >= 50  # north_star: >= 50x
    assert c["pose_parity_max"]["dt_m"] < 1e-3 and c["pose_parity_max"]["dr_rad"] < 1e-3
    c4 = line["c4"]
    assert c4["pairs"] == 64 and c4["converged"] == 64 and "ncclAllGather" in c4["collective"]
    # the reference arm of the same round prints the same config keys
    with open(os.path.join(ROOT, "profiles", "h100_bench_lines.jsonl")) as f:
        ref = [json.loads(x) for x in f][1]
    assert ref["impl"] == "reference" and ref["config"] == line["config"]
