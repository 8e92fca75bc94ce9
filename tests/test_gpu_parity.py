"""GPU parity tests: the CUDA path through the C-ABI (include/b200reg.h) against the CPU oracle on identical
inputs, plus the committed golden fixtures. Run on an H100 with `pytest -m gpu`.

Tolerances
  * integer / index results (leaf indices, point counts, NN indices): bit exact
  * f64 voxel moments: 1e-9 relative (f64 atomics change the summation order only)
  * derivative sums: 2e-5 of the largest Hessian entry (f32 per-pair math, re-associated on the GPU)
  * poses: 1e-3 m / 1e-3 rad (BASELINE.json north_star)
"""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POSE_TOL_T = 1e-3
POSE_TOL_R = 1e-3


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


def _mk(b200, oracle_mod, src, tgt, res, method=2, eps=0.01, max_it=35):
    g = b200.NormalDistributionsTransform()
    g.setResolution(res)
    g.setTransformationEpsilon(eps)
    g.setMaximumIterations(max_it)
    g.setNeighborhoodSearchMethod(method)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    o = oracle_mod.NDT(resolution=res, transformation_epsilon=eps, max_iterations=max_it, search_method=method)
    o.set_target(tgt)
    o.set_source(src)
    return g, o


def test_library_loaded_is_in_tree(b200):
    import os

    assert os.path.exists(b200.LIB_PATH) and b200.LIB_PATH.endswith("lidarslam_ros2_b200/csrc/libb200reg.so")


def test_voxel_map_parity(b200, oracle_mod, pair_small):
    src, tgt, _ = pair_small
    for res in (2.0, 5.0):
        g, o = _mk(b200, oracle_mod, src, tgt, res)
        vg, vo = g.voxels(), o.voxels()
        np.testing.assert_array_equal(vg["idx"], vo["idx"])  # same leaves, ascending leaf index
        np.testing.assert_array_equal(vg["npts"], vo["npts"])
        np.testing.assert_allclose(vg["mean"], vo["mean"], rtol=0, atol=1e-9)
        scale = np.abs(vo["icov"]).max(axis=(1, 2), keepdims=True)
        assert np.max(np.abs(vg["icov"] - vo["icov"]) / scale) < 1e-7
        np.testing.assert_allclose(vg["centroid"], vo["centroid"], atol=2e-4)


@pytest.mark.parametrize("method", [2, 3, 1, 0], ids=["DIRECT7", "DIRECT1", "DIRECT26", "KDTREE"])
def test_derivatives_parity(b200, oracle_mod, pair_small, method):
    src, tgt, _ = pair_small
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0, method=method)
    for p in (np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02]), np.array([-0.4, 0.3, -0.1, 2.9, 0.01, -0.3])):
        T = oracle_mod.pose_to_matrix(p)
        for hess in (True, False):
            sg, gg, Hg = g.derivatives(T, p, hess)
            so, go, Ho = o.derivatives(T, p, hess)
            scale = max(np.abs(Ho).max(), np.abs(go).max(), 1.0) if hess else max(np.abs(go).max(), 1.0)
            assert abs(sg - so) <= 1e-6 * max(1.0, abs(so))
            assert np.abs(gg - go).max() <= 2e-5 * scale
            if hess:
                assert np.abs(Hg - Ho).max() <= 2e-5 * scale
            else:
                assert np.all(Hg == 0)


def test_derivatives_deterministic(b200, oracle_mod, pair_small):
    src, tgt, _ = pair_small
    g, _ = _mk(b200, oracle_mod, src, tgt, 2.0)
    p = np.array([0.1, 0.05, -0.02, 0.003, 0.002, -0.01])
    T = oracle_mod.pose_to_matrix(p)
    a = g.derivatives(T, p)
    b = g.derivatives(T, p)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_hessian_radius_parity(b200, oracle_mod, pair_tiny):
    src, tgt, _ = pair_tiny
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0)
    p = np.array([0.2, -0.1, 0.03, 0.004, -0.006, 0.015])
    T = oracle_mod.pose_to_matrix(p)
    Hg, Ho = g.hessian_radius(T, p), o.hessian_radius(T, p)
    assert np.abs(Hg - Ho).max() <= 1e-9 * np.abs(Ho).max()


def _check_pose(T_gpu, T_cpu):
    from lidarslam_ros2_b200 import synth

    dt, dr = synth.pose_error(T_gpu, T_cpu)
    assert dt < POSE_TOL_T and dr < POSE_TOL_R, (dt, dr)


@pytest.mark.parametrize("cfg,res", [("tiny", 2.0), ("small", 2.0), ("small", 5.0), ("c1", 5.0)])
def test_align_parity_synthetic(b200, oracle_mod, cfg, res):
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair(cfg, res)
    g, o = _mk(b200, oracle_mod, src, tgt, res)
    Tg, To = g.align(), o.align()
    _check_pose(Tg, To)
    assert g.hasConverged() == o.converged
    assert g.getFinalNumIteration() == o.iterations
    assert abs(g.getTransformationProbability() - o.trans_probability) <= 1e-5 * max(1.0, abs(o.trans_probability))
    # with a non-identity guess (frontend: previous pose, scanmatcher_component.cpp:331-353)
    guess = synth.pose_matrix((0.1, -0.05, 0.02), (0.002, -0.001, 0.01)).astype(np.float32)
    _check_pose(g.align(guess), o.align(guess))
    # negative roll: Eigen's eulerAngles(0,1,2) folds the first angle into [0, pi] (ndt_omp_impl.hpp:109)
    guess = synth.pose_matrix((0.05, 0.05, 0.0), (-0.004, 0.002, 0.01)).astype(np.float32)
    _check_pose(g.align(guess), o.align(guess))
    assert g.getFinalNumIteration() == o.iterations


@pytest.mark.parametrize("name,method", [("DIRECT7", 2), ("DIRECT1", 3), ("KDTREE", 0)])
def test_align_golden_pcd(b200, oracle_mod, golden, name, method):
    # apps/align.cpp on the vendored scans: resolution 1.0, defaults (eps 0.1, 35 iterations), identity guess
    g = b200.NormalDistributionsTransform()
    g.setResolution(1.0)
    g.setNeighborhoodSearchMethod(method)
    g.setInputTarget(golden["target"])
    g.setInputSource(golden["source"])
    T = g.align()
    ref = golden["ndt"][name]
    _check_pose(T, np.array(ref["final_transformation"]))
    assert g.hasConverged() and g.getFinalNumIteration() == ref["iterations"]
    # the README's printed fitness (Thirdparty/ndt_omp_ros2/README.md:24-52) through the GPU 1-NN
    assert abs(g.getFitnessScore() - golden["readme_fitness"][name]) < 2e-4


def test_more_thuente_path_parity(b200, oracle_mod, pair_tiny):
    # step_max <= step_min (transformation_epsilon >= 2 * step_size) makes interval_converged false
    # (ndt_omp_impl.hpp:803): the MT loop and the f64 radius Hessian (K2) run.
    src, tgt, _ = pair_tiny
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0, eps=0.2, max_it=6)
    _check_pose(g.align(), o.align())
    assert g.getFinalNumIteration() == o.iterations
    assert g.stats()["evaluations"] == o.evaluations


def test_fitness_and_nn_parity(b200, oracle_mod, pair_small):
    src, tgt, _ = pair_small
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0)
    g.align()
    o.align()
    assert abs(g.getFitnessScore() - o.fitness()) <= 1e-4 * o.fitness() + 1e-6
    assert abs(g.getFitnessScore(1.0) - o.fitness(1.0)) <= 1e-4 * o.fitness(1.0) + 1e-6
    idx_g, d2_g = g.nearest(src)
    idx_o, d2_o = oracle_mod.nn1(tgt, src)
    np.testing.assert_array_equal(idx_g, idx_o)  # exact NN, ties to the lower index
    np.testing.assert_array_equal(d2_g, d2_o)    # same un-fused f32 accumulation


def test_calculate_score_parity(b200, oracle_mod, pair_tiny):
    src, tgt, _ = pair_tiny
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0)
    sg, so = g.calculateScore(src), o.calculate_score(np.eye(4))
    assert abs(sg - so) <= 1e-9 * max(1.0, abs(so))


def test_voxelgrid_parity(b200, oracle_mod, golden):
    raw = golden["raw"]
    for leaf in (0.1, 0.5, 2.5):
        out_g = b200.voxel_grid_filter(raw, leaf)
        out_o = oracle_mod.voxelgrid(raw, leaf)
        assert out_g.shape == out_o.shape  # same occupied leaves, same (ascending) order
        np.testing.assert_allclose(out_g, out_o, rtol=1e-5, atol=5e-5)
    # idempotence property at full size: filtering an already filtered cloud keeps every point
    again = b200.voxel_grid_filter(out_g, 2.5)
    assert len(again) == len(out_g)


def test_edge_cases(b200, oracle_mod, pair_tiny):
    src, tgt, _ = pair_tiny
    g = b200.NormalDistributionsTransform()
    # align without target/source: PCL soft-fails, converged stays false, final = identity
    T = g.align()
    assert not g.hasConverged() and np.array_equal(T, np.eye(4, dtype=np.float32))
    g.setInputTarget(np.zeros((0, 3), dtype=np.float32))  # empty cloud ignored
    g.setResolution(2.0)
    g.setInputTarget(tgt)
    T = g.align()
    assert not g.hasConverged()
    # a target too sparse for any voxel to reach 6 points: first solve gives delta_p = 0 → converged, final = guess
    sparse = tgt[::400]
    g.setInputTarget(sparse)
    g.setInputSource(src)
    guess = np.eye(4, dtype=np.float32)
    guess[0, 3] = 0.25
    T = g.align(guess)
    o = oracle_mod.NDT(resolution=2.0)
    o.set_target(sparse)
    o.set_source(src)
    To = o.align(guess)
    np.testing.assert_allclose(T, To, atol=1e-6)
    assert g.hasConverged() == o.converged
    # ragged stride: PointXYZI layout (32-byte points)
    wide = np.zeros((len(src), 8), dtype=np.float32)
    wide[:, :3] = src
    wide[:, 3] = 1.0
    wide[:, 4] = 7.0
    g2, o2 = _mk(b200, oracle_mod, wide, tgt, 2.0)
    _check_pose(g2.align(), o2.align())


def test_kdtree_mode_dense_target(b200, oracle_mod):
    """KDTREE mode (radiusSearch over voxel centroids, voxel_grid_covariance_omp.h:470-499) on a dense target: the voxel
    centroid is the f32 cast of an order-independent f64 sum here and a float running sum in the reference
    (voxel_grid_covariance_omp_impl.hpp:262, 287) — a documented deviation of a few float ulp that could flip a voxel sitting
    exactly on the search radius. Poses must still agree within the north_star tolerance, the hit counts within 1e-4."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("c2", 2.0)
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0, method=0)
    vg, vo = g.voxels(), o.voxels()
    np.testing.assert_array_equal(vg["idx"], vo["idx"])
    assert np.abs(vg["centroid"] - vo["centroid"]).max() < 5e-4  # well-populated voxels: float-sum rounding of the reference
    _check_pose(g.align(), o.align())
    assert g.getFinalNumIteration() == o.iterations
    p = np.array([0.2, -0.1, 0.03, 0.004, -0.003, 0.015])
    T = oracle_mod.pose_to_matrix(p)
    sg, gg, Hg = g.derivatives(T, p, True)
    so, go, Ho = o.derivatives(T, p, True)
    assert abs(sg - so) <= 1e-4 * abs(so)


def test_invalid_strides_are_rejected(b200):
    """Records hold float fields: a stride or an intensity offset that is not a multiple of 4 would fault inside the unpack
    kernel (misaligned address poisons the CUDA context) — it must be refused at the boundary instead."""
    import ctypes as C

    from lidarslam_ros2_b200 import _capi

    L = _capi.lib()
    g = b200.NormalDistributionsTransform()
    buf = np.zeros(4000, dtype=np.uint8)
    assert L.b200reg_set_input_target(g._h, buf.ctypes.data, 100, 14) == _capi.ERR_ARG
    assert L.b200reg_set_input_source(g._h, buf.ctypes.data, 100, 18) == _capi.ERR_ARG
    m = C.c_size_t(0)
    out = np.zeros(4000, dtype=np.uint8)
    assert L.b200reg_voxelgrid(0, buf.ctypes.data, 100, 16, 13, 0.5, out.ctypes.data, 100, C.byref(m)) == _capi.ERR_ARG
    # and the context is still healthy
    src, tgt, _ = b200.synth.registration_pair("tiny", 2.0) if hasattr(b200, "synth") else (None, None, None)
    if src is None:
        from lidarslam_ros2_b200 import synth
        src, tgt, _ = synth.registration_pair("tiny", 2.0)
    g.setResolution(2.0)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    g.align()
    assert g.hasConverged()


def test_cpp_adapter_end_to_end(b200):
    """The C++ adapter (include/b200reg_pcl.hpp) driven like apps/align.cpp: recovers a known shift on the GPU."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "cpp", "adapter_smoke")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "adapter_smoke.cpp"), "-o", exe,
                           "-L" + os.path.join(root, "lidarslam_ros2_b200", "csrc"), "-lb200reg",
                           "-Wl,-rpath," + os.path.join(root, "lidarslam_ros2_b200", "csrc")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


def test_cpp_adapter_pcl_mode_keeps_the_host_tree_out(b200):
    """PCL mode of the adapter against the PCL-1.12-shaped stub (tests/cpp/fake_pcl): align() through the base-class pointer
    runs pcl::Registration::initCompute(), which would build a host kd-tree over the whole target if the adapter armed
    target_cloud_updated_. The stub counts those builds; the program exits non-zero if one happens, if the fitness came from
    the host tree, or if the aligned-cloud copy is not opt-in."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "cpp", "adapter_pcl_mode")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-DB200REG_WITH_PCL",
                           "-I" + os.path.join(root, "tests", "cpp", "fake_pcl"), "-I" + os.path.join(root, "include"),
                           os.path.join(root, "tests", "cpp", "adapter_pcl_mode.cpp"), "-o", exe,
                           "-L" + os.path.join(root, "lidarslam_ros2_b200", "csrc"), "-lb200reg",
                           "-Wl,-rpath," + os.path.join(root, "lidarslam_ros2_b200", "csrc")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout + out.stderr)


@pytest.mark.parametrize("cfg", ["c2", "headline"])
def test_align_parity_full_size(b200, oracle_mod, cfg):
    """BASELINE.json's full sizes (C2: ~60k vs 500k; headline: ~100k vs 1M), res 2.0, node parameters: pose and iteration
    parity with the CPU path, determinism of repeated solves, and the voxel-count invariant."""
    from lidarslam_ros2_b200 import synth

    src, tgt, T_gt = synth.registration_pair(cfg, 2.0)
    g, o = _mk(b200, oracle_mod, src, tgt, 2.0)
    Tg, To = g.align(), o.align()
    _check_pose(Tg, To)
    assert g.getFinalNumIteration() == o.iterations and g.hasConverged() == o.converged
    assert len(g.voxels()["idx"]) == len(o.voxels()["idx"])
    assert np.array_equal(g.align(), Tg)  # bitwise deterministic
    dt, dr = synth.pose_error(Tg, T_gt)
    assert dt < 0.15 and dr < 5e-3  # and it is a registration: close to the pose the scan was ray-cast from
    assert abs(g.getFitnessScore(1.0) - o.fitness(1.0)) <= 1e-4 * o.fitness(1.0) + 1e-6
