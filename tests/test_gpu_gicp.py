"""GPU parity tests of the GICP path (K5 kNN covariances, K6 correspondences, K7 cost/gradient + BFGS) against the CPU
oracle's restatement of pclomp::GeneralizedIterativeClosestPoint. Parity unpinned beyond the oracle (see
oracle/gicp.hpp): PCL's BFGS and FLANN are external; the pose tolerance is BASELINE.json's 1e-3 m / 1e-3 rad."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


def _surface(n, seed):
    rng = np.random.default_rng(seed)
    u = rng.uniform(-3, 3, size=(n, 2))
    z = 0.3 * np.sin(u[:, 0]) + 0.2 * np.cos(1.7 * u[:, 1])
    wall = rng.uniform(-3, 3, size=(n // 3, 2))
    a = np.stack([u[:, 0], u[:, 1], z], axis=1)
    b = np.stack([wall[:, 0], np.full(len(wall), 3.0) + 0.05 * np.sin(3 * wall[:, 0]), 1.5 + 0.5 * wall[:, 1]], axis=1)
    return np.concatenate([a, b]).astype(np.float32)


def _pair(seed=17):
    from lidarslam_ros2_b200 import synth

    tgt = _surface(6000, seed)
    T_gt = synth.pose_matrix((0.08, -0.05, 0.03), (0.01, -0.015, 0.02))
    Ti = np.linalg.inv(T_gt)
    src = (tgt[::2].astype(np.float64) @ Ti[:3, :3].T + Ti[:3, 3]).astype(np.float32)
    return src, tgt, T_gt


def test_gicp_covariances_parity(b200, oracle_mod):
    src, tgt, _ = _pair()
    g = b200.GeneralizedIterativeClosestPoint()
    g.setInputTarget(tgt)
    g.setInputSource(src)
    g.align()
    o = oracle_mod.GICP()
    o.set_target(tgt)
    o.set_source(src)
    o.align()
    import covref as CR

    for which, cloud in (("source", src), ("target", tgt)):
        cg, co = g.covariances(which), o.covariances(which)
        assert cg.shape == co.shape
        # every point: within the per-point bound of the float64 reference where the smallest-variance direction is
        # determined by the moments, by the projector invariants where it is not (tests/covref.py); the oracle likewise
        ref, info = CR.reference(cloud, 20)
        for what, got in (("gpu", cg), ("oracle", co)):
            bad, _, _ = CR.check(got, ref, info)
            assert not bad.any(), (which, what, int(bad.sum()), np.flatnonzero(bad)[:5])


def test_gicp_align_parity(b200, oracle_mod):
    from lidarslam_ros2_b200 import synth

    src, tgt, T_gt = _pair()
    g = b200.GeneralizedIterativeClosestPoint()
    g.setInputTarget(tgt)
    g.setInputSource(src)
    Tg = g.align()
    o = oracle_mod.GICP()
    o.set_target(tgt)
    o.set_source(src)
    To = o.align()
    dt, dr = synth.pose_error(Tg, To)
    assert dt < 1e-3 and dr < 1e-3, (dt, dr)
    assert g.hasConverged() and o.converged
    assert g.numCorrespondences() == o.num_correspondences()
    # and both recover the known transform
    dt, dr = synth.pose_error(Tg, T_gt)
    assert dt < 5e-3 and dr < 5e-3
    assert abs(g.getFitnessScore() - o.fitness()) <= 1e-3 * max(o.fitness(), 1e-6) + 1e-7
    # with a guess and the node's parameters (scanmatcher_component.cpp:116-120)
    guess = synth.pose_matrix((0.05, -0.02, 0.0), (0.0, -0.005, 0.01)).astype(np.float32)
    g.setMaxCorrespondenceDistance(5.0)
    g.setTransformationEpsilon(1e-8)
    o.set("max_correspondence_distance", 5.0)
    o.set("transformation_epsilon", 1e-8)
    g.setMaximumIterations(30)
    o.set("max_iterations", 30)
    dt, dr = synth.pose_error(g.align(guess), o.align(guess))
    assert dt < 1e-3 and dr < 1e-3, (dt, dr)


@pytest.mark.parametrize("cfg", ["tiny", "small", "c1"])
def test_gicp_on_lidar_scene(b200, oracle_mod, cfg):
    """LiDAR-like scenes (ray-cast rings against the street canyon): the weakly constrained direction along the canyon makes
    the capped inner BFGS (20 iterations, gicp_omp_impl.hpp:218-230) path-dependent — its line search compares f32 cost
    values (:264-270) — so parity needs the same un-fused float arithmetic on both sides (gicp.cu is built with -fmad=false;
    round 1 compared 5e-2 m here). Node parameters (scanmatcher_component.cpp:116-120) and the class defaults."""
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair(cfg, 2.0)
    for eps in (1e-8, None):
        g = b200.GeneralizedIterativeClosestPoint()
        g.setMaxCorrespondenceDistance(5.0)
        o = oracle_mod.GICP(max_correspondence_distance=5.0)
        if eps is not None:
            g.setTransformationEpsilon(eps)
            o.set("transformation_epsilon", eps)
        g.setInputTarget(tgt)
        g.setInputSource(src)
        o.set_target(tgt)
        o.set_source(src)
        Tg, To = g.align(), o.align()
        dt, dr = synth.pose_error(Tg, To)
        assert g.hasConverged() == o.converged
        assert dt < 1e-3 and dr < 1e-3, (cfg, eps, dt, dr, g.stats()["iterations"], o.iterations)
        assert g.numCorrespondences() == o.num_correspondences()
        assert abs(g.getFitnessScore() - o.fitness()) <= 1e-3 * o.fitness()


def test_gicp_parity_baseline_c3_size(b200, oracle_mod):
    """BASELINE config 3 at full size: GICP, 64-ring scan (~94k pts) against the 1M-point map, corr_dist_threshold 5.0,
    transformation_epsilon 1e-8 (sm.cpp:118-119), k = 20; outer iterations bounded to keep the CPU side to about a minute."""
    from lidarslam_ros2_b200 import synth

    src, tgt, T_gt = synth.registration_pair("headline", 2.0)
    g = b200.GeneralizedIterativeClosestPoint()
    g.setMaxCorrespondenceDistance(5.0)
    g.setTransformationEpsilon(1e-8)
    g.setMaximumIterations(6)
    o = oracle_mod.GICP(max_correspondence_distance=5.0, transformation_epsilon=1e-8, max_iterations=6)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    o.set_target(tgt)
    o.set_source(src)
    Tg, To = g.align(), o.align()
    dt, dr = synth.pose_error(Tg, To)
    assert dt < 1e-3 and dr < 1e-3, (dt, dr)
    assert g.numCorrespondences() == o.num_correspondences()
    et, er = synth.pose_error(Tg, T_gt)
    assert et < 0.15 and er < 5e-3  # and it registers: close to the pose the scan was ray-cast from
