"""GICP's k-NN covariances (K5, gicp_cov_kernel) point by point against the float64 reference of tests/covref.py, on
every point of source and target, with no point exempt: at the c3 sizes, on the surface pair, and on fixtures built to
reach K5's edges (far-face ring stops, tied k-th neighbours, zero and rank-deficient covariances, non-finite rows, km
offsets, clouds of k, k + 1 and 2k points), for k in {3, 4, 20, 31, 32} and gicp_epsilon in {1e-3, 0.25}. Also the
k / epsilon setters and the per-cloud cache, and the exact-NN ring search of nearest(), getFitnessScore and the
correspondence pass (K8, K6) on the far-face fixtures, against brute force. Run on an H100 with -m gpu."""
import numpy as np
import pytest

import covref as CR
import gridref as GR

pytestmark = pytest.mark.gpu

F32 = np.float32
KS = (3, 4, 20, 31, 32)


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


def _handle(b200, target, source, k=20, eps=None):
    g = b200.GeneralizedIterativeClosestPoint()
    g.setCorrespondenceRandomness(k)
    if eps is not None:
        g.setEpsilon(eps)
    g.setInputTarget(target)
    g.setInputSource(source)
    g.correspondences()  # align()'s prelude computes both clouds' covariances
    return g


def _failures(got, cloud, k, eps, what, log):
    ref, info = CR.reference(cloud, k, eps)
    assert got.shape == ref.shape, what
    bad, ratio, n_inv = CR.check(got, ref, info)
    log.append((what, ratio, n_inv, int(bad.sum())))
    return [(what, int(bad.sum()), np.flatnonzero(bad)[:6].tolist())] if bad.any() else []


@pytest.mark.parametrize("eps", [1e-3, 0.25])
@pytest.mark.parametrize("k", KS)
def test_k5_fixtures_every_point(b200, k, eps):
    log, fails = [], []
    for name, c in CR.cov_fixtures(k).items():
        g = _handle(b200, c, c, k, eps)
        for which in ("target", "source"):
            fails += _failures(g.covariances(which), c, k, eps, (name, which), log)
    worst = max(log, key=lambda r: r[1])
    print(f"k={k} eps={eps}: worst |dcov|/bound {worst[1]:.3g} at {worst[0]}, invariant-checked points "
          f"{sum(r[2] for r in log)}")
    assert not fails, fails


def test_k5_c3_sizes_and_surface_pair(b200):
    from lidarslam_ros2_b200 import synth
    import gicpref

    scenes = {"surface": gicpref.surface_pair()}
    src, tgt, _ = synth.registration_pair("headline", 2.0)
    scenes["c3"] = (np.ascontiguousarray(src[:, :3]), np.ascontiguousarray(tgt[:, :3]))
    assert len(scenes["c3"][1]) >= 1_000_000 and len(scenes["c3"][0]) >= 90_000
    log, fails = [], []
    for name, (s, t) in scenes.items():
        g = _handle(b200, t, s)
        for which, c in (("target", t), ("source", s)):
            fails += _failures(g.covariances(which), c, 20, 1e-3, (name, which), log)
    for r in log:
        print(f"{r[0]}: worst |dcov|/bound {r[1]:.3g}, invariant-checked points {r[2]}")
    assert not fails, fails


def test_k5_nonfinite_rows_change_nothing(b200):
    clean = CR.scene(2000, seed=8)
    bad, ok = GR.with_nonfinite_rows(clean, seed=8)
    bad = np.ascontiguousarray(bad[:, :3])
    for k in (3, 20, 32):
        cb = _handle(b200, bad, bad, k).covariances("target")
        cc = _handle(b200, clean, clean, k).covariances("target")
        np.testing.assert_array_equal(cb[ok], cc, err_msg=str(k))
        assert np.isfinite(cb[~ok]).all(), k


def test_k5_setters_and_cache(b200):
    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    g = b200.GeneralizedIterativeClosestPoint()
    for k in (2, 33):
        with pytest.raises(B200RegError) as e:
            g.setCorrespondenceRandomness(k)
        assert e.value.code == _capi.ERR_ARG
    rng = np.random.default_rng(5)
    t = CR.scene(3000, seed=5)
    srcs = [(t[rng.choice(len(t), 1500, replace=False)] + rng.normal(0, 0.01, (1500, 3))).astype(F32) for _ in range(3)]
    g.setInputTarget(t)
    launches = []

    def run(s, k, eps):
        g.setInputSource(s)
        before = g.stats()["kernel_launches"]
        g.correspondences()
        launches.append(g.stats()["kernel_launches"] - before)
        fails = _failures(g.covariances("target"), t, k, eps, ("target", k, eps), [])
        fails += _failures(g.covariances("source"), s, k, eps, ("source", k, eps), [])
        assert not fails, fails

    run(srcs[0], 20, 1e-3)
    run(srcs[1], 20, 1e-3)  # a new source alone: the target's covariances stay cached
    run(srcs[2], 20, 1e-3)
    g.setCorrespondenceRandomness(7)
    run(srcs[1], 7, 1e-3)  # both clouds recomputed for the new k
    g.setEpsilon(0.25)
    run(srcs[2], 7, 0.25)  # and for the new epsilon
    assert launches[1] == launches[2] and launches[3] == launches[1] + 1 == launches[4], launches


def _far_face_targets():
    out = {"1nn": CR.far_face_case("1nn"), "gated": CR.far_face_gated()}
    out.update({("knn", k): CR.far_face_case("knn", k) for k in (3, 20, 32)})
    return out


def test_far_face_nearest_fitness_correspondences(b200):
    cases = _far_face_targets()
    for name, f in cases.items():
        g = b200.GeneralizedIterativeClosestPoint()
        g.setInputTarget(f["target"])
        idx, d2 = g.nearest(f["query"])
        ri, rd = GR.nn1_ref(f["target"], f["query"])
        if name == "1nn":
            assert ri[0] == f["want"]
        assert idx[0] == ri[0] and d2[0] == rd[0], (name, idx, ri, d2, rd)
        g.setInputSource(f["query"])
        assert g.getFitnessScore() == float(rd[0]), name
    f = cases["gated"]
    dB = float(f["d2"])
    g = b200.GeneralizedIterativeClosestPoint()
    g.setInputTarget(f["target"])
    g.setInputSource(f["query"])
    # max_range = d2(q, B) exactly: inclusive, and its 1.0001 search slack stays below h^2 0.99999
    assert g.getFitnessScore(dB) == dB
    assert g.getFitnessScore(float(np.nextafter(F32(dB), F32(0)))) != dB
    corr_dist = float(np.sqrt(dB)) * (1 + 1e-12)
    assert dB < corr_dist * corr_dist and F32(F32(corr_dist * corr_dist) * F32(1.0001)) < CR.ring_b2(1, f["geometry"], "old")
    g.setMaxCorrespondenceDistance(corr_dist)
    corr, _, m = g.correspondences()
    assert m == 1 and corr[0] == f["want"], (corr, m)


def test_face_queries_up_to_the_last_cell(b200):
    targets = {name: f["target"] for name, f in _far_face_targets().items()}
    targets["corridor"] = CR.corridor()
    targets["line"] = np.c_[np.random.default_rng(9).uniform(-5, 5, 400), np.zeros(400), np.zeros(400)].astype(F32)
    for name, t in targets.items():
        q = CR.face_queries(t, seed=3)
        assert len(q), name
        g = b200.GeneralizedIterativeClosestPoint()
        g.setInputTarget(t)
        idx, d2 = g.nearest(q)
        ri, rd = GR.nn1_ref(t, q)
        bad = (idx != ri) | (d2 != rd)
        assert not bad.any(), (name, int(bad.sum()), np.flatnonzero(bad)[:5])
