"""Global localisation in a prior map: the pose scorer b200reg_ndt_score_poses (csrc/ndt_score.cu) against the float64
reference tests/ndtref.py and against the solver's own derivative pass, its determinism (a pose's score does not depend on
the batch it is in), its error paths; and the session's b200sm_localize_global against the plain calls and the replay of
tests/globalref.py (grid, scores, choice, refinement and adoption bit for bit), its recovery from a pose metres off with
the heading wrong, and its limits. Run on an H100 with -m gpu."""
import math

import numpy as np
import pytest

import globalref as GR
import gridref as R
import localizeref as L
import ndtref as N
import test_gpu_localize as TL
from lidarslam_ros2_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
METHODS = [(2, "DIRECT7"), (3, "DIRECT1"), (1, "DIRECT26"), (0, "KDTREE")]
TILE, WARPS = 1024, 8  # SCORE_TILE and SCORE_WARPS of csrc/ndt_score.cu
SCAN_SIZES = (1, 31, 32, 33, TILE - 1, TILE, TILE + 1)
POSES6 = [np.zeros(6), np.array([0.21, -0.13, 0.04, 0.006, -0.004, 0.02]), np.array([-0.4, 0.3, -0.1, 0.05, 0.01, -0.3])]


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


@pytest.fixture(scope="module")
def pair():
    return synth.registration_pair("small", 2.0)[:2]


def _ndt(b200, tgt, src, method=2):
    g = b200.NormalDistributionsTransform()
    g.setResolution(2.0)
    g.setNeighborhoodSearchMethod(method)
    g.setInputTarget(tgt)
    g.setInputSource(src)
    return g


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64 if np.asarray(a).dtype.itemsize == 8 else np.uint32)


def _random_poses(n, seed, spread=(1.0, 0.3)):
    import oracle

    rng = np.random.default_rng(seed)
    out = np.zeros((n, 4, 4), dtype=F32)
    for k in range(n):
        p = np.concatenate([rng.uniform(-spread[0], spread[0], 3), rng.uniform(-spread[1], spread[1], 3)])
        out[k] = oracle.pose_to_matrix(p)
    return out


# ---- 1. scores against the reference and against the derivative pass ----------------------------------------------------
@pytest.mark.parametrize("method", [m for m, _ in METHODS], ids=[n for _, n in METHODS])
def test_scores_against_reference(b200, pair, method):
    import oracle

    src_all, tgt = pair
    worst = 0.0
    for n in SCAN_SIZES:
        src = np.ascontiguousarray(src_all[:n])
        g = _ndt(b200, tgt, src, method)
        vox, geom = g.voxels(), R.leaf_geometry(tgt, 2.0)
        Ts = np.stack([oracle.pose_to_matrix(p) for p in POSES6]).astype(F32)
        scores, hits = g.scorePoses(Ts)
        for k, p in enumerate(POSES6):
            ref = N.derivatives(src, Ts[k][:3], p, 2.0, vox, geom, method, compute_hessian=False)
            if ref["near_threshold"] == 0:
                assert hits[k] == ref["hits"], (n, k, hits[k], ref["hits"])
            tol = ref["tol_score"]
            assert abs(scores[k] - ref["score"]) <= tol or scores[k] == ref["score"], (n, k, scores[k], ref["score"], tol)
            if tol:
                worst = max(worst, abs(scores[k] - ref["score"]) / tol)
            s, _, _ = g.derivatives(Ts[k], p, False)
            assert g.stats()["hits"] == hits[k], (n, k)
            assert abs(s - scores[k]) <= 2 * tol or s == scores[k], (n, k, s, scores[k])
    print(f"\nmax |score - ref| / bound, method {method}: {worst:.3g}")


# ---- 2. determinism ---------------------------------------------------------------------------------------------------
def test_determinism(b200, pair):
    import torch

    src, tgt = pair
    g = _ndt(b200, tgt, src)
    n_ctas = torch.cuda.get_device_properties(0).multi_processor_count
    P = _random_poses(3000, 7)
    s_all, h_all = g.scorePoses(P)
    perm = np.random.default_rng(8).permutation(len(P))
    s_perm, h_perm = g.scorePoses(P[perm])
    assert np.array_equal(_bits(s_perm), _bits(s_all[perm])) and np.array_equal(h_perm, h_all[perm])
    s_again, h_again = g.scorePoses(P)
    assert np.array_equal(_bits(s_again), _bits(s_all)) and np.array_equal(h_again, h_all)
    for k in range(0, len(P), 150):  # alone
        s1, h1 = g.scorePoses(P[k:k + 1])
        assert _bits(s1)[0] == _bits(s_all)[k] and h1[0] == h_all[k], k
    for count in (1, WARPS - 1, WARPS, WARPS + 1, WARPS * n_ctas - 1, WARPS * n_ctas, WARPS * n_ctas + 1):
        s, h = g.scorePoses(P[:count])
        assert np.array_equal(_bits(s), _bits(s_all[:count])) and np.array_equal(h, h_all[:count]), count
    assert (h_all > 0).all() and np.unique(s_all).size > len(P) // 2


# ---- 3. error paths -----------------------------------------------------------------------------------------------------
def test_error_paths(b200, pair):
    import ctypes as C

    from lidarslam_ros2_b200 import _capi
    from lidarslam_ros2_b200.registration import B200RegError

    src, tgt = pair
    g = _ndt(b200, tgt, src)
    s, h = g.scorePoses(np.zeros((0, 4, 4), dtype=F32))
    assert len(s) == 0 and len(h) == 0
    bad = _random_poses(3, 1)
    bad[1, 0, 3] = np.nan
    for v in (np.nan, np.inf):
        bad[1, 0, 3] = v
        with pytest.raises(B200RegError) as e:
            g.scorePoses(bad)
        assert e.value.code == _capi.ERR_ARG
    lib = _capi.lib()
    P = np.ascontiguousarray(_random_poses(1, 2).transpose(0, 2, 1))
    out = np.zeros(1)
    gi = b200.GeneralizedIterativeClosestPoint()
    gi.setInputTarget(tgt)
    gi.setInputSource(src)
    assert lib.b200reg_ndt_score_poses(gi._h, 1, P.ctypes.data, out.ctypes.data, None) == _capi.ERR_ARG
    assert lib.b200reg_ndt_score_poses(g._h, -1, P.ctypes.data, out.ctypes.data, None) == _capi.ERR_ARG
    e0 = b200.NormalDistributionsTransform()
    assert lib.b200reg_ndt_score_poses(e0._h, 1, P.ctypes.data, out.ctypes.data, None) == _capi.ERR_NO_TARGET
    e0.setInputTarget(tgt)
    assert lib.b200reg_ndt_score_poses(e0._h, 1, P.ctypes.data, out.ctypes.data, None) == _capi.ERR_NO_SOURCE
    assert lib.b200reg_ndt_score_poses(e0._h, 0, None, None, None) == _capi.OK
    # no voxel holds 6 points: every score and hit count is 0
    sparse = _ndt(b200, tgt[::400][:40] * F32(30.0), src)
    assert sparse.voxels()["idx"].size == 0
    s, h = sparse.scorePoses(_random_poses(5, 3))
    assert np.array_equal(s, np.zeros(5)) and np.array_equal(h, np.zeros(5, dtype=np.int64))
    assert np.array_equal(out, np.zeros(1)) and C.sizeof(C.c_longlong) == 8


# ---- 4. the session against the plain calls --------------------------------------------------------------------------------
def _start(T_true, offset, dyaw):
    yaw = math.atan2(float(T_true[1, 0]), float(T_true[0, 0])) + dyaw
    pos = [float(T_true[0, 3]) + offset[0], float(T_true[1, 3]) + offset[1], float(T_true[2, 3])]
    return pos, (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))


def test_session_against_plain_calls(world_g):
    sm, prior, frames = world_g
    scan, T_true = frames[2]
    pos, quat = _start(T_true, (1.5, -1.0), 0.4)
    radius, step, yaw_steps, top_k = 3.0, 1.0, 8, 5
    g = TL._session(sm, prior)
    g.setInitialPose(pos, quat)
    best, cand, rows, info = g.localizeGlobal(scan, radius, step, yaw_steps, top_k)
    poses, scores, hits = g.globalSearch()
    want = GR.grid(pos, quat, radius, step, yaw_steps)
    assert info["n_hypotheses"] == len(want) == len(scores) and info["n_refined"] == top_k == len(rows)
    assert np.array_equal(_bits(poses), _bits(want))
    assert info["hits_total"] == int(hits.sum()) and info["score_ms"] > 0
    plain = TL._plain(sm, "NDT")
    plain.setInputTarget(g.cutCloud())
    plain.setInputSource(g.filteredScan())
    s2, h2 = plain.scorePoses(poses)
    assert np.array_equal(_bits(s2), _bits(scores)) and np.array_equal(h2, hits)
    assert cand.tolist() == GR.select(scores, top_k)
    for r, row in enumerate(rows):
        final = plain.align(poses[cand[r]])
        assert np.array_equal(_bits(row["final"]), _bits(final)), r
        assert row["converged"] == plain.hasConverged() and row["trans_probability"] == plain.getTransformationProbability(), r
    assert best == L.choose_hypothesis([(r["converged"], r["trans_probability"], r["status"]) for r in rows])
    # the rows are localizeInit's for the same guesses
    g2 = TL._session(sm, prior)
    g2.setInitialPose(pos, quat)
    b2, rows2 = g2.localizeInit(scan, poses[cand])
    assert b2 == best and all(np.array_equal(_bits(a["final"]), _bits(b["final"])) and
                              a["trans_probability"] == b["trans_probability"] for a, b in zip(rows, rows2))
    # the next frame starts from the adopted pose
    loc = L.Localizer(prior, TL.CROP, 1e9, position=pos, quat_xyzw=quat)
    assert loc.begin()
    if best >= 0:
        loc.adopt_pose(rows[best]["final"])
    g.setLocalizationParams(TL.CROP, 1e9)
    _, final, _ = g.localizeCloud(frames[3][0])
    plain.setInputTarget(g.cutCloud())
    plain.setInputSource(g.filteredScan())
    assert np.array_equal(_bits(final), _bits(plain.align(loc.sim_trans())))


@pytest.fixture(scope="module")
def world_g():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    from lidarslam_ros2_b200 import scanmatcher

    return scanmatcher, TL.canyon_map(), TL.drive(6)


# ---- 5. recovery ----------------------------------------------------------------------------------------------------------
RECOVERY = ((6.0, -4.0), math.radians(120.0), 10.0, 1.0, 72)  # offset, heading error, radius, step, yaw_steps


def test_recovery_from_metres_off_and_a_wrong_heading(world_g):
    """tests/test_localize_global_fixture_cpu.py checks on the CPU that the hypothesis nearest the truth scores highest here."""
    sm, prior, frames = world_g
    scan, T_true = frames[2]
    offset, dyaw, radius, step, yaw_steps = RECOVERY
    pos, quat = _start(T_true, offset, dyaw)
    g = TL._session(sm, prior)
    g.setInitialPose(pos, quat)
    best, cand, rows, info = g.localizeGlobal(scan, radius, step, yaw_steps, 8)
    assert info["n_hypotheses"] > 300 * 72
    assert best >= 0
    dt, dr = synth.pose_error(rows[best]["final"], T_true)
    print(f"\nrecovery: best row {best} (hypothesis {cand[best]}), dt {dt:.4f} m, dr {dr:.5f} rad, "
          f"{info['n_hypotheses']} hypotheses scored in {info['score_ms']:.3f} ms")
    assert dt < 0.3 and dr < 0.02, (dt, dr)


# ---- 6. errors and limits ---------------------------------------------------------------------------------------------------
def test_errors_and_limits(world_g):
    """After every refused call the pose, the cut and the engine's target are what they were. The pose is read through a
    radius-0 search, whose only hypothesis is the pose itself (GICP: through the next localizeCloud frame, bitwise that of a
    fresh session started at the same pose)."""
    from lidarslam_ros2_b200.registration import B200RegError

    sm, prior, frames = world_g
    scan, T_true = frames[2]
    E = sm._capi
    pos, quat = _start(T_true, (0.5, -0.5), 0.0)

    def pose_is(g, p, q):
        g.localizeGlobal(scan, 0.0, 1.0, 1, 1)  # adopts a pose: callers set theirs again afterwards
        return np.array_equal(_bits(g.globalSearch()[0]), _bits(GR.grid(p, q, 0.0, 1.0, 1)))

    g = TL._session(sm, None)
    g.setInitialPose(pos, quat)
    with pytest.raises(B200RegError) as e:
        g.localizeGlobal(scan, 1.0, 1.0, 4, 2)
    assert e.value.code == E.ERR_NO_TARGET
    g.setPriorMap(prior)  # leaves the pose alone
    assert pose_is(g, pos, quat)
    g.setInitialPose(pos, quat)
    g.localizeCloud(scan)  # a cut and a target to keep
    g.setInitialPose(pos, quat)
    g.localizeCloud(scan)
    g.setInitialPose(pos, quat)
    cut0, st0, n_t0 = g.cutCloud(), g.localizeStats(), g.registration.stats()["n_target"]
    for spec in ((math.nan, 1.0, 4, 2), (-1.0, 1.0, 4, 2), (1.0, 0.0, 4, 2), (1.0, math.inf, 4, 2), (1.0, 1.0, 0, 2),
                 (1.0, 1.0, 4097, 2), (1.0, 1.0, 4, 0), (1.0, 1.0, 4, 1025), (4097.0, 1.0, 1, 1), (100.0, 0.1, 72, 8)):
        with pytest.raises(B200RegError) as e:
            g.localizeGlobal(scan, *spec)
        assert e.value.code == E.ERR_ARG, spec
        assert np.array_equal(_bits(g.cutCloud()), _bits(cut0)) and g.localizeStats() == st0, spec
        assert g.registration.stats()["n_target"] == n_t0, spec
    assert pose_is(g, pos, quat)
    # a GICP handle: refused before anything changes, so the next frame is that of a session that never made the call
    gi, fresh = TL._session(sm, prior, "GICP"), TL._session(sm, prior, "GICP")
    for s_ in (gi, fresh):
        s_.setInitialPose(pos, quat)
    with pytest.raises(B200RegError) as e:
        gi.localizeGlobal(scan, 1.0, 1.0, 4, 2)
    assert e.value.code == E.ERR_ARG
    assert gi.localizeStats()["n_cuts"] == 0
    pa, Ta, _ = gi.localizeCloud(scan)
    pb, Tb, _ = fresh.localizeCloud(scan)
    assert np.array_equal(pa, pb) and np.array_equal(_bits(Ta), _bits(Tb))
    # No converged row (best = -1) cannot be produced through the NDT solver: it reports a registration converged once it
    # has used up its iterations, so even a one-iteration refinement from far off gives converged rows; only a status
    # failure of the batch launch would leave every row out. The choice is still the replay's.
    g.registration.setMaximumIterations(1)
    far = _start(T_true, (3.0, 2.0), 0.3)
    g.setInitialPose(*far)
    best, _, rows, _ = g.localizeGlobal(scan, 0.0, 1.0, 1, 1)
    assert all(r["converged"] and r["status"] == 0 for r in rows)
    assert best == L.choose_hypothesis([(r["converged"], r["trans_probability"], r["status"]) for r in rows]) == 0
