"""The replay of the localising frontend (tests/localizeref.py) on the CPU: it is self-consistent on the fixtures the GPU
tests use (tests/test_gpu_localize.py), and every named mutation of it — a subtly wrong session — changes an outcome on
those fixtures, so the GPU tests that compare the device with the replay on them can tell such a session from the right one."""
import math

import numpy as np

import localizeref as L
import test_gpu_localize as G
from lidarslam_ros2_b200 import synth

F32 = np.float32


def _replay(prior, poses, recrop, mut=()):
    """The drive with the ground-truth poses (cast to float, as align() returns them) standing in for the device's finals."""
    loc = L.Localizer(prior, G.CROP, recrop, position=(G.X_START, 0.0, 0.0))
    recs = [loc.frame(T.astype(F32), mut) for T in poses]
    return loc, recs


def _world():
    prior = G.canyon_map()
    d = math.pi / 180.0
    poses = []
    for k in range(G.N_FRAMES):  # synth.drive_stream's poses in the map frame, without ray-casting the scans
        yaw = 1.0 * d * math.sin(2.0 * math.pi * k / 40.0)
        poses.append(synth.pose_matrix((G.X_START + G.STEP * k, 0.3 * math.sin(2.0 * math.pi * k / 60.0), 0.0), (0.0, 0.0, yaw)))
    return prior, poses


def test_drive_poses_are_the_fixture_drive():
    _, poses = _world()
    got = G.drive(3)
    for k in range(3):
        assert np.allclose(got[k][1], poses[k], atol=1e-12)


def test_replay_of_the_drive():
    prior, poses = _world()
    loc, recs = _replay(prior, poses, G.RECROP)
    assert loc.n_cuts >= 3 and all(r is not None for r in recs)
    recut_frames = [k for k, r in enumerate(recs) if r["recut"]]
    assert [k for k, _ in loc.adopted_at] == [0] + [k + 1 for k in recut_frames if k + 1 < len(recs)]
    for k, r in enumerate(recs):
        assert r["recut"] == (r["dist"] >= G.RECROP)
        assert np.array_equal(r["pose7"][:3], poses[k].astype(F32)[:3, 3].astype(np.float64))
    # the cut follows the pose: its rows are within the radius of its centre, and it is a strict subset of the map
    cut = loc.cut()
    d = np.hypot(cut[:, 0].astype(np.float64) - loc.centre[0], cut[:, 1].astype(np.float64) - loc.centre[1])
    assert 0 < len(cut) < len(prior) and d.max() <= G.CROP * (1 + 1e-12)


def test_recut_at_equality_and_its_mutation():
    prior, poses = _world()
    _, free = _replay(prior, poses[:4], 1e9)
    d = free[2]["dist"]
    assert free[1]["dist"] < d
    _, at = _replay(prior, poses[:4], d)
    assert [r["recut"] for r in at[:3]] == [False, False, True]
    _, above = _replay(prior, poses[:3], math.nextafter(d, 1e9))
    assert not any(r["recut"] for r in above)
    _, mut = _replay(prior, poses[:4], d, mut={"recut_gt"})
    assert [r["recut"] for r in mut[:3]] == [False, False, False]


def test_adoption_timing_mutation():
    prior, poses = _world()
    loc, _ = _replay(prior, poses, G.RECROP)
    bad, _ = _replay(prior, poses, G.RECROP, mut={"adopt_same_frame"})
    assert loc.adopted_at != bad.adopted_at and [c for _, c in loc.adopted_at] == [c for _, c in bad.adopted_at][:len(loc.adopted_at)]


def test_cut_mutations_show_on_the_edge_maps():
    prior = G.edge_map(G.TILE + 1, "mixed")
    right = L.cut_mask(prior, *G.CENTRE, G.RADIUS)
    assert right[3] and right[5] and not right[7] and right[9]
    lt = L.cut_mask(prior, *G.CENTRE, G.RADIUS, mut={"radius_lt"})
    assert not lt[3] and not lt[5] and np.array_equal(np.delete(lt, [3, 5]), np.delete(right, [3, 5]))
    z = L.cut_mask(prior, *G.CENTRE, G.RADIUS, mut={"with_z"})
    assert z.sum() < right.sum() and right[15] and not z[15]  # a NaN z is ignored by the right cut only
    cx, cy, r = G.fused_case()
    assert L.cut_mask(prior, cx, cy, r)[23] and not L.cut_mask(prior, cx, cy, r, mut={"fused"})[23]
    # non-finite x or y never pass
    assert not right[[11, 13, 17, 19]].any()


def test_cut_mutations_show_on_the_canyon_map():
    prior = G.canyon_map()
    right = L.cut_mask(prior, G.X_START, 0.0, G.CROP)
    assert L.cut_mask(prior, G.X_START, 0.0, G.CROP, mut={"with_z"}, cz=0.0).sum() < right.sum()


def test_hypothesis_choice_and_its_mutation():
    rows = [(True, 2.5, 0), (True, 3.0, 0), (False, 9.0, 0), (True, 3.0, 0), (True, 9.5, -5)]
    assert L.choose_hypothesis(rows) == 1 and L.choose_hypothesis(rows, mut={"tie_last"}) == 3
    assert L.choose_hypothesis([(False, 1.0, 0), (True, 2.0, -5)]) == -1
    same = [(True, 4.0, 0)] * 3  # the equal hypotheses of the GPU test
    assert L.choose_hypothesis(same) == 0 and L.choose_hypothesis(same, mut={"tie_last"}) == 2


def test_every_mutation_is_covered():
    import inspect

    src = inspect.getsource(inspect.getmodule(test_every_mutation_is_covered))
    for m in L.MUTATIONS:
        assert f'"{m}"' in src, m


def test_empty_first_cut():
    prior, _ = _world()
    loc = L.Localizer(prior, G.CROP, G.RECROP, position=(1000.0, 0.0, 0.0))
    assert loc.frame(np.eye(4, dtype=F32)) is None and loc.n_cuts == 0 and not loc.have_cut
