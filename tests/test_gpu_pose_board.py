"""GPU tests of the pose board (include/b200comm.h, b200reg_ndt_attach_pose_board): the batched NDT launch publishes its
poses to every rank's board from inside the solver kernel. The gathered poses must be BITWISE the poses the batch call
returns (they are the same 16 floats), on one GPU (world 1: the stores go to the rank's own board) and — when the box
has two GPUs — across two processes over NVLink peer memory."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def b200():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("no CUDA device: the gpu tests need an H100 (there is no CPU fallback)")
    import lidarslam_ros2_b200 as m

    return m


def _problem(m, n):
    from lidarslam_ros2_b200 import synth

    src, tgt, _ = synth.registration_pair("small", 2.0)
    rng = np.random.default_rng(11)
    scans = []
    for k in range(n):
        s = src[rng.random(len(src)) < (1.0 - 0.05 * (k % 3))][:, :3].copy()
        s += rng.normal(0, 0.004, size=s.shape).astype(np.float32)
        scans.append(np.ascontiguousarray(s))
    g = m.NormalDistributionsTransform()
    g.setResolution(2.0)
    g.setTransformationEpsilon(0.01)
    g.setNeighborhoodSearchMethod(m.DIRECT7)
    g.setInputTarget(tgt)
    return g, scans


def test_board_world1_matches_batch_results(b200):
    from lidarslam_ros2_b200 import batch

    g, scans = _problem(b200, 7)
    plain = g.alignBatch(scans)
    comm = batch.RowComm(0, 1, 0)
    board = comm.create_board(16)
    g.attachPoseBoard(board)
    for rep in range(3):  # the tag advances, both parities of the double buffer are used
        n = 7 - 2 * rep
        r = g.alignBatch(scans[:n])
        poses, counts = g.gatheredPoses()
        assert counts.tolist() == [n]
        assert poses.shape == (1, n, 4, 4)
        assert np.array_equal(poses[0], r["pose"])
        assert np.array_equal(r["pose"], plain["pose"][:n])  # and attaching a board does not change the registration
    # the prepared form of the call carries the gathered poses itself
    call = g.prepareBatch(scans[:5])
    for _ in range(2):
        r = call()
        assert r["gathered_counts"].tolist() == [5]
        assert np.array_equal(r["gathered"][0, :5], r["pose"])
    # too many registrations for the board: refused, nothing launched
    with pytest.raises(Exception):
        g.alignBatch(scans * 3)
    g.attachPoseBoard(None)
    with pytest.raises(Exception):
        g.gatheredPoses()
    assert np.array_equal(g.alignBatch(scans)["pose"], plain["pose"])
    board.close()


def test_board_two_ranks_over_nvlink(b200):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (tools/multi_gpu_check.sh 2 runs it on a 2-GPU box)")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tools", "check_pose_board.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "pose board ok" in p.stdout
