"""tests/cpp/adapter_octomap.cpp: the OctoMap methods of b200reg::ScanMatcherSession (include/b200reg_pcl.hpp) build
against the C-ABI; without a GPU the program refuses to run (exit code 3), on the H100 it builds the OctoMap of a corridor
and saves it as a .bt file."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    """Into out_dir (a temporary directory: the tree may be read-only)."""
    exe = os.path.join(out_dir, "adapter_octomap")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "adapter_octomap.cpp"), "-o", exe,
                           "-L" + os.path.join(ROOT, "lidarslam_ros2_b200", "csrc"), "-lb200reg",
                           "-Wl,-rpath," + os.path.join(ROOT, "lidarslam_ros2_b200", "csrc")])
    return exe


def test_adapter_builds_and_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("covered by the gpu test")
    with tempfile.TemporaryDirectory() as tmp:
        out = subprocess.run([_build(tmp), tmp], capture_output=True, text=True)
    assert out.returncode == 3 and "no CUDA device" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_adapter_octomapes_a_corridor():
    with tempfile.TemporaryDirectory() as tmp:
        out = subprocess.run([_build(tmp), tmp], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
