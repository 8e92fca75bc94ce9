import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def golden(golden_dir):
    import json

    import numpy as np

    with open(os.path.join(golden_dir, "golden.json")) as f:
        g = json.load(f)
    g["target"] = np.load(os.path.join(golden_dir, "pcd_target_ds.npy"))
    g["source"] = np.load(os.path.join(golden_dir, "pcd_source_ds.npy"))
    g["raw"] = np.load(os.path.join(golden_dir, "pcd_source_raw_head.npy"))
    return g


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle

    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def pair_tiny():
    from lidarslam_ros2_b200 import synth

    return synth.registration_pair("tiny", 2.0)


@pytest.fixture(scope="session")
def pair_small():
    from lidarslam_ros2_b200 import synth

    return synth.registration_pair("small", 2.0)
