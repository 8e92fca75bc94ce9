"""lidarslam_ros2_b200 — H100-native scan registration behind lidarslam_ros2's pcl::Registration surface.

Only what the hot path needs lives here: csrc/ (hand-written sm_90a CUDA kernels + the C-ABI of
include/b200reg.h) and the host-side mirror of the reference's registration interface (registration.py).
"""
from ._capi import DIRECT1, DIRECT7, DIRECT26, KDTREE, LIB_PATH, build  # noqa: F401
from .pcd import encode_pcd_ascii, read_pcd  # noqa: F401
from .registration import (  # noqa: F401
    B200RegError,
    GeneralizedIterativeClosestPoint,
    NormalDistributionsTransform,
    align_batch,
    voxel_grid_filter,
)
