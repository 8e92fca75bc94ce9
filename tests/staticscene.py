"""The moving-object drive of the static-map tests: a sensor driving down synth.make_scene()'s canyon, one ray-cast submap
every STEP metres at its true pose, with two cars that are not part of the scene: one oncoming in the other lane while
submaps ONCOMING are taken, and one parked ahead of the start while submaps PARKED are taken, which then leaves. The drive
continues well past both. Every point carries a label: the car it hit, the ground, or the rest of the static scene."""
from __future__ import annotations

import numpy as np

from lidarslam_ros2_b200 import synth

N_SUB, STEP, X0, Y0 = 30, 1.5, -30.0, 3.0  # the street at y = 3 m is clear of the scene's boxes over the whole drive
RINGS, AZIMUTHS = 16, 625
ONCOMING = range(4, 21)
PARKED = range(0, 7)
STATIC, GROUND, CAR = 0, 1, 2
CAR_SIZE = (4.4, 1.8, 1.5)


def _car(xc, yc):
    lx, ly, lz = CAR_SIZE
    return [xc - lx / 2, yc - ly / 2, 0.0, xc + lx / 2, yc + ly / 2, lz]


def cars(k):
    """The car boxes present while submap k is taken (world frame)."""
    out = []
    if k in ONCOMING:
        out.append(_car(X0 + STEP * ONCOMING[0] + 25.0 - STEP * (k - ONCOMING[0]), Y0 - 4.6))
    if k in PARKED:
        out.append(_car(X0 + 12.0, Y0 + 3.0))
    return np.array(out, dtype=np.float64).reshape(-1, 6)


def pose(k):
    return synth.pose_matrix((X0 + STEP * k, Y0 + 0.15 * np.sin(0.3 * k), synth.SENSOR_HEIGHT), (0.0, 0.0, 0.01 * np.sin(0.5 * k)))


def drive():
    """Returns (scans, poses, labels): per submap the sensor-frame points (n, 4) float32 with the label in the fourth
    column, the true pose, and the labels (n,) int8."""
    scene = synth.make_scene()
    el = np.deg2rad(np.linspace(-25.0, 15.0, RINGS))
    az = np.arange(AZIMUTHS) * (2 * np.pi / AZIMUTHS)
    E, A = np.meshgrid(el, az, indexing="ij")
    ds = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], axis=-1).reshape(-1, 3)
    scans, poses, labels = [], [], []
    for k in range(N_SUB):
        P = pose(k)
        R, t = P[:3, :3], P[:3, 3]
        dw = ds @ R.T
        r_static = synth._ray_cast(scene, t, dw, 100.0)
        with_cars = synth.Scene(boxes=np.vstack([scene.boxes, cars(k)]), cylinders=scene.cylinders)
        r = synth._ray_cast(with_cars, t, dw, 100.0)
        car = r < r_static
        z_world = t[2] + r * dw[:, 2]
        lab = np.where(car, CAR, np.where(np.abs(z_world) < 0.05, GROUND, STATIC)).astype(np.int8)
        rn = r + 0.02 * synth.Rng(8800 + k).normal(len(r))
        keep = np.isfinite(rn) & (rn > 0.5)
        pts = np.zeros((int(keep.sum()), 4), dtype=np.float32)
        pts[:, :3] = ds[keep] * rn[keep, None]
        pts[:, 3] = lab[keep]
        scans.append(pts)
        poses.append(P)
        labels.append(lab[keep])
    return scans, poses, labels
