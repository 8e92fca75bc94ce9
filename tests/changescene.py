"""The two-day drive of the map-change tests: two recordings of synth.make_scene()'s canyon, built like staticscene's
moving-object drive (one ray-cast submap every STEP metres at its true pose).

  day 1  a car is parked beside the street for the whole drive;
  day 2  the drive runs 0.4 m further to the side with a different pose wobble; the parked car is gone, a 2 x 2 x 2.5 m
         container stands elsewhere beside the street, and an oncoming car passes in the other lane.

Every point carries a label: the static scene, the ground, the car that vanished, the container that appeared, or the
passing car."""
from __future__ import annotations

import numpy as np

from lidarslam_ros2_b200 import synth

N_SUB, STEP, X0, Y0 = 30, 1.5, -30.0, 3.0  # the street at y = 3 m is clear of the scene's boxes over the whole drive
DAY2_SHIFT = 0.4
RINGS, AZIMUTHS = 16, 625
STATIC, GROUND, VANISHED_CAR, CONTAINER, TRANSIENT = 0, 1, 2, 3, 4
PARKED = [-18.2, 5.3, 0.0, -13.8, 7.1, 1.5]      # day 1: 4.4 x 1.8 x 1.5 m, the whole drive
CONTAINER_BOX = [0.0, 6.0, 0.0, 2.0, 8.0, 2.5]  # day 2: 2 x 2 x 2.5 m
ONCOMING = range(4, 21)                          # day 2: the submaps the oncoming car is seen in


def objects(day, k):
    """(label, box) of the objects that are not part of the scene while submap k of `day` (1 or 2) is taken."""
    if day == 1:
        return [(VANISHED_CAR, PARKED)]
    out = [(CONTAINER, CONTAINER_BOX)]
    if k in ONCOMING:
        xc = X0 + STEP * ONCOMING[0] + 25.0 - STEP * (k - ONCOMING[0])
        yc = Y0 + DAY2_SHIFT - 4.6
        out.append((TRANSIENT, [xc - 2.2, yc - 0.9, 0.0, xc + 2.2, yc + 0.9, 1.5]))
    return out


def pose(day, k):
    if day == 1:
        return synth.pose_matrix((X0 + STEP * k, Y0 + 0.15 * np.sin(0.3 * k), synth.SENSOR_HEIGHT), (0.0, 0.0, 0.01 * np.sin(0.5 * k)))
    return synth.pose_matrix((X0 + STEP * k + 0.3, Y0 + DAY2_SHIFT + 0.12 * np.sin(0.4 * k + 1.3), synth.SENSOR_HEIGHT + 0.02),
                             (0.0, 0.0, 0.012 * np.sin(0.7 * k + 2.0)))


def day(d):
    """Recording d (1 or 2): (scans, poses, labels), per submap the sensor-frame points (n, 4) float32 with the label in the
    fourth column, the true pose, and the labels (n,) int8."""
    scene = synth.make_scene()
    el = np.deg2rad(np.linspace(-25.0, 15.0, RINGS))
    az = np.arange(AZIMUTHS) * (2 * np.pi / AZIMUTHS)
    E, A = np.meshgrid(el, az, indexing="ij")
    ds = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], axis=-1).reshape(-1, 3)
    scans, poses, labels = [], [], []
    for k in range(N_SUB):
        P = pose(d, k)
        R, t = P[:3, :3], P[:3, 3]
        dw = ds @ R.T
        r = synth._ray_cast(scene, t, dw, 100.0)
        lab = np.where(np.abs(t[2] + r * dw[:, 2]) < 0.05, GROUND, STATIC).astype(np.int8)
        for name, box in objects(d, k):
            rb = synth._ray_cast(synth.Scene(boxes=np.vstack([scene.boxes, [box]]), cylinders=scene.cylinders), t, dw, 100.0)
            nearer = rb < r
            lab[nearer] = name
            r = np.minimum(r, rb)
        rn = r + 0.02 * synth.Rng(9100 + 100 * d + k).normal(len(r))
        keep = np.isfinite(rn) & (rn > 0.5)
        pts = np.zeros((int(keep.sum()), 4), dtype=np.float32)
        pts[:, :3] = ds[keep] * rn[keep, None]
        pts[:, 3] = lab[keep]
        scans.append(pts)
        poses.append(P)
        labels.append(lab[keep])
    return scans, poses, labels
