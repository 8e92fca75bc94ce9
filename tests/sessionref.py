"""TEST INFRASTRUCTURE. A float64 replay of the frontend session around align() (csrc/scanmatcher.cu, b200sm_*), driven by
what the device hands back: its `final` of every frame, its submap clouds and poses read back. Written from the reference
(scanmatcher/src/scanmatcher_component.cpp = sm.cpp, graph_based_slam/src/graph_based_slam_component.cpp = gbs.cpp) and
from Eigen's formulas, one scalar operation at a time. Python floats and numpy float32 / float64 elementwise arithmetic are
IEEE and un-fused, so every expression below is evaluated exactly as written, and the session's arithmetic is deterministic
given those inputs: the tests compare the device with this replay bit for bit.

  range_keep            cloud_callback's range filter (sm.cpp:211-219)
  quat_from_rot         Eigen::Quaterniond(Matrix3d), publishMapAndPose (sm.cpp:396-398)
  pose_matrix           tf2::fromMsg(pose, Affine3d) = Translation3d * Quaterniond(...).toRotationMatrix()
  Bookkeeping           publishMapAndPose's position / quaternion / trans / update decision (sm.cpp:391-434),
                        updateMap's latest_distance_ += trans_ (:474), getTransformation (:493-499), initializeMap
  targeted              updateMap's targeted cloud (sm.cpp:438-463)
  loop_candidates, closest, window, loop_target, relative_pose, shard
                        searchLoop (gbs.cpp:144-258) and b200sm_search_loop_all's dealing of the candidates

Every function takes `mut`, a set of mutation names (MUTATIONS): a replay of a subtly wrong session, used by
tests/test_sessionref_cpu.py to show that the fixtures tell such a session from the right one.
Nothing here needs a GPU.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32

MUTATIONS = (
    "update_gt",       # `>` instead of `>=` in the map-update decision (sm.cpp:423)
    "travel_ge",       # `>=` instead of `>` on the travelled distance (gbs.cpp:195)
    "range_le",        # `<=` instead of `<` on the search range (gbs.cpp:196)
    "last_wins",       # `<=` instead of `<` when picking the closest candidate: the last one wins a tie (gbs.cpp:199)
    "upper_unchecked",  # only the negative window indices skipped (gbs.cpp:210; b200reg.h skips both ends)
    "f64_reassoc",     # transform_f64 summed right to left, m0 x + (m1 y + (m2 z + m3))
    "f64_fused",       # transform_f64 with one rounding per coordinate (a fused dot product)
    "rel_full_inverse",  # relative_pose with the general 4x4 inverse instead of Isometry's R^T, -R^T t
    "hypot",           # np.hypot instead of sqrt(x * x + y * y) in the range filter
)


# ---- cloud callback -------------------------------------------------------------------------------------------------
def range_keep(cloud, rmin, rmax, mut=()) -> np.ndarray:
    """sm.cpp:213-215: r = sqrt(pow(x, 2.0) + pow(y, 2.0)) in double (pow(v, 2.0) is v * v exactly), kept when
    rmin < r < rmax. NaN rows fail both comparisons. Returns the boolean mask; the device keeps the same rows as a set
    (its warp-aggregated append reorders them)."""
    c = np.asarray(cloud, dtype=F32)
    x, y = c[:, 0].astype(np.float64), c[:, 1].astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.hypot(x, y) if "hypot" in mut else np.sqrt(x * x + y * y)
        return (rmin < r) & (r < rmax)


# ---- pose arithmetic ------------------------------------------------------------------------------------------------
def quat_from_rot(R) -> list:
    """Eigen::Quaterniond(Matrix3d) (quaternionbase_assign_impl<3x3>): the trace branch, else the largest diagonal i with
    j = i + 1, k = j + 1 (mod 3). Returns [x, y, z, w] as Python floats."""
    m = [[float(R[r][c]) for c in range(3)] for r in range(3)]
    q = [0.0, 0.0, 0.0, 0.0]
    t = (m[0][0] + m[1][1]) + m[2][2]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (m[2][1] - m[1][2]) * t
        q[1] = (m[0][2] - m[2][0]) * t
        q[2] = (m[1][0] - m[0][1]) * t
    else:
        i = 0
        if m[1][1] > m[0][0]:
            i = 1
        if m[2][2] > m[i][i]:
            i = 2
        j = (i + 1) % 3
        k = (j + 1) % 3
        t = math.sqrt(((m[i][i] - m[j][j]) - m[k][k]) + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (m[k][j] - m[j][k]) * t
        q[j] = (m[j][i] + m[i][j]) * t
        q[k] = (m[k][i] + m[i][k]) * t
    return q


def pose_matrix(position, quat_xyzw) -> np.ndarray:
    """Translation3d(p) * Quaterniond(w, x, y, z): Eigen's toRotationMatrix, 4x4 float64."""
    x, y, z, w = (float(v) for v in quat_xyzw)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy, float(position[0])],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx, float(position[1])],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy), float(position[2])],
                     [0.0, 0.0, 0.0, 1.0]])


def distance3(a, b) -> float:
    """(a - b).norm() of two Vector3d: sqrt((dx * dx + dy * dy) + dz * dz)."""
    dx, dy, dz = float(a[0]) - float(b[0]), float(a[1]) - float(b[1]), float(a[2]) - float(b[2])
    return math.sqrt((dx * dx + dy * dy) + dz * dz)


class Bookkeeping:
    """The ScanMatcherComponent members the session keeps on the host: the pose of the last frame, previous_position_,
    latest_distance_, trans_, and per submap the pose matrix and distance it was stored with."""

    def __init__(self, position=(0.0, 0.0, 0.0), quat_xyzw=(0.0, 0.0, 0.0, 1.0), trans_for_mapupdate=1.5):
        self.position = [float(v) for v in position]
        self.quat = [float(v) for v in quat_xyzw]
        self.previous_position = list(self.position)
        self.latest_distance = 0.0
        self.trans = 0.0
        self.trans_for_mapupdate = float(trans_for_mapupdate)
        self.initial = False
        self.poses, self.distances = [], []

    def sim_trans(self) -> np.ndarray:
        """getTransformation (:493-499): the pose's Affine3d matrix cast to float."""
        return pose_matrix(self.position, self.quat).astype(F32)

    def _store_submap(self):
        self.poses.append(pose_matrix(self.position, self.quat))
        self.distances.append(self.latest_distance)

    def initialize(self) -> np.ndarray:
        """initializeMap (:257-297): the first scan at the initial pose becomes submap 0 (distance 0). Returns the float
        transform its targeted cloud is moved by."""
        self.initial = True
        self._store_submap()
        return self.sim_trans()

    def frame(self, final, mut=()) -> dict:
        """publishMapAndPose (:391-434) for the float 4x4 `final` of align(); a map update stores the submap."""
        final = np.asarray(final, dtype=F32)
        pos = [float(final[r, 3]) for r in range(3)]
        self.quat = quat_from_rot(final[:3, :3])
        self.position = pos
        self.trans = distance3(pos, self.previous_position)
        updated = (self.trans > self.trans_for_mapupdate) if "update_gt" in mut else (self.trans >= self.trans_for_mapupdate)
        if updated:
            self.previous_position = list(pos)
            self.latest_distance += self.trans  # updateMap :474
            self._store_submap()
        return {"pose7": np.array(self.position + self.quat), "updated": updated, "trans": self.trans,
                "latest_distance": self.latest_distance}

    def update_map_external(self, position, quat_xyzw):
        """b200sm_update_map, the caller-driven updateMap: the distance to the previous update's position is added to
        latest_distance_ except for the first submap."""
        position = [float(v) for v in position]
        if self.poses:
            self.trans = distance3(position, self.previous_position)
            self.latest_distance += self.trans
        self.previous_position = list(position)
        self.position, self.quat = position, [float(v) for v in quat_xyzw]
        self.initial = True
        self._store_submap()

    def import_submap(self, pose, distance):
        """b200sm_import_submap: the submap is appended as received and its distance becomes latest_distance_; the
        position a later updateMap measures from (previous_position_) is not touched."""
        self.poses.append(np.asarray(pose, dtype=np.float64).copy())
        self.distances.append(float(distance))
        self.latest_distance = float(distance)


# ---- cloud transforms -----------------------------------------------------------------------------------------------
def transform_f32(cloud, T) -> np.ndarray:
    """pcl::transformPointCloud(Matrix4f): ((m0 x + m1 y) + m2 z) + m3 in float; the intensity is copied."""
    T = np.asarray(T, dtype=F32)
    c = np.asarray(cloud, dtype=F32)
    out = c.copy()
    x, y, z = c[:, 0], c[:, 1], c[:, 2]
    for r in range(3):
        out[:, r] = ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
    return out


def transform_f64(cloud, M, mut=()) -> np.ndarray:
    """pcl::transformPointCloud(Matrix4d) (updateMap :462): Transformer<double>, static_cast<float> of
    ((m0 x + m1 y) + m2 z) + m3 in double; the intensity is copied."""
    M = np.asarray(M, dtype=np.float64)
    c = np.asarray(cloud, dtype=F32)
    out = c.copy()
    x, y, z = (c[:, a].astype(np.float64) for a in range(3))
    for r in range(3):
        if "f64_reassoc" in mut:
            v = M[r, 0] * x + (M[r, 1] * y + (M[r, 2] * z + M[r, 3]))
        elif "f64_fused" in mut:  # the exact dot product, one rounding (long double carries 64 bits)
            L = np.longdouble
            v = (((L(M[r, 0]) * x.astype(L) + L(M[r, 1]) * y.astype(L)) + L(M[r, 2]) * z.astype(L)) + L(M[r, 3])).astype(np.float64)
        else:
            v = ((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3]
        out[:, r] = v.astype(F32)
    return out


def targeted(new_cloud, final, submaps, num_targeted_cloud, mut=()) -> np.ndarray:
    """updateMap :449-463: the new submap's cloud (VoxelGrid(vg_size_for_map) of the scan, as read back) moved by the
    float `final`, then the previous num_targeted_cloud - 1 submaps, newest first, each moved by its double pose.
    `submaps` is the list of (cloud, pose) BEFORE the new one was appended."""
    parts = [transform_f32(new_cloud, final)]
    n_sub = len(submaps)
    for i in range(num_targeted_cloud - 1):
        if n_sub - 1 - i < 0:
            continue
        c, M = submaps[n_sub - 1 - i]
        parts.append(transform_f64(c, M, mut))
    return np.concatenate(parts, axis=0)


# ---- searchLoop (gbs.cpp:144-258) -----------------------------------------------------------------------------------
def loop_candidates(poses, distances, distance_loop_closure, range_of_searching_loop_closure, mut=()) -> list:
    """gbs.cpp:190-205: every submap i with latest.distance - distance_i > distance_loop_closure and
    |latest.position - position_i| < range_of_searching_loop_closure, ascending id. Returns [(i, dist)]."""
    n = len(poses)
    if n == 0:
        return []
    lp, ld = poses[-1], float(distances[-1])
    out = []
    for i in range(n):
        dist = distance3(lp[:3, 3], poses[i][:3, 3])
        travel = ld - float(distances[i])
        g1 = travel >= distance_loop_closure if "travel_ge" in mut else travel > distance_loop_closure
        g2 = dist <= range_of_searching_loop_closure if "range_le" in mut else dist < range_of_searching_loop_closure
        if g1 and g2:
            out.append((i, dist))
    return out


def closest(cands, mut=()):
    """gbs.cpp:187-204: id_min / min_dist start at 0 / DBL_MAX; a candidate replaces them when dist < min_dist, so the
    first one wins a tie. None when there is no candidate."""
    if not cands:
        return None
    id_min, min_dist = 0, np.finfo(np.float64).max
    for i, d in cands:
        if (d <= min_dist) if "last_wins" in mut else (d < min_dist):
            id_min, min_dist = i, d
    return id_min, min_dist


def window(id_min, search_submap_num, n_sub, mut=()) -> list:
    """gbs.cpp:209-211: indices id_min - search_submap_num .. id_min + search_submap_num in order; negative ones are
    skipped, and so are those past the newest submap (the reference reads past its array there, b200reg.h)."""
    out = []
    for j in range(2 * search_submap_num + 1):
        idx = id_min + j - search_submap_num
        if idx < 0 or (idx >= n_sub and "upper_unchecked" not in mut):
            continue
        out.append(idx)
    return out


def loop_source(cloud, pose) -> np.ndarray:
    """gbs.cpp:172-181: the newest submap moved by its pose cast to float."""
    return transform_f32(cloud, np.asarray(pose, dtype=np.float64).astype(F32))


def loop_target_parts(clouds, poses, idxs) -> np.ndarray:
    """gbs.cpp:208-222: the window's submaps, each moved by its pose cast to float, concatenated in window order (the
    VoxelGrid of gbs.cpp:224-226 is applied by the caller: gridref.voxelgrid_ref). An index past the array raises."""
    parts = [transform_f32(clouds[i], np.asarray(poses[i], dtype=np.float64).astype(F32)) for i in idxs]
    return np.concatenate(parts, axis=0) if parts else np.zeros((0, 4), F32)


def _matmul4(A, B) -> list:
    """4x4 product in Python floats, each entry summed k = 0..3 left to right from 0.0."""
    C = [[0.0] * 4 for _ in range(4)]
    for r in range(4):
        for c in range(4):
            a = 0.0
            for k in range(4):
                a += A[r][k] * B[k][c]
            C[r][c] = a
    return C


def relative_pose(final, latest_pose, from_pose, mut=()) -> np.ndarray:
    """gbs.cpp:235-246: to = getFinalTransformation().cast<double>() * init_affine.matrix(), then from.inverse() * to
    with Isometry3d's inverse (R^T, -R^T t, t summed ((r0 t0 + r1 t1) + r2 t2))."""
    F = [[float(v) for v in row] for row in np.asarray(final, dtype=F32)]
    L = [[float(v) for v in row] for row in np.asarray(latest_pose, dtype=np.float64)]
    fr = np.asarray(from_pose, dtype=np.float64)
    to = _matmul4(F, L)
    if "rel_full_inverse" in mut:
        inv = np.linalg.inv(fr).tolist()
    else:
        R = [[float(fr[r, c]) for c in range(3)] for r in range(3)]
        t = [float(fr[r, 3]) for r in range(3)]
        inv = [[R[0][r], R[1][r], R[2][r], 0.0] for r in range(3)] + [[0.0, 0.0, 0.0, 1.0]]
        for r in range(3):
            inv[r][3] = -((inv[r][0] * t[0] + inv[r][1] * t[1]) + inv[r][2] * t[2])
    return np.array(_matmul4(inv, to))


def accepted(fitness, threshold_loop_closure_score) -> bool:
    """gbs.cpp:233."""
    return fitness < threshold_loop_closure_score


def shard(cands, rank, world) -> list:
    """b200sm_search_loop_all: candidate k (ascending id) belongs to rank k mod world."""
    return [c for k, c in enumerate(cands) if k % world == rank]


# ---- fixture generators ---------------------------------------------------------------------------------------------
def range_edge_cloud(rmin=5.0, rmax=25.0, seed=0) -> np.ndarray:
    """Points on separated (x, y) positions: Pythagorean ones exactly at rmin and rmax (3-4-5 and 7-24-25 scaled),
    each also one float ulp inside and outside, NaN / inf rows, large |z|, and points where np.hypot and the explicit sum
    disagree right at a bound (rmin and rmax are then their explicit-sum radii). Returns (cloud (N, 4), rmin, rmax)."""
    rng = np.random.default_rng(seed)
    s_min, s_max = rmin / 5.0, rmax / 25.0
    rows = []
    for a, b, s in ((3, 4, s_min), (4, 3, s_min), (-3, 4, s_min), (7, 24, s_max), (-24, -7, s_max), (24, 7, s_max)):
        x, y = F32(a * s), F32(b * s)
        for dx in (x, np.nextafter(x, F32(np.inf)), np.nextafter(x, F32(-np.inf))):
            rows.append((dx, y))
    pts = [(x, y, F32(0.25 * i - 2.0)) for i, (x, y) in enumerate(rows)]  # distinct z: a leaf of its own
    pts += [(F32(1e4), F32(1e4), F32(1.0)), (F32(0.0), F32(0.0), F32(0.0))]  # far outside, at the origin
    pts += [(F32(6.0), F32(0.5), F32(3.0e4)), (F32(-6.5), F32(1.5), F32(-3.0e4))]  # large |z|, inside
    nan, inf = F32(np.nan), F32(np.inf)
    pts += [(nan, F32(6.0), F32(0.0)), (F32(6.0), nan, F32(0.0)), (F32(6.0), F32(7.0), nan), (inf, F32(1.0), F32(0.0)),
            (F32(1.0), -inf, F32(0.0)), (F32(8.0), F32(2.0), inf)]
    cloud = np.array(pts, dtype=F32)
    return np.c_[cloud, rng.uniform(0, 100, len(cloud)).astype(F32)], rmin, rmax


def hypot_disagreements(n=4, lo=8.0, hi=20.0, seed=0) -> np.ndarray:
    """n points in the annulus lo < r < hi where np.hypot(x, y) != sqrt(x * x + y * y) in double."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        r, th = rng.uniform(lo, hi, 4096), rng.uniform(0, 2 * np.pi, 4096)
        x, y = (r * np.cos(th)).astype(F32), (r * np.sin(th)).astype(F32)
        xd, yd = x.astype(np.float64), y.astype(np.float64)
        d = np.flatnonzero(np.hypot(xd, yd) != np.sqrt(xd * xd + yd * yd))
        out += [(x[i], y[i]) for i in d[: n - len(out)]]
    return np.array(out, dtype=F32)


def cancelling_submap(n=4096, seed=0):
    """A submap far from its pose's origin along the direction the rotation maps onto the y axis: row 0 of the transform
    sums two large terms that cancel to a small x, where the order and rounding of the double sum show in the float cast.
    Returns (cloud (n, 4) float32, pose 4x4 float64)."""
    rng = np.random.default_rng(seed)
    yaw = 0.7853981633974483 + 1e-3
    c, s = math.cos(yaw), math.sin(yaw)
    M = np.eye(4)
    M[:2, :2] = [[c, -s], [s, c]]
    M[:3, 3] = [0.3, -1.25, 0.5]
    d = rng.uniform(2.0e5, 8.0e5, n)
    e = rng.uniform(-3.0, 3.0, n)
    x, y = d * s + e * c, d * c - e * s  # R (x, y) = (e, d) up to rounding
    cloud = np.c_[x, y, rng.uniform(-2, 2, n), rng.uniform(0, 100, n)].astype(F32)
    return cloud, M


def out_and_back(n_out=5, step=2.0, rings=16, azimuths=300):
    """Scans at ground-truth poses: n_out submaps down the canyon, then back over the same ground 0.3 m to the side.
    Yields (scan, pose 4x4 float64)."""
    from lidarslam_ros2_b200 import synth

    scene = synth.make_scene()
    xs = [step * k for k in range(n_out)] + [step * k for k in range(n_out - 2, -1, -1)]
    ys = [0.0] * n_out + [0.3] * (n_out - 1)
    S0 = synth.sensor_pose(synth.pose_matrix((0, 0, 0), (0, 0, 0)), -40.0)
    for k, (x, y) in enumerate(zip(xs, ys)):
        Sk = synth.sensor_pose(synth.pose_matrix((x, y, 0.0), (0.0, 0.0, 0.01 * k)), -40.0)
        yield synth.make_scan(scene, rings, azimuths, Sk, stream=8800 + k), np.linalg.inv(S0) @ Sk


GATE_L = np.array([10.0, -20.0, 1.5])
# (offset from the newest submap, travelled distance), for range 13, distance_loop_closure 20, the newest at 60
GATES = [((5, 12, 0), 0.0),   # 0: |d| = 13 = range: excluded
         ((0, 6, 8), 40.0),   # 1: travelled 20 = distance_loop_closure: excluded
         ((6, 8, 0), 10.0),   # 2: |d| = 10, candidate
         ((8, 0, 6), 5.0),    # 3: |d| = 10, candidate, ties with 2
         ((9, 12, 0), 1.0),   # 4: |d| = 15: excluded
         ((0, 0, 0), 60.0)]   # 5: the newest


def gate_fixture(rotated=False):
    """Submap poses and travelled distances of GATES: identity rotations (lattice clouds then move exactly), or small
    yaws when rotated. Every distance between the positions is a Pythagorean integer."""
    poses, dists = [], []
    for i, (off, d) in enumerate(GATES):
        q = (0.0, 0.0, math.sin(0.05 * i), math.cos(0.05 * i)) if rotated else (0.0, 0.0, 0.0, 1.0)
        poses.append(pose_matrix(GATE_L + np.array(off, dtype=float), q))
        dists.append(d)
    return poses, dists


def lattice_cloud(n_side=4, spacing=0.5, offset=0.25, seed=0) -> np.ndarray:
    """n_side^3 points at offset + k * spacing (dyadic, off every 0.2 leaf edge), random intensity: moved by a
    pose with the identity rotation and a dyadic translation, every point lands exactly and alone in its leaf."""
    k = np.arange(n_side, dtype=np.float64) * spacing + offset
    g = np.stack(np.meshgrid(k, k, k, indexing="ij"), axis=-1).reshape(-1, 3)
    rng = np.random.default_rng(seed)
    return np.c_[g, rng.uniform(0, 100, len(g))].astype(F32)
