"""Host-side mirror of the reference's frontend node for the path around align():
`ScanMatcherComponent` (scanmatcher/src/scanmatcher_component.cpp) without ROS — cloud callback, initializeMap,
receiveCloud, publishMapAndPose, updateMap — on top of the `b200sm_*` session of the C-ABI (include/b200reg.h).
The submaps and the targeted cloud live on the GPU; a frame costs one host-to-device copy.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _capi
from .registration import B200RegError, GeneralizedIterativeClosestPoint, NormalDistributionsTransform, _as_cloud, _ptr


def _loop_edges(loop_edges):
    """(from, to, relative_pose 4x4) tuples as a b200sm_loop_edge array (at least one element)."""
    edges = (_capi.SmLoopEdge * max(1, len(loop_edges)))()
    for k, (f, t, Z) in enumerate(loop_edges):
        edges[k].from_, edges[k].to = int(f), int(t)
        edges[k].relative_pose[:] = np.asarray(Z, dtype=np.float64).T.reshape(16).tolist()
    return edges


class ScanMatcher:
    """Parameters carry the reference's names and defaults (scanmatcher_component.cpp:26-50)."""

    def __init__(self, registration_method: str = "NDT", ndt_resolution: float = 5.0, ndt_num_threads: int = 0,
                 gicp_corr_dist_threshold: float = 5.0, trans_for_mapupdate: float = 1.5, vg_size_for_input: float = 0.2,
                 vg_size_for_map: float = 0.1, use_min_max_filter: bool = False, scan_min_range: float = 0.1,
                 scan_max_range: float = 100.0, num_targeted_cloud: int = 10, device: int = 0):
        self._lib = _capi.lib()
        if registration_method == "NDT":  # scanmatcher_component.cpp:97-107
            reg = NormalDistributionsTransform(device=device)
            reg.setResolution(ndt_resolution)
            reg.setTransformationEpsilon(0.01)
            reg.setNeighborhoodSearchMethod(2)  # pclomp::DIRECT7
            if ndt_num_threads > 0:
                reg.setNumThreads(ndt_num_threads)
        elif registration_method == "GICP":  # :108-115
            reg = GeneralizedIterativeClosestPoint(device=device)
            reg.setMaxCorrespondenceDistance(gicp_corr_dist_threshold)
            reg.setTransformationEpsilon(1e-8)
        else:
            raise ValueError("registration_method must be NDT or GICP")
        self.registration = reg
        h = C.c_void_p()
        rc = self._lib.b200sm_create(int(device), C.byref(h))
        if rc != 0:
            raise B200RegError(rc, "b200sm_create failed (no CUDA device? there is no CPU fallback)")
        self._h = h
        self._check(self._lib.b200sm_set_params(self._h, float(vg_size_for_input), float(vg_size_for_map), int(num_targeted_cloud),
                                                float(trans_for_mapupdate), int(bool(use_min_max_filter)),
                                                float(scan_min_range), float(scan_max_range)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.b200sm_destroy(h)
            self._h = None

    def _check(self, rc):
        if rc != 0:
            raise B200RegError(rc, self._lib.b200sm_last_error(self._h).decode())

    def setInitialPose(self, position, quat_xyzw):
        p = np.ascontiguousarray(position, dtype=np.float64)
        q = np.ascontiguousarray(quat_xyzw, dtype=np.float64)
        self._check(self._lib.b200sm_set_initial_pose(self._h, _ptr(p), _ptr(q)))

    def receiveCloud(self, points):
        """One frame (x, y, z[, intensity] rows). Returns (pose7 = position + quaternion xyzw, final 4x4, map_updated)."""
        p = _as_cloud(points)
        n, w = p.shape
        pose = np.zeros(7, dtype=np.float64)
        fin = np.zeros(16, dtype=np.float32)
        upd = C.c_int(0)
        self._check(self._lib.b200sm_receive_cloud(self._h, self.registration._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1,
                                                   _ptr(pose), _ptr(fin), C.byref(upd)))
        return pose, fin.reshape(4, 4).T.copy(), bool(upd.value)

    # ---- localisation in a prior map (b200sm_set_prior_map*, b200sm_localize_*) ----
    def setPriorMap(self, cloud) -> int:
        """The map to localise in, from host rows (x, y, z[, intensity]); it stays on the device. Returns its points."""
        p = _as_cloud(cloud)
        n, w = p.shape
        self._check(self._lib.b200sm_set_prior_map(self._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1))
        return n

    def setPriorMapPCD(self, path) -> int:
        """The map to localise in, from a PCD file (e.g. the one saveMapPCDASCII wrote), parsed onto the device. Returns
        POINTS. A file that cannot be read or parsed raises with ERR_IO / ERR_FORMAT and leaves the previous map."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_set_prior_map_pcd(self._h, os.fsencode(path), C.byref(n)))
        return int(n.value)

    def setLocalizationParams(self, crop_radius: float, recrop_distance: float):
        """Horizontal radius of the target cut around the pose, and how far the pose may move from the cut's centre before
        the target is cut again. Keep crop_radius >= scan_max_range + recrop_distance."""
        self._check(self._lib.b200sm_set_localization_params(self._h, float(crop_radius), float(recrop_distance)))

    def localizeCloud(self, points):
        """One frame registered against the cut of the prior map around the pose (b200sm_localize_cloud). Returns
        (pose7 = position + quaternion xyzw, final 4x4, target_recut)."""
        p = _as_cloud(points)
        n, w = p.shape
        pose = np.zeros(7, dtype=np.float64)
        fin = np.zeros(16, dtype=np.float32)
        recut = C.c_int(0)
        self._check(self._lib.b200sm_localize_cloud(self._h, self.registration._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1,
                                                    _ptr(pose), _ptr(fin), C.byref(recut)))
        return pose, fin.reshape(4, 4).T.copy(), bool(recut.value)

    def localizeInit(self, points, guesses):
        """The initial pose from several hypotheses (NDT): `guesses` (K, 4, 4) registered in one batch launch against the
        cut around the current position; the converged one with the highest transformation probability becomes the pose.
        Returns (best index or -1, list of per-guess dicts: final, trans_probability, converged, iterations, status)."""
        p = _as_cloud(points)
        n, w = p.shape
        G = np.ascontiguousarray(np.asarray(guesses, dtype=np.float32).reshape(-1, 4, 4).transpose(0, 2, 1))
        res = (_capi.BatchResult * len(G))()
        best = C.c_int(-1)
        self._check(self._lib.b200sm_localize_init(self._h, self.registration._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1,
                                                   _ptr(G), len(G), res, C.byref(best)))
        rows = [{"final": np.array(r.final_T, dtype=np.float32).reshape(4, 4).T.copy(),
                 "trans_probability": float(r.trans_probability), "converged": bool(r.converged),
                 "iterations": int(r.iterations), "status": int(r.status)} for r in res]
        return int(best.value), rows

    def localizeGlobal(self, points, radius: float, step: float, yaw_steps: int, top_k: int):
        """The pose without a precise guess (NDT, b200sm_localize_global): an (x, y, yaw) grid around the current pose —
        positions within `radius` at spacing `step`, `yaw_steps` headings each — scored on the device in one launch, the
        `top_k` best refined in one batch launch; the converged one with the highest transformation probability becomes the
        pose. Returns (best row or -1, candidates (hypothesis index per row), rows as localizeInit's, info dict:
        n_hypotheses, hits_total, n_refined, score_ms)."""
        p = _as_cloud(points)
        n, w = p.shape
        spec = _capi.SmGlobalSearch(float(radius), float(step), int(yaw_steps), int(top_k))
        k = max(int(top_k), 1)
        cand = np.full(k, -1, dtype=np.int32)
        res = (_capi.BatchResult * k)()
        out = _capi.SmGlobalResult()
        self._check(self._lib.b200sm_localize_global(self._h, self.registration._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1,
                                                     C.byref(spec), _ptr(cand), res, C.byref(out)))
        m = out.n_refined
        rows = [{"final": np.array(r.final_T, dtype=np.float32).reshape(4, 4).T.copy(),
                 "trans_probability": float(r.trans_probability), "converged": bool(r.converged),
                 "iterations": int(r.iterations), "status": int(r.status)} for r in res[:m]]
        info = dict(n_hypotheses=int(out.n_hypotheses), hits_total=int(out.hits_total), n_refined=int(m),
                    score_ms=float(out.score_ms))
        return int(out.best), cand[:m].copy(), rows, info

    def globalSearch(self):
        """The grid of the last localizeGlobal: (poses (H, 4, 4) float32, scores float64 (H,), hits int64 (H,))."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_global_search(self._h, 0, C.byref(n), None, None, None))
        H = n.value
        poses = np.empty((H, 16), dtype=np.float32)
        scores = np.empty(H, dtype=np.float64)
        hits = np.empty(H, dtype=np.int64)
        self._check(self._lib.b200sm_get_global_search(self._h, H, C.byref(n), _ptr(poses), _ptr(scores), _ptr(hits)))
        return poses.reshape(H, 4, 4).transpose(0, 2, 1).copy(), scores, hits

    def relocalize(self, points, **params):
        """The pose anywhere in the prior map (b200sm_relocalize; NDT or GICP): an exact branch-and-bound (x, y, yaw) search of
        the filtered scan over the map's 2D projection, the best tiles refined against the map cut around them; the
        converged row with the lowest fitness under accept_fitness becomes the pose. `params` override
        _capi.RELOCALIZE_DEFAULTS (resolution, z_min, z_max, yaw_steps, num_levels, min_score, top_k, accept_fitness).
        Returns (best row or -1, rows (dicts), info dict)."""
        p = _as_cloud(points)
        n, w = p.shape
        kw = dict(_capi.RELOCALIZE_DEFAULTS, **params)
        spec = _capi.SmRelocalizeParams(float(kw["resolution"]), float(kw["z_min"]), float(kw["z_max"]), int(kw["yaw_steps"]),
                                        int(kw["num_levels"]), float(kw["min_score"]), int(kw["top_k"]), float(kw["accept_fitness"]))
        cap = max(int(kw["top_k"]), 1)
        rows = (_capi.SmRelocalizeRow * cap)()
        out = _capi.SmRelocalizeResult()
        self._check(self._lib.b200sm_relocalize(self._h, self.registration._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1,
                                                C.byref(spec), rows, cap, C.byref(out)))
        res = [{"yaw_index": r.yaw_index, "cell": (r.cell_i, r.cell_j), "score": r.score,
                "guess": np.array(r.guess, dtype=np.float32).reshape(4, 4).T.copy(),
                "final": np.array(r.final_T, dtype=np.float32).reshape(4, 4).T.copy(), "fitness": float(r.fitness),
                "trans_probability": float(r.trans_probability), "converged": bool(r.converged), "iterations": int(r.iterations),
                "status": int(r.status)} for r in rows[:out.n_rows]]
        info = dict(width=int(out.width), height=int(out.height), origin_cell=(int(out.origin_cell[0]), int(out.origin_cell[1])),
                    m=int(out.m), t0=int(out.t0), t=int(out.t), leaves=int(out.leaves), nodes=[int(v) for v in out.nodes],
                    pyramid_builds=int(out.pyramid_builds), search_ms=float(out.search_ms))
        return int(out.best), res, info

    def relocalizeGrid(self, level: int = 0) -> np.ndarray:
        """Level `level` of the relocalisation pyramid: (H + 2^level - 1, W + 2^level - 1) uint8, row r / column c holding cell
        (c - 2^level + 1, r - 2^level + 1) of the grid."""
        w, h = C.c_longlong(0), C.c_longlong(0)
        self._check(self._lib.b200sm_get_relocalize_grid(self._h, int(level), None, 0, C.byref(w), C.byref(h)))
        out = np.zeros((h.value, w.value), dtype=np.uint8)
        self._check(self._lib.b200sm_get_relocalize_grid(self._h, int(level), _ptr(out), out.size, C.byref(w), C.byref(h)))
        return out

    def relocalizeScoreNodes(self, level: int, nodes) -> np.ndarray:
        """score_level of (heading, i, j) nodes with the last relocalize search's discretised scan, int32."""
        kij = np.ascontiguousarray(np.asarray(nodes, dtype=np.int32).reshape(-1, 3))
        out = np.zeros(len(kij), dtype=np.int32)
        self._check(self._lib.b200sm_relocalize_score_nodes(self._h, int(level), len(kij), _ptr(kij), _ptr(out)))
        return out

    def localizeStats(self) -> dict:
        st = _capi.SmLocalizeStats()
        self._check(self._lib.b200sm_get_localize_stats(self._h, C.byref(st)))
        out = {k: getattr(st, k) for k, _ in _capi.SmLocalizeStats._fields_}
        out["cut_centre"] = (float(st.cut_centre[0]), float(st.cut_centre[1]))
        return out

    def cutCloud(self) -> np.ndarray:
        """The current cut of the prior map, in map order (the newest cut: pending or already the target)."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_cut(self._h, None, 0, C.byref(n)))
        out = np.empty((n.value, 4), dtype=np.float32)
        self._check(self._lib.b200sm_get_cut(self._h, _ptr(out), n.value, C.byref(n)))
        return out

    # ---- the pieces, for callers that drive the steps themselves ----
    def setScan(self, points) -> int:
        p = _as_cloud(points)
        n, w = p.shape
        m = C.c_size_t(0)
        self._check(self._lib.b200sm_set_scan(self._h, self.registration._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1, C.byref(m)))
        return int(m.value)

    def deskewNextScan(self, scan_time: float):
        """use_imu: de-skew the next frame on the device before the range filter (b200sm_deskew_next_scan)."""
        self._check(self._lib.b200sm_deskew_next_scan(self._h, float(scan_time)))

    def setSensorTransform(self, position, quat_xyzw):
        """cloud_callback's tf2::doTransform into the robot frame (sm.cpp:188-199), on the device for every later frame:
        position / quat_xyzw are lookupTransform(robot_frame_id, cloud frame_id). setSensorTransform(None, None) turns it
        off (b200sm_set_sensor_transform)."""
        if position is None and quat_xyzw is None:
            self._check(self._lib.b200sm_set_sensor_transform(self._h, None, None))
            return
        p = np.ascontiguousarray(position, dtype=np.float64).reshape(3)
        q = np.ascontiguousarray(quat_xyzw, dtype=np.float64).reshape(4)
        self._check(self._lib.b200sm_set_sensor_transform(self._h, _ptr(p), _ptr(q)))

    def odomNextScan(self, position, quat_xyzw):
        """use_odom: the odometry lookupTransform(odom_frame_id, robot_frame_id) for the next receiveCloud, whose guess
        becomes pose * previous_odom^-1 * odom (sm.cpp:333-348; b200sm_odom_next_scan)."""
        p = np.ascontiguousarray(position, dtype=np.float64).reshape(3)
        q = np.ascontiguousarray(quat_xyzw, dtype=np.float64).reshape(4)
        self._check(self._lib.b200sm_odom_next_scan(self._h, _ptr(p), _ptr(q)))

    def updateMap(self, final_transformation, position, quat_xyzw, adopt_now: bool = True):
        T = np.ascontiguousarray(np.asarray(final_transformation, dtype=np.float32).T).reshape(16)
        p = np.ascontiguousarray(position, dtype=np.float64)
        q = np.ascontiguousarray(quat_xyzw, dtype=np.float64)
        self._check(self._lib.b200sm_update_map(self._h, self.registration._h, _ptr(T), _ptr(p), _ptr(q), int(adopt_now)))

    def searchLoop(self, registration, voxel_leaf_size: float = 0.2, threshold_loop_closure_score: float = 1.0,
                   distance_loop_closure: float = 20.0, range_of_searching_loop_closure: float = 20.0,
                   search_submap_num: int = 3) -> dict:
        """GraphBasedSlamComponent::searchLoop (graph_based_slam_component.cpp:144-258) over the session's device-resident
        submaps; `registration` is the backend's engine (see backend_registration()). Parameter names and defaults are the
        node's (gbs.cpp:23-39)."""
        r = _capi.SmLoopResult()
        self._check(self._lib.b200sm_search_loop(self._h, registration._h, float(voxel_leaf_size), float(threshold_loop_closure_score),
                                                 float(distance_loop_closure), float(range_of_searching_loop_closure),
                                                 int(search_submap_num), C.byref(r)))
        out = {"is_candidate": bool(r.is_candidate), "id_min": int(r.id_min), "accepted": bool(r.accepted)}
        if r.is_candidate:
            out.update(min_dist=float(r.min_dist), fitness=float(r.fitness), n_source=int(r.n_source), n_target=int(r.n_target),
                       final=np.array(r.final_T, dtype=np.float32).reshape(4, 4).T.copy())
            if r.accepted:
                out["relative_pose"] = np.array(r.relative_pose, dtype=np.float64).reshape(4, 4).T.copy()
        return out

    def importSubmap(self, cloud, pose_matrix, distance: float):
        """Append a submap received as a message (filtered cloud, 4x4 pose, travelled distance): b200sm_import_submap."""
        p = _as_cloud(cloud)
        n, w = p.shape
        M = np.ascontiguousarray(np.asarray(pose_matrix, dtype=np.float64).T).reshape(16)
        self._check(self._lib.b200sm_import_submap(self._h, _ptr(p), n, 4 * w, 12 if w >= 4 else -1, _ptr(M), float(distance)))

    def searchLoopAll(self, registration, voxel_leaf_size: float = 0.2, threshold_loop_closure_score: float = 1.0,
                      distance_loop_closure: float = 20.0, range_of_searching_loop_closure: float = 20.0,
                      search_submap_num: int = 3, shard_rank: int = 0, shard_world: int = 1) -> list:
        """Every gated candidate instead of the closest one (b200sm_search_loop_all); one dict per candidate, ascending id."""
        cap = max(1, self.numSubmaps())
        arr = (_capi.SmLoopResult * cap)()
        n, tot = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_search_loop_all(self._h, registration._h, float(voxel_leaf_size), float(threshold_loop_closure_score),
                                                     float(distance_loop_closure), float(range_of_searching_loop_closure),
                                                     int(search_submap_num), int(shard_rank), int(shard_world), arr, cap,
                                                     C.byref(n), C.byref(tot)))
        out = []
        for k in range(n.value):
            r = arr[k]
            d = {"is_candidate": True, "id_min": int(r.id_min), "accepted": bool(r.accepted), "min_dist": float(r.min_dist),
                 "fitness": float(r.fitness), "n_source": int(r.n_source), "n_target": int(r.n_target),
                 "final": np.array(r.final_T, dtype=np.float32).reshape(4, 4).T.copy(), "n_candidates_total": int(tot.value)}
            if r.accepted:
                d["relative_pose"] = np.array(r.relative_pose, dtype=np.float64).reshape(4, 4).T.copy()
            out.append(d)
        return out

    # ---- place recognition (b200sm_search_loop_place): Scan Context descriptors, a search that ignores the drifted poses ----
    def setScanContextParams(self, num_rings: int = 20, num_sectors: int = 60, max_radius: float = 80.0, lidar_height: float = 2.0):
        """The descriptor's grid: num_rings x num_sectors bins out to max_radius metres; a bin holds the largest
        z + lidar_height of its points. Drops every descriptor built so far (they are rebuilt at the next use)."""
        p = _capi.SmScanContextParams(int(num_rings), int(num_sectors), float(max_radius), float(lidar_height))
        self._check(self._lib.b200sm_set_scan_context_params(self._h, C.byref(p)))
        self._scp = (int(num_rings), int(num_sectors))

    def scanContext(self, index: int) -> np.ndarray:
        """The descriptor of submap `index`, (num_rings, num_sectors) float32 (built on the device if it is not yet)."""
        R, S = getattr(self, "_scp", (20, 60))
        out = np.empty((R, S), dtype=np.float32)
        self._check(self._lib.b200sm_get_scan_context(self._h, int(index), _ptr(out), out.size))
        return out

    def searchLoopPlace(self, registration, voxel_leaf_size: float = 0.2, threshold_loop_closure_score: float = 1.0,
                        distance_loop_closure: float = 20.0, search_submap_num: int = 3, sc_threshold: float = 0.4,
                        top_k: int = 3, capacity=None):
        """The newest submap against every older one more than distance_loop_closure behind it along the path, by Scan
        Context distance and whatever the poses say; the top_k best under sc_threshold are verified by the registration from
        the heading the descriptors give (b200sm_search_loop_place). Returns (rows, n_scored): one dict per verified
        candidate, best first, with searchLoopAll's keys plus sc_distance, shift and guess (4x4)."""
        cap = int(top_k) if capacity is None else int(capacity)
        arr = (_capi.SmPlaceResult * max(1, cap))()
        n, scored = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_search_loop_place(self._h, registration._h, float(voxel_leaf_size),
                                                       float(threshold_loop_closure_score), float(distance_loop_closure),
                                                       int(search_submap_num), float(sc_threshold), int(top_k), arr, cap,
                                                       C.byref(n), C.byref(scored)))
        out = []
        for k in range(n.value):
            p = arr[k]
            r = p.loop
            d = {"is_candidate": True, "id_min": int(r.id_min), "accepted": bool(r.accepted), "min_dist": float(r.min_dist),
                 "fitness": float(r.fitness), "n_source": int(r.n_source), "n_target": int(r.n_target),
                 "final": np.array(r.final_T, dtype=np.float32).reshape(4, 4).T.copy(), "sc_distance": float(p.sc_distance),
                 "shift": int(p.shift), "guess": np.array(p.guess, dtype=np.float32).reshape(4, 4).T.copy()}
            if r.accepted:
                d["relative_pose"] = np.array(r.relative_pose, dtype=np.float64).reshape(4, 4).T.copy()
            out.append(d)
        return out, int(scored.value)

    def placeScores(self):
        """The last searchLoopPlace's per-submap (D float64, s* int32); D is NaN and s* -1 where a submap was not eligible."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_place_scores(self._h, 0, C.byref(n), None, None))
        D = np.empty(n.value, dtype=np.float64)
        S = np.empty(n.value, dtype=np.int32)
        self._check(self._lib.b200sm_get_place_scores(self._h, n.value, C.byref(n), _ptr(D), _ptr(S)))
        return D, S

    def poseAdjust(self, loop_edges, num_adjacent_pose_cnstraints: int = 5, max_iterations: int = 10):
        """GraphBasedSlamComponent::doPoseAdjustment's pose-graph solve (gbs.cpp:262-319) over the session's submap poses:
        loop_edges is a list of (from, to, relative_pose 4x4), e.g. (r["id_min"], numSubmaps() - 1, r["relative_pose"]) of
        an accepted searchLoop. Returns (adjusted poses (N, 4, 4) float64, result dict); the session's poses are unchanged."""
        edges = (_capi.SmLoopEdge * max(1, len(loop_edges)))()
        for k, (f, t, Z) in enumerate(loop_edges):
            edges[k].from_, edges[k].to = int(f), int(t)
            edges[k].relative_pose[:] = np.asarray(Z, dtype=np.float64).T.reshape(16).tolist()
        n = self.numSubmaps()
        poses = np.zeros((max(1, n), 16), dtype=np.float64)
        r = _capi.SmPoseAdjustResult()
        self._check(self._lib.b200sm_pose_adjust(self._h, int(num_adjacent_pose_cnstraints), edges, len(loop_edges),
                                                 int(max_iterations), _ptr(poses), C.byref(r)))
        return (poses[:n].reshape(n, 4, 4).transpose(0, 2, 1).copy(),
                {k: getattr(r, k) for k, _ in _capi.SmPoseAdjustResult._fields_})

    # ---- merging a second session (b200sm_merge_session) ----
    def mergeSession(self, other, registration, loop_edges=(), capacity=None, **params):
        """Merge session `other` (another recording, in a frame of its own) into this one: Scan Context scores of every
        pair on the device, the best candidates verified by `registration`, a consistent set of them kept, the joint pose
        adjustment, and on success `other`'s submaps appended as a new segment at their rigid placement. params: the fields
        of b200sm_merge_params (defaults in _capi.MERGE_DEFAULTS). loop_edges: (from, to, relative_pose 4x4) in merged
        numbering (this session's submaps, then other's at numSubmaps() + b). Returns (rows, poses, result): one dict per
        verified pair in verification order (searchLoopPlace's keys plus src_id, inlier, inlier_rank), the adjusted poses
        (n_A + n_B, 4, 4) or None when the merge did not succeed, and the result dict (T as a 4x4, edges: the inter-session
        loop edges in rank order, ready for poseAdjust)."""
        unknown = set(params) - set(_capi.MERGE_DEFAULTS)
        if unknown:
            raise TypeError(f"mergeSession: unknown parameters {sorted(unknown)}")
        p = _capi.SmMergeParams(**{**_capi.MERGE_DEFAULTS, **params})
        edges = (_capi.SmLoopEdge * max(1, len(loop_edges)))()
        for k, (f, t, Z) in enumerate(loop_edges):
            edges[k].from_, edges[k].to = int(f), int(t)
            edges[k].relative_pose[:] = np.asarray(Z, dtype=np.float64).T.reshape(16).tolist()
        nA, nB = self.numSubmaps(), other.numSubmaps()
        cap = int(p.max_verifications) if capacity is None else int(capacity)
        arr = (_capi.SmMergeRow * max(1, cap))()
        poses = np.zeros((max(1, nA + nB), 16), dtype=np.float64)
        n = C.c_size_t(0)
        r = _capi.SmMergeResult()
        self._check(self._lib.b200sm_merge_session(self._h, other._h, registration._h, C.byref(p), edges, len(loop_edges), arr, cap,
                                                   C.byref(n), _ptr(poses), C.byref(r)))
        rows = []
        for k in range(n.value):
            m = arr[k]
            q, lp = m.place, m.place.loop
            d = {"id_min": int(lp.id_min), "src_id": int(m.src_id), "accepted": bool(lp.accepted), "min_dist": float(lp.min_dist),
                 "fitness": float(lp.fitness), "n_source": int(lp.n_source), "n_target": int(lp.n_target),
                 "final": np.array(lp.final_T, dtype=np.float32).reshape(4, 4).T.copy(), "sc_distance": float(q.sc_distance),
                 "shift": int(q.shift), "guess": np.array(q.guess, dtype=np.float32).reshape(4, 4).T.copy(),
                 "inlier": m.inlier >= 0, "inlier_rank": int(m.inlier)}
            if lp.accepted:
                d["relative_pose"] = np.array(lp.relative_pose, dtype=np.float64).reshape(4, 4).T.copy()
            rows.append(d)
        res = {k: getattr(r, k) for k, _ in _capi.SmMergeResult._fields_ if k not in ("T", "adjust")}
        res["merged"] = bool(r.merged)
        res["T"] = np.array(r.T, dtype=np.float64).reshape(4, 4).T.copy()
        res["adjust"] = {k: getattr(r.adjust, k) for k, _ in _capi.SmPoseAdjustResult._fields_}
        res["edges"] = [(d["id_min"], nA + d["src_id"], d["relative_pose"]) for d in sorted(
            (d for d in rows if d["inlier"]), key=lambda d: d["inlier_rank"])]
        out = poses[:nA + nB].reshape(nA + nB, 4, 4).transpose(0, 2, 1).copy() if r.merged else None
        return rows, out, res

    def mergeScores(self):
        """The last mergeSession's score matrix: (D (n_B, n_A) float64, s* (n_B, n_A) int32), row b = the other session's
        submap b."""
        nq, nc = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_get_merge_scores(self._h, 0, C.byref(nq), C.byref(nc), None, None))
        D = np.empty((nq.value, nc.value), dtype=np.float64)
        S = np.empty((nq.value, nc.value), dtype=np.int32)
        self._check(self._lib.b200sm_get_merge_scores(self._h, D.size, C.byref(nq), C.byref(nc), _ptr(D), _ptr(S)))
        return D, S

    def segments(self) -> list:
        """The first submap of every segment (one per recording merged into this session)."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_segments(self._h, None, 0, C.byref(n)))
        out = np.zeros(max(1, n.value), dtype=np.uint64)
        self._check(self._lib.b200sm_get_segments(self._h, _ptr(out), n.value, C.byref(n)))
        return [int(v) for v in out[:n.value]]

    # ---- saving and loading a session (b200sm_save_session / b200sm_load_session) ----
    def saveSession(self, dir, loop_edges=(), num_adjacent_pose_cnstraints: int = 5, poses=None) -> dict:
        """Save the session into directory `dir`: session.txt (the manifest), pose_graph.g2o (the reference's
        optimizer.save output) and submaps/%06zu.pcd (binary PCD, sensor frame). loop_edges: (from, to, relative_pose 4x4)
        as poseAdjust takes them; poses: the adjusted poses (N, 4, 4) or None. Returns the info dict (n_bytes: all files)."""
        edges = _loop_edges(loop_edges)
        n = self.numSubmaps()
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 4, 4).transpose(0, 2, 1)).reshape(-1)
            if P.size != 16 * n:
                raise ValueError(f"saveSession: {P.size // 16} poses for {n} submaps")
        info = _capi.SmSessionIoInfo()
        self._check(self._lib.b200sm_save_session(self._h, os.fsencode(dir), int(num_adjacent_pose_cnstraints), edges,
                                                  len(loop_edges), _ptr(P) if P is not None else None, C.byref(info)))
        return {k: getattr(info, k) for k, _ in _capi.SmSessionIoInfo._fields_}

    def loadSession(self, dir):
        """Load a directory saveSession wrote into this (empty) session. Returns (loop_edges, poses, k, info): the graph it
        was saved with (edges as (from, to, relative_pose 4x4), the adjusted poses (N, 4, 4) or None,
        num_adjacent_pose_cnstraints) and the info dict."""
        info = _capi.SmSessionIoInfo()
        self._check(self._lib.b200sm_load_session(self._h, os.fsencode(dir), C.byref(info)))
        with open(os.path.join(dir, "session.txt"), "rb") as f:  # the restored descriptor grid: line 2 of the manifest
            f.readline()
            tok = f.readline().split()
        self._scp = (int(tok[1]), int(tok[2]))
        L, n = int(info.n_loop_edges), int(info.n_submaps)
        edges = (_capi.SmLoopEdge * max(1, L))()
        got, k = C.c_size_t(0), C.c_int(0)
        P = np.zeros((max(1, n), 16), dtype=np.float64)
        self._check(self._lib.b200sm_get_session_graph(self._h, edges, L, C.byref(got), _ptr(P), C.byref(k)))
        out = [(int(e.from_), int(e.to), np.array(e.relative_pose, dtype=np.float64).reshape(4, 4).T.copy()) for e in edges[:L]]
        poses = P[:n].reshape(n, 4, 4).transpose(0, 2, 1).copy() if info.adjusted else None
        return out, poses, int(k.value), {k_: getattr(info, k_) for k_, _ in _capi.SmSessionIoInfo._fields_}

    def assembleMap(self, poses=None, capacity=None):
        """The map of every submap moved by its pose cast to float (publishMap sm.cpp:529-552 when poses is None, else the
        modified map of gbs.cpp:321-368), assembled on the device in one launch. Returns (cloud (M, 4) float32, offsets
        (N + 1,) int64): submap i is cloud[offsets[i]:offsets[i + 1]]. capacity: copy at most that many points."""
        n_sub = self.numSubmaps()
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(n_sub, 4, 4).transpose(0, 2, 1))
        offsets = np.zeros(n_sub + 1, dtype=np.uint64)
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_assemble_map(self._h, _ptr(P) if P is not None else None, None, 0, C.byref(n), _ptr(offsets)))
        cap = n.value if capacity is None else min(int(capacity), n.value)
        out = np.empty((max(cap, 1), 4), dtype=np.float32)
        self._check(self._lib.b200sm_assemble_map(self._h, _ptr(P) if P is not None else None, _ptr(out), cap, C.byref(n), None))
        return out[:cap], offsets.astype(np.int64)

    def saveMapPCDASCII(self, path, poses=None):
        """pcl::io::savePCDFileASCII(path, map) of the map assembleMap(poses) returns (the map_save service, gbs.cpp:90-103,
        369): assembled and formatted on the device, written chunk by chunk. Returns (points, file bytes). An empty map
        raises with ERR_ARG and creates no file; a file that cannot be opened or written raises with ERR_IO."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        n, size = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_save_map_pcd_ascii(self._h, _ptr(P) if P is not None else None, os.fsencode(path),
                                                        C.byref(n), C.byref(size)))
        return int(n.value), int(size.value)

    # ---- occupancy grid for a navigation stack (b200sm_build_occupancy_grid, csrc/occupancy_grid.hpp) ----
    def buildOccupancyGrid(self, poses=None, resolution: float = 0.05, z_min: float = 0.2, z_max: float = 2.0,
                           max_range: float = 100.0, sensor_origin=(0.0, 0.0, 0.0), occupied_thresh: float = 0.65,
                           free_thresh: float = 0.25) -> dict:
        """The 2D occupancy grid of every submap at its own pose (poses None) or at `poses` (N, 4, 4), e.g. poseAdjust's:
        free space ray-cast on the device from each submap's sensor origin (sensor_origin: the LiDAR in the robot frame),
        hits and frees counted per submap in the map-frame height band [z_min, z_max]. Returns the build's info as a dict
        (width, height, origin (x, y), resolution, n_rays, n_skipped, n_batches, n_occupied, n_free, n_unknown)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        so = (C.c_double * 3)(*[float(v) for v in sensor_origin])
        prm = _capi.SmOccupancyParams(float(resolution), float(z_min), float(z_max), float(max_range), so, float(occupied_thresh),
                                      float(free_thresh))
        info = _capi.SmOccupancyInfo()
        self._check(self._lib.b200sm_build_occupancy_grid(self._h, _ptr(P) if P is not None else None, C.byref(prm),
                                                          C.byref(info)))
        self._og = info
        return _occupancy_info(info)

    def occupancyGrid(self) -> dict:
        """The last grid: data (height, width) int8 (-1 unknown, else 0..100; row 0 is the bottom row, as
        nav_msgs/OccupancyGrid.data), hits and frees (height, width) uint32, and the build's info."""
        info = getattr(self, "_og", None)
        W, H = (int(info.width), int(info.height)) if info is not None else (0, 0)
        data = np.empty((H, W), dtype=np.int8)
        hits = np.empty((H, W), dtype=np.uint32)
        frees = np.empty((H, W), dtype=np.uint32)
        self._check(self._lib.b200sm_get_occupancy_grid(self._h, _ptr(data), _ptr(hits), _ptr(frees), W * H))
        return dict(data=data, hits=hits, frees=frees, **_occupancy_info(info))

    def saveOccupancyMap(self, pgm_path, yaml_path):
        """nav2 map_server's map.pgm + map.yaml pair of the last grid (trinary)."""
        self._check(self._lib.b200sm_save_occupancy_map(self._h, os.fsencode(pgm_path), os.fsencode(yaml_path)))

    # ---- elevation / traversability map for non-flat ground (b200sm_build_elevation_map, csrc/elevation_map.hpp) ----
    def buildElevationMap(self, poses=None, resolution: float = 0.1, max_range: float = 100.0, sensor_origin=(0.0, 0.0, 0.0),
                          clearance: float = 2.0, min_points: int = 2, window_cells: int = 3, min_cells: int = 6,
                          max_slope: float = 20.0, max_step: float = 0.15, max_roughness: float = 0.05,
                          occupied_thresh: float = 0.65, free_thresh: float = 0.25) -> dict:
        """The 2.5D elevation map of every submap at its own pose (poses None) or at `poses` (N, 4, 4), built on the device:
        per cell the highest point within `clearance` of its lowest one, and over the observed cells within window_cells
        of it the step, slope (max_slope in degrees) and roughness, classified -1 / 0..99 / 100 (lethal). Returns the
        build's info as a dict (width, height, origin (x, y), resolution, n_points, n_skipped, n_overhang, n_observed,
        n_lethal, n_traversable, n_unknown)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        so = (C.c_double * 3)(*[float(v) for v in sensor_origin])
        prm = _capi.SmElevationParams(float(resolution), float(max_range), so, float(clearance), int(min_points),
                                      int(window_cells), int(min_cells), float(max_slope), float(max_step),
                                      float(max_roughness), float(occupied_thresh), float(free_thresh))
        info = _capi.SmElevationInfo()
        self._check(self._lib.b200sm_build_elevation_map(self._h, _ptr(P) if P is not None else None, C.byref(prm),
                                                         C.byref(info)))
        self._el = info
        return _struct_dict(info)

    def elevationMap(self) -> dict:
        """The last map as (height, width) arrays, row 0 the bottom row: n uint32 (points per cell), h and lo int64 (surface
        and lowest height in 2^16-per-cell fixed point), step, tan_slope, roughness float32 (metres; NaN where unknown),
        value int8 (-1, 0..99, 100), and the build's info."""
        info = getattr(self, "_el", None)
        W, H = (int(info.width), int(info.height)) if info is not None else (0, 0)
        out = dict(n=np.empty((H, W), dtype=np.uint32), h=np.empty((H, W), dtype=np.int64), lo=np.empty((H, W), dtype=np.int64),
                   step=np.empty((H, W), dtype=np.float32), tan_slope=np.empty((H, W), dtype=np.float32),
                   roughness=np.empty((H, W), dtype=np.float32), value=np.empty((H, W), dtype=np.int8))
        self._check(self._lib.b200sm_get_elevation_map(self._h, *[_ptr(out[k]) for k in ("n", "h", "lo", "step", "tan_slope",
                                                                                         "roughness", "value")], W * H))
        return dict(out, **(_struct_dict(info) if info is not None else {}))

    def saveTraversabilityMap(self, pgm_path, yaml_path):
        """nav2 map_server's pgm + yaml pair of the last elevation map (trinary: lethal black, traversable white)."""
        self._check(self._lib.b200sm_save_traversability_map(self._h, os.fsencode(pgm_path), os.fsencode(yaml_path)))

    # ---- static map: what moved while the map was recorded removed (b200sm_build_static_map, csrc/static_map.hpp) ----
    def buildStaticMap(self, poses=None, resolution: float = 0.2, max_range: float = 100.0, sensor_origin=(0.0, 0.0, 0.0),
                       ray_fraction: float = 0.85, min_frees: int = 2, dynamic_thresh: float = 0.4) -> dict:
        """The map without its dynamic points, every submap at its own pose (poses None) or at `poses` (N, 4, 4), e.g.
        poseAdjust's: each point is a ray from its submap's sensor origin (sensor_origin: the LiDAR in the robot frame) through
        a 3D voxel grid; the first ray_fraction of each ray frees the voxels it crosses, and a voxel freed by at least
        min_frees submaps and hit by at most dynamic_thresh of those that saw it is dynamic. Returns the build's info as a
        dict (box_origin, box_dims, n_rays, n_skipped, n_voxels, n_dynamic_voxels, n_points, n_static_points, n_batches)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        so = (C.c_double * 3)(*[float(v) for v in sensor_origin])
        prm = _capi.SmStaticMapParams(float(resolution), float(max_range), so, float(ray_fraction), int(min_frees),
                                      float(dynamic_thresh))
        info = _capi.SmStaticMapInfo()
        self._check(self._lib.b200sm_build_static_map(self._h, _ptr(P) if P is not None else None, C.byref(prm), C.byref(info)))
        self._sm_sub = self.numSubmaps()
        return _struct_dict(info)

    def staticMap(self, capacity=None):
        """The last static map: (cloud (M, 4) float32 in the assembled map's order, offsets (N + 1,) int64 per submap, N the
        submaps at the build). capacity: copy at most that many points."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_static_map(self._h, None, 0, C.byref(n), None))
        m = n.value if capacity is None else min(int(capacity), n.value)
        offsets = np.zeros(getattr(self, "_sm_sub", 0) + 1, dtype=np.uint64)
        out = np.empty((max(m, 1), 4), dtype=np.float32)
        self._check(self._lib.b200sm_get_static_map(self._h, _ptr(out), m, C.byref(n), _ptr(offsets)))
        return out[:m], offsets.astype(np.int64)

    def mapVoxels(self) -> dict:
        """The occupied voxels of the last build in rank order: ijk (V, 3) int32, hits, frees (V,) uint32, dynamic (V,) bool."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_map_voxels(self._h, None, None, None, None, 0, C.byref(n)))
        V = n.value
        ijk = np.empty((max(V, 1), 3), dtype=np.int32)
        hits = np.empty(max(V, 1), dtype=np.uint32)
        frees = np.empty(max(V, 1), dtype=np.uint32)
        dyn = np.empty(max(V, 1), dtype=np.uint8)
        self._check(self._lib.b200sm_get_map_voxels(self._h, _ptr(ijk), _ptr(hits), _ptr(frees), _ptr(dyn), V, C.byref(n)))
        return dict(ijk=ijk[:V], hits=hits[:V], frees=frees[:V], dynamic=dyn[:V].astype(bool))

    def saveStaticMapPcd(self, path):
        """pcl::io::savePCDFileASCII(path, static map) of the last build, as saveMapPCDASCII writes a map. Returns (points,
        file bytes)."""
        n, size = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_save_static_map_pcd_ascii(self._h, os.fsencode(path), C.byref(n), C.byref(size)))
        return int(n.value), int(size.value)

    # ---- map changes: what appeared and vanished between two recordings (b200sm_build_map_changes, csrc/map_changes.hpp) ----
    UNCHANGED, APPEARED, VANISHED = 0, 1, 2

    def buildMapChanges(self, poses=None, split_submap: int = -1, resolution: float = 0.2, max_range: float = 100.0,
                        sensor_origin=(0.0, 0.0, 0.0), ray_fraction: float = 0.85, min_frees: int = 2,
                        dynamic_thresh: float = 0.4) -> dict:
        """What changed between the submaps before split_submap and those from it on (-1: the first submap of the last
        segment, e.g. the recording mergeSession added), every submap at its own pose (poses None) or at `poses` (N, 4, 4).
        The rays and parameters are buildStaticMap's; each voxel's hits and frees are counted per epoch, and a voxel
        occupied in one epoch and free in the other APPEARED or VANISHED. Returns the build's info as a dict (box_origin,
        box_dims, split_submap, n_rays, n_skipped, n_voxels, n_appeared_voxels, n_vanished_voxels, n_points,
        n_appeared_points, n_vanished_points, n_updated_points, n_batches)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        so = (C.c_double * 3)(*[float(v) for v in sensor_origin])
        prm = _capi.SmStaticMapParams(float(resolution), float(max_range), so, float(ray_fraction), int(min_frees),
                                      float(dynamic_thresh))
        info = _capi.SmMapChangeInfo()
        self._check(self._lib.b200sm_build_map_changes(self._h, _ptr(P) if P is not None else None, C.byref(prm), int(split_submap),
                                                       C.byref(info)))
        self._ch_sub = self.numSubmaps()
        return _struct_dict(info)

    def mapChanges(self) -> np.ndarray:
        """The label of every point of the last build in map order (M,) uint8: UNCHANGED, APPEARED or VANISHED."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_map_changes(self._h, None, 0, C.byref(n)))
        out = np.empty(max(n.value, 1), dtype=np.uint8)
        self._check(self._lib.b200sm_get_map_changes(self._h, _ptr(out), n.value, C.byref(n)))
        return out[:n.value]

    def changeVoxels(self) -> dict:
        """The occupied voxels of the last build in rank order: ijk (V, 3) int32, hits_before, frees_before, hits_after,
        frees_after (V,) uint32, label (V,) uint8."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_change_voxels(self._h, None, None, None, None, None, None, 0, C.byref(n)))
        V = n.value
        out = dict(ijk=np.empty((max(V, 1), 3), dtype=np.int32), label=np.empty(max(V, 1), dtype=np.uint8))
        for k in ("hits_before", "frees_before", "hits_after", "frees_after"):
            out[k] = np.empty(max(V, 1), dtype=np.uint32)
        self._check(self._lib.b200sm_get_change_voxels(self._h, *[_ptr(out[k]) for k in ("ijk", "hits_before", "frees_before",
                                                                                       "hits_after", "frees_after", "label")],
                                                        V, C.byref(n)))
        return {k: v[:V] for k, v in out.items()}

    def updatedMap(self, capacity=None):
        """The last build's updated map (the assembled map without its VANISHED points): (cloud (M, 4) float32 in the
        assembled map's order, offsets (N + 1,) int64 per submap, N the submaps at the build). capacity: copy at most that
        many points."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_updated_map(self._h, None, 0, C.byref(n), None))
        m = n.value if capacity is None else min(int(capacity), n.value)
        offsets = np.zeros(getattr(self, "_ch_sub", 0) + 1, dtype=np.uint64)
        out = np.empty((max(m, 1), 4), dtype=np.float32)
        self._check(self._lib.b200sm_get_updated_map(self._h, _ptr(out), m, C.byref(n), _ptr(offsets)))
        return out[:m], offsets.astype(np.int64)

    def saveUpdatedMapPcd(self, path):
        """pcl::io::savePCDFileASCII(path, updated map) of the last build: the prior map to localise in next time
        (setPriorMapPcd). Returns (points, file bytes)."""
        n, size = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_save_updated_map_pcd_ascii(self._h, os.fsencode(path), C.byref(n), C.byref(size)))
        return int(n.value), int(size.value)

    # ---- surface mesh: a TSDF of the submaps' rays, extracted by surface nets (b200sm_build_mesh, csrc/mesh.hpp) ----
    def buildMesh(self, poses=None, resolution: float = 0.2, truncation: float = 0.6, max_range: float = 100.0,
                  sensor_origin=(0.0, 0.0, 0.0), min_weight: int = 2) -> dict:
        """The surface mesh of every submap at its own pose (poses None) or at `poses` (N, 4, 4), built on the device: each
        ray fuses its signed distance into the voxels within `truncation` of its endpoint, and surface nets extracts the
        zero crossing of the voxels at least `min_weight` rays observed. Returns the build's info as a dict (box_origin,
        box_dims, n_points, n_rays, n_skipped, n_walked, n_band_voxels, n_observed_voxels, n_vertices, n_faces)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        so = (C.c_double * 3)(*[float(v) for v in sensor_origin])
        prm = _capi.SmMeshParams(float(resolution), float(truncation), float(max_range), so, int(min_weight))
        info = _capi.SmMeshInfo()
        self._check(self._lib.b200sm_build_mesh(self._h, _ptr(P) if P is not None else None, C.byref(prm), C.byref(info)))
        return _struct_dict(info)

    def mesh(self):
        """The last build's mesh: (vertices (V, 3) float32 in the map frame, faces (F, 3) uint32, counter-clockwise seen
        from free space)."""
        nv, nf = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_get_mesh(self._h, None, 0, C.byref(nv), None, 0, C.byref(nf)))
        V, F = nv.value, nf.value
        xyz = np.empty((max(V, 1), 3), dtype=np.float32)
        faces = np.empty((max(F, 1), 3), dtype=np.uint32)
        self._check(self._lib.b200sm_get_mesh(self._h, _ptr(xyz), V, C.byref(nv), _ptr(faces), F, C.byref(nf)))
        return xyz[:V], faces[:F]

    def meshVoxels(self) -> dict:
        """The last build's band voxels in rank order: ijk (B, 3) int32, sdf_sum (B,) int64 (2^-16 voxel units), weight (B,)
        uint32."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_mesh_voxels(self._h, None, None, None, 0, C.byref(n)))
        B = n.value
        out = dict(ijk=np.empty((max(B, 1), 3), dtype=np.int32), sdf_sum=np.empty(max(B, 1), dtype=np.int64),
                   weight=np.empty(max(B, 1), dtype=np.uint32))
        self._check(self._lib.b200sm_get_mesh_voxels(self._h, _ptr(out["ijk"]), _ptr(out["sdf_sum"]), _ptr(out["weight"]), B,
                                                     C.byref(n)))
        return {k: v[:B] for k, v in out.items()}

    def saveMeshPly(self, path) -> int:
        """The last build's mesh as binary little-endian PLY (MeshLab, CloudCompare, Open3D, Blender). Returns the file's
        bytes."""
        size = C.c_size_t(0)
        self._check(self._lib.b200sm_save_mesh_ply(self._h, os.fsencode(path), C.byref(size)))
        return int(size.value)

    # ---- OctoMap: free and occupied voxels pruned into OctoMap's key tree (b200sm_build_octomap, csrc/octomap.hpp) ----
    def buildOctoMap(self, poses=None, resolution: float = 0.2, max_range: float = 100.0, sensor_origin=(0.0, 0.0, 0.0),
                     ray_fraction: float = 0.85, min_frees: int = 2, dynamic_thresh: float = 0.4) -> dict:
        """The OctoMap of every submap at its own pose (poses None) or at `poses` (N, 4, 4), built on the device from the
        static map's rays and parameters: a voxel is OCCUPIED when the static map keeps it as an occupied, non-dynamic
        voxel, FREE when a ray's freed part crosses it or a ray ends in it and it is not OCCUPIED, UNKNOWN otherwise; the
        known voxels pruned into OctoMap's depth-16 key tree. Returns the build's info as a dict (box_origin, box_dims,
        n_rays, n_skipped, n_occupied_voxels, n_dynamic_voxels, n_free_voxels, n_inner_nodes, n_occupied_leaves,
        n_free_leaves, tree_size, n_bytes, n_batches)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        so = (C.c_double * 3)(*[float(v) for v in sensor_origin])
        prm = _capi.SmStaticMapParams(float(resolution), float(max_range), so, float(ray_fraction), int(min_frees),
                                      float(dynamic_thresh))
        info = _capi.SmOctoMapInfo()
        self._check(self._lib.b200sm_build_octomap(self._h, _ptr(P) if P is not None else None, C.byref(prm), C.byref(info)))
        self._om_box = (tuple(info.box_origin), tuple(info.box_dims))
        return _struct_dict(info)

    def octoMapStates(self) -> dict:
        """The last build's box: box_origin (3,) voxel of its lower corner, and states (D, H, W) uint8 indexed [k, j, i]:
        0 UNKNOWN, 1 FREE, 2 OCCUPIED."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_octomap_states(self._h, None, 0, C.byref(n)))
        out = np.empty(max(n.value, 1), dtype=np.uint8)
        self._check(self._lib.b200sm_get_octomap_states(self._h, _ptr(out), n.value, C.byref(n)))
        origin, (W, H, D) = getattr(self, "_om_box", ((0, 0, 0), (0, 0, 0)))
        return dict(box_origin=np.array(origin, dtype=np.int64), states=out[:n.value].reshape(D, H, W))

    def octoMapBytes(self) -> bytes:
        """The last build's OctoMap .bt file, header and data."""
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_octomap_bt(self._h, None, 0, C.byref(n)))
        out = np.empty(max(n.value, 1), dtype=np.uint8)
        self._check(self._lib.b200sm_get_octomap_bt(self._h, _ptr(out), n.value, C.byref(n)))
        return out[:n.value].tobytes()

    def saveOctoMapBt(self, path) -> int:
        """The last build's OctoMap as a .bt file (octomap_server, MoveIt, rviz). Returns the file's bytes."""
        size = C.c_size_t(0)
        self._check(self._lib.b200sm_save_octomap_bt(self._h, os.fsencode(path), C.byref(size)))
        return int(size.value)

    # ---- map consistency: neighbourhood entropy and plane variance (b200sm_build_map_consistency, csrc/map_consistency.hpp) ----
    def buildMapConsistency(self, poses=None, radius: float = 0.5, min_neighbors: int = 10, query_stride: int = 1) -> dict:
        """How crisp the map of every submap at its own pose (poses None) or at `poses` (N, 4, 4) is, built on the device:
        per query point the entropy h and plane variance of its neighbours within `radius`, and their means MME and MPV
        over the valid queries. Returns the build's info as a dict (box_origin, box_dims, n_points, n_skipped, n_cells,
        n_queries, n_valid, n_neighbors, n_candidates, sum_h_q, sum_plane_q, mme, mpv)."""
        P = None
        if poses is not None:
            P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(self.numSubmaps(), 4, 4).transpose(0, 2, 1))
        prm = _capi.SmMapConsistencyParams(float(radius), int(min_neighbors), int(query_stride))
        info = _capi.SmMapConsistencyInfo()
        self._check(self._lib.b200sm_build_map_consistency(self._h, _ptr(P) if P is not None else None, C.byref(prm),
                                                           C.byref(info)))
        self._mc = (int(info.n_points), self.numSubmaps())
        return _struct_dict(info)

    def mapConsistency(self) -> dict:
        """The per-point layers of the last build in map order: n uint32 (neighbours of a query, 0 otherwise), h float64
        (nats) and plane_var float64 (m^2), NaN for an invalid query and for every other point."""
        M = getattr(self, "_mc", (0, 0))[0]
        out = dict(n=np.empty(M, dtype=np.uint32), h=np.empty(M, dtype=np.float64), plane_var=np.empty(M, dtype=np.float64))
        self._check(self._lib.b200sm_get_map_consistency(self._h, _ptr(out["n"]), _ptr(out["h"]), _ptr(out["plane_var"]), M))
        return out

    def submapConsistency(self) -> dict:
        """The per-submap rows of the last build as arrays of length N (submaps at the build): n_points, n_queries, n_valid,
        n_neighbors (uint64), sum_h_q, sum_plane_q (int64), mme, mpv (float64, NaN without a valid query)."""
        N = getattr(self, "_mc", (0, 0))[1]
        rows = (_capi.SmSubmapConsistency * max(N, 1))()
        self._check(self._lib.b200sm_get_submap_consistency(self._h, rows, N))
        out = {}
        for k, t in _capi.SmSubmapConsistency._fields_:
            dt = np.float64 if t is C.c_double else (np.int64 if t is C.c_longlong else np.uint64)
            out[k] = np.array([getattr(rows[i], k) for i in range(N)], dtype=dt)
        return out

    def saveMapConsistencyPcd(self, path):
        """pcl::io::savePCDFileASCII(path, map) of the map at the last build's poses with its intensity replaced by h (NaN
        where invalid), for a heat map in a viewer. Returns (points, file bytes)."""
        n, size = C.c_size_t(0), C.c_size_t(0)
        self._check(self._lib.b200sm_save_map_consistency_pcd_ascii(self._h, os.fsencode(path), C.byref(n), C.byref(size)))
        return int(n.value), int(size.value)

    # ---- read-back ----
    def stats(self) -> dict:
        st = _capi.SmStats()
        self._check(self._lib.b200sm_get_stats(self._h, C.byref(st)))
        return {k: getattr(st, k) for k, _ in _capi.SmStats._fields_}

    def numSubmaps(self) -> int:
        v = C.c_size_t(0)
        self._check(self._lib.b200sm_num_submaps(self._h, C.byref(v)))
        return int(v.value)

    def targetedCloud(self) -> np.ndarray:
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_targeted(self._h, None, 0, C.byref(n)))
        out = np.empty((n.value, 4), dtype=np.float32)
        self._check(self._lib.b200sm_get_targeted(self._h, _ptr(out), n.value, C.byref(n)))
        return out

    def filteredScan(self) -> np.ndarray:
        n = C.c_size_t(0)
        self._check(self._lib.b200sm_get_filtered_scan(self._h, None, 0, C.byref(n)))
        out = np.empty((n.value, 4), dtype=np.float32)
        self._check(self._lib.b200sm_get_filtered_scan(self._h, _ptr(out), n.value, C.byref(n)))
        return out

    def submap(self, index: int):
        n = C.c_size_t(0)
        pose = np.zeros(16, dtype=np.float64)
        dist = C.c_double(0)
        self._check(self._lib.b200sm_get_submap(self._h, index, None, 0, C.byref(n), _ptr(pose), C.byref(dist)))
        out = np.empty((n.value, 4), dtype=np.float32)
        self._check(self._lib.b200sm_get_submap(self._h, index, _ptr(out), n.value, C.byref(n), _ptr(pose), C.byref(dist)))
        return out, pose.reshape(4, 4).T.copy(), float(dist.value)


def _occupancy_info(info) -> dict:
    return {k: (tuple(getattr(info, k)) if k == "origin" else getattr(info, k)) for k, _ in _capi.SmOccupancyInfo._fields_}


def _struct_dict(st) -> dict:
    return {k: (tuple(getattr(st, k)) if hasattr(getattr(st, k), "_length_") else getattr(st, k)) for k, _ in st._fields_}


def backend_registration(registration_method: str = "NDT", ndt_resolution: float = 5.0, ndt_num_threads: int = 0, device: int = 0):
    """The backend node's registration object (graph_based_slam_component.cpp:44-70)."""
    if registration_method == "NDT":
        reg = NormalDistributionsTransform(device=device)
        reg.setMaximumIterations(100)
        reg.setResolution(ndt_resolution)
        reg.setTransformationEpsilon(0.01)
        reg.setNeighborhoodSearchMethod(2)  # pclomp::DIRECT7
        if ndt_num_threads > 0:
            reg.setNumThreads(ndt_num_threads)
        return reg
    if registration_method == "GICP":
        reg = GeneralizedIterativeClosestPoint(device=device)
        reg.setMaxCorrespondenceDistance(30)
        reg.setMaximumIterations(100)
        reg.setTransformationEpsilon(1e-8)
        reg.setEuclideanFitnessEpsilon(1e-6)
        reg.setRANSACIterations(0)
        return reg
    raise ValueError("registration_method must be NDT or GICP")


class LidarUndistortion:
    """scanmatcher/include/scanmatcher/lidar_undistortion.hpp on the GPU session (b200sm_imu_*): getImu keeps the IMU ring
    on the host like the reference, adjustDistortion runs as CUDA kernels on the uploaded scan."""

    def __init__(self, device: int = 0, scan_period: float = 0.1, session=None):
        import ctypes as C

        from . import _capi

        self._C, self._lib = C, _capi.lib()
        self._own = session is None
        if session is None:
            h = C.c_void_p()
            rc = self._lib.b200sm_create(int(device), C.byref(h))
            if rc != 0:
                raise RuntimeError(f"b200sm_create failed ({rc}): no CUDA device? there is no CPU fallback")
            self._s = h
        else:
            self._s = session
        self.setScanPeriod(scan_period)

    def __del__(self):
        if getattr(self, "_own", False) and getattr(self, "_s", None):
            self._lib.b200sm_destroy(self._s)
            self._s = None

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"b200sm error {rc}: {self._lib.b200sm_last_error(self._s).decode()}")

    def setScanPeriod(self, scan_period: float):
        self._check(self._lib.b200sm_imu_set_scan_period(self._s, float(scan_period)))

    def getImu(self, angular_velo, acc, quat_xyzw, imu_time: float):
        a = np.ascontiguousarray(angular_velo, dtype=np.float32)
        b = np.ascontiguousarray(acc, dtype=np.float32)
        q = np.ascontiguousarray(quat_xyzw, dtype=np.float32)
        self._check(self._lib.b200sm_imu_push(self._s, a.ctypes.data, b.ctypes.data, q.ctypes.data, float(imu_time)))

    def adjustDistortion(self, cloud, scan_time: float) -> np.ndarray:
        """cloud: (N, >=3) float32 in firing order; returns the corrected copy (other columns untouched)."""
        c = np.array(cloud, dtype=np.float32, copy=True, order="C")
        ioff = 12 if c.shape[1] >= 4 else -1
        self._check(self._lib.b200sm_imu_adjust_distortion(self._s, c.ctypes.data, len(c), c.strides[0], ioff, float(scan_time)))
        return c

    def pointers(self):
        C = self._C
        a, b, c = C.c_int(0), C.c_int(0), C.c_int(0)
        self._check(self._lib.b200sm_imu_get_state(self._s, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def sample(self, index: int):
        C = self._C
        t = C.c_double(0)
        rpy, sh, ve = (np.zeros(3, dtype=np.float32) for _ in range(3))
        self._check(self._lib.b200sm_imu_get_sample(self._s, int(index), C.byref(t), rpy.ctypes.data, sh.ctypes.data, ve.ctypes.data))
        return t.value, rpy, sh, ve

    def trace(self) -> dict:
        """The last adjustDistortion's per-point scratch (b200sm_imu_get_trace): rel_time (float32), t (float64), front
        (ring index after the walk), skip (bool), k_first (first index that set half_passed, n if none) and rounds
        (passes of the skipped-set fix point, 0 after a literal walk). n = 0 when no kernel ran."""
        C = self._C
        n, k, r = C.c_size_t(0), C.c_int(0), C.c_int(0)
        self._check(self._lib.b200sm_imu_get_trace(self._s, 0, C.byref(n), None, None, None, None, C.byref(k), C.byref(r)))
        m = n.value
        rel, t = np.zeros(m, dtype=np.float32), np.zeros(m, dtype=np.float64)
        front, skip = np.zeros(m, dtype=np.int32), np.zeros(m, dtype=np.uint8)
        if m:
            self._check(self._lib.b200sm_imu_get_trace(self._s, m, C.byref(n), rel.ctypes.data, t.ctypes.data,
                                                       front.ctypes.data, skip.ctypes.data, None, None))
        return {"n": m, "rel_time": rel, "t": t, "front": front, "skip": skip.astype(bool), "k_first": k.value,
                "rounds": r.value}
