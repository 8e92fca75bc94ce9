"""ORACLE — TEST INFRASTRUCTURE ONLY (parity unpinned; see oracle/ndt.hpp header and DESIGN.md).

ctypes binding of ``oracle/liboracle.so``, the dependency-free CPU/OpenMP restatement of the
reference's registration path (pclomp NDT / GICP, pcl::VoxelGrid, getFitnessScore).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this package — and there only as the checker / timed CPU baseline. Nothing under
``lidarslam_ros2_b200/`` imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

KDTREE, DIRECT26, DIRECT7, DIRECT1 = 0, 1, 2, 3


def build(force: bool = False) -> str:
    """Compile oracle/liboracle.so with the committed Makefile (g++ -O3 -fopenmp)."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".hpp", ".cpp"))]
    stale = (not os.path.exists(_LIB_PATH)) or any(
        os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs
    )
    if force or stale:
        subprocess.check_call(["make", "-s", "-C", _HERE] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        fp, dp, ip = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int)
        vp, sz = C.c_void_p, C.c_size_t
        L.oracle_max_threads.restype = C.c_int
        L.oracle_voxelgrid.restype = sz
        L.oracle_voxelgrid.argtypes = [vp, sz, sz, C.c_long, C.c_float, vp, sz]
        L.oracle_ndt_create.restype = vp
        L.oracle_ndt_destroy.argtypes = [vp]
        L.oracle_ndt_set.argtypes = [vp, C.c_char_p, C.c_double]
        L.oracle_ndt_set.restype = C.c_int
        L.oracle_ndt_set_target.argtypes = [vp, vp, sz, sz]
        L.oracle_ndt_set_source.argtypes = [vp, vp, sz, sz]
        L.oracle_ndt_align.argtypes = [vp, vp, vp, ip, ip, dp, ip]
        L.oracle_ndt_fitness.argtypes = [vp, C.c_double]
        L.oracle_ndt_fitness.restype = C.c_double
        L.oracle_ndt_derivatives.argtypes = [vp, vp, vp, C.c_int, vp, vp]
        L.oracle_ndt_derivatives.restype = C.c_double
        L.oracle_ndt_hessian.argtypes = [vp, vp, vp, vp]
        L.oracle_ndt_calculate_score.argtypes = [vp, vp]
        L.oracle_ndt_calculate_score.restype = C.c_double
        L.oracle_ndt_num_voxels.argtypes = [vp]
        L.oracle_ndt_num_voxels.restype = sz
        L.oracle_ndt_num_leaves.argtypes = [vp]
        L.oracle_ndt_num_leaves.restype = sz
        L.oracle_ndt_get_voxels.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.oracle_ndt_grid_geom.argtypes = [vp, vp, vp]
        L.oracle_ndt_gauss.argtypes = [vp, vp]
        L.oracle_euler_angles_012.argtypes = [vp, vp]
        L.oracle_pose_to_matrix.argtypes = [vp, vp]
        L.oracle_sym_eigen3.argtypes = [vp, vp, vp]
        L.oracle_svd6_solve.argtypes = [vp, vp, vp]
        L.oracle_mat3_inverse.argtypes = [vp, vp]
        L.oracle_mt_trial.argtypes = [vp]
        L.oracle_mt_trial.restype = C.c_double
        L.oracle_mt_update.argtypes = [vp, vp]
        L.oracle_mt_update.restype = C.c_int
        L.oracle_angle_tables.argtypes = [vp, vp, vp]
        L.oracle_nn1.argtypes = [vp, sz, sz, vp, sz, sz, vp, vp]
        L.oracle_gicp_create.restype = vp
        L.oracle_gicp_destroy.argtypes = [vp]
        L.oracle_gicp_set.argtypes = [vp, C.c_char_p, C.c_double]
        L.oracle_gicp_set.restype = C.c_int
        L.oracle_gicp_set_target.argtypes = [vp, vp, sz, sz]
        L.oracle_gicp_set_source.argtypes = [vp, vp, sz, sz]
        L.oracle_gicp_align.argtypes = [vp, vp, vp, ip, ip]
        L.oracle_gicp_fitness.argtypes = [vp, C.c_double]
        L.oracle_gicp_fitness.restype = C.c_double
        L.oracle_gicp_get_covariances.argtypes = [vp, C.c_int, vp]
        L.oracle_gicp_get_covariances.restype = sz
        L.oracle_gicp_fdf.argtypes = [vp, vp, vp]
        L.oracle_gicp_fdf.restype = C.c_double
        L.oracle_gicp_num_correspondences.argtypes = [vp]
        L.oracle_gicp_num_correspondences.restype = C.c_int
        L.oracle_gicp_f_only.argtypes = [vp, vp]
        L.oracle_gicp_f_only.restype = C.c_double
        L.oracle_gicp_apply_state.argtypes = [vp, vp, vp]
        L.oracle_gicp_correspondences.argtypes = [vp, vp, vp, vp]
        L.oracle_gicp_set_trace.argtypes = [vp, C.c_int]
        L.oracle_gicp_get_trace.argtypes = [vp, vp, C.c_int]
        L.oracle_gicp_get_trace.restype = C.c_int
        _lib = L
    return _lib


def _cloud(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] >= 3
    return a


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _colmajor(T) -> np.ndarray:
    """row-major numpy 4x4 -> 16 floats column-major (Eigen data() order)."""
    return np.ascontiguousarray(np.asarray(T, dtype=np.float32).T).reshape(16)


def _from_colmajor(buf: np.ndarray) -> np.ndarray:
    return buf.reshape(4, 4).T.copy()


def max_threads() -> int:
    return int(lib().oracle_max_threads())


def voxelgrid(points, leaf: float) -> np.ndarray:
    """pcl::VoxelGrid centroid downsample. points: (N,3) xyz or (N,4) xyz+intensity -> (M,4)."""
    p = _cloud(points)
    n, w = p.shape
    out = np.empty((max(n, 1), 4), dtype=np.float32)
    m = lib().oracle_voxelgrid(_ptr(p), n, w * 4, 12 if w >= 4 else -1, float(leaf), _ptr(out), n)
    return out[:m].copy()


def nn1(target, query):
    t, q = _cloud(target), _cloud(query)
    idx = np.empty(len(q), dtype=np.int32)
    d2 = np.empty(len(q), dtype=np.float32)
    lib().oracle_nn1(_ptr(t), len(t), t.shape[1] * 4, _ptr(q), len(q), q.shape[1] * 4, _ptr(idx), _ptr(d2))
    return idx, d2


class NDT:
    """CPU restatement of pclomp::NormalDistributionsTransform (ndt_omp.h:70-497)."""

    def __init__(self, **params):
        self._h = lib().oracle_ndt_create()
        self.final_transformation = np.eye(4, dtype=np.float32)
        self.converged = False
        self.iterations = 0
        self.trans_probability = 0.0
        self.evaluations = 0
        for k, v in params.items():
            self.set(k, v)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().oracle_ndt_destroy(self._h)
            self._h = None

    def set(self, key: str, value: float):
        if lib().oracle_ndt_set(self._h, key.encode(), float(value)) != 0:
            raise KeyError(key)

    def set_target(self, pts):
        p = _cloud(pts)
        lib().oracle_ndt_set_target(self._h, _ptr(p), len(p), p.shape[1] * 4)

    def set_source(self, pts):
        p = _cloud(pts)
        lib().oracle_ndt_set_source(self._h, _ptr(p), len(p), p.shape[1] * 4)

    def align(self, guess=None) -> np.ndarray:
        g = _colmajor(guess) if guess is not None else None
        out = np.empty(16, dtype=np.float32)
        conv, it, ne = C.c_int(0), C.c_int(0), C.c_int(0)
        tp = C.c_double(0)
        lib().oracle_ndt_align(self._h, _ptr(g) if g is not None else None, _ptr(out), C.byref(conv), C.byref(it),
                               C.byref(tp), C.byref(ne))
        self.final_transformation = _from_colmajor(out)
        self.converged, self.iterations = bool(conv.value), it.value
        self.trans_probability, self.evaluations = tp.value, ne.value
        return self.final_transformation

    def fitness(self, max_range: float = np.finfo(np.float64).max) -> float:
        return float(lib().oracle_ndt_fitness(self._h, float(max_range)))

    def derivatives(self, T, p6, compute_hessian: bool = True):
        Tc = _colmajor(T)
        p = np.ascontiguousarray(p6, dtype=np.float64)
        g = np.zeros(6)
        H = np.zeros((6, 6))
        s = lib().oracle_ndt_derivatives(self._h, _ptr(Tc), _ptr(p), int(compute_hessian), _ptr(g), _ptr(H))
        return float(s), g, H

    def hessian_radius(self, T, p6):
        Tc = _colmajor(T)
        p = np.ascontiguousarray(p6, dtype=np.float64)
        H = np.zeros((6, 6))
        lib().oracle_ndt_hessian(self._h, _ptr(Tc), _ptr(p), _ptr(H))
        return H

    def calculate_score(self, T) -> float:
        Tc = _colmajor(T)
        return float(lib().oracle_ndt_calculate_score(self._h, _ptr(Tc)))

    def voxels(self):
        n = lib().oracle_ndt_num_voxels(self._h)
        idx = np.empty(n, dtype=np.int32)
        npts = np.empty(n, dtype=np.int32)
        mean = np.empty((n, 3))
        cov = np.empty((n, 3, 3))
        icov = np.empty((n, 3, 3))
        cen = np.empty((n, 3), dtype=np.float32)
        lib().oracle_ndt_get_voxels(self._h, _ptr(idx), _ptr(npts), _ptr(mean), _ptr(cov), _ptr(icov), _ptr(cen))
        return dict(idx=idx, npts=npts, mean=mean, cov=cov, icov=icov, centroid=cen)

    def num_leaves(self) -> int:
        return int(lib().oracle_ndt_num_leaves(self._h))

    def grid_geom(self):
        mb = np.zeros(3, dtype=np.int32)
        db = np.zeros(3, dtype=np.int32)
        lib().oracle_ndt_grid_geom(self._h, _ptr(mb), _ptr(db))
        return mb, db

    def gauss(self):
        d = np.zeros(3)
        lib().oracle_ndt_gauss(self._h, _ptr(d))
        return tuple(d)


class GICP:
    """CPU restatement of pclomp::GeneralizedIterativeClosestPoint (gicp_omp.h:60-369)."""

    # GicpTraceRec (oracle/gicp.hpp), the layout of the engine's b200reg_gicp_trace_record
    TRACE_DTYPE = np.dtype([(k, np.int32) for k in (
        "type", "outer", "inner", "evaluation", "want_grad", "status", "m", "nr_iterations", "converged", "last")]
        + [("x", np.float64, (6,)), ("f", np.float64), ("g", np.float64, (6,)), ("x0", np.float64, (6,)),
           ("delta", np.float64), ("T", np.float32, (12,)), ("final_T", np.float32, (16,))])

    def __init__(self, **params):
        self._h = lib().oracle_gicp_create()
        self.final_transformation = np.eye(4, dtype=np.float32)
        self.converged = False
        self.iterations = 0
        for k, v in params.items():
            self.set(k, v)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().oracle_gicp_destroy(self._h)
            self._h = None

    def set(self, key: str, value: float):
        if lib().oracle_gicp_set(self._h, key.encode(), float(value)) != 0:
            raise KeyError(key)

    def set_target(self, pts):
        p = _cloud(pts)
        lib().oracle_gicp_set_target(self._h, _ptr(p), len(p), p.shape[1] * 4)

    def set_source(self, pts):
        p = _cloud(pts)
        lib().oracle_gicp_set_source(self._h, _ptr(p), len(p), p.shape[1] * 4)

    def align(self, guess=None) -> np.ndarray:
        g = _colmajor(guess) if guess is not None else None
        out = np.empty(16, dtype=np.float32)
        conv, it = C.c_int(0), C.c_int(0)
        lib().oracle_gicp_align(self._h, _ptr(g) if g is not None else None, _ptr(out), C.byref(conv), C.byref(it))
        self.final_transformation = _from_colmajor(out)
        self.converged, self.iterations = bool(conv.value), it.value
        return self.final_transformation

    def fitness(self, max_range: float = np.finfo(np.float64).max) -> float:
        return float(lib().oracle_gicp_fitness(self._h, float(max_range)))

    def set_trace(self, on: bool = True):
        """Record the optimiser's functor calls, BFGS steps and outer iterations of every following align()."""
        lib().oracle_gicp_set_trace(self._h, int(bool(on)))

    def trace(self) -> np.ndarray:
        """The records of the last align() as a TRACE_DTYPE record array."""
        n = lib().oracle_gicp_get_trace(self._h, None, 0)
        out = np.zeros(n, dtype=self.TRACE_DTYPE)
        if n:
            lib().oracle_gicp_get_trace(self._h, _ptr(out), n)
        return out

    def covariances(self, which: str):
        w = 1 if which == "target" else 0
        n = lib().oracle_gicp_get_covariances(self._h, w, None)
        out = np.empty((n, 3, 3))
        lib().oracle_gicp_get_covariances(self._h, w, _ptr(out))
        return out

    def fdf(self, x6):
        x = np.ascontiguousarray(x6, dtype=np.float64)
        g = np.zeros(6)
        f = lib().oracle_gicp_fdf(self._h, _ptr(x), _ptr(g))
        return float(f), g

    def num_correspondences(self) -> int:
        return int(lib().oracle_gicp_num_correspondences(self._h))

    def f_only(self, x6) -> float:
        """The functor's operator() (f32 residual and M r, f64 sum) at state x on the last correspondences."""
        x = np.ascontiguousarray(x6, dtype=np.float64)
        return float(lib().oracle_gicp_f_only(self._h, _ptr(x)))

    def apply_state(self, x6) -> np.ndarray:
        """applyState(base_transformation_, x): the f32 transform the functor evaluates at, row-major 4x4."""
        x = np.ascontiguousarray(x6, dtype=np.float64)
        out = np.empty(16, dtype=np.float32)
        lib().oracle_gicp_apply_state(self._h, _ptr(x), _ptr(out))
        return _from_colmajor(out)

    def correspondences(self):
        """(src_idx, tgt_idx, mahalanobis (m, 3, 3) float32) of the last outer iteration."""
        m = self.num_correspondences()
        s = np.empty(m, dtype=np.int32)
        t = np.empty(m, dtype=np.int32)
        M = np.empty((m, 3, 3), dtype=np.float32)
        if m:
            lib().oracle_gicp_correspondences(self._h, _ptr(s), _ptr(t), _ptr(M))
        return s, t, M


# ---- known-answer hooks ----
def euler_angles_012(R) -> np.ndarray:
    r = np.ascontiguousarray(R, dtype=np.float32).reshape(9)
    out = np.zeros(3, dtype=np.float32)
    lib().oracle_euler_angles_012(_ptr(r), _ptr(out))
    return out


def pose_to_matrix(p6) -> np.ndarray:
    p = np.ascontiguousarray(p6, dtype=np.float64)
    out = np.zeros(16, dtype=np.float32)
    lib().oracle_pose_to_matrix(_ptr(p), _ptr(out))
    return _from_colmajor(out)


def sym_eigen3(A):
    a = np.ascontiguousarray(A, dtype=np.float64).reshape(9)
    ev = np.zeros(3)
    V = np.zeros((3, 3))
    lib().oracle_sym_eigen3(_ptr(a), _ptr(ev), _ptr(V))
    return ev, V


def svd6_solve(A, b) -> np.ndarray:
    a = np.ascontiguousarray(A, dtype=np.float64).reshape(36)
    bb = np.ascontiguousarray(b, dtype=np.float64)
    x = np.zeros(6)
    lib().oracle_svd6_solve(_ptr(a), _ptr(bb), _ptr(x))
    return x


def mat3_inverse(A) -> np.ndarray:
    a = np.ascontiguousarray(A, dtype=np.float64).reshape(9)
    out = np.zeros((3, 3))
    lib().oracle_mat3_inverse(_ptr(a), _ptr(out))
    return out


def mt_trial(a_l, f_l, g_l, a_u, f_u, g_u, a_t, f_t, g_t) -> float:
    v = np.array([a_l, f_l, g_l, a_u, f_u, g_u, a_t, f_t, g_t], dtype=np.float64)
    return float(lib().oracle_mt_trial(_ptr(v)))


def mt_update(a_l, f_l, g_l, a_u, f_u, g_u, a_t, f_t, g_t):
    v = np.array([a_l, f_l, g_l, a_u, f_u, g_u], dtype=np.float64)
    t = np.array([a_t, f_t, g_t], dtype=np.float64)
    conv = lib().oracle_mt_update(_ptr(v), _ptr(t))
    return bool(conv), v


def angle_tables(p6):
    p = np.ascontiguousarray(p6, dtype=np.float64)
    j = np.zeros((8, 3), dtype=np.float32)
    h = np.zeros((15, 3), dtype=np.float32)
    lib().oracle_angle_tables(_ptr(p), _ptr(j), _ptr(h))
    return j, h
