"""A numpy float64 restatement of the backend's pose adjustment, GraphBasedSlamComponent::doPoseAdjustment
(graph_based_slam/src/graph_based_slam_component.cpp:262-319): the SE3 pose graph, g2o's EdgeSE3 error and Jacobians and
Levenberg-Marquardt, solved densely (the product factors an envelope; a dense factorisation is fine at test sizes).
Nothing here needs a GPU.

g2o is not vendored in the reference. Everything marked *g2o* is restated from upstream g2o (types/slam3d EdgeSE3 /
VertexSE3 / isometry3d_mappings, core/optimization_algorithm_levenberg.cpp) and cannot be checked against source here; the
product's csrc/pose_graph.hpp carries the same note.

Poses are 4x4 row-major float64 matrices. Products are written out left to right, ((a0 b0 + a1 b1) + a2 b2), like
csrc/pose_graph.hpp: then compose(inverse(P), P) has an exactly zero translation and an exactly symmetric rotation, so an
edge built from the current estimates has an error of exactly zero.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from oracle.scanmatcher import pose_matrix, quat_from_matrix

DBL_MAX = np.finfo(np.float64).max


def compose(A, B):
    C = np.eye(4)
    for i in range(3):
        for j in range(3):
            C[i, j] = (A[i, 0] * B[0, j] + A[i, 1] * B[1, j]) + A[i, 2] * B[2, j]
        C[i, 3] = ((A[i, 0] * B[0, 3] + A[i, 1] * B[1, 3]) + A[i, 2] * B[2, 3]) + A[i, 3]
    return C


def inverse(A):
    """Isometry3d::inverse(): R^T, -(R^T t)."""
    B = np.eye(4)
    B[:3, :3] = A[:3, :3].T
    for i in range(3):
        B[i, 3] = -((A[0, i] * A[0, 3] + A[1, i] * A[1, 3]) + A[2, i] * A[2, 3])
    return B


def from_vector_mqt(d):
    """*g2o* internal::fromVectorMQT: translation d[:3], rotation fromCompactQuaternion(d[3:]) (identity if |v| > 1)."""
    d = np.asarray(d, dtype=np.float64)
    v = d[3:]
    w2 = 1.0 - ((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
    q = [0.0, 0.0, 0.0, 1.0] if w2 < 0.0 else [v[0], v[1], v[2], np.sqrt(w2)]
    return pose_matrix(d[:3], q)


def compact_quaternion(R):
    """*g2o* internal::toCompactQuaternion: Quaternion(R) normalised, w >= 0. Returns (w, xyz)."""
    q = quat_from_matrix(R)
    n = np.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    q = q / n
    if q[3] < 0.0:
        q = -q
    return q[3], q[:3].copy()


def edge_error(Xf, Xt, Zinv):
    """*g2o* EdgeSE3::computeError: toVectorMQT(Z^-1 * X_from^-1 * X_to), evaluated as Z^-1 * (X_from^-1 * X_to)."""
    E = compose(Zinv, compose(inverse(Xf), Xt))
    _, v = compact_quaternion(E[:3, :3])
    return np.concatenate([E[:3, 3], v]), E


def _skew(a):
    return np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])


def edge_jacobians(E, Zinv):
    """d e / d delta for X <- X * fromVectorMQT(delta) of both vertices at delta = 0 (closed form; see pose_graph.hpp)."""
    w, q = compact_quaternion(E[:3, :3])
    RA, tA = Zinv[:3, :3], Zinv[:3, 3]
    Jf, Jt = np.zeros((6, 6)), np.zeros((6, 6))
    Jt[:3, :3] = E[:3, :3]
    Jt[3:, 3:] = w * np.eye(3) + _skew(q)
    Jf[:3, :3] = -RA
    Jf[:3, 3:] = _skew(2.0 * (E[:3, 3] - tA)) @ RA
    Jf[3:, 3:] = -(w * np.eye(3) - _skew(q)) @ RA
    return Jf, Jt


def graph_edges(n, k):
    """The odometry edges of gbs.cpp:289-305, literally: for i > k, (i - k + j, i) for j = 0..k-1."""
    return [(i - k + j, i) for i in range(n) if i > k for j in range(k)]


def build_edges(poses, k, loop_edges=()):
    """(from, to, Z^-1) of every edge: odometry with Z = pose_from^-1 * pose_to, then loop edges (from, to, Z)."""
    E = [(f, t, inverse(compose(inverse(poses[f]), poses[t]))) for f, t in graph_edges(len(poses), k)]
    E += [(int(f), int(t), inverse(np.asarray(Z, dtype=np.float64))) for f, t, Z in loop_edges]
    return E


def chi2(X, edges):
    s = 0.0
    for f, t, Zinv in edges:
        e, _ = edge_error(X[f], X[t], Zinv)
        s += float(np.sum(e * e))
    return s


def optimize(poses, edges, max_iterations=10):
    """*g2o* SparseOptimizer::optimize + OptimizationAlgorithmLevenberg::solve (rules in pose_graph.hpp). Returns
    (poses, result dict, trials [(iteration, accepted, lambda, chi2_after)])."""
    X = [np.array(P, dtype=np.float64) for P in poses]
    n = len(X)
    touched = set()
    for f, t, _ in edges:
        touched.update((f, t))
    free = [i for i in range(1, n) if i in touched]
    pos = {v: p for p, v in enumerate(free)}
    current = chi2(X, edges)
    res = {"chi2_initial": current, "chi2_final": current, "iterations": 0, "trials": 0}
    trace = []
    if not free or max_iterations <= 0:
        return X, res, trace
    m = 6 * len(free)
    lam, nu = 0.0, 2.0
    for it in range(max_iterations):
        current = chi2(X, edges)
        H, b = np.zeros((m, m)), np.zeros(m)
        for f, t, Zinv in edges:
            e, E = edge_error(X[f], X[t], Zinv)
            Jf, Jt = edge_jacobians(E, Zinv)
            for vu, Ju in ((f, Jf), (t, Jt)):
                if vu not in pos:
                    continue
                pu = 6 * pos[vu]
                b[pu:pu + 6] -= Ju.T @ e
                for vw, Jw in ((f, Jf), (t, Jt)):
                    if vw in pos:
                        pw = 6 * pos[vw]
                        H[pu:pu + 6, pw:pw + 6] += Ju.T @ Jw
        if it == 0:
            lam, nu = 1e-5 * np.abs(np.diag(H)).max(), 2.0
        q, rho = 0, 0.0
        while True:
            backup = [x.copy() for x in X]
            try:
                dx = scipy.linalg.cho_solve(scipy.linalg.cho_factor(H + lam * np.eye(m), lower=True), b)
                ok = bool(np.all(np.isfinite(dx)))
            except np.linalg.LinAlgError:
                ok = False
            if ok:
                for v, p in pos.items():
                    X[v] = compose(X[v], from_vector_mqt(dx[6 * p:6 * p + 6]))
                chi_new = chi2(X, edges)
            else:
                dx, chi_new = np.zeros(m), DBL_MAX
            scale = float(np.sum(dx * (lam * dx + b)))
            rho = (current - chi_new) / (scale + 1e-3)
            used = lam
            accept = rho > 0 and np.isfinite(chi_new)
            if accept:
                lam *= max(1.0 / 3.0, min(1.0 - (2.0 * rho - 1.0) ** 3, 2.0 / 3.0))
                nu = 2.0
                current = chi_new
            else:
                lam *= nu
                nu *= 2.0
                X = backup
            res["trials"] += 1
            trace.append((it, int(accept), used, chi_new))
            if not accept and not np.isfinite(lam):
                break
            q += 1
            if not (rho < 0 and q < 10):
                break
        res["iterations"] += 1
        if q == 10 or rho == 0 or not np.isfinite(lam):
            break
    res["chi2_final"] = current
    return X, res, trace


def pose_adjust(poses, k=5, loop_edges=(), max_iterations=10):
    """doPoseAdjustment's solve (gbs.cpp:267-319) on submap poses (N, 4, 4): returns (adjusted poses, result, trials)."""
    return optimize(poses, build_edges(poses, k, loop_edges), max_iterations)
