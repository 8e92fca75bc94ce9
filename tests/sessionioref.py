"""A Python restatement of csrc/session_io.hpp, the on-disk form of a mapping session (b200sm_save_session): the manifest
session.txt, the binary PCD header of a submap file, and pose_graph.g2o as the reference's optimizer.save writes it
(graph_based_slam_component.cpp:319). Nothing here needs a GPU.

g2o is not vendored in the reference. The g2o writer below (*g2o* OptimizableGraph::save with VertexSE3 / EdgeSE3 write:
token order, the space g2o leaves after every number, "FIX 0" after vertex 0, toVectorQT's normalised quaternion without a
sign change, ostream default precision) is restated from upstream g2o and cannot be checked against its source here; the
product's csrc/session_io.hpp carries the same note.

Poses are 4x4 row-major float64 matrices; the manifest prints them column-major. MUTATIONS names subtly wrong variants,
each of which the CPU tests show changes an output:
  precision16   doubles printed with %.16g (they no longer read back bitwise)
  segment_off   the odometry edges of every segment but the first start one submap early (an edge crosses the boundary)
  rowmajor      the manifest's poses printed row-major
  no_fix        no "FIX 0" line after vertex 0
"""
from __future__ import annotations

import numpy as np

import posegraphref as PG
from oracle.scanmatcher import quat_from_matrix

MUTATIONS = ("precision16", "segment_off", "rowmajor", "no_fix")


def _exact(x, mutations=()):
    return ("%.16g" if "precision16" in mutations else "%.17g") % float(x)


def _col16(P, mutations=()):
    P = np.asarray(P, dtype=np.float64)
    return (P.reshape(16) if "rowmajor" in mutations else P.T.reshape(16)).tolist()


def pcd_binary_header(n):
    """pcl::io::savePCDFileBinary's header for a dense PointXYZI cloud of n points."""
    return ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\n"
            f"TYPE F F F F\nCOUNT 1 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")


def submap_file(xyzi):
    """The bytes of a submap file: header, then the float32 rows (x, y, z, intensity)."""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    return pcd_binary_header(len(xyzi)).encode() + xyzi.tobytes()


def write_manifest(sc, seg_first, points, distances, poses, k, loops=(), adjusted=None, mutations=()):
    """sc = (num_rings, num_sectors, max_radius, lidar_height); poses / adjusted: (n, 4, 4); loops: (from, to, Z 4x4)."""
    e = lambda x: _exact(x, mutations)  # noqa: E731
    n = len(points)
    out = ["b200sm_session 1", f"scan_context {int(sc[0])} {int(sc[1])} {e(sc[2])} {e(sc[3])}", f"submaps {n}",
           " ".join(["segments", str(len(seg_first))] + [str(int(f)) for f in seg_first])]
    for i in range(n):
        out.append(" ".join(["submap", str(i), str(int(points[i])), e(distances[i])] + [e(v) for v in _col16(poses[i], mutations)]))
    out.append(f"odometry {int(k)}")
    out.append(f"loops {len(loops)}")
    for f, t, Z in loops:
        out.append(" ".join(["loop", str(int(f)), str(int(t))] + [e(v) for v in _col16(Z, mutations)]))
    out.append("adjusted 1" if adjusted is not None else "adjusted 0")
    if adjusted is not None:
        for i in range(n):
            out.append(" ".join(["pose", str(i)] + [e(v) for v in _col16(adjusted[i], mutations)]))
    return "".join(line + "\n" for line in out)


def graph_edges(poses, k, seg_first, loops=(), mutations=()):
    """(from, to, Z) of every edge in the order b200sm_pose_adjust builds them: odometry per segment (for local i > k, (i-k+j,
    i), j = 0..k-1) with Z = P_from^-1 P_to of the submaps' own poses, then the loop edges as given."""
    n = len(poses)
    E = []
    for s, f0 in enumerate(seg_first):
        f1 = seg_first[s + 1] if s + 1 < len(seg_first) else n
        if "segment_off" in mutations and s > 0:
            f0 -= 1
        for i in range(k + 1, f1 - f0):
            for j in range(k):
                f, t = f0 + i - k + j, f0 + i
                E.append((f, t, PG.compose(PG.inverse(poses[f]), poses[t])))
    E += [(int(f), int(t), np.asarray(Z, dtype=np.float64)) for f, t, Z in loops]
    return E


def _qt(P):
    """*g2o* toVectorQT: x y z, then Quaterniond(R) normalised (qx qy qz qw), each as '%g '."""
    q = quat_from_matrix(P[:3, :3])
    nq = np.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    return "".join("%g " % float(v) for v in [P[0, 3], P[1, 3], P[2, 3], q[0] / nq, q[1] / nq, q[2] / nq, q[3] / nq])


def write_g2o(poses, k, seg_first, loops=(), adjusted=None, mutations=()):
    out = []
    V = adjusted if adjusted is not None else poses
    for i in range(len(poses)):
        out.append(f"VERTEX_SE3:QUAT {i} " + _qt(np.asarray(V[i], dtype=np.float64)) + "\n")
        if i == 0 and "no_fix" not in mutations:
            out.append("FIX 0\n")
    info = "".join("1 " if r == c else "0 " for r in range(6) for c in range(r, 6))
    for f, t, Z in graph_edges(poses, k, seg_first, loops, mutations):
        out.append(f"EDGE_SE3:QUAT {f} {t} " + _qt(Z) + info + "\n")
    return "".join(out)
