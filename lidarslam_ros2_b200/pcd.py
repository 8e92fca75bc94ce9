"""Minimal reader for binary PCD files (the two fixtures of Thirdparty/ndt_omp_ros2/data/, FIELDS x y z intensity,
DATA binary) — what apps/align.cpp:55-62 loads with pcl::io::loadPCDFile — the ASCII PCD text that
pcl::io::savePCDFileASCII writes, formatted on the GPU (b200reg_encode_pcd_ascii), and loadPCDFile itself with the text
parsed on the GPU (read_pcd, b200reg_load_pcd)."""
from __future__ import annotations

import ctypes as C

import numpy as np


def load_pcd(path: str) -> np.ndarray:
    with open(path, "rb") as f:
        data = f.read()
    marker = b"DATA binary\n"
    k = data.index(marker) + len(marker)
    header = data[:k].decode("ascii", "replace").splitlines()
    fields = next(l for l in header if l.startswith("FIELDS")).split()[1:]
    sizes = [int(v) for v in next(l for l in header if l.startswith("SIZE")).split()[1:]]
    n = int(next(l for l in header if l.startswith("POINTS")).split()[1])
    if any(s != 4 for s in sizes):
        raise ValueError("only 4-byte fields supported")
    return np.frombuffer(data[k:k + n * 4 * len(fields)], dtype=np.float32).reshape(n, len(fields)).copy()


def encode_pcd_ascii(cloud, device: int = 0) -> bytes:
    """The bytes savePCDFileASCII writes for a pcl::PointCloud<PointXYZI>: cloud is (N, >=4) float32 rows of x, y, z,
    intensity (N >= 1). The floats are formatted by CUDA kernels on `device`; there is no CPU fallback."""
    from . import _capi
    from .registration import B200RegError

    p = np.ascontiguousarray(cloud, dtype=np.float32)
    if p.ndim != 2 or p.shape[1] < 4:
        raise ValueError("cloud must be (N, >=4) float32: x, y, z, intensity")
    L = _capi.lib()
    n, w = p.shape
    size = C.c_size_t(0)
    args = (int(device), p.ctypes.data_as(C.c_void_p), n, 4 * w, 12)
    rc = L.b200reg_encode_pcd_ascii(*args, None, 0, C.byref(size))
    if rc != 0:
        raise B200RegError(rc, "b200reg_encode_pcd_ascii failed")
    out = bytearray(size.value)
    rc = L.b200reg_encode_pcd_ascii(*args, (C.c_char * len(out)).from_buffer(out), len(out), C.byref(size))
    if rc != 0:
        raise B200RegError(rc, "b200reg_encode_pcd_ascii failed")
    return bytes(out)


def read_pcd(path: str, device: int = 0) -> np.ndarray:
    """pcl::io::loadPCDFile into a PointXYZI cloud: (N, 4) float32 rows of x, y, z, intensity (0 when the file has none).
    DATA ascii is parsed and DATA binary unpacked by CUDA kernels on `device` (contract: b200reg_load_pcd in
    include/b200reg.h); there is no CPU fallback. Raises B200RegError (ERR_IO, ERR_FORMAT) like loadPCDFile returns -1."""
    import os

    from . import _capi
    from .registration import B200RegError

    L = _capi.lib()
    p = os.fsencode(path)
    n = C.c_size_t(0)
    rc = L.b200reg_load_pcd(int(device), p, None, 0, C.byref(n))
    if rc != 0:
        raise B200RegError(rc, f"b200reg_load_pcd failed on {path}")
    out = np.empty((n.value, 4), dtype=np.float32)
    if n.value:
        rc = L.b200reg_load_pcd(int(device), p, out.ctypes.data_as(C.c_void_p), n.value, C.byref(n))
        if rc != 0:
            raise B200RegError(rc, f"b200reg_load_pcd failed on {path}")
    return out
