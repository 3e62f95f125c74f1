"""ctypes front-end of the field-averaging voxel-grid checker (oracle_fields/fields_oracle.c).

TEST INFRASTRUCTURE ONLY, like `oracle`: the serial pcl::ApproximateVoxelGrid<PointT> with per-point float fields, the reference
for vgicp_prep_approximate_voxel_grid_fields and the serial C filter scripts/bench_raw_scans.py times as the host route; and the
serial pcl::VoxelGrid<PointT> (the exact grid), the reference for vgicp_prep_voxel_grid.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libfields_oracle.so")
_SRC = os.path.join(_HERE, "fields_oracle.c")
# the oracle's flags (oracle/Makefile): no contraction, no fast math
CFLAGS = ["-O2", "-std=c11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wall"]


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
        env = {k: v for k, v in os.environ.items() if k not in ("CC", "CFLAGS")}
        subprocess.check_call([cc] + CFLAGS + ["-shared", "-o", _LIB_PATH, _SRC, "-lm"], env=env)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.orc_approximate_voxel_grid_fields.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_float, C.c_int, C.c_int, C.c_void_p]
        L.orc_approximate_voxel_grid_fields.restype = C.c_int
        L.orc_voxel_grid_fields.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_float, C.c_int, C.c_uint, C.c_void_p]
        L.orc_voxel_grid_fields.restype = C.c_int
        _lib = L
    return _lib


def approximate_voxel_grid_fields(records, leaf, cols, remove_near_origin=False, histsize=512):
    """records: (n, k) float32, x y z in columns 0 1 2; cols: the field columns -> (m, 3 + len(cols)) float32 in the order the
    serial filter emits them (optionally after align.cpp's near-origin filter)."""
    r = np.ascontiguousarray(records, dtype=np.float32)
    if r.ndim != 2 or r.shape[1] < 3:
        raise ValueError("records must be (n, k >= 3)")
    c = np.ascontiguousarray(cols, dtype=np.int32).reshape(-1)
    out = np.empty((len(r), 3 + len(c)), dtype=np.float32)
    m = lib().orc_approximate_voxel_grid_fields(r.ctypes.data, len(r), r.shape[1], c.ctypes.data_as(C.POINTER(C.c_int)), len(c), C.c_float(leaf), int(histsize),
                                                int(bool(remove_near_origin)), out.ctypes.data)
    if m < 0:
        raise ValueError("orc_approximate_voxel_grid_fields: bad field columns or count")
    return out[:m].copy()


class Refused(ValueError):
    """The exact grid refuses the cloud: a kept cell outside the int range, or more than INT32_MAX cells in the box."""


def voxel_grid_fields(records, leaf, cols, remove_near_origin=False, min_points=0):
    """pcl::VoxelGrid (the exact grid) of (n, k) float32 records, x y z in columns 0 1 2, averaging the field columns `cols`
    -> (m, 3 + len(cols)) float32 in ascending voxel index.  Raises Refused where vgicp_prep_voxel_grid returns status 1 for the
    cloud itself."""
    r = np.ascontiguousarray(records, dtype=np.float32)
    if r.ndim != 2 or r.shape[1] < 3:
        raise ValueError("records must be (n, k >= 3)")
    c = np.ascontiguousarray(cols, dtype=np.int32).reshape(-1)
    out = np.empty((len(r), 3 + len(c)), dtype=np.float32)
    m = lib().orc_voxel_grid_fields(r.ctypes.data, len(r), r.shape[1], c.ctypes.data_as(C.POINTER(C.c_int)), len(c), C.c_float(leaf), int(bool(remove_near_origin)),
                                    int(min_points), out.ctypes.data)
    if m == -2:
        raise Refused("orc_voxel_grid_fields: a cell lies outside the int range or the box holds more than INT32_MAX cells")
    if m < 0:
        raise ValueError("orc_voxel_grid_fields: bad field columns or count, or a leaf that is not finite and positive")
    return out[:m].copy()
