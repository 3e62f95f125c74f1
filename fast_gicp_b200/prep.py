"""ctypes binding of lib/libvgicp_prep_b200.so (include/vgicp_prep_b200.h): device-side input preparation -- the near-origin
filter and pcl::ApproximateVoxelGrid the reference's callers run on the host before setInputTarget / setInputSource
(src/align.cpp:128-147, src/kitti.cpp:80-82, src/python/main.cpp:46-62).  Independent of the registration library; requires the
built CUDA library (no CPU fallback)."""
import ctypes as C
import os

import numpy as np

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libvgicp_prep_b200.so")
EXPORTED_SYMBOLS = ["vgicp_prep_create", "vgicp_prep_destroy", "vgicp_prep_last_error", "vgicp_prep_approximate_voxel_grid"]
_lib = None


class PrepError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"vgicp_prep status {code}: {msg}")
        self.code = code


def load_library():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python build_native.py` (the CUDA library is required; there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.vgicp_prep_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.vgicp_prep_destroy.argtypes = [C.c_void_p]
        L.vgicp_prep_destroy.restype = None
        L.vgicp_prep_last_error.argtypes = [C.c_void_p]
        L.vgicp_prep_last_error.restype = C.c_char_p
        L.vgicp_prep_approximate_voxel_grid.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_size_t, C.c_int,
                                                        C.POINTER(C.c_size_t)]
        _lib = L
    return _lib


class InputPrep:
    """One preparation context (stream + grow-only scratch) on a device."""

    def __init__(self, device=0):
        self._lib = load_library()
        self._h = C.c_void_p()
        rc = self._lib.vgicp_prep_create(int(device), C.byref(self._h))
        if rc:
            self._h = None
            raise PrepError(rc, "vgicp_prep_create failed (no sm_90a device?)")

    def close(self):
        if getattr(self, "_h", None):
            self._lib.vgicp_prep_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def approximate_voxel_grid(self, points, leaf, remove_near_origin=False):
        """pcl::ApproximateVoxelGrid(leaf) of an (n, >=3) float32 host array, optionally after align.cpp's near-origin filter;
        returns the (m, 3) float32 output in the order the serial filter emits it."""
        p = np.asarray(points)
        if p.dtype != np.float32 or p.ndim != 2 or p.shape[1] < 3 or not p.flags.c_contiguous:
            p = np.ascontiguousarray(np.asarray(points, dtype=np.float32)[:, :3])
        n = len(p)
        out = np.empty((n, 3), dtype=np.float32)
        m = C.c_size_t(0)
        rc = self._lib.vgicp_prep_approximate_voxel_grid(self._h, p.ctypes.data, n, p.strides[0] if n else 12, 0, C.c_float(leaf), int(bool(remove_near_origin)),
                                                         out.ctypes.data, n, 0, C.byref(m))
        if rc:
            raise PrepError(rc, self._lib.vgicp_prep_last_error(self._h).decode())
        return out[: m.value].copy()
