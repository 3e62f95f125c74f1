"""ctypes binding of lib/libvgicp_prep_b200.so (include/vgicp_prep_b200.h): device-side input preparation -- the near-origin
filter and pcl::ApproximateVoxelGrid the reference's callers run on the host before setInputTarget / setInputSource
(src/align.cpp:128-147, src/kitti.cpp:80-82, src/python/main.cpp:46-62), and pcl::VoxelGrid, the exact grid.  Independent of the registration library; requires the
built CUDA library (no CPU fallback)."""
import ctypes as C
import os

import numpy as np

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libvgicp_prep_b200.so")
EXPORTED_SYMBOLS = ["vgicp_prep_create", "vgicp_prep_destroy", "vgicp_prep_last_error", "vgicp_prep_approximate_voxel_grid",
                    "vgicp_prep_approximate_voxel_grid_fields", "vgicp_prep_voxel_grid"]
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
        L.vgicp_prep_approximate_voxel_grid_fields.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_size_t), C.c_int,
                                                               C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_size_t)]
        L.vgicp_prep_voxel_grid.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_size_t), C.c_int, C.c_uint,
                                            C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_size_t)]
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

    def approximate_voxel_grid_fields(self, points, leaf, fields, remove_near_origin=False):
        """approximate_voxel_grid that also averages per-point float32 fields over each voxel (pcl::ApproximateVoxelGrid<PointT>'s
        default, setDownsampleAllData(true)) -> (m, 3 + F) float32 records x y z f_0 ... f_{F-1}.
          points  a numpy structured array (x, y, z: its first three float32 fields; `fields` name float32 fields), an (n, k)
                  float32 array (`fields` are column indices >= 3), or an (n, k) float32 torch CUDA tensor on this context's device
                  (read in place; the result is then an (m, 3 + F) torch CUDA tensor, the layout set_cloud_device reads)."""

        def run(ptr, n, stride, on_device, offsets, out_ptr, cap, out_on_device):
            return self._run_fields(ptr, n, stride, on_device, leaf, remove_near_origin, offsets, out_ptr, cap, out_on_device)

        return self._records(points, fields, "approximate_voxel_grid_fields", run)

    def voxel_grid(self, points, leaf, fields=(), min_points_per_voxel=0, remove_near_origin=False):
        """pcl::VoxelGrid(leaf), the exact grid (vgicp_prep_voxel_grid): one centroid per occupied voxel, in ascending voxel index,
        x y z and the given per-point float32 fields averaged over the voxel in input order -> (m, 3 + F) float32 records.  Points
        with a non-finite coordinate are dropped, and with remove_near_origin those of align.cpp's near-origin filter; voxels with
        fewer than min_points_per_voxel points are dropped.  `points` and `fields` as for approximate_voxel_grid_fields (a torch
        CUDA tensor is read in place and gives a torch CUDA tensor).  Raises PrepError (code 1) for a cloud whose cells x / leaf
        leave the int range or whose box holds more than INT32_MAX cells."""

        def run(ptr, n, stride, on_device, offsets, out_ptr, cap, out_on_device):
            return self._run_voxel_grid(ptr, n, stride, on_device, leaf, remove_near_origin, offsets, min_points_per_voxel, out_ptr, cap, out_on_device)

        return self._records(points, fields, "voxel_grid", run)

    def _records(self, points, fields, who, run):
        """The input parsing both field filters share: run(ptr, n, stride, on_device, offsets, out_ptr, cap, out_on_device) -> m
        on the records of `points`, into an output of n records of 3 + F floats."""
        fields = list(fields)
        if hasattr(points, "is_cuda") and points.is_cuda:
            return self._records_device(points, fields, who, run)
        p = np.asarray(points)
        if p.dtype.names:
            names = p.dtype.names
            if len(names) < 3 or any(p.dtype.fields[k][0] != np.float32 or p.dtype.fields[k][1] != 4 * j for j, k in enumerate(names[:3])):
                raise ValueError(f"{who}: x y z must be the first three float32 fields, at byte offsets 0, 4, 8")
            offsets = []
            for f in fields:
                if p.dtype.fields[f][0] != np.float32:
                    raise ValueError(f"{who}: field {f!r} is not float32")
                offsets.append(p.dtype.fields[f][1])
            p = np.ascontiguousarray(p)
            stride = p.dtype.itemsize
        else:
            p = np.ascontiguousarray(p, dtype=np.float32)
            if p.ndim != 2:
                raise ValueError(f"{who}: points must be (n, k) or a structured array")
            offsets = [4 * int(c) for c in fields]
            stride = 4 * p.shape[1]
        n = len(p)
        out = np.empty((n, 3 + len(fields)), dtype=np.float32)
        m = run(p.ctypes.data, n, stride, 0, offsets, out.ctypes.data, n, 0)
        return out[:m].copy()

    def _check(self, rc):
        if rc:
            raise PrepError(rc, self._lib.vgicp_prep_last_error(self._h).decode())

    def _run_fields(self, ptr, n, stride, on_device, leaf, remove_near_origin, offsets, out_ptr, cap, out_on_device):
        off = (C.c_size_t * max(len(offsets), 1))(*offsets)
        m = C.c_size_t(0)
        self._check(self._lib.vgicp_prep_approximate_voxel_grid_fields(self._h, ptr, n, stride, int(on_device), C.c_float(leaf), int(bool(remove_near_origin)), off,
                                                                       len(offsets), out_ptr, cap, int(out_on_device), C.byref(m)))
        return m.value

    def _run_voxel_grid(self, ptr, n, stride, on_device, leaf, remove_near_origin, offsets, min_points, out_ptr, cap, out_on_device):
        off = (C.c_size_t * max(len(offsets), 1))(*offsets)
        m = C.c_size_t(0)
        self._check(self._lib.vgicp_prep_voxel_grid(self._h, ptr, n, stride, int(on_device), C.c_float(leaf), int(bool(remove_near_origin)), off, len(offsets),
                                                    int(min_points), out_ptr, cap, int(out_on_device), C.byref(m)))
        return m.value

    def _records_device(self, t, fields, who, run):
        import torch

        if t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
            raise ValueError(f"{who}: a device input must be an (n, k) float32 tensor with contiguous rows")
        n, k = t.shape
        torch.cuda.current_stream(t.device).synchronize()  # the filter runs on this context's own stream: the input must be complete
        out = torch.empty((n, 3 + len(fields)), dtype=torch.float32, device=t.device)
        m = run(t.data_ptr(), n, 4 * (t.stride(0) if n > 1 else k), 1, [4 * int(c) for c in fields], out.data_ptr(), n, 1)
        return out[:m]
