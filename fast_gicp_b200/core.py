"""ctypes binding of the C ABI (include/vgicp_b200.h): `Core` mirrors fast_gicp::cuda::FastVGICPCudaCore
(reference include/fast_gicp/cuda/fast_vgicp_cuda.cuh:28-92) method for method.

There is no CPU fallback: importing this module without the built library, or creating a Core without an H100, raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# Several handles in one process (each owns two streams) alias onto the default 8 hardware work queues and wait on each other; the driver reads
# this when the context is created.  A value the caller has set wins.  C/C++ callers export it themselves (INTEGRATION.md 7).
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
LIB_PATH = os.environ.get("VGICP_B200_LIB") or os.path.join(_HERE, "lib", "libvgicp_b200.so")  # override only for A/B experiments

OK, ERR_INVALID_ARGUMENT, ERR_BAD_STATE, ERR_CUDA, ERR_UNSUPPORTED, ERR_NO_DEVICE, ERR_COMM = range(7)

# gicp_settings.hpp:6,8
REG_NONE, REG_MIN_EIG, REG_NORMALIZED_MIN_EIG, REG_PLANE, REG_FROBENIUS = range(5)
DIRECT27, DIRECT7, DIRECT1, DIRECT_RADIUS = range(4)
REGULARIZATION = {"NONE": REG_NONE, "MIN_EIG": REG_MIN_EIG, "NORMALIZED_MIN_EIG": REG_NORMALIZED_MIN_EIG, "PLANE": REG_PLANE, "FROBENIUS": REG_FROBENIUS}
NEIGHBOR_SEARCH = {"DIRECT27": DIRECT27, "DIRECT7": DIRECT7, "DIRECT1": DIRECT1, "DIRECT_RADIUS": DIRECT_RADIUS}
# vgicp_set_robust_kernel kinds (include/vgicp_b200.h)
ROBUST_NONE, ROBUST_HUBER, ROBUST_CAUCHY, ROBUST_GEMAN_MCCLURE = range(4)
ROBUST_KERNEL = {"NONE": ROBUST_NONE, "HUBER": ROBUST_HUBER, "CAUCHY": ROBUST_CAUCHY, "GEMAN_MCCLURE": ROBUST_GEMAN_MCCLURE}

# every symbol include/vgicp_b200.h declares (tests check the library exports all of them)
EXPORTED_SYMBOLS = [
    "vgicp_create", "vgicp_destroy", "vgicp_last_error", "vgicp_version",
    "vgicp_set_resolution", "vgicp_set_kernel_params", "vgicp_set_neighbor_search_method",
    "vgicp_set_source_cloud", "vgicp_set_target_cloud", "vgicp_swap_source_and_target",
    "vgicp_set_source_neighbors", "vgicp_set_target_neighbors", "vgicp_find_source_neighbors", "vgicp_find_target_neighbors",
    "vgicp_calculate_source_covariances", "vgicp_calculate_target_covariances",
    "vgicp_calculate_source_covariances_rbf", "vgicp_calculate_target_covariances_rbf",
    "vgicp_get_source_covariances", "vgicp_get_target_covariances", "vgicp_get_source_neighbors", "vgicp_get_target_neighbors",
    "vgicp_get_num_source_points", "vgicp_get_num_target_points",
    "vgicp_create_target_voxelmap", "vgicp_get_num_voxels", "vgicp_get_num_buckets",
    "vgicp_get_voxel_num_points", "vgicp_get_voxel_means", "vgicp_get_voxel_covs", "vgicp_get_voxel_buckets",
    "vgicp_update_correspondences", "vgicp_get_voxel_correspondences", "vgicp_compute_error",
    "vgicp_lsq_default_params", "vgicp_align", "vgicp_transform_source",
    "vgicp_get_launch_count", "vgicp_synchronize", "vgicp_get_stream",
    "vgicp_set_source_cloud_device", "vgicp_set_target_cloud_device", "vgicp_set_profiling", "vgicp_get_profile", "vgicp_profile_category_name",
    "vgicp_set_voxel_index", "vgicp_set_speculation", "vgicp_register", "vgicp_get_fitness_score", "vgicp_set_execution_hint", "vgicp_set_problem", "vgicp_ndt_create_voxelmaps",
    "vgicp_comm_export", "vgicp_comm_init", "vgicp_comm_shutdown", "vgicp_comm_error", "vgicp_set_source_shard", "vgicp_clear_source_shard",
    "vgicp_comm_export_arena", "vgicp_comm_init_arena", "vgicp_set_stage1_sharding", "vgicp_set_source_covariances", "vgicp_set_target_covariances",
    "vgicp_align_multi", "vgicp_evaluate_poses", "vgicp_set_robust_kernel",
    "vgicp_append_source_to_target", "vgicp_crop_target", "vgicp_thin_target", "vgicp_deskew_source",
    "vgicp_set_source_timestamps", "vgicp_compute_error_ct", "vgicp_align_ct",
    "vgicp_set_source_timestamps_device", "vgicp_deskew_source_stored", "vgicp_align_sources",
    "vgicp_carve_default_params", "vgicp_carve_target",
]
PROF_NUM_CATEGORIES = 7


class VgicpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"vgicp status {code}: {msg}")
        self.code = code


class LsqParams(C.Structure):
    _fields_ = [
        ("max_iterations", C.c_int),
        ("rotation_epsilon", C.c_double),
        ("transformation_epsilon", C.c_double),
        ("use_gauss_newton", C.c_int),
        ("lm_max_iterations", C.c_int),
        ("lm_init_lambda_factor", C.c_double),
    ]


class CarveParams(C.Structure):
    _fields_ = [
        ("width", C.c_int),
        ("height", C.c_int),
        ("elevation_min", C.c_double),
        ("elevation_max", C.c_double),
        ("window", C.c_int),
        ("margin", C.c_double),
        ("margin_rel", C.c_double),
    ]


class AlignResult(C.Structure):
    _fields_ = [
        ("T", C.c_double * 16),
        ("H", C.c_double * 36),
        ("nr_iterations", C.c_int),
        ("converged", C.c_int),
        ("n_linearize", C.c_int),
        ("n_compute_error", C.c_int),
        ("lm_failed", C.c_int),
    ]


class AlignCtResult(C.Structure):
    _fields_ = [
        ("T", C.c_double * 16),
        ("twist", C.c_double * 6),
        ("H", C.c_double * 144),
        ("nr_iterations", C.c_int),
        ("converged", C.c_int),
        ("n_linearize", C.c_int),
        ("n_compute_error", C.c_int),
        ("lm_failed", C.c_int),
    ]


_lib = None


def load_library():
    """dlopen the native library; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python build_native.py` (the CUDA library is required; there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    hp, fp, ip, dp = C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double)
    sig = {
        "vgicp_create": [C.c_int, C.POINTER(hp)],
        "vgicp_destroy": [hp],
        "vgicp_set_resolution": [hp, C.c_double],
        "vgicp_set_kernel_params": [hp, C.c_double, C.c_double],
        "vgicp_set_robust_kernel": [hp, C.c_int, C.c_double],
        "vgicp_set_neighbor_search_method": [hp, C.c_int, C.c_double],
        "vgicp_set_source_cloud": [hp, C.c_void_p, C.c_size_t, C.c_size_t],
        "vgicp_set_target_cloud": [hp, C.c_void_p, C.c_size_t, C.c_size_t],
        "vgicp_swap_source_and_target": [hp],
        "vgicp_set_source_neighbors": [hp, C.c_int, ip, C.c_size_t],
        "vgicp_set_target_neighbors": [hp, C.c_int, ip, C.c_size_t],
        "vgicp_find_source_neighbors": [hp, C.c_int],
        "vgicp_find_target_neighbors": [hp, C.c_int],
        "vgicp_calculate_source_covariances": [hp, C.c_int],
        "vgicp_calculate_target_covariances": [hp, C.c_int],
        "vgicp_calculate_source_covariances_rbf": [hp, C.c_int],
        "vgicp_calculate_target_covariances_rbf": [hp, C.c_int],
        "vgicp_get_source_covariances": [hp, fp, C.c_size_t],
        "vgicp_get_target_covariances": [hp, fp, C.c_size_t],
        "vgicp_get_source_neighbors": [hp, ip, C.c_size_t, ip],
        "vgicp_get_target_neighbors": [hp, ip, C.c_size_t, ip],
        "vgicp_get_num_source_points": [hp, C.POINTER(C.c_size_t)],
        "vgicp_get_num_target_points": [hp, C.POINTER(C.c_size_t)],
        "vgicp_create_target_voxelmap": [hp],
        "vgicp_get_num_voxels": [hp, ip],
        "vgicp_get_num_buckets": [hp, ip],
        "vgicp_get_voxel_num_points": [hp, ip, C.c_size_t],
        "vgicp_get_voxel_means": [hp, fp, C.c_size_t],
        "vgicp_get_voxel_covs": [hp, fp, C.c_size_t],
        "vgicp_get_voxel_buckets": [hp, ip, ip, C.c_size_t],
        "vgicp_update_correspondences": [hp, dp],
        "vgicp_get_voxel_correspondences": [hp, ip, C.c_size_t, C.POINTER(C.c_size_t)],
        "vgicp_compute_error": [hp, dp, dp, dp, dp],
        "vgicp_lsq_default_params": [C.POINTER(LsqParams)],
        "vgicp_align": [hp, dp, C.POINTER(LsqParams), C.POINTER(AlignResult)],
        "vgicp_align_multi": [hp, dp, C.c_int, C.POINTER(LsqParams), C.POINTER(AlignResult)],
        "vgicp_evaluate_poses": [hp, dp, C.c_int, dp, dp, dp, C.POINTER(C.c_int64)],
        "vgicp_transform_source": [hp, dp, C.c_void_p, C.c_size_t, C.c_size_t],
        "vgicp_get_launch_count": [hp, C.POINTER(C.c_uint64)],
        "vgicp_synchronize": [hp],
        "vgicp_get_stream": [hp, C.POINTER(C.c_uint64)],
        "vgicp_set_source_cloud_device": [hp, C.c_void_p, C.c_size_t, C.c_size_t],
        "vgicp_set_target_cloud_device": [hp, C.c_void_p, C.c_size_t, C.c_size_t],
        "vgicp_set_profiling": [hp, C.c_int],
        "vgicp_set_voxel_index": [hp, C.c_int],
        "vgicp_set_speculation": [hp, C.c_int],
        "vgicp_get_fitness_score": [hp, dp, C.c_double, dp],
        "vgicp_set_execution_hint": [hp, C.c_int],
        "vgicp_set_problem": [hp, C.c_int],
        "vgicp_ndt_create_voxelmaps": [hp],
        "vgicp_comm_export": [hp, C.c_void_p],
        "vgicp_comm_init": [hp, C.c_int, C.c_int, C.c_void_p],
        "vgicp_comm_shutdown": [hp],
        "vgicp_comm_error": [hp, ip],
        "vgicp_set_source_shard": [hp, C.c_size_t, C.c_size_t],
        "vgicp_clear_source_shard": [hp],
        "vgicp_comm_export_arena": [hp, C.c_size_t, C.c_void_p],
        "vgicp_comm_init_arena": [hp, C.c_void_p],
        "vgicp_set_stage1_sharding": [hp, C.c_int],
        "vgicp_set_source_covariances": [hp, fp, C.c_size_t],
        "vgicp_set_target_covariances": [hp, fp, C.c_size_t],
        "vgicp_register": [hp, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, dp, C.POINTER(LsqParams), C.POINTER(AlignResult)],
        "vgicp_get_profile": [hp, dp, C.POINTER(C.c_uint64), C.c_int],
        "vgicp_append_source_to_target": [hp, dp],
        "vgicp_crop_target": [hp, dp, C.c_double, C.c_size_t],
        "vgicp_thin_target": [hp, C.c_double, C.c_int],
        "vgicp_carve_default_params": [C.POINTER(CarveParams)],
        "vgicp_carve_target": [hp, dp, C.POINTER(CarveParams), C.POINTER(C.c_size_t)],
        "vgicp_deskew_source": [hp, C.c_void_p, C.c_size_t, C.c_size_t, dp, C.c_double],
        "vgicp_set_source_timestamps": [hp, C.c_void_p, C.c_size_t, C.c_size_t, C.c_double],
        "vgicp_compute_error_ct": [hp, dp, dp, dp, dp, dp, dp, dp],
        "vgicp_align_ct": [hp, dp, dp, dp, dp, C.POINTER(LsqParams), C.POINTER(AlignCtResult)],
        "vgicp_set_source_timestamps_device": [hp, C.c_void_p, C.c_size_t, C.c_size_t, C.c_double],
        "vgicp_deskew_source_stored": [hp, dp],
        "vgicp_align_sources": [hp, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_size_t, C.c_int, C.c_int, C.c_int, dp, C.c_int, C.POINTER(LsqParams),
                                C.POINTER(AlignResult)],
    }
    for name, argtypes in sig.items():
        fn = getattr(L, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
    L.vgicp_lsq_default_params.restype = None
    L.vgicp_carve_default_params.restype = None
    L.vgicp_last_error.argtypes = [hp]
    L.vgicp_last_error.restype = C.c_char_p
    L.vgicp_profile_category_name.argtypes = [C.c_int]
    L.vgicp_profile_category_name.restype = C.c_char_p
    L.vgicp_version.argtypes = []
    L.vgicp_version.restype = C.c_char_p
    _lib = L
    return L


def default_params(**kw):
    p = LsqParams()
    load_library().vgicp_lsq_default_params(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def carve_params(**kw):
    """vgicp_carve_target's parameters as a dict: the library's defaults (vgicp_carve_default_params), overridden by kw.  Keys:
    width, height, elevation_min, elevation_max (rad), window, margin (m), margin_rel; synthetic.carve_indices takes the same dict."""
    p = CarveParams()
    load_library().vgicp_carve_default_params(C.byref(p))
    out = {name: getattr(p, name) for name, _ in CarveParams._fields_}
    for k, v in kw.items():
        if k not in out:
            raise TypeError(f"unknown carve parameter {k!r}")
        if v is not None:
            out[k] = v
    return out


def pose_to_c(T):
    """(4,4) -> 16 doubles column-major (Eigen::Isometry3d::data())."""
    return np.ascontiguousarray(np.asarray(T, dtype=np.float64).T).reshape(16)


def pose_from_c(buf):
    return np.array(buf, dtype=np.float64).reshape(4, 4).T.copy()


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def twist_from_motion(delta, duration):
    """Constant body twist [omega, v] (rotation first, per time unit) that moves by the 4x4 `delta` in `duration`: the float64
    SE(3) logarithm, the inverse of se3_exp (csrc/lsq_math.hpp), divided by duration.  For a constant-velocity deskew,
    twist_from_motion(inv(T_prev) @ T_cur, dt) with the last two estimated poses."""
    T = np.asarray(delta, dtype=np.float64)
    R, t = T[:3, :3], T[:3, 3]
    # quaternion (Shepperd: divide by the largest of the four candidates), w >= 0
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    k = int(np.argmax([tr, R[0, 0], R[1, 1], R[2, 2]]))
    if k == 0:
        r = np.sqrt(1.0 + tr) * 2.0
        q = np.array([0.25 * r, (R[2, 1] - R[1, 2]) / r, (R[0, 2] - R[2, 0]) / r, (R[1, 0] - R[0, 1]) / r])
    elif k == 1:
        r = np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2.0
        q = np.array([(R[2, 1] - R[1, 2]) / r, 0.25 * r, (R[0, 1] + R[1, 0]) / r, (R[0, 2] + R[2, 0]) / r])
    elif k == 2:
        r = np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2.0
        q = np.array([(R[0, 2] - R[2, 0]) / r, (R[0, 1] + R[1, 0]) / r, 0.25 * r, (R[1, 2] + R[2, 1]) / r])
    else:
        r = np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2.0
        q = np.array([(R[1, 0] - R[0, 1]) / r, (R[0, 2] + R[2, 0]) / r, (R[1, 2] + R[2, 1]) / r, 0.25 * r])
    if q[0] < 0.0:
        q = -q
    w, vec = q[0], q[1:]
    nv = np.linalg.norm(vec)
    theta = 2.0 * np.arctan2(nv, w)
    omega = vec * (theta / nv if nv > 1e-10 else 2.0 / w * (1.0 - nv * nv / (3.0 * w * w)))
    # v solves V v = t with V built exactly as se3_exp builds it (V = R below theta = 1e-10), so that the round trip holds at
    # every angle, the tiny ones included
    th2 = float(omega @ omega)
    th = np.sqrt(th2)
    if th < 1e-10:
        V = R
    else:
        Om = np.array([[0.0, -omega[2], omega[1]], [omega[2], 0.0, -omega[0]], [-omega[1], omega[0], 0.0]])
        V = np.eye(3) + (1.0 - np.cos(th)) / th2 * Om + (th - np.sin(th)) / (th2 * th) * (Om @ Om)
    v = np.linalg.solve(V, t)
    return np.concatenate([omega, v]) / float(duration)


class Core:
    """One FastVGICPCudaCore: owns a CUDA stream and all device state of one registration context."""

    def __init__(self, device=0):
        self._lib = load_library()
        self._h = C.c_void_p()
        rc = self._lib.vgicp_create(int(device), C.byref(self._h))
        if rc != OK:
            self._h = None
            raise VgicpError(rc, "vgicp_create failed (needs a CUDA device with an sm_90a image; no CPU fallback)")

    def close(self):
        if getattr(self, "_h", None):
            self._lib.vgicp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, allow=()):
        if rc != OK and rc not in allow:
            raise VgicpError(rc, self._lib.vgicp_last_error(self._h).decode())
        return rc

    # ---- settings
    def set_resolution(self, resolution):
        self._check(self._lib.vgicp_set_resolution(self._h, float(resolution)))

    def set_kernel_params(self, kernel_width, kernel_max_dist):
        self._check(self._lib.vgicp_set_kernel_params(self._h, float(kernel_width), float(kernel_max_dist)))

    def set_robust_kernel(self, kind, scale=1.0):
        """Robust kernel of the Mahalanobis residual: "NONE" (default), "HUBER", "CAUCHY" or "GEMAN_MCCLURE" (or the
        ROBUST_* value); scale = delta in Mahalanobis units (ignored for NONE).  Kept across set_*_cloud and swap."""
        if isinstance(kind, str):
            kind = ROBUST_KERNEL[kind]
        self._check(self._lib.vgicp_set_robust_kernel(self._h, int(kind), float(scale)))

    def set_neighbor_search_method(self, method, radius=-1.0):
        if isinstance(method, str):
            method = NEIGHBOR_SEARCH[method]
        self._check(self._lib.vgicp_set_neighbor_search_method(self._h, int(method), float(radius)))

    # ---- clouds
    @staticmethod
    def _cloud(points):
        a = np.asarray(points)
        if a.dtype != np.float32 or a.ndim != 2 or a.shape[1] < 3 or not a.flags.c_contiguous:
            a = np.ascontiguousarray(np.asarray(points, dtype=np.float32)[:, :3])
        return a, a.shape[0], a.shape[1] * 4  # (strides of an empty array are not meaningful)

    def set_source_cloud(self, points):
        a, n, stride = self._cloud(points)
        self._check(self._lib.vgicp_set_source_cloud(self._h, a.ctypes.data, n, stride))

    def set_target_cloud(self, points):
        a, n, stride = self._cloud(points)
        self._check(self._lib.vgicp_set_target_cloud(self._h, a.ctypes.data, n, stride))

    def set_cloud_raw(self, which, ptr, n, stride):
        """Host pointer + size straight through (used by bench.py with pinned buffers)."""
        fn = self._lib.vgicp_set_source_cloud if which == "source" else self._lib.vgicp_set_target_cloud
        self._check(fn(self._h, ptr, n, stride))

    def set_cloud_device(self, which, dev_ptr, n, stride):
        """Points already resident in this GPU's memory (e.g. a torch CUDA tensor's data_ptr())."""
        fn = self._lib.vgicp_set_source_cloud_device if which == "source" else self._lib.vgicp_set_target_cloud_device
        self._check(fn(self._h, dev_ptr, n, stride))

    def set_problem(self, problem):
        """0 = VGICP (default), 1 = NDT P2D, 2 = NDT D2D."""
        self._check(self._lib.vgicp_set_problem(self._h, int(problem)))

    def ndt_create_voxelmaps(self):
        self._check(self._lib.vgicp_ndt_create_voxelmaps(self._h))

    def set_execution_hint(self, hint):
        """0 = latency (default), 1 = throughput (many handles share the GPU)."""
        self._check(self._lib.vgicp_set_execution_hint(self._h, int(hint)))

    def set_voxel_index(self, mode):
        """0: direct-mapped voxel index when the map's bounding box fits (default), 1: hash table only."""
        self._check(self._lib.vgicp_set_voxel_index(self._h, int(mode)))

    def set_speculation(self, enable):
        """LM trial evaluations also linearise at the trial pose (default on); results are identical either way."""
        self._check(self._lib.vgicp_set_speculation(self._h, int(bool(enable))))

    def set_profiling(self, enable):
        self._check(self._lib.vgicp_set_profiling(self._h, int(bool(enable))))

    def get_profile(self):
        """-> {category: (total_ms, launches)} since profiling was enabled."""
        ms = (C.c_double * PROF_NUM_CATEGORIES)()
        cnt = (C.c_uint64 * PROF_NUM_CATEGORIES)()
        self._check(self._lib.vgicp_get_profile(self._h, ms, cnt, PROF_NUM_CATEGORIES))
        return {self._lib.vgicp_profile_category_name(i).decode(): (ms[i], cnt[i]) for i in range(PROF_NUM_CATEGORIES)}

    def swap_source_and_target(self):
        self._check(self._lib.vgicp_swap_source_and_target(self._h))

    # ---- stage 1
    def set_source_neighbors(self, k, indices):
        idx = np.ascontiguousarray(indices, dtype=np.int32)
        self._check(self._lib.vgicp_set_source_neighbors(self._h, int(k), idx.ctypes.data_as(C.POINTER(C.c_int)), idx.size))

    def set_target_neighbors(self, k, indices):
        idx = np.ascontiguousarray(indices, dtype=np.int32)
        self._check(self._lib.vgicp_set_target_neighbors(self._h, int(k), idx.ctypes.data_as(C.POINTER(C.c_int)), idx.size))

    def find_source_neighbors(self, k):
        self._check(self._lib.vgicp_find_source_neighbors(self._h, int(k)))

    def find_target_neighbors(self, k):
        self._check(self._lib.vgicp_find_target_neighbors(self._h, int(k)))

    def calculate_source_covariances(self, method=REG_PLANE):
        return self._check(self._lib.vgicp_calculate_source_covariances(self._h, int(method)), allow=(ERR_UNSUPPORTED,))

    def calculate_target_covariances(self, method=REG_PLANE):
        return self._check(self._lib.vgicp_calculate_target_covariances(self._h, int(method)), allow=(ERR_UNSUPPORTED,))

    def calculate_source_covariances_rbf(self, method=REG_PLANE):
        return self._check(self._lib.vgicp_calculate_source_covariances_rbf(self._h, int(method)), allow=(ERR_UNSUPPORTED,))

    def calculate_target_covariances_rbf(self, method=REG_PLANE):
        return self._check(self._lib.vgicp_calculate_target_covariances_rbf(self._h, int(method)), allow=(ERR_UNSUPPORTED,))

    def set_source_covariances(self, cov9):
        """(n, 9) or (n, 3, 3) float32, column-major 3x3 per point (== get_source_covariances())."""
        c = np.ascontiguousarray(np.asarray(cov9, dtype=np.float32).reshape(-1, 9))
        self._check(self._lib.vgicp_set_source_covariances(self._h, c.ctypes.data_as(C.POINTER(C.c_float)), len(c)))

    def set_target_covariances(self, cov9):
        c = np.ascontiguousarray(np.asarray(cov9, dtype=np.float32).reshape(-1, 9))
        self._check(self._lib.vgicp_set_target_covariances(self._h, c.ctypes.data_as(C.POINTER(C.c_float)), len(c)))

    def num_source_points(self):
        n = C.c_size_t(0)
        self._check(self._lib.vgicp_get_num_source_points(self._h, C.byref(n)))
        return n.value

    def num_target_points(self):
        n = C.c_size_t(0)
        self._check(self._lib.vgicp_get_num_target_points(self._h, C.byref(n)))
        return n.value

    def _get_covs(self, fn, n):
        out = np.empty((n, 9), dtype=np.float32)
        self._check(fn(self._h, out.ctypes.data_as(C.POINTER(C.c_float)), n))
        return out

    def get_source_covariances(self):
        return self._get_covs(self._lib.vgicp_get_source_covariances, self.num_source_points())

    def get_target_covariances(self):
        return self._get_covs(self._lib.vgicp_get_target_covariances, self.num_target_points())

    def _get_nbr(self, fn, n):
        k = C.c_int(0)
        fn(self._h, None, 0, C.byref(k))  # query k
        if k.value <= 0:
            self._check(ERR_BAD_STATE)
        out = np.empty((n, k.value), dtype=np.int32)
        self._check(fn(self._h, out.ctypes.data_as(C.POINTER(C.c_int)), out.size, C.byref(k)))
        return out

    def get_source_neighbors(self):
        return self._get_nbr(self._lib.vgicp_get_source_neighbors, self.num_source_points())

    def get_target_neighbors(self):
        return self._get_nbr(self._lib.vgicp_get_target_neighbors, self.num_target_points())

    # ---- stage 2
    def create_target_voxelmap(self):
        self._check(self._lib.vgicp_create_target_voxelmap(self._h))

    def num_voxels(self):
        v = C.c_int(0)
        self._check(self._lib.vgicp_get_num_voxels(self._h, C.byref(v)))
        return v.value

    def num_buckets(self):
        v = C.c_int(0)
        self._check(self._lib.vgicp_get_num_buckets(self._h, C.byref(v)))
        return v.value

    def get_voxel_num_points(self):
        out = np.empty(self.num_voxels(), dtype=np.int32)
        self._check(self._lib.vgicp_get_voxel_num_points(self._h, out.ctypes.data_as(C.POINTER(C.c_int)), out.size))
        return out

    def get_voxel_means(self):
        out = np.empty((self.num_voxels(), 3), dtype=np.float32)
        self._check(self._lib.vgicp_get_voxel_means(self._h, out.ctypes.data_as(C.POINTER(C.c_float)), len(out)))
        return out

    def get_voxel_covs(self):
        out = np.empty((self.num_voxels(), 9), dtype=np.float32)
        self._check(self._lib.vgicp_get_voxel_covs(self._h, out.ctypes.data_as(C.POINTER(C.c_float)), len(out)))
        return out

    def get_voxel_buckets(self):
        B = self.num_buckets()
        coords = np.empty((B, 3), dtype=np.int32)
        ids = np.empty(B, dtype=np.int32)
        self._check(self._lib.vgicp_get_voxel_buckets(self._h, coords.ctypes.data_as(C.POINTER(C.c_int)), ids.ctypes.data_as(C.POINTER(C.c_int)), B))
        return coords, ids

    def voxelmap_as_dict(self):
        coords, ids = self.get_voxel_buckets()
        n, mean, cov = self.get_voxel_num_points(), self.get_voxel_means(), self.get_voxel_covs()
        return {tuple(int(x) for x in coords[b]): (int(n[ids[b]]), mean[ids[b]].copy(), cov[ids[b]].copy()) for b in np.flatnonzero(ids >= 0)}

    # ---- stage 2b + 3
    def update_correspondences(self, T):
        t = pose_to_c(T)
        self._check(self._lib.vgicp_update_correspondences(self._h, _dp(t)))

    def get_voxel_correspondences(self):
        n = C.c_size_t(0)
        self._check(self._lib.vgicp_get_voxel_correspondences(self._h, None, 0, C.byref(n)))
        out = np.empty((max(n.value, 1), 2), dtype=np.int32)
        self._check(self._lib.vgicp_get_voxel_correspondences(self._h, out.ctypes.data_as(C.POINTER(C.c_int)), n.value, C.byref(n)))
        return out[: n.value].copy()

    def compute_error(self, T, want_H=True):
        """-> (err, H(6,6) | None, b(6) | None); want_H=False is the reference's compute_error(trans, nullptr, nullptr)."""
        t = pose_to_c(T)
        err = C.c_double(0.0)
        if want_H:
            H = np.zeros(36)
            b = np.zeros(6)
            self._check(self._lib.vgicp_compute_error(self._h, _dp(t), _dp(H), _dp(b), C.byref(err)))
            return err.value, H.reshape(6, 6).T.copy(), b
        self._check(self._lib.vgicp_compute_error(self._h, _dp(t), None, None, C.byref(err)))
        return err.value, None, None

    def linearize(self, T):
        """FastVGICPCuda::linearize (fast_vgicp_cuda_impl.hpp:170-173)."""
        self.update_correspondences(T)
        return self.compute_error(T, True)

    # ---- extensions
    def align(self, guess=None, params=None):
        g = pose_to_c(np.eye(4) if guess is None else guess)
        params = params or default_params()
        res = AlignResult()
        self._check(self._lib.vgicp_align(self._h, _dp(g), C.byref(params), C.byref(res)))
        return res

    @staticmethod
    def _poses_to_c(poses):
        P = np.asarray(poses, dtype=np.float64)
        if P.ndim != 3 or P.shape[1:] != (4, 4):
            raise ValueError("poses must be (B, 4, 4)")
        return np.ascontiguousarray(P.transpose(0, 2, 1)).reshape(-1)  # B x 16 doubles, column-major each

    def align_multi(self, guesses, params=None):
        """B registrations from the (B, 4, 4) initial guesses, evaluated together -> list of AlignResult;
        result i equals align(guesses[i], params) bit for bit."""
        g = self._poses_to_c(guesses)
        B = len(g) // 16
        params = params or default_params()
        res = (AlignResult * max(B, 1))()
        self._check(self._lib.vgicp_align_multi(self._h, _dp(g), B, C.byref(params), res))
        return list(res)[:B]

    def align_sources(self, sources, guesses=None, k=20, reg=REG_PLANE, params=None):
        """Register each of the B source clouds ((N_i, >=3) arrays) against the current target map, the optimisers' evaluations
        shared across sources -> list of AlignResult.  Result i equals set_source_cloud(sources[i]) + find_source_neighbors(k) +
        calculate_source_covariances(reg) + align(guesses[i], params) bit for bit; the handle's own source is left as it was.
        guesses: (B, 4, 4), None = identity for every source."""
        clouds = [self._cloud(s) for s in sources]
        if len({st for _, _, st in clouds}) > 1:  # one stride for all: repack to xyz
            clouds = [self._cloud(np.ascontiguousarray(np.asarray(a, dtype=np.float32)[:, :3])) for a, _, _ in clouds]
        ptrs = [a.ctypes.data for a, _, _ in clouds]
        ns = [n for _, n, _ in clouds]
        return self.align_sources_raw(ptrs, ns, clouds[0][2] if clouds else 12, False, k, reg, guesses, params)

    def align_sources_raw(self, ptrs, ns, stride=12, on_device=False, k=20, reg=REG_PLANE, guesses=None, params=None):
        """vgicp_align_sources with the B point pointers (host, or device when on_device) and sizes straight through."""
        B = len(ptrs)
        P = (C.c_void_p * max(B, 1))(*[int(p) for p in ptrs])
        N = (C.c_size_t * max(B, 1))(*[int(n) for n in ns])
        g = None
        if guesses is not None:
            g = self._poses_to_c(guesses)
            if len(g) != 16 * B:
                raise ValueError("guesses must be (B, 4, 4) with one pose per source")
        params = params or default_params()
        res = (AlignResult * max(B, 1))()
        self._check(self._lib.vgicp_align_sources(self._h, P, N, int(stride), int(bool(on_device)), int(k), int(reg), _dp(g) if g is not None else None, B,
                                                  C.byref(params), res))
        return list(res)[:B]

    def evaluate_poses(self, poses, want_H=False):
        """-> (err (B,), H (B,6,6) | None, b (B,6) | None, n_corr (B,) int64): per pose what update_correspondences(T) +
        compute_error(T, want_H) return, and the number of correspondences get_voxel_correspondences() would list."""
        t = self._poses_to_c(poses)
        B = len(t) // 16
        err = np.zeros(B)
        n_corr = np.zeros(B, dtype=np.int64)
        H = np.zeros((B, 36)) if want_H else None
        b = np.zeros((B, 6)) if want_H else None
        self._check(self._lib.vgicp_evaluate_poses(self._h, _dp(t), B, _dp(err), _dp(H) if want_H else None, _dp(b) if want_H else None,
                                                   n_corr.ctypes.data_as(C.POINTER(C.c_int64))))
        if want_H:
            H = H.reshape(B, 6, 6).transpose(0, 2, 1).copy()
        return err, H, b, n_corr

    def register_raw(self, tgt_ptr, n_t, src_ptr, n_s, stride=12, on_device=False, k=20, reg=REG_PLANE, guess=None, params=None):
        """clear + setInputTarget + setInputSource + align in one C call (pointers: host, or device when on_device)."""
        res = AlignResult()
        g = None if guess is None else _dp(pose_to_c(guess))
        self._check(self._lib.vgicp_register(self._h, tgt_ptr, n_t, src_ptr, n_s, stride, int(on_device), int(k), int(reg), g, C.byref(params) if params is not None else None, C.byref(res)))
        return res

    def register(self, target, source, k=20, reg=REG_PLANE, guess=None, params=None):
        t, nt, st = self._cloud(target)
        s_, ns, ss = self._cloud(source)
        assert st == ss
        return self.register_raw(t.ctypes.data, nt, s_.ctypes.data, ns, st, False, k, reg, guess, params)

    # ---- local map (scan-to-map odometry)
    def append_source_to_target(self, T):
        """Append the current source, transformed by the 4x4 T, to the target on the device and rebuild the voxel map.
        Appended points are transform_source(T)'s; covariances are R C R^T in the order include/vgicp_b200.h documents."""
        t = pose_to_c(T)
        self._check(self._lib.vgicp_append_source_to_target(self._h, _dp(t)))

    def crop_target(self, center, radius, max_points=0):
        """Keep the target points within `radius` of `center` (float32 test), then at most the newest `max_points` of them
        (0 = no cap); rebuild the voxel map.  A crop that would leave no points raises and changes nothing."""
        c = np.ascontiguousarray(np.asarray(center, dtype=np.float64).reshape(3))
        self._check(self._lib.vgicp_crop_target(self._h, _dp(c), float(radius), int(max_points)))

    def thin_target(self, leaf_size, max_points_per_voxel):
        """Keep at most max_points_per_voxel target points per cell floor(p * (1 / leaf_size)) (float32), the oldest in array
        order; rebuild the voxel map.  Kept rows are unchanged and stay in order.  Errors raise and change nothing."""
        self._check(self._lib.vgicp_thin_target(self._h, float(leaf_size), int(max_points_per_voxel)))

    def carve_target(self, T, width=None, height=None, elevation_min=None, elevation_max=None, window=None, margin=None, margin_rel=None):
        """Remove the target points the current source (the scan in its sensor frame, placed by the 4x4 T) sees through: every map
        point clearly in front of the least range measured in its range-image window (include/vgicp_b200.h gives the float32
        rule).  None takes the library's default.  Returns the number of points removed; errors raise and change nothing."""
        p = CarveParams(**carve_params(width=width, height=height, elevation_min=elevation_min, elevation_max=elevation_max, window=window, margin=margin,
                                       margin_rel=margin_rel))
        t = pose_to_c(T)
        removed = C.c_size_t(0)
        self._check(self._lib.vgicp_carve_target(self._h, _dp(t), C.byref(p), C.byref(removed)))
        return removed.value

    # ---- motion compensation
    def deskew_source(self, times, twist, t_ref=0.0):
        """Re-express every source point in the sensor frame at t_ref: point i <- Exp((times[i] - t_ref) twist) p_i, on the device
        (include/vgicp_b200.h documents the float32 arithmetic).  times: one relative timestamp per source point, a 1-D float32
        array or a strided float32 column such as cloud["time"] of a structured array; twist: [omega, v] per time unit.
        Afterwards the source has no neighbours and no covariances, as after set_source_cloud."""
        a, stride = self._times(times)
        xi = np.ascontiguousarray(np.asarray(twist, dtype=np.float64).reshape(6))
        self._check(self._lib.vgicp_deskew_source(self._h, a.ctypes.data, len(a), stride, _dp(xi), float(t_ref)))

    @staticmethod
    def _times(times):
        """A 1-D float32 array (a strided column is passed as it is) -> (array, stride in bytes)."""
        a = np.asarray(times)
        if a.ndim != 1 or a.dtype != np.float32 or a.strides[0] < 4 or a.strides[0] % 4 != 0:
            a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1)
        return a, (a.strides[0] if len(a) > 1 else 4)

    # ---- continuous-time registration
    def set_source_timestamps(self, times, t_ref=0.0):
        """One timestamp per source point (as deskew_source takes them), kept on the device for compute_error_ct / align_ct.
        set_source_cloud and swap_source_and_target drop them; deskew_source keeps them."""
        a, stride = self._times(times)
        self._check(self._lib.vgicp_set_source_timestamps(self._h, a.ctypes.data, len(a), stride, float(t_ref)))

    def set_source_timestamps_device(self, dev_ptr, n, stride, t_ref=0.0):
        """set_source_timestamps with the timestamps already in this GPU's memory (e.g. a torch CUDA tensor's data_ptr(), or the
        time column of a prep output: data_ptr() + 4 * (3 + j), stride (3 + F) * 4); the same state as the host call."""
        self._check(self._lib.vgicp_set_source_timestamps_device(self._h, dev_ptr, n, stride, float(t_ref)))

    def deskew_source_stored(self, twist):
        """deskew_source with the stored timestamps and their t_ref (set_source_timestamps(_device)): no upload; the same points."""
        xi = np.ascontiguousarray(np.asarray(twist, dtype=np.float64).reshape(6))
        self._check(self._lib.vgicp_deskew_source_stored(self._h, _dp(xi)))

    def compute_error_ct(self, T_lin, xi_lin, T_eval, xi_eval, want_H=True):
        """-> (err, H (12,12) | None, b (12,) | None): the data terms at (T_eval, xi_eval) over the correspondences of
        (T_lin, xi_lin), the state ordered [pose step (rotation first), twist step] (include/vgicp_b200.h)."""
        tl, te = pose_to_c(T_lin), pose_to_c(T_eval)
        xl = np.ascontiguousarray(np.asarray(xi_lin, dtype=np.float64).reshape(6))
        xe = np.ascontiguousarray(np.asarray(xi_eval, dtype=np.float64).reshape(6))
        err = C.c_double(0.0)
        if want_H:
            H = np.zeros(144)
            b = np.zeros(12)
            self._check(self._lib.vgicp_compute_error_ct(self._h, _dp(tl), _dp(xl), _dp(te), _dp(xe), _dp(H), _dp(b), C.byref(err)))
            return err.value, H.reshape(12, 12).T.copy(), b
        self._check(self._lib.vgicp_compute_error_ct(self._h, _dp(tl), _dp(xl), _dp(te), _dp(xe), None, None, C.byref(err)))
        return err.value, None, None

    def align_ct(self, guess=None, twist_guess=None, twist_prior=None, twist_weight=None, params=None):
        """Pose at t_ref and the sweep's body twist together -> AlignCtResult (T, twist, H (144), counters).  twist_prior: the
        prior mean (default: the twist guess), twist_weight: its 6 weights > 0 (default 1e-6 each)."""
        g = pose_to_c(np.eye(4) if guess is None else guess)
        tg = np.ascontiguousarray(np.zeros(6) if twist_guess is None else np.asarray(twist_guess, dtype=np.float64).reshape(6))
        tp = tg.copy() if twist_prior is None else np.ascontiguousarray(np.asarray(twist_prior, dtype=np.float64).reshape(6))
        tw = np.full(6, 1e-6) if twist_weight is None else np.ascontiguousarray(np.broadcast_to(np.asarray(twist_weight, dtype=np.float64), (6,)))
        params = params or default_params()
        res = AlignCtResult()
        self._check(self._lib.vgicp_align_ct(self._h, _dp(g), _dp(tg), _dp(tp), _dp(tw), C.byref(params), C.byref(res)))
        return res

    def transform_source(self, T, stride=12, out=None):
        n = self.num_source_points()
        if out is None:
            out = np.zeros((n, stride // 4), dtype=np.float32)
        else:
            assert out.dtype == np.float32 and out.flags.c_contiguous and out.shape[0] >= n
            stride = out.shape[1] * 4
        t = pose_to_c(T)
        self._check(self._lib.vgicp_transform_source(self._h, _dp(t), out.ctypes.data, n, stride))
        return out

    # ---- multi-GPU source sharding
    def comm_export(self):
        buf = (C.c_ubyte * 64)()
        self._check(self._lib.vgicp_comm_export(self._h, buf))
        return bytes(buf)

    def comm_init(self, rank, nranks, all_handles):
        """all_handles: nranks x 64 bytes, rank order (all-gathered from comm_export())."""
        blob = b"".join(all_handles)
        assert len(blob) == 64 * nranks
        arr = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._check(self._lib.vgicp_comm_init(self._h, int(rank), int(nranks), arr))

    def comm_export_arena(self, max_points):
        """Stage-1 sharding: allocate the exchange arena (covariances of both clouds, up to max_points each) and return its IPC handle."""
        buf = (C.c_ubyte * 64)()
        self._check(self._lib.vgicp_comm_export_arena(self._h, int(max_points), buf))
        return bytes(buf)

    def comm_init_arena(self, all_handles):
        blob = b"".join(all_handles)
        arr = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._check(self._lib.vgicp_comm_init_arena(self._h, arr))

    def set_stage1_sharding(self, enable):
        self._check(self._lib.vgicp_set_stage1_sharding(self._h, int(bool(enable))))

    def comm_shutdown(self):
        self._check(self._lib.vgicp_comm_shutdown(self._h))

    def comm_error(self):
        v = C.c_int(0)
        self._check(self._lib.vgicp_comm_error(self._h, C.byref(v)))
        return v.value

    def set_source_shard(self, begin, end):
        self._check(self._lib.vgicp_set_source_shard(self._h, int(begin), int(end)))

    def clear_source_shard(self):
        self._check(self._lib.vgicp_clear_source_shard(self._h))

    def fitness_score(self, T, max_range=float("inf")):
        t = pose_to_c(T)
        out = C.c_double(0.0)
        self._check(self._lib.vgicp_get_fitness_score(self._h, _dp(t), min(float(max_range), 1.7976931348623157e308), C.byref(out)))
        return out.value

    def launch_count(self):
        v = C.c_uint64(0)
        self._check(self._lib.vgicp_get_launch_count(self._h, C.byref(v)))
        return v.value

    def synchronize(self):
        self._check(self._lib.vgicp_synchronize(self._h))

    def stream(self):
        v = C.c_uint64(0)
        self._check(self._lib.vgicp_get_stream(self._h, C.byref(v)))
        return v.value
