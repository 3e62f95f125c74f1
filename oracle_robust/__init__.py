"""ctypes front-end of the robust-kernel CPU checker (oracle_robust/robust_oracle.c).

TEST INFRASTRUCTURE ONLY, like `oracle`: the library compiles oracle/vgicp_oracle.c unchanged and adds the robust kind
(vgicp_set_robust_kernel) to its derivative sum.  Voxel maps are the `oracle.VoxelMap` objects (same structure, same source);
layouts and poses as in `oracle`.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB_PATH = os.path.join(_HERE, "_build", "librobust_oracle.so")
_SRCS = [os.path.join(_HERE, "robust_oracle.c"), os.path.join(_ROOT, "oracle", "vgicp_oracle.c")]

NONE, HUBER, CAUCHY, GEMAN_MCCLURE = range(4)  # VGICP_ROBUST_*
KINDS = {"NONE": NONE, "HUBER": HUBER, "CAUCHY": CAUCHY, "GEMAN_MCCLURE": GEMAN_MCCLURE}
# the oracle's flags (oracle/Makefile): no contraction, no fast math
CFLAGS = ["-O2", "-std=c11", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wno-unused-variable",
          "-Wno-unused-but-set-variable", "-Wno-unused-function"]


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(_LIB_PATH) < os.path.getmtime(s) for s in _SRCS):
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
        env = {k: v for k, v in os.environ.items() if k not in ("CC", "CFLAGS")}
        subprocess.check_call([cc] + CFLAGS + ["-shared", "-o", _LIB_PATH, _SRCS[0], "-lm"], env=env)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        fp, ip, dp, vp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_void_p
        L.orc_robust_rho.argtypes = [C.c_int, C.c_float, fp, C.c_int, fp, fp]
        L.orc_robust_evaluate_f32.restype = C.c_double
        L.orc_robust_evaluate_f32.argtypes = [vp, fp, fp, C.c_int, ip, C.c_int, dp, dp, dp, dp, C.c_int, C.c_float, C.POINTER(C.c_long)]
        L.orc_robust_derivatives.restype = C.c_double
        L.orc_robust_derivatives.argtypes = [vp, fp, fp, ip, C.c_long, dp, dp, dp, dp, C.c_int, C.c_float]
        L.orc_robust_align_f32.argtypes = [vp, fp, fp, C.c_int, ip, C.c_int, C.POINTER(O.LsqParams), dp, C.c_int, C.c_float, C.POINTER(O.LsqResult)]
        _lib = L
    return _lib


def kind_of(robust):
    return KINDS[robust] if isinstance(robust, str) else int(robust)


def scale_sq(scale):
    """delta^2 as the library forms it: (float)(delta * delta)."""
    return np.float32(float(scale) * float(scale))


def rho(robust, scale, s):
    """(rho(s), rho'(s)) in float32, exactly as the kernels form them."""
    s = np.ascontiguousarray(s, dtype=np.float32).reshape(-1)
    r = np.empty_like(s)
    d = np.empty_like(s)
    lib().orc_robust_rho(kind_of(robust), C.c_float(scale_sq(scale)), O._p(s, C.c_float), len(s), O._p(r, C.c_float), O._p(d, C.c_float))
    return r, d


def evaluate(vmap, src, src_cov, offs, T_lin, T_eval, want_H=True, robust=NONE, robust_scale=1.0):
    """oracle.evaluate (double sums) with the robust kind: returns (err, H(6,6), b(6), n_corr)."""
    src, src_cov, offs = O._f32(src), O._f32(src_cov), O._i32(offs)
    H = np.zeros(36)
    b = np.zeros(6)
    nc = C.c_long(0)
    e = lib().orc_robust_evaluate_f32(vmap._h, O._p(src, C.c_float), O._p(src_cov, C.c_float), len(src), O._p(offs, C.c_int), len(offs),
                                      O._p(O._pose_in(T_lin), C.c_double), O._p(O._pose_in(T_eval), C.c_double), O._p(H, C.c_double) if want_H else None,
                                      O._p(b, C.c_double) if want_H else None, kind_of(robust), C.c_float(scale_sq(robust_scale)), C.byref(nc))
    return e, H.reshape(6, 6).T.copy(), b, nc.value


def derivatives(vmap, src, src_cov, pairs, T_lin, T_eval, want_H=True, robust=NONE, robust_scale=1.0):
    """err, H, b at T_eval over a fixed (source index, voxel id) list linearised at T_lin."""
    src, src_cov, pairs = O._f32(src), O._f32(src_cov), O._i32(pairs)
    H = np.zeros(36)
    b = np.zeros(6)
    e = lib().orc_robust_derivatives(vmap._h, O._p(src, C.c_float), O._p(src_cov, C.c_float), O._p(pairs, C.c_int), len(pairs), O._p(O._pose_in(T_lin), C.c_double),
                                     O._p(O._pose_in(T_eval), C.c_double), O._p(H, C.c_double) if want_H else None, O._p(b, C.c_double) if want_H else None,
                                     kind_of(robust), C.c_float(scale_sq(robust_scale)))
    return e, H.reshape(6, 6).T.copy(), b


def align_f32(vmap, src, src_cov, offs, guess=None, params=None, robust=NONE, robust_scale=1.0):
    """oracle.align_f32 (double sums) with the robust kind."""
    src, src_cov, offs = O._f32(src), O._f32(src_cov), O._i32(offs)
    params = params or O.default_params()
    g = O._pose_in(np.eye(4) if guess is None else guess)
    r = O.LsqResult()
    lib().orc_robust_align_f32(vmap._h, O._p(src, C.c_float), O._p(src_cov, C.c_float), len(src), O._p(offs, C.c_int), len(offs), C.byref(params),
                               O._p(g, C.c_double), kind_of(robust), C.c_float(scale_sq(robust_scale)), C.byref(r))
    return O.AlignResult(r)


def register_f32(target, source, k=20, reg=O.REG_PLANE, res=1.0, method=O.DIRECT1, radius=-1.0, guess=None, params=None, accum_double=False, symmetrize=False,
                 robust=NONE, robust_scale=1.0):
    """oracle.register_f32 (k-NN covariances) with the robust kind."""
    tc = O.estimate_covariances(target, k, reg)
    sc = O.estimate_covariances(source, k, reg)
    if symmetrize:
        tc, sc = O.symmetrized(tc), O.symmetrized(sc)
    vm = O.VoxelMap(target, tc, res, accum_double=accum_double)
    return align_f32(vm, source, sc, O.offsets(method, radius), guess, params, robust, robust_scale)
