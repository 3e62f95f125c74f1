"""Robust kernels (vgicp_set_robust_kernel) on the GPU: every evaluation path against the robust CPU checker, registrations
against its LM, bit identity across the paths that must not change results, NONE against a handle that never set a kind, the
error codes, and the public surfaces."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

import oracle as O
import oracle_robust as R
from conftest import pose_error
from test_gpu_multi_hypothesis import assert_same, guesses, setup
from test_oracle_robust import GATE_R, GATE_T, contaminate

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["NONE", "HUBER", "CAUCHY", "GEMAN_MCCLURE"]
ROBUST = KINDS[1:]
METHODS = [(O.DIRECT1, -1.0), (O.DIRECT7, -1.0), (O.DIRECT27, -1.0), (O.DIRECT_RADIUS, 1.5)]


def sym(c9):
    m = c9.reshape(-1, 3, 3)
    return (0.5 * (m + m.transpose(0, 2, 1))).reshape(-1, 9).astype(np.float32)


@pytest.fixture(scope="module")
def prepared(pair02):
    R.build()
    tgt, src = pair02
    t_cov = sym(O.regularize(O.covariances(tgt, O.knn(tgt, 20, "kdtree")), O.REG_PLANE))
    s_cov = sym(O.regularize(O.covariances(src, O.knn(src, 20, "kdtree")), O.REG_PLANE))
    return dict(tgt=tgt, src=src, s_cov=s_cov, vm=O.VoxelMap(tgt, t_cov, 1.0, accum_double=True))


def assert_close(got, want):
    (e, H, b), (e0, H0, b0) = got, want
    assert abs(e - e0) <= 2e-5 * abs(e0)
    if H is not None:
        assert np.abs(H - H0).max() <= 2e-5 * np.abs(H0).max()
        assert np.abs(b - b0).max() <= 2e-5 * max(np.abs(b0).max(), 1e-3 * np.abs(H0).max())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("method,radius", METHODS)
def test_evaluation_matches_the_robust_oracle(prepared, relative_pose, kind, method, radius):
    from fast_gicp_b200.core import Core

    c = setup(Core(0), prepared["tgt"], prepared["src"], method=method, radius=radius)
    c.set_robust_kernel(kind, 1.0)
    offs = O.offsets(method, radius)
    for T in (np.eye(4), relative_pose):
        c.update_correspondences(T)
        for want_H in (True, False):
            e0, H0, b0, _ = R.evaluate(prepared["vm"], prepared["src"], prepared["s_cov"], offs, T, T, want_H, robust=kind, robust_scale=1.0)
            assert_close(c.compute_error(T, want_H), (e0, H0 if want_H else None, b0))
    c.close()


@pytest.mark.parametrize("kind", ROBUST)
def test_align_matches_the_robust_oracle(pair01, relative_pose, kind):
    from fast_gicp_b200.core import Core, pose_from_c

    tgt, src = pair01
    for method in (O.DIRECT1, O.DIRECT7):
        c = setup(Core(0), tgt, src, method=method)
        c.set_robust_kernel(kind, 1.0)
        r = c.align()
        ref = R.register_f32(tgt, src, method=method, accum_double=True, symmetrize=True, robust=kind, robust_scale=1.0)
        assert r.converged and ref.converged
        assert (r.nr_iterations, r.n_linearize, r.n_compute_error) == (ref.iterations, ref.n_linearize, ref.n_error)
        dt, dr = pose_error(ref.T, pose_from_c(r.T))
        assert dt < 1e-4 and dr < 1e-5, (method, dt, dr)
        c.close()


def test_contaminated_source_passes_the_gate_only_with_a_robust_kernel(pair01, relative_pose):
    from fast_gicp_b200.core import Core, pose_from_c

    tgt, src = pair01
    c = setup(Core(0), tgt, contaminate(src), method=O.DIRECT1)
    dt, _ = pose_error(relative_pose, pose_from_c(c.align().T))
    assert dt > GATE_T, dt
    for kind in ROBUST:
        c.set_robust_kernel(kind, 1.0)
        r = c.align()
        dt, dr = pose_error(relative_pose, pose_from_c(r.T))
        assert r.converged and dt < GATE_T and dr < GATE_R, (kind, dt, math.degrees(dr))
    c.close()


@pytest.mark.parametrize("kind", ROBUST)
def test_robust_results_are_path_independent(pair02, relative_pose, kind):
    """speculation on / off, both execution hints, both voxel indexes; align_multi == a loop of align; evaluate_poses == the
    single-pose calls -- all bit for bit with a robust kind set."""
    from fast_gicp_b200.core import Core

    G = guesses(relative_pose)
    base = None
    for spec, hint, index in [(1, 0, 0), (0, 0, 0), (1, 1, 0), (0, 1, 1), (1, 0, 1)]:
        c = Core(0)
        c.set_speculation(spec)
        c.set_execution_hint(hint)
        c.set_voxel_index(index)
        setup(c, *pair02, method=O.DIRECT7)
        c.set_robust_kernel(kind, 1.0)
        res = [c.align(g) for g in G[:6]]
        if base is None:
            base = res
            multi = c.align_multi(G)
            for i, g in enumerate(G):
                assert_same(multi[i], c.align(g), f"{kind} guess {i}")
            err, H, b, n_corr = c.evaluate_poses(G[:6], want_H=True)
            for i, T in enumerate(G[:6]):
                c.update_correspondences(T)
                e1, H1, b1 = c.compute_error(T, True)
                assert err[i] == e1 and np.array_equal(H[i], H1) and np.array_equal(b[i], b1)
                assert n_corr[i] == len(c.get_voxel_correspondences())
        else:
            for a, r in zip(base, res):
                assert_same(a, r, f"{kind} spec={spec} hint={hint} index={index}")
        c.close()


def test_streaming_kernel_matches_the_robust_oracle():
    """1 M-point pair, DIRECT1: the bulk-copy streaming kernel, against the checker fed the GPU's (bit-exact) covariances."""
    from fast_gicp_b200.core import Core
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
    c = setup(Core(0), tgt, src, method=O.DIRECT1, res=0.5)
    vm = O.VoxelMap(tgt, c.get_target_covariances(), 0.5, accum_double=True)
    s_cov = c.get_source_covariances()
    offs = O.offsets(O.DIRECT1)
    for kind in ("HUBER", "CAUCHY", "GEMAN_MCCLURE"):
        c.set_robust_kernel(kind, 1.0)
        c.update_correspondences(T_gt)
        for want_H in (True, False):
            e0, H0, b0, _ = R.evaluate(vm, src, s_cov, offs, T_gt, T_gt, want_H, robust=kind, robust_scale=1.0)
            assert_close(c.compute_error(T_gt, want_H), (e0, H0 if want_H else None, b0))
    c.close()


def test_none_after_a_robust_kind_equals_a_fresh_handle(pair02, relative_pose):
    """NONE after another kind is bit-identical to a handle that never set one; the setting survives cloud changes and a swap."""
    from fast_gicp_b200.core import Core

    tgt, src = pair02
    fresh = setup(Core(0), tgt, src, method=O.DIRECT27)
    used = setup(Core(0), tgt, src, method=O.DIRECT27)
    robust_ref = setup(Core(0), tgt, src, method=O.DIRECT27)
    robust_ref.set_robust_kernel("CAUCHY", 2.0)
    want_robust = robust_ref.align(relative_pose)
    used.set_robust_kernel("CAUCHY", 2.0)
    used.set_source_cloud(src)  # a setting of the handle, like the resolution
    used.find_source_neighbors(20)
    used.calculate_source_covariances(O.REG_PLANE)
    assert_same(used.align(relative_pose), want_robust)
    used.swap_source_and_target()
    used.swap_source_and_target()
    assert_same(used.align(relative_pose), want_robust)
    used.set_robust_kernel("NONE", 2.0)
    assert_same(used.align(relative_pose), fresh.align(relative_pose))
    for T in (np.eye(4), relative_pose):
        fresh.update_correspondences(T)
        used.update_correspondences(T)
        a, b = fresh.compute_error(T, True), used.compute_error(T, True)
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    for c in (fresh, used, robust_ref):
        c.close()


def test_error_codes_launch_nothing(pair02):
    from fast_gicp_b200.core import ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, OK, AlignResult, Core

    tgt, src = pair02
    c = setup(Core(0), tgt, src, method=O.DIRECT7)
    c.align()
    L, h = c._lib, c._h
    n0 = c.launch_count()
    for kind, scale in [(4, 1.0), (-1, 1.0), (1, 0.0), (2, -1.0), (3, float("nan")), (1, float("inf")), (2, float("-inf"))]:
        assert L.vgicp_set_robust_kernel(h, kind, scale) == ERR_INVALID_ARGUMENT, (kind, scale)
    assert L.vgicp_set_robust_kernel(None, 1, 1.0) == ERR_INVALID_ARGUMENT
    assert L.vgicp_set_robust_kernel(h, 0, float("nan")) == OK  # the scale is ignored for NONE
    assert c.launch_count() == n0
    c.close()
    # NDT with a robust kind: refused before anything is launched
    nd = setup(Core(0), tgt, src, method=O.DIRECT7, problem=2)
    nd.update_correspondences(np.eye(4))
    nd.compute_error(np.eye(4), True)
    nd.set_robust_kernel("HUBER", 1.0)
    L, h = nd._lib, nd._h
    G = np.ascontiguousarray(np.stack([np.eye(4)] * 2).transpose(0, 2, 1)).reshape(-1)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    out, H, b, e = np.zeros(2), np.zeros(72), np.zeros(12), C.c_double(0.0)
    res = (AlignResult * 2)()
    n0 = nd.launch_count()
    rcs = [L.vgicp_compute_error(h, dp(G), dp(H), dp(b), C.byref(e)), L.vgicp_compute_error(h, dp(G), None, None, C.byref(e)),
           L.vgicp_align(h, dp(G), None, res), L.vgicp_align_multi(h, dp(G), 2, None, res),
           L.vgicp_evaluate_poses(h, dp(G), 2, dp(out), None, None, None)]
    assert rcs == [ERR_UNSUPPORTED] * len(rcs)
    assert nd.launch_count() == n0
    nd.set_robust_kernel("NONE")
    nd.align()  # NDT runs again once the kind is NONE
    nd.close()


def _pygicp():
    lib = os.path.join(ROOT, "fast_gicp_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import pygicp

    return pygicp


def test_surfaces_return_the_core_pose(pair02):
    """The Python class (bit for bit: same C call) and pygicp over the C++ mirror (its own LM loop: to rounding)."""
    import fast_gicp_b200 as F
    from fast_gicp_b200.core import Core, pose_from_c

    tgt, src = pair02
    for kind in ROBUST:
        c = setup(Core(0), tgt, src, method=O.DIRECT27)
        c.set_robust_kernel(kind, 1.5)
        T_core = pose_from_c(c.align().T).astype(np.float32)
        c.close()
        reg = F.FastVGICPCuda()
        reg.setNeighborSearchMethod("DIRECT27")
        reg.setRobustKernel(kind, 1.5)
        reg.setInputTarget(tgt)
        reg.setInputSource(src)
        assert np.array_equal(reg.align(), T_core) and reg.hasConverged(), kind
        pg = _pygicp().FastVGICPCuda()
        pg.set_neighbor_search_method("DIRECT27", 0.0)
        pg.set_robust_kernel(kind, 1.5)
        pg.set_input_target(tgt.astype(np.float64))
        pg.set_input_source(src.astype(np.float64))
        dt, dr = pose_error(T_core, pg.align())
        assert pg.has_converged() and dt < 1e-6 and dr < 1e-7, (kind, dt, dr)
    with pytest.raises(ValueError):
        _pygicp().FastVGICPCuda().set_robust_kernel("TUKEY", 1.0)
