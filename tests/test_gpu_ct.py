"""Continuous-time registration on the device: vgicp_compute_error_ct against the float64 model (tests/ct_reference.py), entry by
entry with the tau A scheme, over every neighbour search, both voxel indexes and every robust kind, at source sizes on both sides
of make_lin_launch's thresholds (65 536: where DIRECT1 would stream, the CT evaluation keeps the compacted (1, 1) shape; 400 000:
the lane split); the reduction to vgicp_compute_error / vgicp_align bit for bit with zero time offsets; the distorted scan that
plain registration cannot register; strides, reset rules and error codes (none of which launches anything)."""
import numpy as np
import pytest

import oracle as O
from conftest import pose_error
from ct_reference import assert_close, ct_sums, system12
from eval_reference import KINDS
from test_ct_model import EFFECT_TWIST, _f32pose, deskew_f32, distorted_pair, twist_error
from test_gpu_multi_hypothesis import setup

pytestmark = pytest.mark.gpu

TAU_PLANE = 1e-4  # PLANE covariances (test_gpu_eval_matrix: cond(S) <= 1e3)
METHODS = {"d1": (O.DIRECT1, -1.0), "d7": (O.DIRECT7, -1.0), "d27": (O.DIRECT27, -1.0), "r1.5": (O.DIRECT_RADIUS, 1.5)}
XI = np.array([0.02, -0.03, np.radians(20.0), 9.0, 0.3, -0.1])


def core():
    from fast_gicp_b200.core import Core

    return Core(0)


def model_ref(h, times, T_lin, xi_lin, T_eval, xi_eval, offs, robust):
    q_lin = deskew_f32(h["src"], times, xi_lin, 0.0)
    q_eval = deskew_f32(h["src"], times, xi_eval, 0.0)
    pairs = O.find_correspondences(h["vm"], q_lin, T_lin, offs)
    sums = ct_sums(h["mean"], h["cov"], h["n"], q_eval, h["s_cov"], times, pairs, _f32pose(T_lin), _f32pose(T_eval), robust)
    return system12(sums, _f32pose(T_eval))


def handle(tgt, src, times):
    c = setup(core(), tgt, src, method=O.DIRECT1)
    t_cov = c.get_target_covariances()
    vm = O.VoxelMap(tgt, t_cov, 1.0, accum_double=True)
    assert c.num_voxels() == vm.num_voxels and np.array_equal(c.get_voxel_means(), vm.vox_mean)
    c.set_source_timestamps(times, 0.0)
    return dict(core=c, vm=vm, src=src, s_cov=c.get_source_covariances(), mean=c.get_voxel_means(), cov=c.get_voxel_covs(), n=c.get_voxel_num_points())


def check(h, times, methods, kinds, T_near, what):
    c = h["core"]
    T2 = T_near @ O.se3_exp(np.array([0.002, -0.001, 0.003, 0.03, 0.02, -0.01]))
    cases = [(T_near, XI, T_near, XI), (T_near, np.zeros(6), T2, XI)]  # lin = eval, lin != eval
    worst = 0.0
    for m in methods:
        c.set_neighbor_search_method(*METHODS[m])
        offs = O.offsets(*METHODS[m])
        for Tl, xl, Te, xe in cases:
            refs = {k: model_ref(h, times, Tl, xl, Te, xe, offs, None if k == "NONE" else k) for k in kinds}
            for k in kinds:
                c.set_robust_kernel(k, 1.0)
                for index in (0, 1):
                    c.set_voxel_index(index)
                    got = c.compute_error_ct(Tl, xl, Te, xe, True)
                    tag = f"{what} {m} {k} index={index} lin{'=' if Tl is Te else '!='}eval"
                    worst = max(worst, assert_close(got, refs[k], TAU_PLANE, tag))
                    e_only = c.compute_error_ct(Tl, xl, Te, xe, False)
                    assert_close(e_only, refs[k], TAU_PLANE, tag + " error only")
    c.set_robust_kernel("NONE")
    c.set_voxel_index(0)
    print(f"{what}: worst |x - x_ref| / A {worst:.3g}")


@pytest.fixture(scope="module")
def small():
    tgt, src, ts, T = distorted_pair()
    h = handle(tgt, src, ts)
    yield h, ts, T
    h["core"].close()


def test_compute_error_ct_small(small):
    h, ts, T = small
    check(h, ts, METHODS, KINDS, T, "small")


@pytest.fixture(scope="module")
def big():
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0)
    rng = np.random.default_rng(44)
    tgt = tgt[np.sort(rng.permutation(len(tgt))[:500_000])]
    src = src[rng.permutation(len(src))[:400_000]]
    times = rng.uniform(0.0, 0.1, size=len(src)).astype(np.float32)
    return tgt, src, times, T_gt


@pytest.mark.parametrize("n,method", [(65_535, "d1"), (65_536, "d1"), (399_999, "d7"), (400_000, "d7")])
def test_compute_error_ct_thresholds(big, n, method):
    tgt, src, times, T_gt = big
    h = handle(tgt, src[:n], times[:n])
    check(h, times[:n], [method], ("NONE", "CAUCHY"), T_gt, f"n={n}")
    h["core"].close()


def test_zero_time_offsets_equal_the_single_pose_path(small):
    """s = 0 everywhere: err, H0, b0 are vgicp_compute_error's bit for bit, the coupling blocks exactly zero; align_ct with a zero
    twist guess and prior (W = 1e-6) is vgicp_align: T and counters bit for bit."""
    h, ts, T = small
    c = h["core"]
    c.set_source_timestamps(np.full(len(ts), 0.05, dtype=np.float32), 0.05)
    T2 = T @ O.se3_exp(np.array([0.002, -0.001, 0.003, 0.03, 0.02, -0.01]))
    try:
        for m in METHODS:
            c.set_neighbor_search_method(*METHODS[m])
            for k in ("NONE", "HUBER"):
                c.set_robust_kernel(k, 1.0)
                for index in (0, 1):
                    c.set_voxel_index(index)
                    c.update_correspondences(T)
                    err, H, b = c.compute_error(T2, True)
                    e, H12, b12 = c.compute_error_ct(T, np.zeros(6), T2, np.zeros(6), True)
                    assert e == err and np.array_equal(H12[:6, :6], H) and np.array_equal(b12[:6], b), (m, k, index)
                    assert not H12[:6, 6:].any() and not H12[6:, :6].any() and not H12[6:, 6:].any() and not b12[6:].any()
                    assert c.compute_error_ct(T, np.zeros(6), T2, np.zeros(6), False)[0] == c.compute_error(T2, False)[0]
                    for guess in (np.eye(4), T2):
                        plain = c.align(guess)
                        ct = c.align_ct(guess, np.zeros(6), np.zeros(6), np.full(6, 1e-6))
                        assert np.array_equal(np.array(plain.T), np.array(ct.T)), (m, k, index)
                        assert not np.array(ct.twist).any()
                        for f in ("nr_iterations", "converged", "n_linearize", "n_compute_error", "lm_failed"):
                            assert getattr(plain, f) == getattr(ct, f), (m, k, index, f)
    finally:
        c.set_robust_kernel("NONE")
        c.set_voxel_index(0)
        c.set_source_timestamps(ts, 0.0)


def test_align_ct_registers_the_distorted_scan(small):
    """vgicp_align misses the 0.05 m / 1 deg gate on the raw scan (0.240 m / 0.55 deg with the oracle); align_ct meets it and finds
    the sweep's twist.  The numpy CT-LM (test_ct_model) reaches 0.0016 m / 0.011 deg and 0.15 deg/s / 0.023 m/s of twist error:
    the gates below leave a margin of about 5 over those."""
    h, ts, T = small
    c = h["core"]
    c.set_neighbor_search_method(O.DIRECT7)
    t0, r0 = pose_error(T, np.array(c.align(np.eye(4)).T).reshape(4, 4).T)
    assert not (t0 < 0.05 and r0 < np.radians(1.0)), (t0, np.degrees(r0))
    res = c.align_ct(np.eye(4), np.zeros(6), np.zeros(6), np.full(6, 1e-6))
    t, r = pose_error(T, np.array(res.T).reshape(4, 4).T)
    tw = twist_error(np.array(res.twist), EFFECT_TWIST)
    print(f"align: {t0:.4f} m / {np.degrees(r0):.3f} deg;  align_ct: {t:.4f} m / {np.degrees(r):.4f} deg, twist error {tw[0]:.3f} deg/s / {tw[1]:.4f} m/s, "
          f"{res.n_linearize} + {res.n_compute_error} evaluations")
    assert res.converged and not res.lm_failed
    assert t < 0.01 and r < np.radians(0.05), (t, np.degrees(r))
    assert tw[0] < 0.75 and tw[1] < 0.12, tw


def test_strides_reset_rules_and_errors(small):
    from fast_gicp_b200.core import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, VgicpError

    h, ts, T = small
    c = h["core"]
    c.set_neighbor_search_method(O.DIRECT7)
    args = (T, XI * 0.5, T, XI)
    ref = c.compute_error_ct(*args)
    rec = np.zeros(len(ts), dtype=[("x", np.float32, 3), ("t", np.float32), ("pad", np.float32, 4)])  # 32-byte records
    rec["t"] = ts
    c.set_source_timestamps(rec["t"], 0.0)
    got = c.compute_error_ct(*args)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])

    def code(fn, *a):
        n0 = c.launch_count()
        with pytest.raises(VgicpError) as e:
            fn(*a)
        assert c.launch_count() == n0, "an error path launched a kernel"
        return e.value.code

    W = np.full(6, 1e-6)
    bad_twist = np.array([0.0, 0.0, 20.0, 0.0, 0.0, 0.0])  # 20 rad/s x 0.1 s > pi/2
    assert code(c.align_ct, np.eye(4), np.zeros(6), np.zeros(6), np.zeros(6)) == ERR_INVALID_ARGUMENT  # W = 0
    assert code(c.align_ct, np.eye(4), np.zeros(6), np.zeros(6), -W) == ERR_INVALID_ARGUMENT
    assert code(c.align_ct, np.eye(4), np.full(6, np.nan), np.zeros(6), W) == ERR_INVALID_ARGUMENT
    assert code(c.align_ct, np.full((4, 4), np.inf), np.zeros(6), np.zeros(6), W) == ERR_INVALID_ARGUMENT
    assert code(c.align_ct, np.eye(4), bad_twist, np.zeros(6), W) == ERR_INVALID_ARGUMENT
    assert code(c.align_ct, np.eye(4), np.zeros(6), bad_twist, W) == ERR_INVALID_ARGUMENT
    assert code(c.compute_error_ct, T, bad_twist, T, np.zeros(6)) == ERR_INVALID_ARGUMENT
    assert code(c.set_source_timestamps, ts[:-1], 0.0) == ERR_INVALID_ARGUMENT
    bad = ts.copy()
    bad[3] = np.inf
    assert code(c.set_source_timestamps, bad, 0.0) == ERR_INVALID_ARGUMENT
    assert code(c.set_source_timestamps, ts, 1e39) == ERR_INVALID_ARGUMENT
    # deskew keeps the timestamps (then the covariances are recomputed); set_source_cloud and swap drop them
    c.deskew_source(ts, XI * 0.5, 0.0)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)
    c.compute_error_ct(T, XI * 0.5, T, XI * 0.5)
    c.set_source_cloud(h["src"])
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)
    assert code(c.align_ct, np.eye(4), np.zeros(6), np.zeros(6), W) == ERR_BAD_STATE
    assert code(c.compute_error_ct, *args) == ERR_BAD_STATE
    c.set_source_timestamps(ts, 0.0)
    c.swap_source_and_target()
    c.swap_source_and_target()
    assert code(c.align_ct, np.eye(4), np.zeros(6), np.zeros(6), W) == ERR_BAD_STATE
    c.set_source_timestamps(ts, 0.0)
    got = c.compute_error_ct(*args)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1])
    # NDT and sharding
    c.set_problem(1)
    assert code(c.align_ct, np.eye(4), np.zeros(6), np.zeros(6), W) == ERR_UNSUPPORTED
    c.set_problem(0)
    c.set_source_shard(0, len(ts) // 2)
    assert code(c.compute_error_ct, *args) == ERR_UNSUPPORTED
    c.clear_source_shard()
    got = c.compute_error_ct(*args)
    assert got[0] == ref[0]


def test_twist_prior(small):
    """A prior weight large enough to matter.  W = 1e12 pins the twist to the prior mean (from a zero guess: the prior's terms in
    err, H and b all have to be right for the step to land there).  A moderate W pulls the estimate away from the free one, and the
    device follows the numpy CT-LM of test_ct_model with the same prior."""
    from test_ct_model import ct_lm, problem

    h, ts, T = small
    c = h["core"]
    c.set_neighbor_search_method(O.DIRECT7)
    xi0 = EFFECT_TWIST * 0.7
    pinned = c.align_ct(np.eye(4), np.zeros(6), xi0, np.full(6, 1e12))
    assert np.max(np.abs(np.array(pinned.twist) - xi0)) <= 1e-6 * np.max(np.abs(xi0)), (list(pinned.twist), xi0)
    free = np.array(c.align_ct(np.eye(4), np.zeros(6), np.zeros(6), np.full(6, 1e-6)).twist)
    W = np.full(6, 1e4)
    res = c.align_ct(np.eye(4), np.zeros(6), np.zeros(6), W)
    vm, src, sc, ts_m, _ = problem()
    T_m, xi_m, it, conv = ct_lm(vm, src, sc, ts_m, O.offsets(O.DIRECT7), np.eye(4), np.zeros(6), np.zeros(6), W)
    got_T = np.array(res.T).reshape(4, 4).T
    t, r = pose_error(T_m, got_T)
    dw, dv = twist_error(np.array(res.twist), xi_m)
    pw, pv = twist_error(np.array(res.twist), free)
    print(f"W = 1e4: device vs model {t:.2e} m / {np.degrees(r):.2e} deg, twist {dw:.3g} deg/s / {dv:.3g} m/s; the prior moved the twist by {pw:.3g} deg/s / {pv:.3g} m/s")
    assert res.converged and conv
    assert t < 2e-3 and r < np.radians(0.02) and dw < 0.05 and dv < 0.01, (t, np.degrees(r), dw, dv)
    assert pw > 0.5 or pv > 0.1, (pw, pv)


def test_python_class_cpp_mirror_and_pygicp_equal_core():
    """FastVGICPCuda.alignCT (Python), and pygicp's align_ct over the C++ mirror's alignCT, return Core.align_ct's T (as float, like
    align), twist, H and counters; a new input source drops the timestamps in every layer, the same one keeps them."""
    import os
    import sys

    from fast_gicp_b200 import FastVGICPCuda
    from fast_gicp_b200.core import ERR_BAD_STATE, VgicpError, pose_from_c

    tgt, src, ts, _ = distorted_pair()
    xi0, W = EFFECT_TWIST * 0.8, np.full(6, 1e-2)
    a = setup(core(), tgt, src, method=O.DIRECT7)
    a.set_source_timestamps(ts, 0.0)
    want = a.align_ct(np.eye(4), xi0, xi0, W)
    a.close()
    want_T = pose_from_c(want.T).astype(np.float32)
    want_H = np.array(want.H).reshape(12, 12).T
    counters = ("nr_iterations", "converged", "n_linearize", "n_compute_error", "lm_failed")

    def same(d, what):
        assert np.array_equal(np.asarray(d["T"], dtype=np.float32), want_T), what
        assert np.array_equal(d["twist"], np.array(want.twist)) and np.array_equal(d["H"], want_H), what
        assert tuple(int(d[f]) for f in counters) == tuple(int(getattr(want, f)) for f in counters), what

    reg = FastVGICPCuda()
    reg.setNeighborSearchMethod("DIRECT7")
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    reg.setSourceTimestamps(ts)
    same(reg.alignCT(np.eye(4), xi0, xi0, W), "python class")
    assert np.array_equal(reg.getFinalTransformation(), want_T) and reg.hasConverged() == bool(want.converged)
    reg.setInputSource(src)  # the same cloud: nothing is reloaded, the timestamps stay
    same(reg.alignCT(np.eye(4), xi0, xi0, W), "python class, same source")
    reg.setInputSource(src.copy())
    with pytest.raises(VgicpError) as e:
        reg.alignCT(np.eye(4), xi0, xi0, W)
    assert e.value.code == ERR_BAD_STATE

    lib = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fast_gicp_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import pygicp

    p = pygicp.FastVGICPCuda()
    p.set_neighbor_search_method("DIRECT7", 1.5)
    p.set_input_target(tgt.astype(np.float64))
    p.set_input_source(src.astype(np.float64))
    p.set_source_timestamps(ts)
    same(p.align_ct(np.eye(4, dtype=np.float32), xi0, xi0, W), "pygicp")
    p.set_input_source(src.astype(np.float64))  # a new cloud: reloaded, the timestamps dropped
    with pytest.raises(RuntimeError):
        p.align_ct(np.eye(4, dtype=np.float32), xi0, xi0, W)
