"""Motion compensation on the device: vgicp_deskew_source.

The deskewed points are read back with transform_source(identity) (exact up to the sign of zero) and compared with deskew_f32,
the numpy float32 restatement of the header's recipe (tests/test_deskew_model.py).  For the state afterwards, handle A deskews on
the device and handle B is given the restated points with set_source_cloud: both must then hold and evaluate the same bytes."""
import ctypes
import os
import sys

import numpy as np
import pytest

import oracle as O
from conftest import pose_error
from test_deskew_model import EFFECT_TWIST, deskew_f32, distorted_pair, random_twist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fast_gicp_b200", "lib")

pytestmark = pytest.mark.gpu

# a PointXYZIT-like 32-byte point: the timestamps are read straight out of it
POINT_XYZIT = np.dtype({"names": ["x", "y", "z", "intensity", "time", "ring"], "formats": ["<f4", "<f4", "<f4", "<f4", "<f4", "<u2"],
                        "offsets": [0, 4, 8, 12, 16, 20], "itemsize": 32})


def _core(method="DIRECT7"):
    from fast_gicp_b200.core import Core

    c = Core(0)
    c.set_resolution(1.0)
    c.set_neighbor_search_method(method)
    return c


def _load_target(c, pts):
    c.set_target_cloud(pts)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()


def _covs(c):
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)


def _source_points(c):
    return c.transform_source(np.eye(4))


def _res_tuple(r):
    return (bytes(r.T), bytes(r.H), r.nr_iterations, r.converged, r.n_linearize, r.n_compute_error, r.lm_failed)


def _times_and_twist(rng, n, max_theta=1.2):
    times = rng.uniform(0.0, 0.1, size=n).astype(np.float32)
    return times, random_twist(rng, max_theta, 0.1)


# ------------------------------------------------------------------------------------------------------------ bytes
@pytest.mark.parametrize("layout", ["contiguous", "point_struct"])
def test_device_equals_restatement(pair02, layout):
    _, src = pair02
    rng = np.random.default_rng(21)
    c = _core()
    for trial in range(4):
        times, xi = _times_and_twist(rng, len(src))
        t_ref = float(rng.uniform(0.0, 0.1))
        c.set_source_cloud(src)
        if layout == "contiguous":
            c.deskew_source(times, xi, t_ref)
        else:
            cloud = np.zeros(len(src), dtype=POINT_XYZIT)
            cloud["x"], cloud["y"], cloud["z"], cloud["time"] = src[:, 0], src[:, 1], src[:, 2], times
            assert cloud["time"].strides[0] == 32
            c.deskew_source(cloud["time"], xi, t_ref)
        assert np.array_equal(_source_points(c), deskew_f32(src, times, xi, t_ref)), trial
    c.close()


def test_quarter_turn_edge_and_zero_twist(pair02):
    from fast_gicp_b200.core import Core

    _, src = pair02
    rng = np.random.default_rng(4)
    times = rng.uniform(0.0, 0.1, size=len(src)).astype(np.float32)
    times[0], times[1] = 0.0, 0.1
    span = float(np.float32(0.1))
    w = rng.normal(size=3)
    w *= (np.pi / 2) / span / np.linalg.norm(w) * (1.0 - 1e-12)  # |omega| * max |t_i - t_ref| = pi/2
    xi = np.concatenate([w, [20.0, -3.0, 0.5]])
    c = Core(0)
    c.set_source_cloud(src)
    c.deskew_source(times, xi, 0.0)
    assert np.array_equal(_source_points(c), deskew_f32(src, times, xi, 0.0))
    c.set_source_cloud(src)
    c.deskew_source(times, np.zeros(6), 0.05)
    assert np.array_equal(_source_points(c), src)
    c.close()


# ------------------------------------------------------------------------------------------------------------ state
def _pair_of_handles(tgt, src, times, xi, problem=0, robust=None):
    """A deskews on the device, B is given the restated points; both then compute their source state the same way."""
    a, b = _core(), _core()
    for c in (a, b):
        if problem:
            c.set_problem(problem)
        if robust:
            c.set_robust_kernel(robust, 1.0)
        c.set_target_cloud(tgt)
        if not problem:
            c.find_target_neighbors(20)
            c.calculate_target_covariances(O.REG_PLANE)
            c.create_target_voxelmap()
    a.set_source_cloud(src)
    if not problem:
        _covs(a)  # covariances of the raw scan: the deskew must drop them
    a.deskew_source(times, xi, 0.05)
    b.set_source_cloud(deskew_f32(src, times, xi, 0.05))
    for c in (a, b):
        if problem:
            c.ndt_create_voxelmaps()
        else:
            _covs(c)
    return a, b


def _assert_same_evaluations(a, b, poses, with_align=True):
    for T in poses:
        a.update_correspondences(T)
        b.update_correspondences(T)
        ea, Ha, ba = a.compute_error(T)
        eb, Hb, bb = b.compute_error(T)
        assert ea == eb and Ha.tobytes() == Hb.tobytes() and ba.tobytes() == bb.tobytes()
    if with_align:
        assert _res_tuple(a.align(poses[0])) == _res_tuple(b.align(poses[0]))
    ma, mb = a.align_multi(np.stack(poses)), b.align_multi(np.stack(poses))
    assert [_res_tuple(r) for r in ma] == [_res_tuple(r) for r in mb]
    for want_H in (False, True):
        ra, rb = a.evaluate_poses(np.stack(poses), want_H), b.evaluate_poses(np.stack(poses), want_H)
        for x, y in zip(ra, rb):
            assert (x is None and y is None) or x.tobytes() == y.tobytes()


@pytest.mark.parametrize("robust", [None, "CAUCHY"])
def test_deskewed_handle_equals_uploaded_points(pair02, relative_pose, robust):
    tgt, src = pair02
    rng = np.random.default_rng(8)
    times, xi = _times_and_twist(rng, len(src), 0.3)
    xi[3:] *= 0.05  # keep the pair registrable
    a, b = _pair_of_handles(tgt, src, times, xi, robust=robust)
    assert a.get_source_covariances().tobytes() == b.get_source_covariances().tobytes()
    assert a.get_source_neighbors().tobytes() == b.get_source_neighbors().tobytes()
    _assert_same_evaluations(a, b, [relative_pose, np.eye(4)])
    a.close()
    b.close()


def test_deskew_under_ndt_p2d(pair02, relative_pose):
    tgt, src = pair02
    rng = np.random.default_rng(9)
    times, xi = _times_and_twist(rng, len(src), 0.3)
    xi[3:] *= 0.05
    a, b = _pair_of_handles(tgt, src, times, xi, problem=1)
    assert np.array_equal(_source_points(a), _source_points(b))
    _assert_same_evaluations(a, b, [relative_pose, np.eye(4)])
    a.close()
    b.close()


def test_errors_change_nothing(pair02):
    from fast_gicp_b200 import core as K

    _, src = pair02
    n = len(src)
    c = _core()
    c.set_source_cloud(src)
    _covs(c)
    pts0, cov0, launches = _source_points(c), c.get_source_covariances(), c.launch_count()
    lib, h = c._lib, c._h
    dp = lambda x: x.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    times = np.linspace(0.0, 0.1, n, dtype=np.float32)
    xi = np.array([0.0, 0.0, 1.0, 10.0, 0.0, 0.0])

    def call(t=times, nn=n, stride=4, tw=xi, t_ref=0.0):
        return lib.vgicp_deskew_source(h, None if t is None else t.ctypes.data, nn, stride, None if tw is None else dp(tw), t_ref)

    assert call(t=None) == K.ERR_INVALID_ARGUMENT
    assert call(tw=None) == K.ERR_INVALID_ARGUMENT
    assert call(nn=n - 1) == K.ERR_INVALID_ARGUMENT
    assert call(nn=n + 1) == K.ERR_INVALID_ARGUMENT
    for stride in (0, 2, 6):
        assert call(stride=stride) == K.ERR_INVALID_ARGUMENT
    for bad in (np.nan, np.inf):
        tb = times.copy()
        tb[n // 2] = bad
        assert call(t=tb) == K.ERR_INVALID_ARGUMENT
        xb = xi.copy()
        xb[4] = bad
        assert call(tw=xb) == K.ERR_INVALID_ARGUMENT
        assert call(t_ref=bad) == K.ERR_INVALID_ARGUMENT
    xb = xi.copy()
    xb[3] = 1e300  # finite in double, not in float
    assert call(tw=xb) == K.ERR_INVALID_ARGUMENT
    xb = xi.copy()
    xb[2] = 16.0  # 16 rad/s over 0.1 s > pi/2
    assert call(tw=xb) == K.ERR_INVALID_ARGUMENT
    xb[2] = 0.99 * (np.pi / 2) / 0.1  # within the bound over [0, 0.1] from t_ref = 0, beyond it from t_ref = -0.01
    assert call(tw=xb, t_ref=-0.01) == K.ERR_INVALID_ARGUMENT
    assert c.launch_count() == launches
    assert np.array_equal(_source_points(c), pts0) and c.get_source_covariances().tobytes() == cov0.tobytes()
    e = K.Core(0)
    assert e._lib.vgicp_deskew_source(e._h, times.ctypes.data, 0, 4, dp(xi), 0.0) == K.ERR_BAD_STATE
    e.set_source_cloud(np.zeros((0, 3), dtype=np.float32))
    assert e._lib.vgicp_deskew_source(e._h, times.ctypes.data, 0, 4, dp(xi), 0.0) == K.ERR_BAD_STATE
    e.close()
    # success: no covariances, no neighbour rows, as after set_source_cloud
    c.deskew_source(times, xi, 0.0)
    for get in (c.get_source_covariances, c.get_source_neighbors):
        with pytest.raises(K.VgicpError) as err:
            get()
        assert err.value.code == K.ERR_BAD_STATE
    c.close()


def test_append_then_deskew_appends_the_raw_source(pair02, relative_pose):
    tgt, src = pair02
    c = _core()
    _load_target(c, tgt)
    c.set_source_cloud(src)
    _covs(c)
    want = c.transform_source(relative_pose)
    rng = np.random.default_rng(12)
    times, xi = _times_and_twist(rng, len(src))
    c.append_source_to_target(relative_pose)
    c.deskew_source(times, xi, 0.0)
    c.swap_source_and_target()
    got = c.transform_source(np.eye(4))
    assert np.array_equal(got[len(tgt):], want)
    c.swap_source_and_target()
    assert np.array_equal(_source_points(c), deskew_f32(src, times, xi, 0.0))
    c.close()


# ------------------------------------------------------------------------------------------------------------ effect
def test_distorted_pair_matches_oracle_and_gate():
    from fast_gicp_b200.core import pose_from_c

    tgt, src, ts, T_gt = distorted_pair()
    for deskew in (False, True):
        c = _core()
        _load_target(c, tgt)
        c.set_source_cloud(src)
        if deskew:
            c.deskew_source(ts, EFFECT_TWIST, 0.0)
        _covs(c)
        r = c.align()
        T = pose_from_c(r.T)
        ref = O.register_f32(tgt, deskew_f32(src, ts, EFFECT_TWIST, 0.0) if deskew else src, method=O.DIRECT7, accum_double=True)
        dt, dr = pose_error(ref.T, T)
        assert r.converged and dt < 1e-4 and dr < 1e-5, (deskew, dt, dr)
        gt_t, gt_r = pose_error(T_gt, T)
        assert (gt_t < 0.05 and gt_r < np.radians(1.0)) == deskew, (deskew, gt_t, np.degrees(gt_r))
        c.close()


# ------------------------------------------------------------------------------------------------------------ surfaces
def test_python_mirror_and_pygicp_equal_the_core_route():
    from fast_gicp_b200 import FastVGICPCuda
    from fast_gicp_b200.core import pose_from_c

    tgt, src, ts, _ = distorted_pair()
    a = _core("DIRECT1")
    _load_target(a, tgt)
    a.set_source_cloud(src)
    a.deskew_source(ts, EFFECT_TWIST, 0.0)
    _covs(a)
    reg = FastVGICPCuda()
    reg.setNeighborSearchMethod("DIRECT1")
    want = pose_from_c(a.align(np.eye(4), reg._params()).T).astype(np.float32)
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    reg.deskewSource(ts, EFFECT_TWIST, 0.0)
    got = reg.align()
    assert np.array_equal(got, want)
    reg.setInputSource(src)  # the device source is the deskewed cloud: this reloads the raw one
    assert np.array_equal(reg.vgicp_cuda_.transform_source(np.eye(4)), src)
    a.close()

    if LIB not in sys.path:
        sys.path.insert(0, LIB)
    import pygicp

    p = pygicp.FastVGICPCuda()
    p.set_neighbor_search_method("DIRECT1", 1.5)
    p.set_input_target(tgt.astype(np.float64))
    p.set_input_source(src.astype(np.float64))
    p.deskew_source(ts, EFFECT_TWIST, 0.0)
    assert np.array_equal(p.align(), want)
