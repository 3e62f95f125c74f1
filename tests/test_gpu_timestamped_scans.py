"""Timestamped scans on the device: the voxel grid with per-point fields (vgicp_prep_approximate_voxel_grid_fields), source
timestamps read from device memory (vgicp_set_source_timestamps_device) and the deskew with the stored timestamps
(vgicp_deskew_source_stored), each held bit for bit to a path already trusted: the C restatement of the serial filter
(oracle_fields), vgicp_set_source_timestamps and vgicp_deskew_source.  The prep part runs in a child process, as
test_input_prep does: a fault there cannot poison the CUDA context of the other GPU tests."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
import oracle_fields as OF
from test_deskew_model import EFFECT_POSE, EFFECT_TWIST, distorted_pair, syn
from test_gpu_multi_hypothesis import setup
from test_input_prep import raw_like_cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
XYZIT = np.dtype([("x", np.float32), ("y", np.float32), ("z", np.float32), ("intensity", np.float32), ("time", np.float32), ("ring", np.float32),
                  ("pad", np.float32, 2)])  # a 32-byte PointXYZIT-like record
COUNTERS = ("nr_iterations", "converged", "n_linearize", "n_compute_error", "lm_failed")
METHODS = {"DIRECT1": O.DIRECT1, "DIRECT7": O.DIRECT7, "DIRECT27": O.DIRECT27}


def raw_sweep(seed=42):
    """A raw distorted sweep (64 x 2083 rays) as PointXYZIT-like records with a synthetic intensity, and the sensor pose at t = 0."""
    world = syn._make_world(np.random.default_rng(seed))
    yaw = np.radians(EFFECT_POSE[2])
    T = np.eye(4)
    T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
    T[:3, 3] = [EFFECT_POSE[0], EFFECT_POSE[1], 0.0]
    pts, times = syn.distorted_scan(world, 64, 2083, T, EFFECT_TWIST, 0.1, np.random.default_rng(seed + 1))
    rec = np.zeros(len(pts), dtype=XYZIT)
    rec["x"], rec["y"], rec["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    rec["time"] = times
    rng = np.random.default_rng(seed + 2)
    rec["intensity"] = (200.0 / (1.0 + np.linalg.norm(pts, axis=1)) + rng.uniform(0.0, 5.0, len(pts))).astype(np.float32)
    return rec, T


def as_floats(rec):
    return rec.view(np.float32).reshape(len(rec), -1)


# ------------------------------------------------------------------------------------------------------------------ prep
def _prep_child():
    import torch

    from fast_gicp_b200.prep import InputPrep

    p = InputPrep(0)

    def check(rec, leaf, cols, flt, what):
        want = OF.approximate_voxel_grid_fields(rec, leaf, cols, flt)
        xyz = p.approximate_voxel_grid(np.ascontiguousarray(rec[:, :3]), leaf, flt)
        assert np.array_equal(want[:, :3], xyz), what  # the oracle's xyz are the existing entry's bytes
        got_h = p.approximate_voxel_grid_fields(rec, leaf, cols, flt)  # host in, host out
        assert got_h.shape == want.shape and np.array_equal(got_h, want), what
        d = torch.from_numpy(rec).cuda()
        got_d = p.approximate_voxel_grid_fields(d, leaf, cols, flt)  # device in, device out
        assert got_d.is_cuda and np.array_equal(got_d.cpu().numpy(), want), what
        # device in, host out and host in, device out: the C entry point with the other two combinations
        out = np.empty((len(rec), 3 + len(cols)), dtype=np.float32)
        m = p._run_fields(d.data_ptr(), len(rec), rec.strides[0], 1, leaf, flt, [4 * c for c in cols], out.ctypes.data, len(rec), 0)
        assert np.array_equal(out[:m], want), what
        dout = torch.empty((max(len(rec), 1), 3 + len(cols)), dtype=torch.float32, device="cuda")
        m = p._run_fields(rec.ctypes.data, len(rec), rec.strides[0], 0, leaf, flt, [4 * c for c in cols], dout.data_ptr(), len(rec), 1)
        assert np.array_equal(dout[:m].cpu().numpy(), want), what
        return want

    cases = 0
    for n in (1, 3000, 9000, 40000):  # 3000, 9000, 40000: not multiples of the 2048-point tile; 9000 and 40000 hold the origin run
        pts = raw_like_cloud(n + 3, n)  # and a > 16-point run of one entry
        rng = np.random.default_rng(n)
        for nf, stride_f in ((1, 4), (2, 8), (8, 12)):  # strides 16, 32, 48 bytes
            rec = np.zeros((n, stride_f), dtype=np.float32)
            rec[:, :3] = pts
            rec[:, 3:] = rng.uniform(-1.0, 100.0, (n, stride_f - 3)).astype(np.float32)
            cols = list(range(stride_f - 1, stride_f - 1 - nf, -1))  # the last nf columns, in reverse order
            for leaf, flt in ((0.1, True), (0.25, False), (1.0, True)):
                check(rec, leaf, cols, flt, (n, nf, stride_f, leaf, flt))
                cases += 1
    # n = 0, host and device
    assert p.approximate_voxel_grid_fields(np.zeros((0, 4), np.float32), 0.25, [3]).shape == (0, 4)
    assert tuple(p.approximate_voxel_grid_fields(torch.zeros((0, 4), device="cuda"), 0.25, [3]).shape) == (0, 4)
    # a raw distorted sweep as 32-byte records: time and intensity, from the structured array and from its float view
    rec, _ = raw_sweep()
    want = check(as_floats(rec), 0.25, [4, 3], True, "sweep")
    assert np.array_equal(p.approximate_voxel_grid_fields(rec, 0.25, ["time", "intensity"], True), want)
    # bad arguments
    for cols in ([2], [8], list(range(3, 12))):
        try:
            p.approximate_voxel_grid_fields(as_floats(rec), 0.25, cols)
        except Exception as e:
            assert getattr(e, "code", None) == 1, e
        else:
            raise AssertionError(f"columns {cols} accepted")
    print(f"prep fields ok: {cases} cases")


@pytest.mark.gpu
def test_gpu_prep_with_fields_matches_the_oracle_bit_for_bit():
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_gpu_timestamped_scans as t; t._prep_child()"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "prep fields ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------------------------ timestamps
def core():
    from fast_gicp_b200.core import Core

    return Core(0)


def target_only(tgt):
    """A handle with the target, its covariances and voxel map as setup() makes them, and no source yet."""
    c = core()
    c.set_resolution(1.0)
    c.set_neighbor_search_method(O.DIRECT7)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()
    return c


def same_ct(a, b, what):
    for f in ("T", "twist", "H"):
        assert np.array_equal(np.array(getattr(a, f)), np.array(getattr(b, f))), (what, f)
    assert tuple(getattr(a, f) for f in COUNTERS) == tuple(getattr(b, f) for f in COUNTERS), what


@pytest.fixture(scope="module")
def scan():
    """The clean target, the sweep's device prep output (x y z time intensity, a torch CUDA tensor), its host copy, and the pose."""
    import torch

    from fast_gicp_b200.prep import InputPrep

    tgt = distorted_pair()[0]
    rec, T = raw_sweep()
    p = InputPrep(0)
    out = p.approximate_voxel_grid_fields(torch.from_numpy(as_floats(rec)).cuda(), 0.25, [4, 3], True)
    torch.cuda.synchronize()
    yield tgt, out, out.cpu().numpy(), T
    p.close()


def test_device_timestamps_equal_host_timestamps(scan):
    """Two handles on the same scan, one given the host timestamps, one reading the prep output's time column in place: the same
    compute_error_ct (err, H, b) and align_ct (T, twist, H, counters) bytes."""
    tgt, out, host, T = scan
    m, stride = len(host), host.strides[0]
    a = setup(core(), tgt, np.ascontiguousarray(host[:, :3]))
    b = setup(core(), tgt, np.ascontiguousarray(host[:, :3]))
    a.set_source_timestamps(np.ascontiguousarray(host[:, 3]), 0.05)
    b.set_source_timestamps_device(out.data_ptr() + 12, m, stride, 0.05)
    xi = EFFECT_TWIST * 0.9
    T2 = T @ O.se3_exp(np.array([0.002, -0.001, 0.003, 0.03, 0.02, -0.01]))
    for name, method in METHODS.items():
        for k in ("NONE", "CAUCHY"):
            for c in (a, b):
                c.set_neighbor_search_method(method)
                c.set_robust_kernel(k, 1.0)
            for args in ((T, xi, T, xi), (T, np.zeros(6), T2, xi)):
                ea, Ha, ba = a.compute_error_ct(*args)
                eb, Hb, bb = b.compute_error_ct(*args)
                assert ea == eb and np.array_equal(Ha, Hb) and np.array_equal(ba, bb), (name, k)
            W = np.full(6, 1e-3)
            same_ct(a.align_ct(np.eye(4), EFFECT_TWIST * 0.5, EFFECT_TWIST * 0.5, W), b.align_ct(np.eye(4), EFFECT_TWIST * 0.5, EFFECT_TWIST * 0.5, W), (name, k))
    a.close()
    b.close()


def test_device_timestamp_errors(scan):
    import torch

    from fast_gicp_b200.core import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, VgicpError

    tgt, out, host, T = scan
    m, stride = len(host), host.strides[0]
    c = setup(core(), tgt, np.ascontiguousarray(host[:, :3]))
    c.set_neighbor_search_method(O.DIRECT7)
    c.set_source_timestamps_device(out.data_ptr() + 12, m, stride, 0.0)
    args = (T, EFFECT_TWIST * 0.5, T, EFFECT_TWIST)
    ref = c.compute_error_ct(*args)

    def code(fn, *a, launches=0):
        n0 = c.launch_count()
        with pytest.raises(VgicpError) as e:
            fn(*a)
        assert c.launch_count() == n0 + launches, "an error path launched an unexpected number of kernels"
        return e.value.code

    # found by the kernel (one launch, the gather): the previous timestamps stay in place
    for bad in (np.nan, np.inf, -np.inf):
        t = torch.from_numpy(np.ascontiguousarray(host[:, 3])).cuda()
        t[m // 2] = bad
        assert code(c.set_source_timestamps_device, t.data_ptr(), m, 4, 0.0, launches=1) == ERR_INVALID_ARGUMENT
        got = c.compute_error_ct(*args)
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
    # before any launch
    assert code(c.set_source_timestamps_device, out.data_ptr() + 12, m - 1, stride, 0.0) == ERR_INVALID_ARGUMENT
    assert code(c.set_source_timestamps_device, out.data_ptr() + 12, m, 2, 0.0) == ERR_INVALID_ARGUMENT
    assert code(c.set_source_timestamps_device, out.data_ptr() + 12, m, 18, 0.0) == ERR_INVALID_ARGUMENT
    assert code(c.set_source_timestamps_device, None, m, stride, 0.0) == ERR_INVALID_ARGUMENT
    assert code(c.set_source_timestamps_device, out.data_ptr() + 12, m, stride, 1e39) == ERR_INVALID_ARGUMENT
    got = c.compute_error_ct(*args)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1])
    # the stored deskew needs stored timestamps: a new source drops them
    c.set_source_cloud(np.ascontiguousarray(host[:, :3]))
    assert code(c.deskew_source_stored, EFFECT_TWIST) == ERR_BAD_STATE
    c.close()
    e = core()
    n0 = e.launch_count()
    with pytest.raises(VgicpError) as r:
        e.set_source_timestamps_device(out.data_ptr() + 12, m, stride, 0.0)
    assert r.value.code == ERR_BAD_STATE and e.launch_count() == n0
    with pytest.raises(VgicpError) as r:
        e.deskew_source_stored(EFFECT_TWIST)
    assert r.value.code == ERR_BAD_STATE and e.launch_count() == n0
    e.close()


@pytest.mark.parametrize("route", ["host", "device"])
def test_stored_deskew_equals_deskew_source(scan, route):
    """deskew_source_stored(xi) after set_source_timestamps(_device)(t, t_ref) against deskew_source(t, xi, t_ref): the same points
    (read back through transform_source(I)), then the same covariances, align and align_ct (the timestamps kept); both refuse the
    same twist beyond the series bound."""
    from fast_gicp_b200.core import ERR_INVALID_ARGUMENT, VgicpError

    tgt, out, host, T = scan
    m, stride = len(host), host.strides[0]
    src, ts = np.ascontiguousarray(host[:, :3]), np.ascontiguousarray(host[:, 3])
    t_ref = 0.05
    a = setup(core(), tgt, src)
    b = setup(core(), tgt, src)
    if route == "host":
        a.set_source_timestamps(ts, t_ref)
    else:
        a.set_source_timestamps_device(out.data_ptr() + 12, m, stride, t_ref)
    b.set_source_timestamps(ts, t_ref)
    bad = np.array([0.0, 0.0, 40.0, 0.0, 0.0, 0.0])  # 40 rad/s x 0.05 s > pi/2
    for c, call in ((a, lambda: a.deskew_source_stored(bad)), (b, lambda: b.deskew_source(ts, bad, t_ref))):
        n0 = c.launch_count()
        with pytest.raises(VgicpError) as e:
            call()
        assert e.value.code == ERR_INVALID_ARGUMENT and c.launch_count() == n0
    a.deskew_source_stored(EFFECT_TWIST)
    b.deskew_source(ts, EFFECT_TWIST, t_ref)
    pa, pb = a.transform_source(np.eye(4)), b.transform_source(np.eye(4))
    assert np.array_equal(pa, pb)
    assert not np.array_equal(pa, src)
    for c in (a, b):
        c.find_source_neighbors(20)
        c.calculate_source_covariances(O.REG_PLANE)
    assert np.array_equal(a.get_source_covariances(), b.get_source_covariances())
    ra, rb = a.align(np.eye(4)), b.align(np.eye(4))
    assert np.array_equal(np.array(ra.T), np.array(rb.T)) and np.array_equal(np.array(ra.H), np.array(rb.H))
    W = np.full(6, 1e-3)
    same_ct(a.align_ct(np.eye(4), np.zeros(6), np.zeros(6), W), b.align_ct(np.eye(4), np.zeros(6), np.zeros(6), W), route)
    # a second stored deskew works from the same timestamps (kept), as a second deskew_source would
    a.deskew_source_stored(EFFECT_TWIST * -0.1)
    b.deskew_source(ts, EFFECT_TWIST * -0.1, t_ref)
    assert np.array_equal(a.transform_source(np.eye(4)), b.transform_source(np.eye(4)))
    a.close()
    b.close()


def test_end_to_end_device_front_end_equals_the_host_calls(scan):
    """Raw sweep -> device prep with time and intensity -> set_source_cloud_device + set_source_timestamps_device -> covariances ->
    align_ct -> deskew_source_stored, against the same pipeline fed the oracle's arrays through the host calls: bit for bit."""
    tgt, out, host, T = scan
    rec, _ = raw_sweep()
    ref = OF.approximate_voxel_grid_fields(as_floats(rec), 0.25, [4, 3], True)
    assert np.array_equal(host, ref)
    m, stride = len(host), host.strides[0]
    W = np.full(6, 1e-3)
    d, h = target_only(tgt), target_only(tgt)
    d.set_cloud_device("source", out.data_ptr(), m, stride)
    d.set_source_timestamps_device(out.data_ptr() + 12, m, stride, 0.0)
    h.set_source_cloud(np.ascontiguousarray(ref[:, :3]))
    h.set_source_timestamps(np.ascontiguousarray(ref[:, 3]), 0.0)
    res = []
    for c in (d, h):
        c.find_source_neighbors(20)
        c.calculate_source_covariances(O.REG_PLANE)
        res.append(c.align_ct(np.eye(4), np.zeros(6), np.zeros(6), W))
    same_ct(res[0], res[1], "end to end")
    xi = np.array(res[0].twist)
    d.deskew_source_stored(xi)
    h.deskew_source(np.ascontiguousarray(ref[:, 3]), xi, 0.0)
    assert np.array_equal(d.transform_source(np.eye(4)), h.transform_source(np.eye(4)))
    d.close()
    h.close()


def test_python_class_cpp_mirror_and_pygicp():
    """FastVGICPCuda.deskewSourceStored (Python) and pygicp's deskew_source_stored (over the C++ mirror) register as deskewSource /
    deskew_source do in the same layer, bit for bit; pygicp.downsample_fields returns the oracle's records."""
    from fast_gicp_b200 import FastVGICPCuda

    tgt, src, ts, _ = distorted_pair()
    xi = EFFECT_TWIST * 0.9
    out = []
    for stored in (False, True):
        reg = FastVGICPCuda()
        reg.setNeighborSearchMethod("DIRECT7")
        reg.setInputTarget(tgt)
        reg.setInputSource(src)
        reg.setSourceTimestamps(ts, 0.02)
        if stored:
            reg.deskewSourceStored(xi)
        else:
            reg.deskewSource(ts, xi, 0.02)
        reg.align()
        out.append(reg.getFinalTransformation())
    assert np.array_equal(out[0], out[1])

    lib = os.path.join(ROOT, "fast_gicp_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import pygicp

    got = []
    for stored in (False, True):
        p = pygicp.FastVGICPCuda()
        p.set_neighbor_search_method("DIRECT7", 1.5)
        p.set_input_target(tgt.astype(np.float64))
        p.set_input_source(src.astype(np.float64))
        p.set_source_timestamps(ts, 0.02)
        if stored:
            p.deskew_source_stored(xi)
        else:
            p.deskew_source(ts, xi, 0.02)
        got.append(p.align(np.eye(4, dtype=np.float32)))
    assert np.array_equal(got[0], got[1])
    rec, _ = raw_sweep()
    f = as_floats(rec)
    assert np.array_equal(pygicp.downsample_fields(f, 0.25, [4, 3]), OF.approximate_voxel_grid_fields(f, 0.25, [4, 3]))
