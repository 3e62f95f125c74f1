"""The exact grid on the device (vgicp_prep_voxel_grid, pcl::VoxelGrid with per-point fields) against its C checker
(oracle_fields.voxel_grid_fields), bit for bit, at the sizes, strides, field counts and key widths that change the code path; its
refusals; pygicp.voxel_grid; and the exact grid's device output driving the continuous-time registration exactly as the same
arrays given through the host calls.  The prep calls run in a child process, as test_input_prep does: a fault there cannot poison
the CUDA context of the other GPU tests."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
import oracle_fields as OF
from test_gpu_timestamped_scans import as_floats, raw_sweep, same_ct, target_only
from test_deskew_model import distorted_pair
from test_input_prep import raw_like_cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
SENTINEL = F32(-12345.5)


def with_fields(pts, stride_f, seed):
    """(n, stride_f) float32 records: x y z, then uniform noise with a few NaN and inf field values."""
    rng = np.random.default_rng(seed)
    r = np.zeros((len(pts), stride_f), F32)
    r[:, :3] = pts
    r[:, 3:] = rng.uniform(-1.0, 100.0, (len(pts), stride_f - 3)).astype(F32)
    if stride_f > 3 and len(pts) > 100:
        r[rng.choice(len(pts), 3, replace=False), stride_f - 1] = [np.nan, np.inf, -np.inf]
    return r


def same(got, want):
    """Bit for bit, except that a NaN is any NaN: the device's float adds return the canonical NaN where the host's keep an
    operand's payload (the recipe says that non-finite values propagate, not which NaN results)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape or not np.array_equal(np.isnan(got), np.isnan(want)):
        return False
    ok = ~np.isnan(want)
    return got[ok].tobytes() == want[ok].tobytes()


def box_cloud(div, n, seed):
    """Points in a box of exactly div cells at leaf 1 (a point at both corners), some NaN and inf points: the key widths 9, 18, 27
    and 31 bits (1, 2, 3 and 4 sort passes) with the dropped points' key V = div_x * div_y * div_z."""
    rng = np.random.default_rng(seed)
    d = np.asarray(div)
    p = (np.floor(rng.uniform(0, 1, (n, 3)) * d) + rng.uniform(0.1, 0.9, (n, 3))).astype(F32)
    p[0], p[1] = 0.5, d - 0.5
    p[2, 0], p[3, 1], p[4, 2] = np.nan, np.inf, -np.inf
    return p


def _child():
    import torch

    from fast_gicp_b200.prep import InputPrep, PrepError

    p = InputPrep(0)
    cases = 0

    def check(rec, leaf, cols, flt, mp, what):
        nonlocal cases
        rec = np.ascontiguousarray(rec, dtype=F32)
        n, k = rec.shape
        want = OF.voxel_grid_fields(rec, leaf, cols, flt, mp)
        R = 3 + len(cols)
        offs = [4 * c for c in cols]
        got = p.voxel_grid(rec, leaf, cols, mp, flt)  # host in, host out
        assert same(got, want), what
        d = torch.from_numpy(rec).cuda()
        got = p.voxel_grid(d, leaf, cols, mp, flt)  # device in, device out
        assert got.is_cuda and same(got.cpu().numpy(), want), what
        out = np.full((max(n, 1), R), SENTINEL, F32)  # device in, host out
        m = p._run_voxel_grid(d.data_ptr(), n, 4 * k, 1, leaf, flt, offs, mp, out.ctypes.data, n, 0)
        assert same(out[:m], want) and (out[m:] == SENTINEL).all(), what
        dout = torch.full((max(n, 1), R), float(SENTINEL), device="cuda")  # host in, device out
        m = p._run_voxel_grid(rec.ctypes.data, n, 4 * k, 0, leaf, flt, offs, mp, dout.data_ptr(), n, 1)
        dout = dout.cpu().numpy()
        assert same(dout[:m], want) and (dout[m:] == SENTINEL).all(), what
        cases += 1
        return want

    # sizes around the 2048-key sort tile, a scan, the raw sweep and 1 M points; strides 12, 16, 32, 48 bytes with F = 0, 1, 2, 8
    for n in (1, 2, 2047, 2048, 2049, 40000, 1000000):
        pts = raw_like_cloud(n + 5, n)
        for stride_f, cols in ((3, []), (4, [3]), (8, [7, 4]), (12, [11, 3, 4, 5, 6, 7, 8, 9])):
            rec = with_fields(pts, stride_f, n)
            for leaf, flt, mp in ((0.1, True, 0), (0.25, False, 3), (1.0, True, 1)):
                if n == 1000000 and leaf == 0.1 and stride_f != 12:
                    continue
                check(rec, leaf, cols, flt, mp, (n, stride_f, leaf, flt, mp))
    sweep, _ = raw_sweep()
    want = check(as_floats(sweep), 0.25, [4, 3], True, 0, "sweep")
    assert p.voxel_grid(sweep, 0.25, ["time", "intensity"], remove_near_origin=True).tobytes() == want.tobytes()  # structured array
    for mp in (2, 5):
        check(as_floats(sweep), 0.1, [4, 3, 5], False, mp, ("sweep", mp))
    # 1, 2, 3 and 4 sort passes
    for div in ((8, 8, 7), (64, 64, 63), (512, 512, 511), (1290, 1290, 1290)):
        check(with_fields(box_cloud(div, 40000, div[0]), 5, 1), 1.0, [3, 4], False, 0, div)
    # one voxel holding 200 k points (and a few NaN / inf ones)
    rng = np.random.default_rng(9)
    one = rng.uniform(0.01, 0.24, (200000, 3)).astype(F32)
    one[7], one[11] = np.nan, np.inf
    check(with_fields(one, 6, 9), 0.25, [3, 5], False, 0, "one voxel")
    check(with_fields(one, 6, 9), 0.25, [3, 5], False, 200001, "one voxel below the minimum")
    # every point dropped: the near-origin filter, non-finite coordinates
    zero = np.zeros((5000, 4), F32)
    zero[::3, 0] = np.nan
    check(zero, 0.25, [3], True, 0, "all dropped")
    assert p.voxel_grid(zero[:, :3].copy(), 0.25, remove_near_origin=False).shape == (1, 3)
    # n = 0, host and device
    assert p.voxel_grid(np.zeros((0, 4), F32), 0.25, [3]).shape == (0, 4)
    assert tuple(p.voxel_grid(torch.zeros((0, 4), device="cuda"), 0.25, [3]).shape) == (0, 4)

    # refusals: status 1, *n_out = 0 (m when only the capacity is short), out untouched
    L, C = p._lib, __import__("ctypes")
    rec = with_fields(raw_like_cloud(3, 3000), 4, 3)
    n = len(rec)
    m_ok = len(OF.voxel_grid_fields(rec, 0.25, [3]))
    hout = np.full((n, 4), SENTINEL, F32)
    dout = torch.full((n, 4), float(SENTINEL), device="cuda")
    drec = torch.from_numpy(rec).cuda()
    ok_box = np.array([[0.25, 0.25, 0.25, 1.0], [1289.5, 1289.5, 1289.5, 2.0]], F32)
    over_box = ok_box.copy()
    over_box[1, 0] = 1290.5
    far = np.array([[2.0**31, 0.0, 0.0, 1.0], [1.0, 0.0, 0.0, 1.0]], F32)
    assert len(p.voxel_grid(ok_box, 1.0, [3])) == 2

    def refused(src, on_dev, stride, leaf, offs, nf, cap, n_out_expected, npts=None):
        for out, out_dev in ((hout, 0), (dout, 1)):
            off = (C.c_size_t * 9)(*offs) if offs is not None else None
            m = C.c_size_t(77)
            ptr = out.ctypes.data if out_dev == 0 else out.data_ptr()
            rc = L.vgicp_prep_voxel_grid(p._h, src, npts if npts is not None else n, stride, on_dev, C.c_float(leaf), 0, off, nf, 0, ptr, cap, out_dev, C.byref(m))
            assert rc == 1 and m.value == n_out_expected, (rc, m.value)
        assert (hout == SENTINEL).all() and bool((dout == float(SENTINEL)).all())

    for on_dev, src in ((0, rec.ctypes.data), (1, drec.data_ptr())):
        refused(src, on_dev, 14, 0.25, [12], 1, n, 0)       # stride not a multiple of 4
        refused(src, on_dev, 8, 0.25, [], 0, n, 0)          # stride < 12
        refused(src, on_dev, 16, 0.25, [10], 1, n, 0)       # offset not a multiple of 4
        refused(src, on_dev, 16, 0.25, [8], 1, n, 0)        # offset inside x y z
        refused(src, on_dev, 16, 0.25, [16], 1, n, 0)       # offset beyond the stride
        refused(src, on_dev, 16, 0.25, [12] * 9, 9, n, 0)   # nine fields
        refused(src, on_dev, 16, 0.25, None, 1, n, 0)       # null field offsets
        refused(src, on_dev, 16, 0.25, [12], -1, n, 0)      # negative field count
        for leaf in (0.0, -0.25, float("inf"), float("nan")):
            refused(src, on_dev, 16, leaf, [12], 1, n, 0)
        refused(src, on_dev, 16, 0.25, [12], 1, m_ok - 1, m_ok)  # capacity one short
        refused(src, on_dev, 16, 0.25, [12], 1, n, 0, npts=2**31 - 4096 + 1)  # too many points
    refused(None, 0, 16, 0.25, [12], 1, n, 0)  # null input
    for bad in (over_box, far):
        dbad = torch.from_numpy(bad).cuda()
        refused(bad.ctypes.data, 0, 16, 1.0, [12], 1, n, 0, npts=2)
        refused(dbad.data_ptr(), 1, 16, 1.0, [12], 1, n, 0, npts=2)
        try:
            p.voxel_grid(bad, 1.0, [3])
        except PrepError as e:
            assert e.code == 1
        else:
            raise AssertionError("refused cloud accepted")
    m = C.c_size_t(0)
    assert L.vgicp_prep_voxel_grid(p._h, rec.ctypes.data, n, 16, 0, C.c_float(0.25), 0, None, 0, 0, hout.ctypes.data, n, 0, None) == 1  # null n_out
    assert L.vgicp_prep_voxel_grid(p._h, rec.ctypes.data, n, 16, 0, C.c_float(0.25), 0, None, 0, 0, None, n, 0, C.byref(m)) == 1  # null out
    assert L.vgicp_prep_voxel_grid(None, rec.ctypes.data, n, 16, 0, C.c_float(0.25), 0, None, 0, 0, hout.ctypes.data, n, 0, C.byref(m)) == 1  # null handle
    assert (hout == SENTINEL).all()
    # and the context still works after every refusal
    check(rec, 0.25, [3], True, 0, "after the refusals")
    print(f"voxel grid ok: {cases} cases")


@pytest.mark.gpu
def test_gpu_voxel_grid_matches_the_checker_bit_for_bit():
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_gpu_voxel_grid as t; t._child()"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "voxel grid ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_pygicp_voxel_grid_returns_the_checkers_records():
    lib = os.path.join(ROOT, "fast_gicp_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import pygicp

    f = as_floats(raw_sweep()[0])
    for cols, mp in (([], 0), ([4, 3], 0), ([4, 3], 3)):
        assert pygicp.voxel_grid(f, 0.25, cols, mp).tobytes() == OF.voxel_grid_fields(f, 0.25, cols, False, mp).tobytes()
    assert pygicp.voxel_grid(f, 0.5).tobytes() == OF.voxel_grid_fields(f, 0.5, []).tobytes()


def test_end_to_end_exact_grid_on_the_device_equals_the_host_calls():
    """Raw sweep -> the exact grid on the device with time and intensity -> set_source_cloud_device + set_source_timestamps_device
    -> covariances -> align_ct -> deskew_source_stored, against the same pipeline fed the checker's arrays through the host calls:
    bit for bit."""
    import torch

    from fast_gicp_b200.prep import InputPrep

    tgt = distorted_pair()[0]
    rec, _ = raw_sweep()
    p = InputPrep(0)
    out = p.voxel_grid(torch.from_numpy(as_floats(rec)).cuda(), 0.25, [4, 3], remove_near_origin=True)
    torch.cuda.synchronize()
    ref = OF.voxel_grid_fields(as_floats(rec), 0.25, [4, 3], True)
    assert out.cpu().numpy().tobytes() == ref.tobytes()
    m, stride = ref.shape[0], 4 * ref.shape[1]
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
    p.close()
