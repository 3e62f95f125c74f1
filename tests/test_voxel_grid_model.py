"""pcl::VoxelGrid, the exact grid with per-point fields (vgicp_prep_voxel_grid), on the CPU: its C checker (oracle_fields
orc_voxel_grid_fields) against a numpy float32 restatement of the recipe in include/vgicp_prep_b200.h, byte for byte; a hand-built
known answer; the float64 exact grid synthetic.voxel_downsample_values at power-of-two leaves; input permutations; and the refusal
edges (cell range, cell product, far coordinates)."""
import os

import numpy as np
import pytest

import oracle_fields as OF
from fast_gicp_b200 import synthetic as syn
from test_gpu_timestamped_scans import as_floats, raw_sweep
from test_input_prep import raw_like_cloud
from test_prep_fields import records

F32 = np.float32
INT32_MAX = 2**31 - 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def restate(rec, leaf, cols, remove_near_origin=False):
    """The recipe in numpy float32 -> (centroids of every voxel in ascending index, their counts, their indices).  Sums run in
    input order (numpy's own float32 reductions are pairwise, so the adds are done one point per voxel per round); raises
    OF.Refused where the device refuses the cloud."""
    r = np.ascontiguousarray(rec, dtype=F32)
    cols = list(cols)
    R = 3 + len(cols)
    x, y, z = r[:, 0], r[:, 1], r[:, 2]
    with np.errstate(over="ignore", invalid="ignore"):
        keep = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
        if remove_near_origin:
            keep &= ~(((x * x + y * y) + z * z) < F32(1e-3))
        src = np.flatnonzero(keep)
        c = np.floor(r[src, :3] * (F32(1.0) / F32(leaf)))
    if len(src) == 0:
        return np.zeros((0, R), F32), np.zeros(0, np.int64), np.zeros(0, np.int64)
    if not ((c >= -2.0**31) & (c < 2.0**31)).all():
        raise OF.Refused("cell outside the int range")
    g = c.astype(np.int64)
    lo, div = g.min(axis=0), g.max(axis=0) - g.min(axis=0) + 1
    if int(div[0]) * int(div[1]) * int(div[2]) > INT32_MAX:
        raise OF.Refused("more than INT32_MAX cells")
    idx = (g[:, 0] - lo[0]) + (g[:, 1] - lo[1]) * div[0] + (g[:, 2] - lo[2]) * div[0] * div[1]
    order = np.argsort(idx, kind="stable")  # stable: input order inside a voxel
    idx_s = idx[order]
    starts = np.flatnonzero(np.r_[True, idx_s[1:] != idx_s[:-1]])
    counts = np.diff(np.r_[starts, len(idx_s)])
    vals = r[src[order]][:, [0, 1, 2] + cols]
    # round k adds the k-th point of every voxel holding more than k points: s = 0.0f, then s = s + v in order
    by_size = np.argsort(-counts, kind="stable")
    st, sc = starts[by_size], counts[by_size]
    acc = np.zeros((len(starts), R), F32)
    for k in range(int(sc[0])):
        a = int(np.count_nonzero(sc > k))
        acc[:a] = acc[:a] + vals[st[:a] + k]
    sums = np.empty_like(acc)
    sums[by_size] = acc
    return sums / counts.astype(F32)[:, None], counts, idx_s[starts]


def restated(rec, leaf, cols, remove_near_origin=False, min_points=0):
    out, counts, _ = restate(rec, leaf, cols, remove_near_origin)
    return out[counts >= min_points]


_SWEEP = []


def sweep_records():
    """The raw distorted sweep (64 x 2083 rays, about 124.5 k points) as 11-float records: x y z, time, intensity, 6 noise columns."""
    if not _SWEEP:
        rec, _ = raw_sweep()
        f = as_floats(rec)
        r = records(f[:, :3], 8, 3)
        r[:, 3], r[:, 4] = f[:, 4], f[:, 3]
        _SWEEP.append(r)
    return _SWEEP[0]


def cloud(name):
    return sweep_records() if name == "sweep" else records(raw_like_cloud(31, 40000), 8, 31)


COLS8 = [3, 4, 5, 6, 7, 8, 9, 10]


@pytest.mark.parametrize("flt", [False, True])
@pytest.mark.parametrize("leaf", [0.1, 0.25, 1.0])
@pytest.mark.parametrize("name", ["raw_like", "sweep"])
def test_checker_equals_the_numpy_restatement(name, leaf, flt):
    rec = cloud(name)
    out, counts, _ = restate(rec, leaf, COLS8, flt)
    assert counts.sum() == len(rec) - (np.count_nonzero(((rec[:, 0] * rec[:, 0] + rec[:, 1] * rec[:, 1]) + rec[:, 2] * rec[:, 2]) < F32(1e-3)) if flt else 0)
    for nf, cols in ((0, []), (1, [3]), (2, [4, 3]), (8, COLS8)):
        sel = [0, 1, 2] + [COLS8.index(c) + 3 for c in cols]
        for mp in (0, 1, 3):
            got = OF.voxel_grid_fields(rec, leaf, cols, flt, mp)
            want = out[counts >= mp][:, sel]
            assert got.shape == want.shape and got.tobytes() == want.tobytes(), (nf, mp)


def test_known_answer():
    """A dozen points at leaf 0.5: negative coordinates, points exactly on leaf multiples, a NaN and an inf point, two near-origin
    points, a duplicate, a lone point that min_points drops, and a NaN field value that propagates."""
    P = [(-0.5, -0.5, 0.0, 1.0),    # a  cell (-1, -1, 0), on leaf multiples
         (-0.25, -0.1, 0.4, 2.0),   # b  (-1, -1, 0)
         (0.0, 0.0, 0.0, 100.0),    # c  (0, 0, 0), near the origin
         (0.01, 0.01, 0.01, 200.0),  # d  (0, 0, 0), near the origin (3e-4 < 1e-3)
         (0.5, 0.0, 0.0, 3.0),      # e  (1, 0, 0), on leaf multiples
         (np.nan, 1.0, 1.0, 7.0),   # dropped: not finite
         (0.75, 0.25, 0.25, 4.0),   # f  (1, 0, 0)
         (1.0, np.inf, 1.0, 7.0),   # dropped: not finite
         (0.9, 0.4, 0.1, np.nan),   # g  (1, 0, 0), a NaN field
         (1.0, 1.0, -1.0, 5.0),     # j  (2, 2, -2), alone
         (-0.5, -0.5, 0.0, 6.0)]    # k  (-1, -1, 0), a's duplicate
    rec = np.array(P, F32)
    # box: x -1..2, y -1..2, z -2..0 -> div (4, 4, 3); idx j = 3 + 3*4 + 0 = 15, a/b/k = 0 + 0 + 2*16 = 32, c/d = 1 + 4 + 32 = 37,
    # e/f/g = 2 + 4 + 32 = 38
    r = rec

    def cen(*rows):
        s = np.zeros(4, F32)
        for i in rows:
            s = s + r[i]
        return s / F32(len(rows))

    abk, cd, efg, j = cen(0, 1, 10), cen(2, 3), cen(4, 6, 8), r[9]
    assert np.isnan(efg[3]) and abk[0] == F32(np.float32(-1.25) / F32(3))
    cases = {(False, 0): [j, abk, cd, efg], (True, 0): [j, abk, efg], (False, 2): [abk, cd, efg], (True, 2): [abk, efg], (True, 3): [abk, efg],
             (False, 4): []}
    for (flt, mp), want in cases.items():
        want = np.array(want, F32).reshape(-1, 4)
        for got in (OF.voxel_grid_fields(rec, 0.5, [3], flt, mp), restated(rec, 0.5, [3], flt, mp)):
            assert got.tobytes() == want.tobytes(), (flt, mp, got, want)
    _, counts, idx = restate(rec, 0.5, [3])
    assert idx.tolist() == [15, 32, 37, 38] and counts.tolist() == [1, 3, 2, 3]
    # no kept point: the empty result
    assert OF.voxel_grid_fields(rec[[2, 3, 5, 7]], 0.5, [3], True).shape == (0, 4)
    assert OF.voxel_grid_fields(rec[:0], 0.5, [3]).shape == (0, 4)


@pytest.mark.parametrize("leaf", [0.25, 0.5, 1.0])
def test_power_of_two_leaves_agree_with_the_float64_exact_grid(leaf):
    """At a power-of-two leaf x * (1 / leaf) is x / leaf exactly, so synthetic.voxel_downsample_values (float64 sums, division by
    the leaf) has the same voxels in the same order; its centroids agree within the float32 error of in-order sums."""
    pts = raw_like_cloud(77, 40000)
    rec = records(pts, 1, 77)
    got = OF.voxel_grid_fields(rec, leaf, [3])
    ref_p, ref_v = syn.voxel_downsample_values(pts, rec[:, 3], leaf)
    assert got.shape == (len(ref_p), 4)
    _, counts, _ = restate(rec, leaf, [3])
    u = 2.0**-24
    gamma = (counts - 1) * u / (1 - (counts - 1) * u)
    for want, g, mag in ((ref_p, got[:, :3], leaf + np.abs(ref_p)), (ref_v[:, None], got[:, 3:], np.full((len(counts), 1), 200.0))):
        # |fl(sum) - sum| <= gamma_{c-1} sum|v|, then one division and the float64 reference's own rounding, each <= u |result|
        bound = gamma[:, None] * mag + 2 * u * np.abs(want) + 1e-30
        assert (np.abs(g.astype(np.float64) - want.astype(np.float64)) <= bound).all()
    # the same voxels: every output centroid lies in the cell of the voxel the float64 grid put at that rank
    cells = np.floor(ref_p.astype(np.float64) / leaf)
    assert (np.floor(got[:, :3].astype(np.float64) / leaf) == cells).all()


def test_a_permuted_input_gives_the_same_voxels_and_counts():
    rec = records(raw_like_cloud(5, 20000), 2, 5)
    perm = np.random.default_rng(0).permutation(len(rec))
    for leaf, flt in ((0.1, True), (0.25, False), (1.0, True)):
        a, ca, ia = restate(rec, leaf, [3, 4], flt)
        b, cb, ib = restate(rec[perm], leaf, [3, 4], flt)
        assert np.array_equal(ia, ib) and np.array_equal(ca, cb)
        assert np.allclose(a, b, rtol=1e-5, atol=1e-4)
        for mp in (0, 3):
            assert OF.voxel_grid_fields(rec[perm], leaf, [3, 4], flt, mp).tobytes() == restated(rec[perm], leaf, [3, 4], flt, mp).tobytes()


def test_refusal_edges():
    # 1290^3 = 2 146 689 000 cells (<= INT32_MAX) is accepted; 1291 x 1290 x 1290 = 2 148 353 100 is refused
    ok = np.array([[0.25, 0.25, 0.25], [1289.5, 1289.5, 1289.5]], F32)
    got = OF.voxel_grid_fields(ok, 1.0, [])
    assert got.tobytes() == ok.tobytes() and got.tobytes() == restated(ok, 1.0, []).tobytes()
    _, _, idx = restate(ok, 1.0, [])
    assert idx.tolist() == [0, 1290**3 - 1]
    over = ok.copy()
    over[1, 0] = 1290.5
    for f in (lambda: OF.voxel_grid_fields(over, 1.0, []), lambda: restate(over, 1.0, [])):
        with pytest.raises(OF.Refused):
            f()
    # a coordinate at x / leaf = 2^31 is refused; -2^31 is the lowest cell and is accepted
    far = np.array([[2.0**31, 0.0, 0.0], [1.0, 0.0, 0.0]], F32)
    with pytest.raises(OF.Refused):
        OF.voxel_grid_fields(far, 1.0, [])
    low = np.array([[-(2.0**31), 0.0, 0.0]], F32)
    assert OF.voxel_grid_fields(low, 1.0, []).tobytes() == low.tobytes()
    # a leaf that is not finite and positive is a bad argument
    for leaf in (0.0, -1.0, np.inf, np.nan):
        with pytest.raises(ValueError):
            OF.voxel_grid_fields(ok, leaf, [])
    # 1e5 m from the origin at leaf 0.005 (|x / leaf| = 2e7 > 2^24): integer indices, in range, equal to the restatement
    rng = np.random.default_rng(3)
    p = (np.array([1e5, -1e5, 50.0]) + rng.uniform(-2.0, 2.0, (5000, 3))).astype(F32)
    rec = records(p, 1, 3)
    got = OF.voxel_grid_fields(rec, 0.005, [3])
    out, counts, idx = restate(rec, 0.005, [3])
    assert got.tobytes() == out.tobytes() and idx.max() < INT32_MAX and counts.sum() == len(p)


def test_the_product_never_imports_the_checker():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "fast_gicp_b200")):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".hpp")):
                assert "oracle_fields" not in open(os.path.join(dirpath, f), errors="replace").read(), f
