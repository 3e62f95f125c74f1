"""pcl::ApproximateVoxelGrid<PointT> with per-point float fields (vgicp_prep_approximate_voxel_grid_fields), on the CPU.

The C restatement (oracle_fields) against a Python serial restatement; its x y z against orc_approximate_voxel_grid's bytes; and
the formulation the CUDA kernels implement with fields -- 512 independent history chains walked in tiles of 2048 points, tile-local
lists filled in arbitrary order and sorted back, the scan fallback for more than 16 matches of one entry in a tile, flushed field
centroids stored at the index of the flushing point, the held ones in entry order -- against the serial filter."""
import numpy as np
import pytest

import oracle as O
import oracle_fields as OF
from test_input_prep import kCap, kHist, kTile, raw_like_cloud

F32 = np.float32


def records(pts, n_fields, seed, stride_f=None):
    """(n, stride_f) float32 records: x y z, then n_fields fields (a time ramp, then uniform noise), then padding."""
    rng = np.random.default_rng(seed)
    n = len(pts)
    stride_f = stride_f or 3 + n_fields
    r = np.zeros((n, stride_f), dtype=F32)
    r[:, :3] = pts
    if n_fields:
        r[:, 3] = np.linspace(0.0, 0.1, n, dtype=F32)
    if n_fields > 1:
        r[:, 4:3 + n_fields] = rng.uniform(-50.0, 200.0, (n, n_fields - 1)).astype(F32)
    return r


def serial_fields(rec, leaf, cols, remove_near_origin):
    """The serial filter restated in Python float32 scalars: every field summed in input order next to x y z, one division by
    (float)count at each flush, the held voxels in entry order at the end."""
    inv = F32(1.0) / F32(leaf)
    hist = [None] * 512
    out = []

    def emit(e):
        c = F32(e["count"])
        out.append([e["s"][j] / c for j in range(len(e["s"]))])

    for r in rec:
        x, y, z = r[0], r[1], r[2]
        if remove_near_origin and (x * x + y * y) + z * z < F32(1e-3):
            continue
        key = (int(np.floor(x * inv)), int(np.floor(y * inv)), int(np.floor(z * inv)))
        h = (key[0] * 7171 + key[1] * 3079 + key[2] * 4231) & 511
        e = hist[h]
        if e is not None and e["count"] and e["key"] != key:
            emit(e)
            e = None
        if e is None or not e["count"]:
            e = hist[h] = {"key": key, "count": 0, "s": [F32(0.0)] * (3 + len(cols))}
        e["key"] = key
        e["count"] += 1
        vals = [x, y, z] + [r[c] for c in cols]
        e["s"] = [F32(e["s"][j] + vals[j]) for j in range(len(vals))]
    for e in hist:
        if e is not None and e["count"]:
            emit(e)
    return np.asarray(out, dtype=F32).reshape(-1, 3 + len(cols))


def walk_kernel_fields(rec, leaf, cols, flt, seed=0):
    """k_prep_walk<F> / k_prep_scatter<F> / k_prep_tail<F> restated step by step (test_input_prep.emulate_walk_kernel with fields)."""
    rng = np.random.default_rng(seed)
    p = rec[:, :3].astype(F32)
    fv = rec[:, cols].astype(F32) if len(cols) else np.zeros((len(rec), 0), F32)
    n, nf = len(p), len(cols)
    inv = F32(1.0) / F32(leaf)
    ijk = np.floor(p * inv).astype(np.int64)
    ent = ((ijk[:, 0] * 7171 + ijk[:, 1] * 3079 + ijk[:, 2] * 4231) & 511).astype(np.int64)
    if flt:
        sq = (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]
        ent = np.where(sq < F32(1e-3), 0xFFFF, ent)
    flushed = np.zeros((n, 4), F32)     # xyz + flag, at the flushing point's index
    fflushed = np.zeros((n, nf), F32)   # the side array of field centroids, same index
    E = [dict(k=None, c=0, s=np.zeros(3, F32), f=np.zeros(nf, F32)) for _ in range(kHist)]

    def step(e, i):
        k = tuple(ijk[i])
        if e["c"] and e["k"] != k:
            c = F32(e["c"])
            flushed[i, :3] = e["s"] / c
            flushed[i, 3] = 1
            fflushed[i] = e["f"] / c
            e["c"] = 0
            e["s"] = np.zeros(3, F32)
            e["f"] = np.zeros(nf, F32)
        e["k"] = k
        e["c"] += 1
        e["s"] = e["s"] + p[i]
        e["f"] = e["f"] + fv[i]

    for base in range(0, n, kTile):
        cnt = np.zeros(kHist, int)
        lst = np.full((kHist, kCap), -1, int)
        sh = np.full(kTile, 0xFFFF, int)
        for j in rng.permutation(kTile):  # arbitrary arrival order of the shared-memory atomics
            i = base + j
            t = ent[i] if i < n else 0xFFFF
            sh[j] = t
            if t != 0xFFFF:
                q = cnt[t]
                cnt[t] += 1
                if q < kCap:
                    lst[t, q] = j
        for h in range(kHist):
            c = cnt[h]
            if 0 < c <= kCap:
                for j in sorted(lst[h, :c]):
                    step(E[h], base + j)
            elif c > kCap:
                for j in range(kTile):
                    if sh[j] == h:
                        step(E[h], base + j)
    out = [np.concatenate([flushed[i, :3], fflushed[i]]) for i in range(n) if flushed[i, 3] != 0]
    for h in range(kHist):
        if E[h]["c"]:
            c = F32(E[h]["c"])
            out.append(np.concatenate([E[h]["s"] / c, E[h]["f"] / c]))
    return np.asarray(out, F32).reshape(-1, 3 + nf)


@pytest.mark.parametrize("n,leaf,nf,flt", [(1, 0.25, 1, False), (700, 0.1, 2, True), (3000, 0.25, 1, False), (3000, 1.0, 3, True)])
def test_oracle_equals_the_python_serial_restatement(n, leaf, nf, flt):
    rec = records(raw_like_cloud(n + 11, n), nf, n)
    cols = list(range(3, 3 + nf))
    got = OF.approximate_voxel_grid_fields(rec, leaf, cols, flt)
    want = serial_fields(rec, leaf, cols, flt)
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.parametrize("nf,stride_f", [(1, 4), (2, 8), (8, 12)])
@pytest.mark.parametrize("flt", [False, True])
def test_oracle_xyz_equal_the_xyz_filter(nf, stride_f, flt):
    pts = raw_like_cloud(21, 20000)
    rec = records(pts, nf, 5, stride_f)
    # fields in reverse column order, padding behind them: the xyz bytes do not depend on which columns are averaged
    cols = list(range(3 + nf - 1, 2, -1))
    got = OF.approximate_voxel_grid_fields(rec, 0.25, cols, flt)
    want = O.approximate_voxel_grid(O.remove_near_origin(pts) if flt else pts, 0.25)
    assert np.array_equal(got[:, :3], want)
    # and a field equal to a coordinate column averages to that coordinate's bytes
    rec[:, 3] = rec[:, 0]
    assert np.array_equal(OF.approximate_voxel_grid_fields(rec, 0.25, [3], flt)[:, 3], want[:, 0])


def test_oracle_rejects_bad_columns():
    rec = records(raw_like_cloud(1, 100), 1, 1)
    for cols in ([2], [4], list(range(3, 3 + 9))):
        with pytest.raises(ValueError):
            OF.approximate_voxel_grid_fields(rec, 0.25, cols)


@pytest.mark.parametrize("n,leaf,nf,flt", [(2048, 1.0, 1, False), (9000, 0.1, 2, True), (9000, 0.25, 8, False)])
def test_walk_kernel_bookkeeping_with_fields_equals_the_serial_filter(n, leaf, nf, flt):
    c = raw_like_cloud(n + 7, n)  # n = 9000 holds both the origin run and a > 16-point run of one entry (scan fallback)
    rec = records(c, nf, n)
    cols = list(range(3, 3 + nf))
    want = OF.approximate_voxel_grid_fields(rec, leaf, cols, flt)
    assert np.array_equal(walk_kernel_fields(rec, leaf, cols, flt), want)
