"""The host model of vgicp_thin_target (synthetic.thin_indices) against the rule spelled as a plain loop: row i is kept iff fewer
than M earlier rows share its cell, cells c = floor(p * (1 / (float)leaf)) in float32.  CPU only."""
import numpy as np
import pytest

from fast_gicp_b200.synthetic import thin_indices


def loop_model(pts, leaf, M):
    inv = np.float32(1.0) / np.float32(leaf)
    counts, keep = {}, []
    for i, p in enumerate(np.asarray(pts, dtype=np.float32)):
        cell = tuple(int(np.floor(np.float32(p[a]) * inv)) for a in range(3))
        if counts.get(cell, 0) < M:
            keep.append(i)
        counts[cell] = counts.get(cell, 0) + 1
    return np.array(keep, dtype=np.int64)


def check(pts, leaf, M):
    got = thin_indices(pts, leaf, M)
    want = loop_model(pts, leaf, M)
    assert np.array_equal(got, want)
    return got


@pytest.mark.parametrize("seed,n,extent,leaf,M", [(0, 2000, 5.0, 0.5, 1), (1, 3000, 20.0, 0.5, 4), (2, 5000, 3.0, 0.25, 2), (3, 1500, 100.0, 1.0, 8),
                                                  (4, 4000, 2.0, 0.5, 20)])
def test_random_clouds(seed, n, extent, leaf, M):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-extent, extent, size=(n, 3)).astype(np.float32)
    keep = check(pts, leaf, M)
    assert 0 < len(keep) <= n


def test_boundaries_negatives_and_signed_zero():
    leaf = 0.5
    vals = np.array([0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 0.49999997, -0.49999997, 0.50000006, -1e-30, 1e-30], dtype=np.float32)
    grid = np.array(np.meshgrid(vals, vals, vals, indexing="ij")).reshape(3, -1).T
    pts = np.vstack([grid, grid[::-1], grid])
    for M in (1, 2, 3):
        keep = check(pts, leaf, M)
        # -0.0 and +0.0 share cell 0; -1e-30 lies in cell -1
        assert len(keep) < len(pts)


def test_product_rounding_onto_an_integer():
    """p * inv rounds up onto an integer in float32 though p / leaf in exact arithmetic lies just below it."""
    leaf = np.float32(0.1)
    inv = np.float32(1.0) / leaf
    # find float32 values p with p < k * leaf exactly but fl(p * inv) == k
    cands = []
    for k in range(1, 200):
        p = np.nextafter(np.float32(k) * leaf, np.float32(0))
        if float(p) < k * float(leaf) and np.floor(p * inv) == k:
            cands.append(p)
    assert cands, "no rounding case found"
    c = np.array(cands, dtype=np.float32)
    pts = np.stack([c, np.zeros_like(c), np.zeros_like(c)], axis=1)
    pts = np.vstack([pts, pts + np.float32(0.0)])
    check(pts, float(leaf), 1)
    # the model uses the float32 product, not the double quotient
    inv64 = np.floor(c.astype(np.float64) / np.float64(leaf))
    assert np.any(np.floor(c * inv) != inv64)


def test_M_one_M_large_and_one_cell():
    rng = np.random.default_rng(9)
    pts = rng.uniform(-3, 3, size=(1000, 3)).astype(np.float32)
    one = check(pts, 1.0, 1)
    assert len(one) == len(np.unique(np.floor(pts * np.float32(1.0)), axis=0))
    assert np.array_equal(check(pts, 1.0, 1000), np.arange(len(pts)))
    same = rng.uniform(0.1, 0.9, size=(50, 3)).astype(np.float32)
    assert np.array_equal(check(same, 1.0, 7), np.arange(7))
    assert np.array_equal(check(same, 1.0, 50), np.arange(50))
    assert np.array_equal(check(same[:1], 1.0, 1), [0])


def test_known_answer():
    pts = np.array([[0.1, 0.1, 0.1],    # cell (0,0,0): 1st
                    [1.2, 0.0, 0.0],    # cell (1,0,0): 1st
                    [0.9, 0.9, 0.9],    # (0,0,0): 2nd
                    [-0.1, 0.0, 0.0],   # (-1,0,0): 1st
                    [0.5, 0.5, 0.5],    # (0,0,0): 3rd -> dropped at M = 2
                    [1.0, 0.99, 0.0],   # (1,0,0): 2nd
                    [1.5, 0.5, 0.5],    # (1,0,0): 3rd -> dropped at M = 2
                    [0.0, -0.0, 0.0]],  # (0,0,0): 4th -> dropped at M = 2
                   dtype=np.float32)
    assert check(pts, 1.0, 2).tolist() == [0, 1, 2, 3, 5]
    assert check(pts, 1.0, 1).tolist() == [0, 1, 3]
    assert check(pts, 1.0, 3).tolist() == [0, 1, 2, 3, 4, 5, 6]


def test_null_handle_is_refused():
    from fast_gicp_b200 import core

    lib = core.load_library()
    assert lib.vgicp_thin_target(None, 0.5, 2) == core.ERR_INVALID_ARGUMENT
