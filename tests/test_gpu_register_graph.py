"""vgicp_register with resident clouds runs stage 1 (k-NN + covariances of both clouds, first voxel-map attempt) as one CUDA graph:
eager on the first call with a given shape, captured on the second, replayed after that.  Every call must return what the eager
path returns, byte for byte, and count the same kernel launches."""
import threading

import numpy as np
import pytest

from fast_gicp_b200.core import REG_PLANE, ROBUST_CAUCHY, ROBUST_NONE, Core

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def _handle(method, robust=ROBUST_NONE, res=1.0):
    c = Core(0)
    c.set_resolution(res)
    c.set_neighbor_search_method(method)
    if robust != ROBUST_NONE:
        c.set_robust_kernel(robust, 1.0)
    return c


def _state(c, r):
    """Everything a registration leaves behind, as bytes."""
    coords, ids = c.get_voxel_buckets()
    out = {"T": np.asarray(r.T), "H": np.asarray(r.H), "it": (r.nr_iterations, r.converged, r.n_linearize, r.n_compute_error),
           "buckets": coords, "ids": ids, "vox_n": c.get_voxel_num_points(), "vox_mean": c.get_voxel_means(), "vox_cov": c.get_voxel_covs(),
           "tcov": c.get_target_covariances(), "scov": c.get_source_covariances(), "tnbr": c.get_target_neighbors(), "snbr": c.get_source_neighbors()}
    return {k: (np.asarray(v).tobytes() if not isinstance(v, tuple) else v) for k, v in out.items()}


def _assert_same(a, b):
    for k in a:
        assert a[k] == b[k], k


def _resident(torch, pts):
    return torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).cuda()


def _register_dev(c, dt, ds):
    l0 = c.launch_count()
    r = c.register_raw(dt.data_ptr(), dt.shape[0], ds.data_ptr(), ds.shape[0], 12, True, 20, REG_PLANE)
    return r, c.launch_count() - l0


def _register_eager(c, tgt, src):
    """Host clouds: the eager path (no graph)."""
    l0 = c.launch_count()
    r = c.register(np.ascontiguousarray(tgt, np.float32), np.ascontiguousarray(src, np.float32), 20, REG_PLANE)
    return r, c.launch_count() - l0


def _moved(pts, yaw, t):
    R = np.array([[np.cos(yaw), -np.sin(yaw), 0.0], [np.sin(yaw), np.cos(yaw), 0.0], [0.0, 0.0, 1.0]])
    return (pts.astype(np.float64) @ R.T + t).astype(np.float32)


@pytest.mark.parametrize("pair", ["pair01", "pair02"])
@pytest.mark.parametrize("method,robust", [("DIRECT27", ROBUST_NONE), ("DIRECT7", ROBUST_NONE), ("DIRECT1", ROBUST_NONE), ("DIRECT27", ROBUST_CAUCHY)])
def test_graph_matches_eager(torch, request, pair, method, robust):
    tgt, src = request.getfixturevalue(pair)
    inputs = [(tgt, src), (_moved(tgt, 0.03, [0.2, -0.1, 0.0]), _moved(src, 0.03, [0.2, -0.1, 0.0])), (_moved(tgt, -0.02, [0.0, 0.3, 0.1]), src)]
    ref = _handle(method, robust)
    c = _handle(method, robust)
    # calls 1..4 on one handle: eager, captured, replayed, replayed -- each against the eager path on another handle
    for j in range(4):
        t, s = inputs[min(j, len(inputs) - 1)] if j < 3 else inputs[0]
        r_ref, n_ref = _register_eager(ref, t, s)
        r, n = _register_dev(c, _resident(torch, t), _resident(torch, s))
        _assert_same(_state(ref, r_ref), _state(c, r))
        assert n == n_ref, (j, n, n_ref)


def test_shape_change_rebuilds(torch, pair01):
    tgt, src = pair01
    shapes = [(tgt, src), (tgt[::2], src[::3]), (tgt, src), (tgt, src), (tgt[::2], src[::3]), (tgt[::2], src[::3]), (tgt[::2], src[::3]), (tgt, src)]
    ref = _handle("DIRECT27")
    c = _handle("DIRECT27")
    for t, s in shapes:
        r_ref, n_ref = _register_eager(ref, t, s)
        r, n = _register_dev(c, _resident(torch, t), _resident(torch, s))
        _assert_same(_state(ref, r_ref), _state(c, r))
        assert n == n_ref


def test_buffer_move_rebuilds(torch, pair01):
    """A crop exchanges the target's arrays: a graph captured before must not be replayed on the old ones."""
    tgt, src = pair01
    ref = _handle("DIRECT7")
    c = _handle("DIRECT7")
    dt, ds = _resident(torch, tgt), _resident(torch, src)
    for _ in range(3):
        _register_dev(c, dt, ds)
    c.crop_target([0.0, 0.0, 0.0], 1e4)
    r, _ = _register_dev(c, dt, ds)
    r_ref, _ = _register_eager(ref, tgt, src)
    _assert_same(_state(ref, r_ref), _state(c, r))


def test_table_growth_fallback(torch):
    """A cloud of 40 k points in distinct voxels needs more than the initial 8192 buckets: the graph enqueues the first attempt,
    the eager finish grows the table."""
    rng = np.random.default_rng(7)
    g = np.stack(np.meshgrid(np.arange(40), np.arange(40), np.arange(25), indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    tgt = (g + rng.uniform(0.2, 0.8, size=g.shape)).astype(np.float32)
    src = _moved(tgt, 0.01, [0.05, 0.02, 0.0])
    ref = _handle("DIRECT1")
    c = _handle("DIRECT1")
    for _ in range(3):
        r_ref, n_ref = _register_eager(ref, tgt, src)
        r, n = _register_dev(c, _resident(torch, tgt), _resident(torch, src))
        assert c.num_buckets() > 8192
        _assert_same(_state(ref, r_ref), _state(c, r))
        assert n == n_ref


def test_profiling_stays_eager(torch, pair02):
    tgt, src = pair02
    c = _handle("DIRECT7")
    dt, ds = _resident(torch, tgt), _resident(torch, src)
    for _ in range(3):
        _register_dev(c, dt, ds)
    c.set_profiling(True)
    _, n = _register_dev(c, dt, ds)
    prof = c.get_profile()
    c.set_profiling(False)
    ref = _handle("DIRECT7")
    ref.set_profiling(True)
    _, n_ref = _register_eager(ref, tgt, src)
    prof_ref = ref.get_profile()
    assert n == n_ref
    assert {k: v[1] for k, v in prof.items()} == {k: v[1] for k, v in prof_ref.items()}
    # events around the stage-1 launches: they ran eagerly
    assert prof["knn"][0] > 0 and prof["covariance"][0] > 0 and prof["voxelmap_build"][0] > 0


def test_concurrent_threads_match_sequential(torch, pair01):
    tgt, src = pair01
    S, per = 8, 4
    rng = np.random.default_rng(3)
    pairs = []
    for i in range(S * per):
        yaw, t = rng.uniform(-0.05, 0.05), rng.uniform(-0.5, 0.5, size=3)
        pairs.append((_moved(tgt, yaw, t), _moved(src, yaw, t)))
    ref = _handle("DIRECT27")
    expect = [_state(ref, _register_eager(ref, t, s)[0]) for t, s in pairs]
    dev = [(_resident(torch, t), _resident(torch, s)) for t, s in pairs]
    torch.cuda.synchronize()
    cores = [_handle("DIRECT27") for _ in range(S)]
    got = [None] * len(pairs)
    errors = []

    def work(ci):
        try:
            for j in range(per):
                i = ci + j * S
                r, _ = _register_dev(cores[ci], *dev[i])
                got[i] = _state(cores[ci], r)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=work, args=(ci,)) for ci in range(S)]
    for t_ in th:
        t_.start()
    for t_ in th:
        t_.join()
    assert not errors, errors
    for i in range(len(pairs)):
        _assert_same(expect[i], got[i])
