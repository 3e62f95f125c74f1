"""Multi-source alignment (vgicp_align_sources): B source clouds against one target map.  Stage 1 runs source by source on the
library's own k-NN and covariance kernels; the optimisers share their evaluation launches, each source a row of blocks with its own
single-pose grid.  So every result must equal set_source_cloud + find_source_neighbors + calculate_source_covariances + align on
the same handle, bit for bit."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle as O
from conftest import random_pose

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("nr_iterations", "converged", "n_linearize", "n_compute_error", "lm_failed")
STAGE1 = ("unpack_points", "knn", "covariance")


def test_null_handle_is_rejected():
    """The entry point refuses a null handle before it touches the device (runs without a GPU)."""
    from fast_gicp_b200 import core

    lib = core.load_library()
    xyz = (C.c_void_p * 1)(None)
    n = (C.c_size_t * 1)(100)
    res = (core.AlignResult * 1)()
    assert lib.vgicp_align_sources(None, xyz, n, 12, 0, 20, O.REG_PLANE, None, 1, None, res) == core.ERR_INVALID_ARGUMENT


def assert_same(a, b, what=""):
    assert np.array_equal(np.array(a.T), np.array(b.T)), what
    assert np.array_equal(np.array(a.H), np.array(b.H)), what
    assert tuple(getattr(a, f) for f in FIELDS) == tuple(getattr(b, f) for f in FIELDS), what


def make_core(tgt, method=O.DIRECT7, radius=-1.0, hint=0, spec=1, index=0, robust=None, res=1.0):
    from fast_gicp_b200.core import Core

    c = Core(0)
    c.set_execution_hint(hint)
    c.set_speculation(spec)
    c.set_voxel_index(index)
    c.set_resolution(res)
    c.set_neighbor_search_method(method, radius)
    if robust:
        c.set_robust_kernel(*robust)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()
    return c


def sources_and_guesses(src, relative_pose, seed=0):
    """Five sources of different sizes (subsets of the fixture source) and a guess near the truth for each."""
    rng = np.random.default_rng(seed)
    S = [src, src[::2].copy(), src[1::3].copy(), src[: len(src) // 2].copy(), src[::5].copy()]
    G = np.stack([relative_pose @ random_pose(rng, 0.08, 0.4) for _ in S])
    return S, G


def loop(c, sources, G, k=20, reg=O.REG_PLANE, params=None):
    out = []
    for s, g in zip(sources, G):
        c.set_source_cloud(s)
        c.find_source_neighbors(k)
        c.calculate_source_covariances(reg)
        out.append(c.align(g, params))
    return out


def launches(c):
    return {name: cnt for name, (_, cnt) in c.get_profile().items()}


def delta(a, b):
    return {k: b[k] - a[k] for k in a}


CASES = {
    "direct1": dict(method=O.DIRECT1),
    "direct7": dict(method=O.DIRECT7),
    "direct27": dict(method=O.DIRECT27),
    "radius": dict(method=O.DIRECT_RADIUS, radius=1.5),
    "hash_table_direct27": dict(method=O.DIRECT27, index=1),
    "hash_table_radius": dict(method=O.DIRECT_RADIUS, radius=1.5, index=1),
    "huber_direct7": dict(method=O.DIRECT7, robust=("HUBER", 1.0)),
    "cauchy_hash_direct1": dict(method=O.DIRECT1, robust=("CAUCHY", 2.0), index=1),
    "gauss_newton": dict(method=O.DIRECT7, gn=1),
    "lm_no_speculation": dict(method=O.DIRECT27, spec=0),
    "throughput_hint": dict(method=O.DIRECT7, hint=1),
    "throughput_no_speculation_huber": dict(method=O.DIRECT1, hint=1, spec=0, robust=("HUBER", 1.0)),
    "normalized_min_eig": dict(method=O.DIRECT7, reg=O.REG_NORMALIZED_MIN_EIG),
    "min_eig_k10": dict(method=O.DIRECT7, reg=O.REG_MIN_EIG, k=10),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_bit_identical_to_the_loop(pair02, relative_pose, case):
    from fast_gicp_b200.core import default_params

    cfg = CASES[case]
    tgt, src = pair02
    c = make_core(tgt, method=cfg["method"], radius=cfg.get("radius", -1.0), hint=cfg.get("hint", 0), spec=cfg.get("spec", 1), index=cfg.get("index", 0),
                  robust=cfg.get("robust"))
    params = default_params(use_gauss_newton=cfg.get("gn", 0))
    k, reg = cfg.get("k", 20), cfg.get("reg", O.REG_PLANE)
    S, G = sources_and_guesses(src, relative_pose)
    res = c.align_sources(S, G, k=k, reg=reg, params=params)
    assert len(res) == len(S)
    ref = loop(c, S, G, k, reg, params)
    for i in range(len(S)):
        assert_same(res[i], ref[i], f"{case} source {i}")
    assert sum(r.converged for r in res) >= 4
    c.close()


@pytest.fixture(scope="module")
def large_pair():
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
    return tgt, src, T_gt


@pytest.mark.gpu
@pytest.mark.parametrize("method", [O.DIRECT1, O.DIRECT7])
def test_mixed_launch_classes(large_pair, method):
    """Sources below and above the DIRECT1 streaming threshold (65 536 points) and one past the G = 1 threshold (400 000 points):
    a round issues one launch per class present, and every result still equals the loop's."""
    from fast_gicp_b200.core import default_params

    tgt, src, T_gt = large_pair
    c = make_core(tgt, method=method, res=0.5)
    rng = np.random.default_rng(7)
    sizes = [20_000, 50_000, 70_000, 150_000, 450_000]
    S = [src[rng.permutation(len(src))[:n]].copy() for n in sizes]
    G = np.stack([T_gt @ random_pose(rng, 0.05, 0.4) for _ in S])
    params = default_params()
    c.synchronize()
    p0 = launches(c)
    res = c.align_sources(S, G, params=params)
    d = delta(p0, launches(c))
    ref = loop(c, S, G, params=params)
    for i in range(len(S)):
        assert_same(res[i], ref[i], f"method {method} source {i}")
    # LM with speculation: per class, one linearisation launch and then one trial launch per round while one of its sources runs
    thr = 65536 if method == O.DIRECT1 else 400000
    classes = {}
    for n, r in zip(sizes, res):
        classes.setdefault(n >= thr, []).append(1 + r.n_compute_error)
    assert len(classes) == 2
    assert d["linearize"] + d["compute_error"] == sum(max(v) for v in classes.values())
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("gn", [0, 1])
def test_launches_are_batched(pair02, relative_pose, gn):
    """One class: evaluation launches = rounds, not the sum over sources; stage 1 launches = those of the loop."""
    from fast_gicp_b200.core import default_params

    tgt, src = pair02
    c = make_core(tgt, method=O.DIRECT27)
    params = default_params(use_gauss_newton=gn)
    rng = np.random.default_rng(3)
    S = [src[rng.permutation(len(src))[: len(src) - 500 * j]].copy() for j in range(8)]
    G = np.stack([relative_pose @ random_pose(rng, 0.1, 0.5) for _ in S])
    c.synchronize()
    p0 = launches(c)
    res = c.align_sources(S, G, params=params)
    p1 = launches(c)
    ref = loop(c, S, G, params=params)
    p2 = launches(c)
    d, dl = delta(p0, p1), delta(p1, p2)
    evals = d["linearize"] + d["compute_error"]
    want = max(r.n_linearize for r in res) if gn else max(1 + r.n_compute_error for r in res)
    assert evals == want
    assert evals < (dl["linearize"] + dl["compute_error"]) / 2
    for cat in STAGE1:
        assert d[cat] == dl[cat] and d[cat] > 0, cat
    assert d["voxelmap_build"] == 0
    for i in range(len(S)):
        assert_same(res[i], ref[i], f"source {i}")
    c.close()


@pytest.mark.gpu
def test_handle_state_is_undisturbed(pair02, relative_pose):
    from fast_gicp_b200.core import Core

    tgt, src = pair02
    c = make_core(tgt, method=O.DIRECT7)
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)
    t = np.linspace(0.0, 0.1, len(src), dtype=np.float32)
    c.set_source_timestamps(t, 0.05)
    cov0, nbr0 = c.get_source_covariances(), c.get_source_neighbors()
    xi = np.array([0.0, 0.0, 0.3, 1.0, 0.0, 0.0])
    ct0 = c.compute_error_ct(relative_pose, xi, relative_pose, xi)
    T_prev = relative_pose @ random_pose(np.random.default_rng(2), 0.05, 0.2)
    c.update_correspondences(T_prev)
    pairs0 = c.get_voxel_correspondences()
    e0, H0, b0 = c.compute_error(T_prev, True)
    S, G = sources_and_guesses(src[::-1].copy(), relative_pose, seed=5)
    c.align_sources(S, G)
    assert c.num_source_points() == len(src)
    assert np.array_equal(c.get_source_covariances().view(np.uint32), cov0.view(np.uint32))
    assert np.array_equal(c.get_source_neighbors(), nbr0)
    ct1 = c.compute_error_ct(relative_pose, xi, relative_pose, xi)
    assert ct1[0] == ct0[0] and np.array_equal(ct1[1], ct0[1]) and np.array_equal(ct1[2], ct0[2])
    assert np.array_equal(c.get_voxel_correspondences(), pairs0)
    e1, H1, b1 = c.compute_error(T_prev, True)
    assert e1 == e0 and np.array_equal(H1, H0) and np.array_equal(b1, b0)
    fresh = make_core(tgt, method=O.DIRECT7)
    fresh.set_source_cloud(src)
    fresh.find_source_neighbors(20)
    fresh.calculate_source_covariances(O.REG_PLANE)
    for g in G[:3]:
        assert_same(c.align(g), fresh.align(g))
    for a, b in zip(c.align_multi(G), fresh.align_multi(G)):
        assert_same(a, b)
    fresh.close()
    c.close()


@pytest.mark.gpu
def test_inputs_host_device_and_strides(pair02, relative_pose):
    import torch

    tgt, src = pair02
    c = make_core(tgt, method=O.DIRECT7)
    S, G = sources_and_guesses(src, relative_pose, seed=1)
    ref = c.align_sources(S, G)  # packed xyz, stride 12
    for width in (4, 8):  # strides 16 and 32
        W = [np.concatenate([s, np.full((len(s), width - 3), 7.0, np.float32)], axis=1) for s in S]
        for r, q in zip(c.align_sources(W, G), ref):
            assert_same(r, q, f"stride {4 * width}")
        dev = [torch.from_numpy(w).cuda() for w in W]
        torch.cuda.synchronize()
        res = c.align_sources_raw([d.data_ptr() for d in dev], [len(s) for s in S], 4 * width, True, guesses=G)
        for r, q in zip(res, ref):
            assert_same(r, q, f"device, stride {4 * width}")
    dev = [torch.from_numpy(s).cuda() for s in S]
    torch.cuda.synchronize()
    for r, q in zip(c.align_sources_raw([d.data_ptr() for d in dev], [len(s) for s in S], 12, True, guesses=G), ref):
        assert_same(r, q, "device, stride 12")
    # NULL guesses = identity guesses
    I = np.tile(np.eye(4), (len(S), 1, 1))
    for r, q in zip(c.align_sources(S), c.align_sources(S, I)):
        assert_same(r, q, "identity")
    # the pool shrinks and grows between calls without changing results
    assert_same(c.align_sources(S[4:], G[4:])[0], ref[4])
    for r, q in zip(c.align_sources(S[::-1], G[::-1]), ref[::-1]):
        assert_same(r, q, "reversed")
    c.close()


@pytest.mark.gpu
def test_errors_launch_nothing(pair02):
    from fast_gicp_b200.core import AlignResult, Core, ERR_BAD_STATE, ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED

    tgt, src = pair02
    B = 4097
    pts = [src[: 1000 + j].copy() for j in range(4)]
    P = (C.c_void_p * B)(*([p.ctypes.data for p in pts] * (B // 4 + 1))[:B])
    N = (C.c_size_t * B)(*([len(p) for p in pts] * (B // 4 + 1))[:B])
    G = np.tile(np.eye(4).reshape(16), B)
    gp = G.ctypes.data_as(C.POINTER(C.c_double))
    res = (AlignResult * B)()

    def call(c, xyz=P, n=N, stride=12, k=20, reg=O.REG_PLANE, guesses=gp, b=4, out=res, h=None):
        return c._lib.vgicp_align_sources(c._h if h is None else h, xyz, n, stride, 0, k, reg, guesses, b, None, out)

    # no voxel map yet: the state error
    c = Core(0)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    n0 = c.launch_count()
    assert call(c) == ERR_BAD_STATE and c.launch_count() == n0
    c.create_target_voxelmap()
    assert call(c, b=1) == 0  # (settles the map build)
    n0 = c.launch_count()
    nullp = (C.c_void_p * 4)(P[0], None, P[2], P[3])
    small = (C.c_size_t * 4)(1000, 1001, 10, 1003)
    huge = (C.c_size_t * 4)(1000, 1001, 1 << 26, 1003)
    bad = [
        call(c, h=C.c_void_p(0)), call(c, xyz=None), call(c, n=None), call(c, out=None), call(c, b=0), call(c, b=B), call(c, b=-2),
        call(c, stride=8), call(c, stride=14), call(c, k=0), call(c, k=65), call(c, n=small), call(c, n=huge), call(c, xyz=nullp),
        call(c, reg=5), call(c, reg=-1),
    ]
    assert bad == [ERR_INVALID_ARGUMENT] * len(bad)
    assert c.launch_count() == n0
    # sharding: unsupported, nothing launched
    c.set_source_shard(0, 500)
    assert call(c) == ERR_UNSUPPORTED and c.launch_count() == n0
    c.clear_source_shard()
    c.set_stage1_sharding(True)
    assert call(c) == ERR_UNSUPPORTED and c.launch_count() == n0
    c.set_stage1_sharding(False)
    # NDT: unsupported
    c.set_problem(2)
    assert call(c) == ERR_UNSUPPORTED and c.launch_count() == n0
    c.set_problem(0)
    # the largest batch is accepted; NULL guesses are the identity
    assert call(c, b=B - 1, guesses=None) == 0
    assert all(np.array_equal(np.array(res[i].T), np.array(res[i % 4].T)) for i in range(B - 1))
    c.close()


@pytest.mark.gpu
def test_communicator_handle_is_unsupported():
    """A handle in a multi-GPU communicator refuses the call with VGICP_ERR_UNSUPPORTED and launches nothing (two GPUs)."""
    import subprocess

    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_multi_gpu import _free_port

    port = _free_port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "align_sources_comm_worker.py")], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.PIPE, text=True))
    for p in procs:
        o, e = p.communicate(timeout=600)
        assert p.returncode == 0, e[-3000:]
        assert o.strip().splitlines()[-1] == "unsupported ok"


# ------------------------------------------------------------------------------------------------------ public surfaces
def _pygicp():
    lib = os.path.join(ROOT, "fast_gicp_b200", "lib")
    if lib not in sys.path:
        sys.path.insert(0, lib)
    import pygicp

    return pygicp


@pytest.mark.gpu
def test_surfaces(pair02, relative_pose):
    import fast_gicp_b200 as F
    from fast_gicp_b200.registration import NearestNeighborMethod

    tgt, src = pair02
    S, G = sources_and_guesses(src, relative_pose, seed=2)

    # Python class: align_sources(S, G)[i] == setInputSource(S[i]) + align(G[i]); the input source and the single state stay
    reg = F.FastVGICPCuda()
    reg.setNeighborSearchMethod("DIRECT27")
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    T_s, conv_s = reg.align_sources(S, G)
    assert T_s.dtype == np.float32 and T_s.shape == (len(S), 4, 4) and conv_s.dtype == bool and conv_s.sum() >= 4
    assert np.array_equal(reg.getFinalTransformation(), np.eye(4, dtype=np.float32)) and not reg.hasConverged()
    T_src = reg.align(G[0])
    for i, s in enumerate(S):
        reg.setInputSource(s)
        assert np.array_equal(reg.align(G[i]), T_s[i]) and reg.hasConverged() == conv_s[i], i
    reg.setInputSource(src)
    assert np.array_equal(reg.align(G[0]), T_src)
    rbf = F.FastVGICPCuda()
    rbf.setNearestNeighborSearchMethod(NearestNeighborMethod.GPU_RBF_KERNEL)
    rbf.setInputTarget(tgt)
    with pytest.raises(RuntimeError, match="RBF"):
        rbf.align_sources(S, G)

    # pygicp (the C++ mirror's alignSources): the same device results; its align (the mirror's own LM loop) agrees to rounding
    pg = _pygicp().FastVGICPCuda()
    pg.set_neighbor_search_method("DIRECT27", 0.0)
    pg.set_input_target(tgt.astype(np.float64))
    T_pg, conv_pg = pg.align_sources([s.astype(np.float64) for s in S], G.astype(np.float32))
    assert np.array_equal(T_pg, T_s) and np.array_equal(conv_pg, conv_s)
    T_id, _ = pg.align_sources([s.astype(np.float64) for s in S[:2]])
    T_py_id, _ = reg.align_sources(S[:2])
    assert np.array_equal(T_id, T_py_id)
    from conftest import pose_error

    for i, s in enumerate(S):
        pg.set_input_source(s.astype(np.float64))
        T = pg.align(G[i].astype(np.float32))
        assert pg.has_converged() == conv_s[i], i
        dt, dr = pose_error(T_s[i], T)
        assert dt < 1e-6 and dr < 1e-7, (i, dt, dr)
