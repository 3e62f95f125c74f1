"""Multi-hypothesis alignment (vgicp_align_multi, vgicp_evaluate_poses): B registrations of one source against one map, the
evaluations of all running hypotheses sharing launches.  Each hypothesis is a row of blocks with the single-pose launch's grid and
the same fixed-order fold, so every result must equal the single-pose call bit for bit."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from conftest import pose_error, random_pose

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("nr_iterations", "converged", "n_linearize", "n_compute_error", "lm_failed")


def sym(c9):
    m = c9.reshape(-1, 3, 3)
    return (0.5 * (m + m.transpose(0, 2, 1))).reshape(-1, 9)


def guesses(relative_pose, seed=0):
    """24 initial guesses: identity, three near the truth, seventeen up to 30 deg / 2 m around it, a duplicate and a far one."""
    rng = np.random.default_rng(seed)
    G = [np.eye(4)]
    G += [relative_pose @ random_pose(rng, 0.05, 0.3) for _ in range(3)]
    G += [relative_pose @ random_pose(rng, np.radians(30.0), 2.0) for _ in range(17)]
    G.append(G[4].copy())
    far = np.eye(4)
    far[:3, :3] = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    far[:3, 3] = [9.0, -7.0, 1.5]
    G.append(far)
    return np.stack(G)


def setup(c, tgt, src, method=O.DIRECT7, radius=-1.0, problem=0, rbf=False, res=1.0):
    c.set_resolution(res)
    if problem:
        c.set_problem(problem)
        c.set_neighbor_search_method(method, radius)
        c.set_target_cloud(tgt)
        c.set_source_cloud(src)
        c.ndt_create_voxelmaps()
        return c
    c.set_neighbor_search_method(method, radius)
    c.set_target_cloud(tgt)
    if rbf:
        c.calculate_target_covariances_rbf(O.REG_PLANE)
    else:
        c.find_target_neighbors(20)
        c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()
    c.set_source_cloud(src)
    if rbf:
        c.calculate_source_covariances_rbf(O.REG_PLANE)
    else:
        c.find_source_neighbors(20)
        c.calculate_source_covariances(O.REG_PLANE)
    return c


def assert_same(a, b, what=""):
    assert np.array_equal(np.array(a.T), np.array(b.T)), what
    assert np.array_equal(np.array(a.H), np.array(b.H)), what
    assert tuple(getattr(a, f) for f in FIELDS) == tuple(getattr(b, f) for f in FIELDS), what


CASES = {
    "direct1": dict(method=O.DIRECT1),
    "direct7": dict(method=O.DIRECT7),
    "direct27": dict(method=O.DIRECT27),
    "radius": dict(method=O.DIRECT_RADIUS, radius=1.5),
    "lm_no_speculation": dict(method=O.DIRECT27, spec=0),
    "gauss_newton": dict(method=O.DIRECT7, gn=1),
    "throughput_hint": dict(method=O.DIRECT27, hint=1),
    "throughput_no_speculation": dict(method=O.DIRECT1, hint=1, spec=0),
    "hash_table": dict(method=O.DIRECT27, index=1),
    "hash_table_radius": dict(method=O.DIRECT_RADIUS, radius=1.5, index=1),
    "rbf": dict(method=O.DIRECT7, rbf=True),
    "ndt_p2d": dict(method=O.DIRECT7, problem=1),
    "ndt_d2d": dict(method=O.DIRECT7, problem=2),
    "ndt_d2d_direct1": dict(method=O.DIRECT1, problem=2, spec=0),
    "lm_no_trials": dict(method=O.DIRECT7, params=dict(lm_max_iterations=0)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_align_multi_is_bit_identical_to_align(pair02, relative_pose, case):
    from fast_gicp_b200.core import Core, default_params

    cfg = CASES[case]
    c = Core(0)
    c.set_execution_hint(cfg.get("hint", 0))
    c.set_speculation(cfg.get("spec", 1))
    c.set_voxel_index(cfg.get("index", 0))
    setup(c, *pair02, method=cfg["method"], radius=cfg.get("radius", -1.0), problem=cfg.get("problem", 0), rbf=cfg.get("rbf", False))
    params = default_params(use_gauss_newton=cfg.get("gn", 0), **cfg.get("params", {}))
    G = guesses(relative_pose)
    multi = c.align_multi(G, params)
    assert len(multi) == len(G)
    for i, g in enumerate(G):
        assert_same(multi[i], c.align(g, params), f"{case} guess {i}")
    assert_same(multi[4], multi[21])  # the duplicated guess
    if params.lm_max_iterations > 0:
        assert sum(r.converged for r in multi) >= 4
    else:  # step_lm tries no step: one linearisation each, then "lm not converged"
        assert all(r.lm_failed and r.n_linearize == 1 and r.n_compute_error == 0 for r in multi)
    c.close()


def test_align_multi_matches_the_oracle(pair02, relative_pose):
    """The hypotheses near the truth against the float oracle: same counters, pose within the north-star tolerance."""
    from fast_gicp_b200.core import Core, pose_from_c

    tgt, src = pair02
    t_cov = O.regularize(O.covariances(tgt, O.knn(tgt, 20, "kdtree")), O.REG_PLANE)
    s_cov = sym(O.regularize(O.covariances(src, O.knn(src, 20, "kdtree")), O.REG_PLANE)).astype(np.float32)
    vm = O.VoxelMap(tgt, sym(t_cov).astype(np.float32), 1.0, accum_double=True)
    G = guesses(relative_pose)[:4]
    for method in (O.DIRECT7, O.DIRECT27):
        c = setup(Core(0), tgt, src, method=method)
        multi = c.align_multi(G)
        for g, r in zip(G, multi):
            ref = O.align_f32(vm, src, s_cov, O.offsets(method), guess=g)
            assert r.converged and ref.converged
            assert (r.nr_iterations, r.n_linearize, r.n_compute_error) == (ref.iterations, ref.n_linearize, ref.n_error)
            dt, dr = pose_error(ref.T, pose_from_c(r.T))
            assert dt < 1e-4 and dr < 1e-5, (dt, dr)
        c.close()


def test_large_cloud_bit_identity():
    """C4-size pair (1 M points): DIRECT1 runs the bulk-copy streaming kernel, DIRECT27 the compacted one; B = 4."""
    from fast_gicp_b200.core import Core
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
    c = setup(Core(0), tgt, src, method=O.DIRECT27, res=0.5)
    rng = np.random.default_rng(4)
    G = np.stack([np.eye(4), T_gt] + [T_gt @ random_pose(rng, 0.1, 0.8) for _ in range(2)])
    for method in (O.DIRECT1, O.DIRECT27):
        c.set_neighbor_search_method(method)
        multi = c.align_multi(G)
        for i, g in enumerate(G):
            assert_same(multi[i], c.align(g), f"method {method} guess {i}")
        # the scoring primitive on the same kernels (hit counts included)
        err, H, b, n_corr = c.evaluate_poses(G[:2], want_H=True)
        for i in range(2):
            c.update_correspondences(G[i])
            e1, H1, b1 = c.compute_error(G[i], True)
            assert err[i] == e1 and np.array_equal(H[i], H1) and np.array_equal(b[i], b1)
            assert n_corr[i] == len(c.get_voxel_correspondences())
    c.close()


@pytest.mark.parametrize("method,radius,problem", [(O.DIRECT1, -1, 0), (O.DIRECT7, -1, 0), (O.DIRECT27, -1, 0), (O.DIRECT_RADIUS, 1.5, 0), (O.DIRECT7, -1, 1), (O.DIRECT7, -1, 2)])
def test_evaluate_poses(pair02, relative_pose, method, radius, problem):
    from fast_gicp_b200.core import Core

    c = setup(Core(0), *pair02, method=method, radius=radius, problem=problem)
    rng = np.random.default_rng(9)
    P = [relative_pose @ random_pose(rng, 0.4, 1.5) for _ in range(15)]
    nowhere = np.eye(4)
    nowhere[:3, 3] = [1000.0, 1000.0, 1000.0]
    P = np.stack(P + [nowhere])
    err, H, b, n_corr = c.evaluate_poses(P, want_H=True)
    e_only, H0, b0, n_corr0 = c.evaluate_poses(P)
    assert H0 is None and b0 is None and np.array_equal(n_corr0, n_corr)
    for i, T in enumerate(P):
        c.update_correspondences(T)
        e1, H1, b1 = c.compute_error(T, True)
        e2, _, _ = c.compute_error(T, False)
        assert err[i] == e1 and np.array_equal(H[i], H1) and np.array_equal(b[i], b1), i
        assert e_only[i] == e2, i
        assert n_corr[i] == len(c.get_voxel_correspondences()), i
    assert err[-1] == 0.0 and n_corr[-1] == 0
    assert n_corr[:-1].min() > 0
    c.close()


@pytest.mark.parametrize("gn", [0, 1])
def test_launches_are_batched(pair02, relative_pose, gn):
    """LM + speculation: one launch per round, rounds = max(1 + n_compute_error); GN: rounds = max(n_linearize)."""
    from fast_gicp_b200.core import Core, default_params

    c = setup(Core(0), *pair02, method=O.DIRECT27)
    params = default_params(use_gauss_newton=gn)
    c.set_profiling(True)  # (resets the counters)
    multi = c.align_multi(guesses(relative_pose), params)
    prof = c.get_profile()
    launches = prof["linearize"][1] + prof["compute_error"][1]
    want = max(r.n_linearize for r in multi) if gn else max(1 + r.n_compute_error for r in multi)
    assert launches == want
    assert launches < sum(r.n_linearize + r.n_compute_error for r in multi) / 2
    c.close()


def test_handle_state_is_undisturbed(pair02, relative_pose):
    from fast_gicp_b200.core import Core

    tgt, src = pair02
    c = setup(Core(0), tgt, src, method=O.DIRECT7)
    T_prev = relative_pose @ random_pose(np.random.default_rng(2), 0.05, 0.2)
    c.update_correspondences(T_prev)
    pairs0 = c.get_voxel_correspondences()
    e0, H0, b0 = c.compute_error(T_prev, True)
    G = guesses(relative_pose)
    c.align_multi(G)
    c.evaluate_poses(G, want_H=True)
    assert np.array_equal(c.get_voxel_correspondences(), pairs0)
    e1, H1, b1 = c.compute_error(T_prev, True)
    assert e1 == e0 and np.array_equal(H1, H0) and np.array_equal(b1, b0)
    fresh = setup(Core(0), tgt, src, method=O.DIRECT7)
    for g in G[:3]:
        assert_same(c.align(g), fresh.align(g))
    fresh.close()
    c.close()


def test_errors_launch_nothing(pair02):
    from fast_gicp_b200.core import AlignResult, Core, ERR_BAD_STATE, ERR_INVALID_ARGUMENT

    tgt, src = pair02
    G = np.tile(np.eye(4).reshape(16), 4097)
    res = (AlignResult * 4097)()
    out = np.zeros(4097 * 43)
    n64 = np.zeros(4097, dtype=np.int64)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    ip = n64.ctypes.data_as(C.POINTER(C.c_int64))

    def calls(c):
        L, h = c._lib, c._h
        return [
            L.vgicp_align_multi(h, dp(G), 4, None, res), L.vgicp_evaluate_poses(h, dp(G), 4, dp(out), None, None, ip),
        ]

    # missing source / map: the documented state errors, nothing launched
    c = Core(0)
    c.set_target_cloud(tgt)
    n0 = c.launch_count()
    assert calls(c) == [ERR_BAD_STATE] * 2
    assert c.launch_count() == n0
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)
    n0 = c.launch_count()
    assert calls(c) == [ERR_BAD_STATE] * 2  # no voxel map yet
    assert c.launch_count() == n0
    nd = Core(0)
    nd.set_problem(2)
    nd.set_source_cloud(src)
    n0 = nd.launch_count()
    assert calls(nd) == [ERR_BAD_STATE] * 2  # NDT without a target
    assert nd.launch_count() == n0
    nd.close()
    # argument errors on a ready handle
    c.create_target_voxelmap()
    c.align_multi(np.eye(4)[None])  # (settles the map build)
    n0 = c.launch_count()
    L, h = c._lib, c._h
    bad = [
        L.vgicp_align_multi(h, dp(G), 0, None, res), L.vgicp_align_multi(h, dp(G), 4097, None, res), L.vgicp_align_multi(h, dp(G), -3, None, res),
        L.vgicp_align_multi(h, None, 4, None, res), L.vgicp_align_multi(h, dp(G), 4, None, None),
        L.vgicp_evaluate_poses(h, dp(G), 0, dp(out), None, None, ip), L.vgicp_evaluate_poses(h, dp(G), 4097, dp(out), None, None, ip),
        L.vgicp_evaluate_poses(h, None, 4, dp(out), None, None, ip), L.vgicp_evaluate_poses(h, dp(G), 4, None, None, None, ip),
        L.vgicp_evaluate_poses(h, dp(G), 4, dp(out), dp(out), None, ip), L.vgicp_evaluate_poses(h, dp(G), 4, dp(out), None, dp(out), ip),
        L.vgicp_align_multi(None, dp(G), 4, None, res), L.vgicp_evaluate_poses(None, dp(G), 4, dp(out), None, None, ip),
    ]
    assert bad == [ERR_INVALID_ARGUMENT] * len(bad)
    assert c.launch_count() == n0
    # the largest batch is accepted
    assert L.vgicp_evaluate_poses(h, dp(G), 4096, dp(out), None, None, ip) == 0 and (n64[:4096] == n64[0]).all()
    c.close()


def test_communicator_handle_is_unsupported():
    """A handle in a multi-GPU communicator refuses both calls with VGICP_ERR_UNSUPPORTED and launches nothing (two GPUs)."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_multi_gpu import _free_port

    port = _free_port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "multi_hypothesis_comm_worker.py")], env=env, stdout=subprocess.PIPE,
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


@pytest.mark.parametrize("cls", ["FastVGICPCuda", "NDTCuda"])
def test_surfaces(pair02, relative_pose, cls):
    import fast_gicp_b200 as F

    tgt, src = pair02
    G = guesses(relative_pose)[:12]

    def py_reg():
        r = getattr(F, cls)()
        if cls == "NDTCuda":
            r.setNeighborSearchMethod("DIRECT7")
        else:
            r.setNeighborSearchMethod("DIRECT27")
        r.setInputTarget(tgt)
        r.setInputSource(src)
        return r

    def pg_reg():
        r = getattr(_pygicp(), cls)()
        r.set_neighbor_search_method("DIRECT7" if cls == "NDTCuda" else "DIRECT27", 0.0)
        r.set_input_target(tgt.astype(np.float64))
        r.set_input_source(src.astype(np.float64))
        return r

    # Python class: align_multi(G)[i] == align(G[i]), and the single-registration state is left alone
    reg = py_reg()
    T_multi, conv_multi = reg.align_multi(G)
    assert T_multi.dtype == np.float32 and T_multi.shape == (len(G), 4, 4) and conv_multi.dtype == bool
    assert np.array_equal(reg.getFinalTransformation(), np.eye(4, dtype=np.float32)) and not reg.hasConverged()
    single = py_reg()
    for i, g in enumerate(G):
        assert np.array_equal(single.align(g), T_multi[i]) and single.hasConverged() == conv_multi[i], i
    # pygicp: the same multi-hypothesis results; its align (the C++ mirror's own LM loop) agrees to rounding
    pg = pg_reg()
    T_pg, conv_pg = pg.align_multi(G.astype(np.float32))
    assert np.array_equal(T_pg, T_multi) and np.array_equal(conv_pg, conv_multi)
    pg_single = pg_reg()
    for i, g in enumerate(G):
        T = pg_single.align(g.astype(np.float32))
        assert pg_single.has_converged() == conv_multi[i], i
        dt, dr = pose_error(T_multi[i], T)
        assert dt < 1e-6 and dr < 1e-7, (i, dt, dr)
    # evaluate_poses through both surfaces
    P = np.stack([relative_pose, np.eye(4), G[5]])
    e_py, n_py = py_reg().evaluate_poses(P)
    e_pg, n_pg = pg_reg().evaluate_poses(P)
    assert np.array_equal(e_py, e_pg) and np.array_equal(n_py, n_pg) and n_py.min() > 0
