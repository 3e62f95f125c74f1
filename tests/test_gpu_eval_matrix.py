"""Every evaluation-kernel variant against a float64 reference, at the cloud sizes that select it.

make_lin_launch (csrc/vgicp_b200.cu) picks the kernel from the source size n, the offset table and the voxel index alone, so the
cases below reach each variant through input sizes: one generated target and exact-size prefixes of one generated source.
selected_kernel() restates that rule as data and test_case_table_reaches_every_kernel checks that the cases reach every shape of
with_lin_shape and the streaming kernel, with robust weights on and off, under both voxel indexes.

Per case, with T_lin != T_eval (update_correspondences(T), then compute_error(T @ small perturbation)) at the identity and near
the ground truth, for every robust kind:
  1. compute_error(.., True / False) against eval64 (tests/eval_reference.py) and against the float oracle, entry by entry with A,
     the sum of |per-correspondence terms| of each entry, as its scale;
  2. evaluate_poses over 3 poses (the multi-row kernels, with hit counts) equals the single-pose calls bit for bit, n_corr equals
     the length of the oracle's correspondence list;
  3. the hash-table index gives the dense index's sums bit for bit where both run the same compacted kernel (DIRECT1 on >= 65 536
     points streams with the dense index only: there the two kernels are each held to the references instead);
  4. (DIRECT1 at 120 k, 450 k and 65 536 points) align with speculation on equals align with it off, and align_multi equals a loop
     of align, bit for bit.

Tolerances (|x - x_ref| <= tau A + 1e-12 max(A)):
  TAU = 1e-5 against the float oracle (the same float32 terms, summed in another order) and against eval64 on the well-conditioned
  covariances (eigenvalues in [0.1, 1]).
  TAU_PLANE = 1e-4 against eval64 on PLANE covariances and for NDT.  The float32 cofactor inverse of S = C_B + R C_A R^T has a
  relative error up to about cond(S) u per term, u = 2^-24; PLANE clamps the eigenvalues at 1e-3 of the largest, so cond(S) <= 1e3
  and a term may be off by 1e3 * 6e-8 = 6e-5 of its size.  Those errors have random signs across correspondences, so the sums
  stay well inside 1e-4 A.
NDT is compared with eval64 over the GPU's own voxel Gaussians (read back from the handle): the oracle's NDT map regularises with
a restated eigen-solver that may differ in the rank-deficient voxels (test_gpu_ndt pins those), which would be a difference of
inputs, not of the evaluation.
"""
import re

import numpy as np
import pytest

import oracle as O
import oracle_robust as R
from conftest import random_pose
from eval_reference import KINDS, assert_close, eval64_kinds
from test_gpu_multi_hypothesis import assert_same, setup

pytestmark = pytest.mark.gpu

TAU = 1e-5
TAU_PLANE = 1e-4

# with_lin_shape's table: (MODE, G), MODE = 1 / 7 / 27 fixed tables, 0 = generic offset list
LIN_SHAPES = {(1, 1), (7, 1), (7, 4), (27, 1), (27, 3), (0, 1), (0, 4), (0, 8)}
MODE_OF = {O.DIRECT1: 1, O.DIRECT7: 7, O.DIRECT27: 27, O.DIRECT_RADIUS: 0}
METHODS = {"d1": (O.DIRECT1, -1.0), "d7": (O.DIRECT7, -1.0), "d27": (O.DIRECT27, -1.0), "r0.5": (O.DIRECT_RADIUS, 0.5),
           "r1": (O.DIRECT_RADIUS, 1.0), "r1.5": (O.DIRECT_RADIUS, 1.5), "r2": (O.DIRECT_RADIUS, 2.0), "r2.5": (O.DIRECT_RADIUS, 2.5)}
# source sizes: pair_0p2; mid (G = 3 / 4 / 8 with several grid-stride sets per warp, DIRECT1 streams); large (G = 1); the thresholds
# of the lane split (400 000) and of the streaming kernel (65 536; 65 537 leaves a final tile of one point)
SIZES = {"small": None, "mid": 120_000, "large": 450_000, "n399999": 399_999, "n400000": 400_000, "n65535": 65_535, "n65536": 65_536,
         "n65537": 65_537}
KERNEL_THREADS, MAX_BLOCKS = 128, 4 * 132  # kLinThreads, kLinMaxBlocks

VGICP_CASES = ([("small", m) for m in METHODS] + [("mid", m) for m in METHODS] + [("large", m) for m in ("d1", "d7", "d27", "r0.5", "r1.5")]
               + [("n399999", "d7"), ("n400000", "d7"), ("n65535", "d1"), ("n65536", "d1"), ("n65537", "d1")])
SPD_CASES = [("mid", m) for m in ("d1", "d7", "d27", "r1.5")] + [("large", m) for m in ("d1", "d27")]
NDT_CASES = [(size, problem, m) for size in ("small", "large") for problem in (1, 2) for m in ("d1", "d7", "d27", "r1.5")]
ALIGN_SIZES = ("mid", "large", "n65536")


def selected_kernel(n, method, radius, dense):
    """make_lin_launch's choice for n source points: "stream" or the compacted kernel's (MODE, G)."""
    mode, n_off = MODE_OF[method], len(O.offsets(method, radius))
    if mode == 1 and dense and n >= 65536:
        return "stream"
    if n >= 400_000 or n_off == 1:
        return (mode, 1)
    return (mode, 3 if mode == 27 else (4 if n_off <= 7 else 8))


def sets_per_warp(n, G):
    """Grid-stride sets of 32 // G points each warp of a compacted kernel walks (the grid is capped at MAX_BLOCKS)."""
    tpw = (32 // G) * G
    warps = min(-(-n * G // (KERNEL_THREADS // 32 * tpw)), MAX_BLOCKS) * (KERNEL_THREADS // 32)
    return -(-n * G // (warps * tpw))


def case_sizes(pair_n):
    return {k: (pair_n if v is None else v) for k, v in SIZES.items()}


def claimed_cells(pair_n):
    """{(kernel, RB, dense)} the cases reach: every case runs every robust kind (RB = kind != NONE; NDT: RB off) on both indexes."""
    n_of = case_sizes(pair_n)
    cells = set()
    for size, m in VGICP_CASES + SPD_CASES:
        for dense in (True, False):
            k = selected_kernel(n_of[size], *METHODS[m], dense)
            cells |= {(k, rb, dense) for rb in (False, True)}
    for size, problem, m in NDT_CASES:
        if problem == 1:  # (D2D evaluates the source voxels: their number decides)
            cells |= {(selected_kernel(n_of[size], *METHODS[m], dense), False, dense) for dense in (True, False)}
    return cells


def test_case_table_reaches_every_kernel(pair02):
    """The cases reach every (MODE, G) of with_lin_shape with RB on and off under both indexes, the streaming kernel (dense index
    only) with RB on and off and with NDT weights, every robust kind at every shape, and wide kernels with >= 3 sets per warp."""
    n_of = case_sizes(len(pair02[1]))
    cells = claimed_cells(len(pair02[1]))
    want = {(s, rb, dense) for s in LIN_SHAPES for rb in (False, True) for dense in (True, False)} | {("stream", rb, True) for rb in (False, True)}
    assert want <= cells, sorted(want - cells, key=str)
    assert not {c for c in cells if c[0] != "stream"} - want
    assert ("stream", False, True) in {(selected_kernel(n_of[s], *METHODS[m], True), False, True) for s, p, m in NDT_CASES if p == 1}
    for G in (3, 4, 8):
        assert any(sets_per_warp(n_of[s], G) >= 3 and selected_kernel(n_of[s], *METHODS[m], True)[1:] == (G,) for s, m in VGICP_CASES), G
    # DIRECT_RADIUS at 2.0 and 2.5 runs the 8-lane kernel over 2 and 3 passes of 32 cells
    assert [len(O.offsets(*METHODS[m])) for m in ("r0.5", "r1", "r1.5", "r2", "r2.5")] == [1, 7, 19, 33, 81]


# ---- inputs ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def big():
    """One 128-beam scan pair.  A scan is ordered beam by beam, so a raw prefix of it is only the ground ring around the sensor:
    the target is a seeded random half-million subset and the source a seeded shuffle, whose prefixes spread over the scene."""
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0)
    rng = np.random.default_rng(44)
    tgt = tgt[np.sort(rng.permutation(len(tgt))[:500_000])]
    src = src[rng.permutation(len(src))[:SIZES["large"]]]
    assert len(tgt) == 500_000 and len(src) == SIZES["large"]
    return tgt, src, T_gt


def spd(n, seed):
    """n symmetric positive definite 3x3 (column-major rows of 9) with eigenvalues in [0.1, 1]."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    C = (Q * rng.uniform(0.1, 1.0, size=(n, 1, 3))) @ Q.transpose(0, 2, 1)
    return (0.5 * (C + C.transpose(0, 2, 1))).astype(np.float32).reshape(n, 9)


def cloud_of(size, pair02, relative_pose, big):
    if size == "small":
        return pair02[0], pair02[1], relative_pose
    tgt, src, T_gt = big
    return tgt, src[:SIZES[size]], T_gt


def pose_pairs(T_near, seed):
    rng = np.random.default_rng(seed)
    return [(T, T @ random_pose(rng, 0.005, 0.05)) for T in (np.eye(4), T_near)]


def assert_same_map(c, vm):
    """The GPU voxel map is the oracle's: buckets, ids, counts and means bit for bit."""
    coords, ids = c.get_voxel_buckets()
    assert c.num_buckets() == vm.num_buckets and c.num_voxels() == vm.num_voxels
    assert np.array_equal(ids, vm.bucket_id) and np.array_equal(coords, vm.bucket_coord)
    assert np.array_equal(c.get_voxel_num_points(), vm.vox_n)
    assert np.array_equal(c.get_voxel_means(), vm.vox_mean)


_HANDLES = {}
WORST = {}  # family -> largest |x - x_ref| / A seen


def record(family, got, ref, tau, what):
    worst = assert_close(got, ref, tau, what)
    WORST[family] = max(WORST.get(family, 0.0), worst)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for c in _HANDLES.values():
        c["core"].close()
    _HANDLES.clear()
    for k in sorted(WORST):
        print(f"worst |x - x_ref| / A  {k}: {WORST[k]:.3g}")


def vgicp_handle(size, covs, pair02, relative_pose, big):
    """A handle with the size's target map and source prefix; covs "plane" (stage 1 on the GPU) or "spd"."""
    key = (size, covs)
    if key in _HANDLES:
        return _HANDLES[key]
    from fast_gicp_b200.core import Core

    tgt, src, T_near = cloud_of(size, pair02, relative_pose, big)
    if covs == "plane":
        c = setup(Core(0), tgt, src, method=O.DIRECT1)
        t_cov, s_cov = c.get_target_covariances(), c.get_source_covariances()
    else:
        t_cov, s_cov = spd(len(tgt), 1), spd(len(src), 2)
        c = Core(0)
        c.set_target_cloud(tgt)
        c.set_target_covariances(t_cov)
        c.create_target_voxelmap()
        c.set_source_cloud(src)
        c.set_source_covariances(s_cov)
    vm = O.VoxelMap(tgt, t_cov, 1.0, accum_double=True)
    assert_same_map(c, vm)
    assert vm.vox_n.min() >= 1  # (so the error-only sums equal the err of the full evaluation)
    h = dict(core=c, vm=vm, src=src, s_cov=s_cov, mean=c.get_voxel_means(), cov=c.get_voxel_covs(), n=c.get_voxel_num_points(),
             poses=pose_pairs(T_near, SIZES[size] or 0), T_near=T_near)
    _HANDLES[key] = h
    return h


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def check_case(h, method_key, family, tau64, oracle):
    """Checks 1-3 on one handle for one neighbour search setting."""
    c, src = h["core"], h["src"]
    method, radius = METHODS[method_key]
    c.set_neighbor_search_method(method, radius)
    offs = O.offsets(method, radius)
    kernels = [selected_kernel(len(src), method, radius, dense) for dense in (True, False)]
    pair_lists = []
    for Tl, Te in h["poses"]:
        pairs = O.find_correspondences(h["vm"], src, Tl, offs)
        pair_lists.append(pairs)
        kinds = ("NONE",) if oracle == "ndt" else KINDS  # (NDT carries its own weight: a robust kind is refused)
        refs = eval64_kinds(h["mean"], h["cov"], h["n"], src, h["s_cov"], pairs, Tl, Te, True, kinds=kinds, ndt=oracle == "ndt", res=1.0)
        for kind in kinds:
            c.set_robust_kernel(kind, 1.0)
            ref = refs[kind]
            orc = R.derivatives(h["vm"], src, h["s_cov"], pairs, Tl, Te, True, robust=kind) if oracle == "float" else None
            got = []
            for index, k in zip((0, 1), kernels):
                c.set_voxel_index(index)
                c.update_correspondences(Tl)
                full, err_only = c.compute_error(Te, True), c.compute_error(Te, False)
                what = f"{method_key} {k} index={index} {kind} n={len(src)} T_lin={'I' if Tl is h['poses'][0][0] else 'near'}"
                record(f"{family} eval64 {k}", full, ref, tau64, what)
                record(f"{family} eval64 {k}", err_only, (ref[0], None, None, ref[3][:1]), tau64, what + " error only")
                if orc is not None:
                    oref = (orc[0], orc[1], orc[2], ref[3])
                    record(f"{family} oracle {k}", full, oref, TAU, what + " vs float oracle")
                    record(f"{family} oracle {k}", err_only, (orc[0], None, None, ref[3][:1]), TAU, what + " error only vs float oracle")
                got.append((full, err_only))
            if kernels[0] == kernels[1]:  # the same compacted kernel over either index: the same voxels in the same order
                assert same(got[0][0], got[1][0]) and got[0][1][0] == got[1][1][0], (method_key, kind)
    # 2. the multi-row kernels (with hit counts) against the single-pose calls
    poses = np.stack([h["poses"][0][0], h["poses"][1][0], h["poses"][1][1]])
    n_pairs = [len(pair_lists[0]), len(pair_lists[1]), len(O.find_correspondences(h["vm"], src, poses[2], offs))]
    for kind in (("NONE",) if oracle == "ndt" else KINDS):
        c.set_robust_kernel(kind, 1.0)
        for index in (0, 1):
            c.set_voxel_index(index)
            for want_H in (True, False):
                err, H, b, n_corr = c.evaluate_poses(poses, want_H)
                assert list(n_corr) == n_pairs, (method_key, kind, index)
                for i, T in enumerate(poses):
                    c.update_correspondences(T)
                    one = c.compute_error(T, want_H)
                    assert err[i] == one[0], (method_key, kind, index, want_H, i)
                    if want_H:
                        assert np.array_equal(H[i], one[1]) and np.array_equal(b[i], one[2]), (method_key, kind, index, i)
    c.set_robust_kernel("NONE")
    c.set_voxel_index(0)


@pytest.mark.parametrize("size,method", VGICP_CASES, ids=[f"{s}-{m}" for s, m in VGICP_CASES])
def test_plane_covariances(pair02, relative_pose, big, size, method):
    h = vgicp_handle(size, "plane", pair02, relative_pose, big)
    check_case(h, method, "plane", TAU_PLANE, "float")


@pytest.mark.parametrize("size,method", SPD_CASES, ids=[f"{s}-{m}" for s, m in SPD_CASES])
def test_well_conditioned_covariances(pair02, relative_pose, big, size, method):
    h = vgicp_handle(size, "spd", pair02, relative_pose, big)
    check_case(h, method, "spd", TAU, "float")


@pytest.mark.parametrize("size,problem,method", NDT_CASES, ids=[f"{s}-{'p2d' if p == 1 else 'd2d'}-{m}" for s, p, m in NDT_CASES])
def test_ndt(pair02, relative_pose, big, size, problem, method):
    from fast_gicp_b200.core import Core

    tgt, src, T_near = cloud_of(size, pair02, relative_pose, big)
    c = setup(Core(0), tgt, src, method=METHODS[method][0], radius=METHODS[method][1], problem=problem)
    tm = O.VoxelMap(tgt, None, 1.0, accum_double=True)
    assert_same_map(c, tm)
    if problem == 2:  # the source Gaussians as the GPU builds them: the same map build, run with the source as the target
        s = setup(Core(0), src, src, method=O.DIRECT1, problem=1)
        assert_same_map(s, O.VoxelMap(src, None, 1.0, accum_double=True))
        s_pts, s_cov = s.get_voxel_means(), s.get_voxel_covs()
        s.close()
    else:
        s_pts, s_cov = src, None
    h = dict(core=c, vm=tm, src=s_pts, s_cov=s_cov, mean=c.get_voxel_means(), cov=c.get_voxel_covs(), n=c.get_voxel_num_points(),
             poses=pose_pairs(T_near, 5 + problem))
    check_case(h, method, "ndt", TAU_PLANE, "ndt")
    c.close()


@pytest.mark.parametrize("size", ALIGN_SIZES)
def test_speculation_and_multi_hypothesis_are_bit_identical(pair02, relative_pose, big, size):
    """DIRECT1 where it streams (k_linearize_stream<kEvalSpec> / k_linearize_stream_multi<kEvalSpec, ..., SRC = false>) and, over the
    hash table, where it does not."""
    h = vgicp_handle(size, "plane", pair02, relative_pose, big)
    c = h["core"]
    c.set_neighbor_search_method(O.DIRECT1)
    G = np.stack([np.eye(4), h["T_near"] @ random_pose(np.random.default_rng(3), 0.02, 0.2)])
    for index in (0, 1):
        c.set_voxel_index(index)
        for kind in ("NONE", "CAUCHY"):
            c.set_robust_kernel(kind, 1.0)
            c.set_speculation(0)
            plain = [c.align(g) for g in G]
            c.set_speculation(1)
            spec = [c.align(g) for g in G]
            for a, b in zip(plain, spec):
                assert_same(a, b, f"{size} index={index} {kind}: speculation")
            for i, r in enumerate(c.align_multi(G)):
                assert_same(r, spec[i], f"{size} index={index} {kind}: align_multi guess {i}")
    c.set_robust_kernel("NONE")
    c.set_voxel_index(0)


# ---- the kernels the table claims are the ones that run ---------------------------------------------------------------------

_LIN = re.compile(r"k_linearize<(\d+), (\d+), (\d+), (true|false)>")
_STREAM = re.compile(r"k_linearize_stream<(\d+), (true|false)>")


def test_profiler_sees_every_claimed_kernel(pair02, relative_pose, big):
    """One pass over the case settings (GPU side only) under torch.profiler: the demangled names of the launched evaluation
    kernels include every (MODE, G, RB) instantiation and both streaming RB variants the table claims.  (The voxel index is a
    branch inside the kernels, not a template argument: it is not visible here.)"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from fast_gicp_b200.core import Core

    torch.cuda.init()
    n_of = case_sizes(len(pair02[1]))
    handles = {size: vgicp_handle(size, "plane", pair02, relative_pose, big) for size in ("small", "mid", "large")}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for size, m in VGICP_CASES:
            if size not in handles:
                continue
            c = handles[size]["core"]
            c.set_neighbor_search_method(*METHODS[m])
            for kind in ("NONE", "HUBER"):
                c.set_robust_kernel(kind, 1.0)
                for index in (0, 1):
                    c.set_voxel_index(index)
                    c.update_correspondences(np.eye(4))
                    c.compute_error(np.eye(4), True)
            c.set_robust_kernel("NONE")
            c.set_voxel_index(0)
        nd = setup(Core(0), big[0], big[1], method=O.DIRECT1, problem=1)
        nd.update_correspondences(np.eye(4))
        nd.compute_error(np.eye(4), True)
        torch.cuda.synchronize()
        nd.close()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    if not names:
        pytest.skip("torch.profiler recorded no device kernel events on this machine")
    seen = {(int(g[0]), int(g[2]), g[3] == "true") for g in (_LIN.search(s).groups() for s in names if _LIN.search(s)) if g[1] == "1"}  # WHAT == kEvalLinearize
    seen |= {("stream", g[1] == "true") for g in (_STREAM.search(s).groups() for s in names if _STREAM.search(s)) if g[0] == "1"}
    want = {(k[0], k[1], rb) for size, m in VGICP_CASES if size in handles for k in [selected_kernel(n_of[size], *METHODS[m], d) for d in (True, False)]
            if k != "stream" for rb in (False, True)}
    want |= {("stream", rb) for rb in (False, True)}
    assert want <= seen, (sorted(want - seen, key=str), sorted(names))
    print("launched evaluation kernels:", sorted(s for s in names if "k_linearize" in s))
