"""Stage 1 (k-NN and RBF covariances, the regularisers) and the voxel Gaussians on the GPU, at the inputs and launch shapes where a
closed-form 3x3 eigen-solver and the RBF kernel's block loop go wrong.  Every case is held twice: to the CPU oracle, bit for bit
(regularised results may differ in one point by a double-rounding tie of the trig step), and to the float64 references of
cov_reference.py within their derived bounds -- so that an error shared by the oracle and the kernels does not pass unseen.
The last test prints the worst ratio |x - x_ref| / scale seen per quantity."""
import numpy as np
import pytest

import oracle as O
import cov_reference as R

pytestmark = pytest.mark.gpu

REGS = (O.REG_NONE, O.REG_PLANE, O.REG_MIN_EIG, O.REG_FROBENIUS)
RBF_SETTINGS = R.RBF_SETTINGS
RBF_QUERIES = 48  # float64 checks per RBF case: a seeded subsample plus queries the origin padding reaches
WORST = {}


def note(quantity, value):
    WORST[quantity] = max(WORST.get(quantity, 0.0), float(value))


@pytest.fixture(scope="module")
def core():
    from fast_gicp_b200.core import Core

    c = Core(0)
    yield c
    c.close()


def assert_matches_oracle(got, raw, method, what):
    """got: the GPU's stored covariances; raw: the oracle's raw covariances of the same cloud."""
    want = O.symmetrized(raw if method == O.REG_NONE else O.regularize(raw, method))
    bad = np.flatnonzero((got != want).any(axis=1))
    if method == O.REG_NONE:
        assert not len(bad), (what, len(bad), bad[:5])
    else:  # a double-rounding coincidence in the double -> float trig step is conceivable (p ~ 1e-8 per point); allow one
        assert len(bad) <= 1, (what, method, len(bad), bad[:5], np.abs(got - want).max())


def assert_regularised_float64(method, raw, got, what):
    for q, v in R.assert_regularised(method, raw, got, what).items():
        note(q, v)


def check_knn_chain(core, raw, ref_raw, what, side="source"):
    """Every regulariser on the rows set on `side`: oracle and float64.  Returns the PLANE covariances."""
    calc = core.calculate_source_covariances if side == "source" else core.calculate_target_covariances
    get = core.get_source_covariances if side == "source" else core.get_target_covariances
    out = None
    for method in REGS:
        calc(method)
        got = get()
        assert_matches_oracle(got, raw, method, what)
        if method == O.REG_NONE:
            r, bad = R.check(R.mat(got), *ref_raw, R.TAU_RAW)
            assert not len(bad), (what, bad[:5], r[bad][:5])
            note("raw k-NN", r.max())
        else:
            assert_regularised_float64(method, raw, got, what)
        if method == O.REG_PLANE:
            out = got
    return out


# ---------------------------------------------------------------------------------------------------------------- a. k-NN
@pytest.mark.parametrize("k", R.KNN_KS)
def test_knn_covariances_on_hand_built_neighbourhoods(core, k):
    """Rows given with set_source_neighbors, so that each is exactly the intended set: identical points, repeated indices, exact
    lines and planes (axis-aligned and rotated), isotropic sets, disks, prolate sets, lidar ring arcs, sets 1e3 and 1e4 m from the
    origin and sets below the MIN_EIG clamp.  The target side runs the same kernel: byte-equal."""
    pts, nbr, kind = R.knn_neighbourhoods(k)
    raw = O.covariances(pts, nbr)
    core.set_source_cloud(pts)
    core.set_source_neighbors(k, nbr)
    plane = check_knn_chain(core, raw, R.raw_knn64(pts, nbr), f"hand-built k={k}")
    core.set_target_cloud(pts)
    core.set_target_neighbors(k, nbr)
    core.calculate_target_covariances(O.REG_PLANE)
    assert np.array_equal(core.get_target_covariances(), plane)


@pytest.mark.parametrize("cloud", ["grid", "whole cloud"])
@pytest.mark.parametrize("k", [3, 33, 64])
def test_knn_chain_from_found_neighbours(core, k, cloud):
    """find_source_neighbors + the covariance kernel = O.covariances(pts, O.knn(pts, k)) regularised.  grid: 3000 points, the grid
    search; whole cloud: 200 points, every query scans the whole cloud block-cooperatively."""
    pts = R.lidar_scan(3000 if cloud == "grid" else 200, seed=k)
    core.set_source_cloud(pts)
    core.find_source_neighbors(k)
    nbr = core.get_source_neighbors()
    assert np.array_equal(nbr, O.knn(pts, k, "bruteforce"))
    check_knn_chain(core, O.covariances(pts, nbr), R.raw_knn64(pts, nbr), f"{cloud} k={k}")


# ---------------------------------------------------------------------------------------------------------------- b. RBF
def check_rbf_case(core, pts, kw, md, what, queries):
    core.set_kernel_params(kw, md)
    core.set_source_cloud(pts)
    raw = O.covariances_rbf(pts, kw, md)
    ref, sc = R.rbf64(pts, queries, kw, md)
    for method in REGS:
        core.calculate_source_covariances_rbf(method)
        got = core.get_source_covariances()
        assert_matches_oracle(got, raw, method, what)
        if method == O.REG_NONE:
            r, bad = R.check(R.mat(got[queries]), ref, sc, R.TAU_RBF)
            assert not len(bad), (what, queries[bad][:5], r[bad][:5])
            note("RBF raw", r.max())
        else:
            assert_regularised_float64(method, raw[queries], got[queries], what)
    return raw


@pytest.mark.parametrize("n", R.RBF_NS)
def test_rbf_covariances_at_every_launch_shape(core, n):
    """n around the 512-point block (padding or none), the 8-block round boundary (4096) and several rounds (20 000), each cloud
    in azimuth order (neighbouring queries share blocks; far blocks are skipped by the box test) and shuffled (every box spans the
    cloud).  All four regularisers bit-equal to the oracle; float64 on a seeded subsample of queries."""
    rng = np.random.default_rng(n)
    base = R.lidar_scan(n, seed=n)
    for order in ("sorted", "shuffled"):
        pts = base if order == "sorted" else base[rng.permutation(n)]
        for kw, md in RBF_SETTINGS:
            near = np.flatnonzero(R.in_range32(np.zeros(3, np.float32), pts, md))
            q = np.unique(np.concatenate([rng.choice(n, size=min(n, RBF_QUERIES), replace=False), near[:16]]))
            check_rbf_case(core, pts, kw, md, f"RBF n={n} {order} ({kw}, {md})", q)


def test_rbf_isolated_points_see_only_themselves(core):
    """Points farther than max_dist from each other and from the origin: each query's weight is its own (w = exp(0) = 1), the
    covariance exactly zero, and every regulariser takes eig3_direct's scale == 0 path."""
    g = np.arange(17, dtype=np.float32)
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)[:4097] + np.float32(3.5)
    raw = check_rbf_case(core, pts, 0.5, 0.25, "RBF isolated", np.arange(0, len(pts), 61))
    assert not raw.any()


# ---------------------------------------------------------------------------------------------------------------- c. voxels
@pytest.mark.parametrize("res", [0.1, 0.5, 1.0])
def test_voxel_gaussians(res):
    """Voxels of exactly 1, 2, 3 and 4 points, collinear and coplanar voxels, 33 points (two rounds of k_voxel_reduce's 32-point
    loop), 10 000 points, and voxels 1e3 and 1e4 m from the origin (the one-pass (S - mu S^T) / n cancels there): the VGICP map
    (caller-supplied covariances) and the NDT map (points alone, MIN_EIG) against the oracle and against float64."""
    from fast_gicp_b200.core import Core

    pts, cov = R.voxel_cloud(res)
    for ndt in (False, True):
        c = Core(0)
        c.set_resolution(res)
        if ndt:
            c.set_problem(2)
            c.set_target_cloud(pts)
            c.set_source_cloud(pts)
            c.ndt_create_voxelmaps()
        else:
            c.set_target_cloud(pts)
            c.set_target_covariances(cov)
            c.create_target_voxelmap()
        what = f"{'NDT' if ndt else 'VGICP'} res={res}"
        vm = O.VoxelMap(pts, None if ndt else cov, res, accum_double=True)
        coords, ids = c.get_voxel_buckets()
        assert np.array_equal(ids, vm.bucket_id) and np.array_equal(coords, vm.bucket_coord), what
        n_got, mean, vcov = c.get_voxel_num_points(), c.get_voxel_means(), c.get_voxel_covs()
        c.close()
        assert np.array_equal(n_got, vm.vox_n) and np.array_equal(mean, vm.vox_mean), what
        bad = np.flatnonzero((vcov != O.symmetrized(vm.vox_cov)).any(axis=1))
        assert len(bad) <= (1 if ndt else 0), (what, len(bad))
        ref = R.voxels64(pts, res, None if ndt else cov)
        v = R.match_voxels(ref["coords"], coords, ids)
        assert (v >= 0).all() and np.array_equal(n_got[v], ref["n"]), what
        rm, bad = R.check(mean[v][:, :, None], ref["mean"][:, :, None], ref["mean_scale"][:, :, None], R.TAU_VOXEL)
        assert not len(bad), (what, "mean", ref["n"][bad][:5])
        rc, bad = R.check(R.mat(vcov[v]), ref["cov"], ref["cov_scale"], R.TAU_VOXEL)
        assert not len(bad), (what, "cov", ref["n"][bad][:5], rc[bad][:5])
        note(f"{'NDT' if ndt else 'VGICP'} voxel mean", rm.max())
        note(f"{'NDT' if ndt else 'VGICP'} voxel covariance", rc.max())
        if ndt:
            assert np.linalg.eigvalsh(R.mat(vcov)).min() > 0.99e-3, what


def test_report_worst_ratios(capsys):
    with capsys.disabled():
        print("\n  [stage1 matrix] worst |x - x_ref| / scale on the GPU: " + ", ".join(f"{q} {v:.3g}" for q, v in sorted(WORST.items())))
