"""GPU parity tests: the CUDA path (through the C ABI, fast_gicp_b200.core.Core) against the CPU oracle on the same inputs.

Tolerances (north_star): voxel-hash values / coordinates / bucket indices bit-exact; final SE(3) within 1e-5 rad / 1e-4 m of
the oracle; reference's own gate 0.05 m / 1 deg against data/relative.txt (src/test/gicp_test.cpp:147-201).
"""
import numpy as np
import pytest

import oracle as O
from conftest import pose_error, random_pose

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-5    # rad, north_star
TRANS_TOL = 1e-4  # m, north_star


@pytest.fixture(scope="module")
def core():
    from fast_gicp_b200.core import Core

    c = Core(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def prepared(pair02):
    """Oracle products for the 0.2 m fixture pair (the reference's test inputs)."""
    tgt, src = pair02
    t_nbr = O.knn(tgt, 20, "kdtree")
    s_nbr = O.knn(src, 20, "kdtree")
    t_raw = O.covariances(tgt, t_nbr)
    s_raw = O.covariances(src, s_nbr)
    t_cov = O.regularize(t_raw, O.REG_PLANE)
    s_cov = O.regularize(s_raw, O.REG_PLANE)
    return dict(tgt=tgt, src=src, t_nbr=t_nbr, s_nbr=s_nbr, t_raw=t_raw, s_raw=s_raw, t_cov=t_cov, s_cov=s_cov)


def sym(c9):
    m = c9.reshape(-1, 3, 3)
    return (0.5 * (m + m.transpose(0, 2, 1))).reshape(-1, 9)


# ---------------------------------------------------------------------------------------------------------- stage 1
def test_knn_matches_oracle_exactly(core, prepared):
    """find_target_neighbors: exact k-NN, rows ascending in (d2, index) -- identical to the oracle (kd-tree and brute force)."""
    core.set_target_cloud(prepared["tgt"])
    core.find_target_neighbors(20)
    got = core.get_target_neighbors()
    assert got.shape == prepared["t_nbr"].shape
    assert np.array_equal(got, prepared["t_nbr"])
    assert np.array_equal(got[:, 0], np.arange(len(got)))  # self is neighbour 0 (H6)


@pytest.mark.parametrize("cloud", ["grid", "small", "far"])
@pytest.mark.parametrize("k", [1, 7, 33, 64])
def test_knn_other_k(core, k, cloud):
    """Both k-NN search paths return the oracle's rows; duplicates tie-break by index.  grid: the warp-per-query grid search;
    small: a cloud below 256 points, every query scans the whole cloud block-cooperatively; far: a few far outliers, whose queries
    (more of them for k = 64) scan all 1500 points block-cooperatively, for k > 32 with the wide kernels."""
    rng = np.random.default_rng(k)
    pts = rng.uniform(-20, 20, size=(200 if cloud == "small" else 1500, 3)).astype(np.float32)
    pts[100:110] = pts[100]  # duplicates: ties broken by index
    if cloud == "far":
        pts[:5] = rng.uniform(2000, 5000, size=(5, 3))
    core.set_source_cloud(pts)
    core.find_source_neighbors(k)
    assert np.array_equal(core.get_source_neighbors(), O.knn(pts, k, "bruteforce"))


@pytest.mark.parametrize("shape", ["line", "clusters", "outliers", "tiny", "identical", "17k"])
def test_knn_grid_hard_cases(core, shape, pair01):
    """Density extremes for the multi-level grid: 1-D line, tight clusters far apart, far outliers, tiny clouds, all-equal points."""
    rng = np.random.default_rng(11)
    if shape == "line":
        pts = np.zeros((3000, 3), dtype=np.float32)
        pts[:, 0] = np.sort(rng.uniform(0, 500, 3000))
    elif shape == "clusters":
        pts = np.concatenate([rng.normal(c, 0.01, size=(400, 3)) for c in rng.uniform(-300, 300, size=(8, 3))]).astype(np.float32)
    elif shape == "outliers":
        pts = rng.normal(0, 1.0, size=(4000, 3)).astype(np.float32)
        pts[:5] = rng.uniform(2000, 5000, size=(5, 3))
    elif shape == "tiny":
        pts = rng.uniform(-1, 1, size=(23, 3)).astype(np.float32)
    elif shape == "identical":
        pts = np.tile(np.array([[1.5, -2.0, 0.25]], dtype=np.float32), (700, 1))
    else:
        pts = pair01[0]
    k = 20
    core.set_source_cloud(pts)
    core.find_source_neighbors(k)
    assert np.array_equal(core.get_source_neighbors(), O.knn(pts, k, "kdtree" if len(pts) > 5000 else "bruteforce"))


def test_raw_covariance_bit_exact(core, prepared):
    """covariance_estimation.cu:26-34 (RegularizationMethod NONE leaves it raw): same fma sequence as the oracle -> bit-exact."""
    core.set_target_cloud(prepared["tgt"])
    core.set_target_neighbors(20, prepared["t_nbr"])
    core.calculate_target_covariances(O.REG_NONE)
    got = core.get_target_covariances()
    assert np.array_equal(got, prepared["t_raw"])


@pytest.mark.parametrize("method", [O.REG_PLANE, O.REG_MIN_EIG, O.REG_FROBENIUS])
def test_regularised_covariance_bit_exact(core, prepared, method):
    """covariance_regularization.cu restated with the same operation order on both sides (stage 1 is compiled with
    --fmad=false, trig evaluated in double and rounded once): the regularised covariances agree bit-for-bit, including on
    line-like neighbourhoods where the closed-form eigen-solver amplifies 1-ulp differences to percent level.  The GPU
    stores the symmetric part of V L V^-1."""
    core.set_target_cloud(prepared["tgt"])
    core.set_target_neighbors(20, prepared["t_nbr"])
    core.calculate_target_covariances(method)
    got = core.get_target_covariances()
    want = sym(O.regularize(prepared["t_raw"], method)).astype(np.float32)
    bad = np.flatnonzero((got != want).any(axis=1))
    # a double-rounding coincidence in the double->float trig step is conceivable (p ~ 1e-8 per point); allow one
    assert len(bad) <= 1, (len(bad), np.abs(got - want).max())


def test_plane_regularisation_identity(core, prepared):
    """C_reg = I - 0.999 n n^T up to rounding (SURVEY 8c-2): eigenvalues (1e-3, 1, 1)."""
    core.set_source_cloud(prepared["src"])
    core.set_source_neighbors(20, prepared["s_nbr"])
    core.calculate_source_covariances(O.REG_PLANE)
    got = core.get_source_covariances().reshape(-1, 3, 3).astype(np.float64)
    w = np.linalg.eigvalsh(got)
    assert np.abs(w[:, 0] - 1e-3).max() < 1e-3
    assert np.abs(w[:, 1:] - 1.0).max() < 1e-3


def test_normalized_min_eig_unsupported(core, prepared):
    from fast_gicp_b200.core import ERR_UNSUPPORTED

    core.set_source_cloud(prepared["src"])
    core.set_source_neighbors(20, prepared["s_nbr"])
    rc = core.calculate_source_covariances(O.REG_NORMALIZED_MIN_EIG)
    assert rc == ERR_UNSUPPORTED  # reference prints "unimplemented ..." and leaves the raw covariance
    assert np.array_equal(core.get_source_covariances(), prepared["s_raw"])


# ---------------------------------------------------------------------------------------------------------- stage 2
@pytest.mark.parametrize("res", [1.0, 0.5, 0.25])
def test_voxelmap_table_bit_exact(prepared, res):
    """calc_voxel_coord, vector3i_hash, bucket = (hash+i) % num_buckets, growth rule: table identical to the oracle's."""
    from fast_gicp_b200.core import Core

    c = Core(0)
    c.set_resolution(res)
    c.set_target_cloud(prepared["tgt"])
    c.set_target_neighbors(20, prepared["t_nbr"])
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()
    vm = O.VoxelMap(prepared["tgt"], sym(prepared["t_cov"]).astype(np.float32), res, accum_double=True)
    assert c.num_buckets() == vm.num_buckets
    assert c.num_voxels() == vm.num_voxels
    coords, ids = c.get_voxel_buckets()
    assert np.array_equal(ids, vm.bucket_id)
    assert np.array_equal(coords, vm.bucket_coord)
    # every occupied bucket sits within 10 probes of its hash (bit-exact hash check on the device-built table)
    occ = np.flatnonzero(ids >= 0)
    h = O.hashes(coords[occ])
    disp = (occ.astype(np.uint64) - (h % np.uint64(len(ids)))) % np.uint64(len(ids))
    assert disp.max() < 10
    assert np.array_equal(c.get_voxel_num_points(), vm.vox_n)
    # means / covs: the points of a voxel are added in index order in double and rounded once on both sides -> bit for bit
    assert np.array_equal(c.get_voxel_means(), vm.vox_mean)
    assert np.array_equal(c.get_voxel_covs(), vm.vox_cov)
    # the reference's float accumulation (any order) stays within float rounding of it
    vmf = O.VoxelMap(prepared["tgt"], sym(prepared["t_cov"]).astype(np.float32), res, accum_double=False)
    assert np.abs(c.get_voxel_means() - vmf.vox_mean).max() < 2e-4
    c.close()


def test_voxelmap_growth_and_drops():
    """Dense random cloud: the 8192-bucket table overflows, the map grows by doubling until <1% of points fail (Q5)."""
    from fast_gicp_b200.core import Core

    rng = np.random.default_rng(7)
    pts = rng.uniform(-40, 40, size=(60000, 3)).astype(np.float32)
    cov = np.tile(np.eye(3, dtype=np.float32).reshape(9), (len(pts), 1))
    nbr = np.tile(np.arange(1, dtype=np.int32), (len(pts), 1))
    c = Core(0)
    c.set_resolution(1.0)
    c.set_target_cloud(pts)
    c.set_target_neighbors(1, nbr)  # k=1 -> zero raw covariance, NONE keeps it
    c.calculate_target_covariances(O.REG_NONE)
    c.create_target_voxelmap()
    vm = O.VoxelMap(pts, np.zeros_like(cov), 1.0, accum_double=True)
    assert vm.num_buckets > 8192
    assert c.num_buckets() == vm.num_buckets and c.num_voxels() == vm.num_voxels
    coords, ids = c.get_voxel_buckets()
    assert np.array_equal(ids, vm.bucket_id) and np.array_equal(coords, vm.bucket_coord)
    assert np.array_equal(c.get_voxel_num_points(), vm.vox_n)
    c.close()


# ------------------------------------------------------------------------------------------------------ stage 2b + 3
def _setup_pair(core, p, method, radius=-1.0, res=1.0):
    core.set_resolution(res)
    core.set_neighbor_search_method(method, radius)
    core.set_target_cloud(p["tgt"])
    core.find_target_neighbors(20)
    core.calculate_target_covariances(O.REG_PLANE)
    core.create_target_voxelmap()
    core.set_source_cloud(p["src"])
    core.find_source_neighbors(20)
    core.calculate_source_covariances(O.REG_PLANE)


@pytest.mark.parametrize("method,radius", [(O.DIRECT1, -1), (O.DIRECT7, -1), (O.DIRECT27, -1), (O.DIRECT_RADIUS, 1.5)])
def test_correspondences_and_linear_system(prepared, relative_pose, method, radius):
    from fast_gicp_b200.core import Core

    c = Core(0)
    _setup_pair(c, prepared, method, radius)
    offs = O.offsets(method, radius)
    vm = O.VoxelMap(prepared["tgt"], sym(prepared["t_cov"]).astype(np.float32), 1.0, accum_double=True)
    s_cov = sym(prepared["s_cov"]).astype(np.float32)
    rng = np.random.default_rng(3)
    poses = [np.eye(4), relative_pose, relative_pose @ random_pose(rng, 0.02, 0.3)]
    for T in poses:
        c.update_correspondences(T)
        got_pairs = c.get_voxel_correspondences()
        want_pairs = O.find_correspondences(vm, prepared["src"], T, offs)
        assert np.array_equal(got_pairs, want_pairs)  # same order (offset-major), same ids
        for Te in (T, T @ random_pose(rng, 0.005, 0.05)):
            err, H, b = c.compute_error(Te, True)
            e0, H0, b0, nc = O.evaluate(vm, prepared["src"], s_cov, offs, T, Te, True)
            assert nc == len(want_pairs)
            assert abs(err - e0) <= 2e-5 * abs(e0)
            assert np.abs(H - H0).max() <= 2e-5 * np.abs(H0).max()
            assert np.abs(b - b0).max() <= 2e-5 * max(np.abs(b0).max(), 1e-3 * np.abs(H0).max())
            assert np.array_equal(H, H.T)
            e1, _, _ = c.compute_error(Te, False)
            assert abs(e1 - e0) <= 2e-5 * abs(e0)
            # bitwise reproducible (fixed-order reduction)
            err2, H2, b2 = c.compute_error(Te, True)
            assert err2 == err and np.array_equal(H2, H) and np.array_equal(b2, b)
            # the reference-layout hash table and the direct-mapped index find the same voxels in the same order
            c.set_voxel_index(1)
            err3, H3, b3 = c.compute_error(Te, True)
            e3, _, _ = c.compute_error(Te, False)
            c.set_voxel_index(0)
            assert err3 == err and np.array_equal(H3, H) and np.array_equal(b3, b) and e3 == e1
    c.close()


def test_voxel_index_falls_back_to_the_hash_table(prepared, relative_pose):
    """A target whose voxel bounding box is too large for the direct-mapped index (one far outlier) is evaluated through the
    hash table alone; the linear system still matches the oracle and the in-box case."""
    from fast_gicp_b200.core import Core

    tgt = np.vstack([prepared["tgt"], np.array([[3.0e6, -2.0e6, 1.0e6]], dtype=np.float32)])
    c = Core(0)
    c.set_neighbor_search_method(O.DIRECT27)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()
    c.set_source_cloud(prepared["src"])
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)
    t_cov = sym(c.get_target_covariances()).astype(np.float32)
    vm = O.VoxelMap(tgt, t_cov, 1.0, accum_double=True)
    offs = O.offsets(O.DIRECT27, -1)
    s_cov = sym(prepared["s_cov"]).astype(np.float32)
    err, H, b = c.linearize(relative_pose)
    e0, H0, b0, _ = O.evaluate(vm, prepared["src"], s_cov, offs, relative_pose, relative_pose, True)
    assert abs(err - e0) <= 2e-5 * abs(e0)
    assert np.abs(H - H0).max() <= 2e-5 * np.abs(H0).max()
    c.set_voxel_index(1)  # no change: the index was never built
    err1, H1, b1 = c.linearize(relative_pose)
    assert err1 == err and np.array_equal(H1, H) and np.array_equal(b1, b)
    c.close()


@pytest.mark.parametrize("method,radius", [(O.DIRECT1, -1), (O.DIRECT7, -1), (O.DIRECT27, -1), (O.DIRECT_RADIUS, 1.5)])
def test_speculative_evaluation_is_invisible(prepared, method, radius):
    """LM with the trial evaluation fused with the next linearisation (default) walks bit-identical iterates to one launch per
    evaluation, with the same evaluation counters and fewer launches; also from a poor guess, where trials get rejected."""
    from fast_gicp_b200.core import Core

    rng = np.random.default_rng(17)
    guesses = [np.eye(4), random_pose(rng, 0.15, 1.5)]
    out = {}
    for spec in (1, 0):
        c = Core(0)
        c.set_speculation(spec)
        _setup_pair(c, prepared, method, radius)
        rows = []
        for g in guesses:
            n0 = c.launch_count()
            r = c.align(guess=g)
            rows.append((np.array(r.T).copy(), np.array(r.H).copy(), r.nr_iterations, r.n_linearize, r.n_compute_error, bool(r.converged), c.launch_count() - n0))
        out[spec] = rows
        c.close()
    for a, b in zip(out[1], out[0]):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert a[2:6] == b[2:6]
        assert a[6] < b[6]  # fewer launches


@pytest.mark.parametrize("method", [O.DIRECT1, O.DIRECT7, O.DIRECT27])
def test_align_matches_oracle_and_ground_truth(prepared, relative_pose, method):
    """Whole registration vs the float oracle (north_star tolerance) and vs data/relative.txt (reference's gate)."""
    from fast_gicp_b200.core import Core

    c = Core(0)
    _setup_pair(c, prepared, method)
    res = c.align()
    from fast_gicp_b200.core import pose_from_c

    T = pose_from_c(res.T)
    vm = O.VoxelMap(prepared["tgt"], sym(prepared["t_cov"]).astype(np.float32), 1.0, accum_double=True)
    ref = O.align_f32(vm, prepared["src"], sym(prepared["s_cov"]).astype(np.float32), O.offsets(method))
    assert res.converged and ref.converged
    assert res.nr_iterations == ref.iterations
    assert (res.n_linearize, res.n_compute_error) == (ref.n_linearize, ref.n_error)
    dt, dr = pose_error(ref.T, T)
    assert dt < TRANS_TOL and dr < ROT_TOL, (dt, dr)
    Hg = np.array(res.H).reshape(6, 6).T
    assert np.abs(Hg - ref.H).max() <= 1e-4 * np.abs(ref.H).max()
    gt_t, gt_r = pose_error(relative_pose, T)
    assert gt_t < 0.05 and gt_r < np.radians(1.0)
    c.close()


def test_align_lm_failure_and_iteration_cap(prepared):
    """max_iterations is honoured, and an LM that may try no step reports the reference's 'lm not converged' state."""
    from fast_gicp_b200.core import Core, default_params

    c = Core(0)
    _setup_pair(c, prepared, O.DIRECT1)
    r = c.align(np.eye(4), default_params(max_iterations=2))
    assert r.n_linearize == 2 and not r.converged and r.nr_iterations == 1
    r = c.align(np.eye(4), default_params(max_iterations=0))
    assert r.n_linearize == 0 and not r.converged
    r = c.align(np.eye(4), default_params(lm_max_iterations=0))
    assert r.lm_failed == 1 and r.n_linearize == 1 and r.n_compute_error == 0 and r.converged == 0
    c.close()


def test_align_17k_pair(pair01, relative_pose):
    """BASELINE config 2 inputs (17k-pt pair, DIRECT27, res 1.0) end to end against the oracle."""
    from fast_gicp_b200.core import Core, pose_from_c

    tgt, src = pair01
    c = Core(0)
    _setup_pair(c, dict(tgt=tgt, src=src), O.DIRECT27)
    res = c.align()
    ref = O.register_f32(tgt, src, method=O.DIRECT27, accum_double=True)
    dt, dr = pose_error(ref.T, pose_from_c(res.T))
    assert res.converged and dt < TRANS_TOL and dr < ROT_TOL, (dt, dr)
    gt_t, gt_r = pose_error(relative_pose, pose_from_c(res.T))
    assert gt_t < 0.05 and gt_r < np.radians(1.0)
    c.close()


# ------------------------------------------------------------------------------------- reference test scenarios (API)
def test_reference_alignment_scenarios(pair02, relative_pose):
    """src/test/gicp_test.cpp:147-201 re-expressed on the FastVGICPCuda mirror: forward, backward, swap+setSource, swap+setTarget."""
    from fast_gicp_b200 import FastVGICPCuda

    target, source = pair02
    t_tol, r_tol = 0.05, np.radians(1.0)

    reg = FastVGICPCuda()
    reg.setInputTarget(target)
    reg.setInputSource(source)
    T = reg.align()
    e = pose_error(relative_pose, T)
    assert e[0] < t_tol and e[1] < r_tol and reg.hasConverged(), "FORWARD TEST"

    reg.setInputTarget(source)
    reg.setInputSource(target)
    T = reg.align()
    e = pose_error(relative_pose, np.linalg.inv(T.astype(np.float64)))
    assert e[0] < t_tol and e[1] < r_tol and reg.hasConverged(), "BACKWARD TEST"

    reg = FastVGICPCuda()
    reg.setInputSource(target)
    reg.swapSourceAndTarget()
    reg.setInputSource(source)
    T = reg.align()
    e = pose_error(relative_pose, T)
    assert e[0] < t_tol and e[1] < r_tol and reg.hasConverged(), "SWAP AND SET SOURCE TEST"

    reg = FastVGICPCuda()
    reg.setInputTarget(source)
    reg.swapSourceAndTarget()
    reg.setInputTarget(target)
    T = reg.align()
    e = pose_error(relative_pose, T)
    assert e[0] < t_tol and e[1] < r_tol and reg.hasConverged(), "SWAP AND SET TARGET TEST"


# ------------------------------------------------------------------------------------------------------- edge cases
def test_error_states_and_edge_cases():
    from fast_gicp_b200.core import Core, VgicpError, ERR_BAD_STATE, ERR_INVALID_ARGUMENT

    c = Core(0)
    with pytest.raises(VgicpError) as e:
        c.find_source_neighbors(20)
    assert e.value.code == ERR_BAD_STATE
    with pytest.raises(VgicpError) as e:
        c.create_target_voxelmap()
    assert e.value.code == ERR_BAD_STATE
    with pytest.raises(VgicpError) as e:
        c.compute_error(np.eye(4))
    assert e.value.code == ERR_BAD_STATE
    pts = np.random.default_rng(0).uniform(-5, 5, (10, 3)).astype(np.float32)
    c.set_source_cloud(pts)
    with pytest.raises(VgicpError) as e:
        c.find_source_neighbors(20)  # k > n
    assert e.value.code == ERR_INVALID_ARGUMENT
    with pytest.raises(VgicpError) as e:
        c.set_source_neighbors(3, np.zeros(7, dtype=np.int32))  # k*n mismatch (the reference asserts)
    assert e.value.code == ERR_INVALID_ARGUMENT
    with pytest.raises(VgicpError) as e:
        c.set_neighbor_search_method(17)  # the reference abort()s
    assert e.value.code == ERR_INVALID_ARGUMENT
    c.set_target_cloud(np.zeros((0, 3), dtype=np.float32))  # empty cloud accepted, map refused
    assert c.num_target_points() == 0
    # strided input (pcl::PointXYZI = 32 bytes/pt)
    rec = np.zeros((10, 8), dtype=np.float32)
    rec[:, :3] = pts
    c.set_source_cloud(rec)
    c.find_source_neighbors(5)
    assert np.array_equal(c.get_source_neighbors(), O.knn(pts, 5, "bruteforce"))
    c.close()


def test_source_outside_map_gives_zero_system(prepared):
    """No correspondences (source far away from every voxel): H = 0, b = 0, err = 0."""
    from fast_gicp_b200.core import Core

    c = Core(0)
    _setup_pair(c, prepared, O.DIRECT7)
    T = np.eye(4)
    T[:3, 3] = [1000.0, 1000.0, 1000.0]
    err, H, b = c.linearize(T)
    assert err == 0.0 and not H.any() and not b.any()
    assert len(c.get_voxel_correspondences()) == 0
    c.close()


# ----------------------------------------------------------------------------- other BASELINE configs as parity cases
def test_c3_synthetic_kitti_pair_matches_oracle():
    """BASELINE config 3 shape (synthetic HDL-64 pair, 0.25 m downsample, ~23k pts): whole registration vs the oracle and vs
    the generator's ground-truth motion."""
    from fast_gicp_b200.core import Core, pose_from_c
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=64, az_steps=2083, seed=42, pose=(0.8, 0.05, 0.7), downsample=0.25)
    c = Core(0)
    _setup_pair(c, dict(tgt=tgt, src=src), O.DIRECT27)
    res = c.align()
    T = pose_from_c(res.T)
    ref = O.register_f32(tgt, src, method=O.DIRECT27, accum_double=True)
    dt, dr = pose_error(ref.T, T)
    assert res.converged and ref.converged and dt < TRANS_TOL and dr < ROT_TOL, (dt, dr)
    gt_t, gt_r = pose_error(T_gt, T)
    assert gt_t < 0.05 and gt_r < np.radians(0.5), (gt_t, gt_r)
    c.close()


def test_large_cloud_size_independent_properties():
    """C4-sized inputs (1M points) cannot be checked against the CPU oracle in seconds; check properties that do not depend on
    size: every point is its own nearest neighbour, neighbour rows are sorted by distance and duplicate-free, spot-checked rows
    equal a brute-force scan, the voxel map conserves the points, H is symmetric positive definite, an evaluation under the
    latency and the throughput execution hints agrees, and the registration recovers the generator's motion."""
    from fast_gicp_b200.core import Core, pose_from_c
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
    c = Core(0)
    c.set_resolution(0.5)
    c.set_neighbor_search_method("DIRECT27")
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    nbr = c.get_target_neighbors()
    assert np.array_equal(nbr[:, 0], np.arange(len(tgt)))  # self first (d2 = 0; duplicates tie-break by index)
    rng = np.random.default_rng(0)
    rows = rng.choice(len(tgt), 400, replace=False)
    p64 = tgt.astype(np.float64)
    for i in rows:
        d2 = ((p64[nbr[i]] - p64[i]) ** 2).sum(axis=1)
        assert np.all(np.diff(d2) >= -1e-9) and len(set(nbr[i].tolist())) == 20
    for i in rows[:25]:  # exact rows against a full scan (float32 distance semantics of the kernel)
        d = tgt - tgt[i]
        dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        want = np.lexsort((np.arange(len(tgt)), dd))[:20]
        assert np.array_equal(nbr[i], want)
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()
    n_vox = c.get_voxel_num_points()
    # the reference's rule (gaussian_voxelmap.cu:265-285, SURVEY Q5): voxels that find no slot within 10 probes are dropped, the
    # table only grows while >= 1% of the POINTS fail -> at most 1% of the points are missing, every kept voxel is populated
    assert 0.99 * len(tgt) < n_vox.sum() <= len(tgt) and n_vox.min() >= 1
    coords, ids = c.get_voxel_buckets()
    uniq = np.unique(O.voxel_coords(tgt, 0.5), axis=0)
    assert (ids >= 0).sum() == c.num_voxels() <= len(uniq)
    kept = {tuple(x) for x in coords[ids >= 0].tolist()}
    assert kept <= {tuple(x) for x in uniq.tolist()}  # every bucket holds a real voxel of the cloud
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)
    e1, H1, b1 = c.linearize(np.eye(4))
    assert np.array_equal(H1, H1.T) and np.all(np.linalg.eigvalsh(H1) > 0)
    c.set_execution_hint(1)
    e2, H2, b2 = c.linearize(np.eye(4))
    c.set_execution_hint(0)
    assert abs(e1 - e2) <= 1e-6 * abs(e1) and np.abs(H1 - H2).max() <= 1e-6 * np.abs(H1).max()
    res = c.align()
    gt_t, gt_r = pose_error(T_gt, pose_from_c(res.T))
    assert res.converged and gt_t < 0.02 and gt_r < np.radians(0.2), (gt_t, gt_r)
    c.close()


def test_c4_matches_the_oracle_golden():
    """BASELINE config 4 (synthetic 1M-pt pair, seeds 44/45, res 0.5) against the oracle's committed outputs
    (tests/golden/c4_golden.json, written by tests/golden/make_c4_golden.py): both 1M x 20 k-NN tables and the regularised
    covariances by SHA-256, the voxel table (buckets, ids, point counts) by SHA-256, one evaluation at the identity and at the
    ground-truth pose (DIRECT27 and DIRECT1) and the whole registration at the north-star tolerance with identical counters."""
    import hashlib
    import json
    import os

    from conftest import GOLDEN
    from fast_gicp_b200.core import Core, pose_from_c
    from fast_gicp_b200.synthetic import kitti_like_pair

    def sha(a):
        return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()

    g = json.load(open(os.path.join(GOLDEN, "c4_golden.json")))
    tgt, src, T_gt = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
    assert (len(tgt), len(src)) == (g["n_target"], g["n_source"]) and sha(tgt) == g["sha_target"] and sha(src) == g["sha_source"]
    c = Core(0)
    c.set_resolution(g["res"])
    c.set_target_cloud(tgt)
    c.find_target_neighbors(g["k"])
    assert sha(c.get_target_neighbors().astype(np.int32)) == g["sha_knn_target"]
    c.calculate_target_covariances(O.REG_PLANE)
    assert sha(c.get_target_covariances()) == g["sha_cov_target"]
    c.create_target_voxelmap()
    assert c.num_buckets() == g["num_buckets"] and c.num_voxels() == g["num_voxels"]
    coords, ids = c.get_voxel_buckets()
    assert sha(coords) == g["sha_bucket_coord"] and sha(ids) == g["sha_bucket_id"]
    assert sha(c.get_voxel_num_points()) == g["sha_voxel_num_points"] and sha(c.get_voxel_means()) == g["sha_voxel_means"]
    c.set_source_cloud(src)
    c.find_source_neighbors(g["k"])
    assert sha(c.get_source_neighbors().astype(np.int32)) == g["sha_knn_source"]
    c.calculate_source_covariances(O.REG_PLANE)
    assert sha(c.get_source_covariances()) == g["sha_cov_source"]
    for name in ("DIRECT27", "DIRECT1"):
        c.set_neighbor_search_method(name)
        rec = g[name]
        for pname, T in (("identity", np.eye(4)), ("gt", np.array(g["T_gt"]))):
            err, H, b = c.linearize(T)
            H0, b0, e0 = np.array(rec[pname]["H"]), np.array(rec[pname]["b"]), rec[pname]["err"]
            assert len(c.get_voxel_correspondences()) == rec[pname]["n_correspondences"]
            assert abs(err - e0) <= 2e-5 * abs(e0), (name, pname)
            assert np.abs(H - H0).max() <= 2e-5 * np.abs(H0).max(), (name, pname)
            assert np.abs(b - b0).max() <= 2e-5 * max(np.abs(b0).max(), 1e-3 * np.abs(H0).max()), (name, pname)
        res = c.align()
        a = rec["align"]
        dt, dr = pose_error(np.array(a["T"]), pose_from_c(res.T))
        assert res.converged and a["converged"] and dt < TRANS_TOL and dr < ROT_TOL, (name, dt, dr)
        assert (res.nr_iterations, res.n_linearize, res.n_compute_error) == (a["iterations"], a["n_linearize"], a["n_error"]), name
    c.close()


def test_direct1_streaming_kernel_matches_the_gather_kernel():
    """DIRECT1 evaluations of clouds >= 64k points run in k_linearize_stream (source staged through shared memory by bulk copies);
    it reads the direct-mapped voxel index, so with the hash table alone (set_voxel_index(1)) the ordinary kernel runs.  The two
    indexes return the same voxel ids (test_correspondences_and_linear_system).  Same correspondences, same per-term arithmetic,
    another summation order: err, H, b agree to float rounding, the registration walks the same iterates, and both match the oracle."""
    from fast_gicp_b200.core import Core, pose_from_c
    from fast_gicp_b200.synthetic import kitti_like_pair

    tgt, src, T_gt = kitti_like_pair(beams=64, az_steps=2083, seed=7, pose=(0.6, 0.1, 0.8), downsample=0.0)
    assert len(src) > 65536
    got = {}
    for stream in (True, False):
        c = Core(0)
        c.set_voxel_index(0 if stream else 1)  # the hash table alone keeps the ordinary kernel
        _setup_pair(c, dict(tgt=tgt, src=src), O.DIRECT1, res=0.5)
        rows = []
        for T in (np.eye(4), T_gt):
            c.update_correspondences(T)
            rows.append(c.compute_error(T, True) + c.compute_error(T, False)[:1])
        res = c.align()
        got[stream] = (rows, pose_from_c(res.T), res.nr_iterations, res.n_linearize, res.n_compute_error, bool(res.converged))
        if stream:
            cov_t, cov_s = c.get_target_covariances(), c.get_source_covariances()
        c.close()
    for (e1, H1, b1, eo1), (e0, H0, b0, eo0) in zip(got[True][0], got[False][0]):
        assert abs(e1 - e0) <= 2e-6 * abs(e0) and abs(eo1 - eo0) <= 2e-6 * abs(eo0)
        assert np.abs(H1 - H0).max() <= 2e-6 * np.abs(H0).max() and np.abs(b1 - b0).max() <= 2e-6 * max(np.abs(b0).max(), 1e-3 * np.abs(H0).max())
    assert got[True][2:] == got[False][2:] and got[True][5]
    dt, dr = pose_error(got[False][1], got[True][1])
    assert dt < 1e-6 and dr < 1e-7, (dt, dr)
    vm = O.VoxelMap(tgt, cov_t, 0.5, accum_double=True)
    e0, H0, b0, _ = O.evaluate(vm, src, cov_s, O.offsets(O.DIRECT1), T_gt, T_gt, True)
    e1, H1, b1, _ = got[True][0][1]
    assert abs(e1 - e0) <= 2e-5 * abs(e0) and np.abs(H1 - H0).max() <= 2e-5 * np.abs(H0).max()


def test_caller_supplied_covariances(prepared, relative_pose):
    """vgicp_set_{source,target}_covariances (FastGICP::setSourceCovariances / setTargetCovariances on the CUDA path): feeding the
    oracle's covariances gives the oracle's voxel map and linear system; the size is checked."""
    from fast_gicp_b200.core import ERR_INVALID_ARGUMENT, Core, VgicpError

    c = Core(0)
    c.set_neighbor_search_method(O.DIRECT7)
    c.set_target_cloud(prepared["tgt"])
    c.set_target_covariances(prepared["t_cov"])
    c.create_target_voxelmap()
    c.set_source_cloud(prepared["src"])
    c.set_source_covariances(prepared["s_cov"])
    assert np.array_equal(c.get_source_covariances(), sym(prepared["s_cov"]).astype(np.float32))
    vm = O.VoxelMap(prepared["tgt"], sym(prepared["t_cov"]).astype(np.float32), 1.0, accum_double=True)
    assert np.array_equal(c.get_voxel_means(), vm.vox_mean) and np.array_equal(c.get_voxel_covs(), vm.vox_cov)
    err, H, b = c.linearize(relative_pose)
    e0, H0, b0, _ = O.evaluate(vm, prepared["src"], sym(prepared["s_cov"]).astype(np.float32), O.offsets(O.DIRECT7), relative_pose, relative_pose, True)
    assert abs(err - e0) <= 2e-5 * abs(e0) and np.abs(H - H0).max() <= 2e-5 * np.abs(H0).max()
    with pytest.raises(VgicpError) as e:
        c.set_source_covariances(prepared["s_cov"][:-1])
    assert e.value.code == ERR_INVALID_ARGUMENT
    c.close()


def test_abi_guards_added_in_round_2(prepared):
    """set_*_neighbors rejects an index outside the cloud (it would be an illegal address in the covariance kernel and poison the
    context of every handle of the process); vgicp_register carries on after NORMALIZED_MIN_EIG like the class wrappers do (the
    reference prints "unimplemented ..." and keeps the raw covariances, covariance_regularization.cu:121-123)."""
    from fast_gicp_b200.core import ERR_INVALID_ARGUMENT, Core, VgicpError

    c = Core(0)
    c.set_source_cloud(prepared["src"])
    bad = prepared["s_nbr"].copy()
    bad[123, 7] = len(prepared["src"])
    with pytest.raises(VgicpError) as e:
        c.set_source_neighbors(20, bad)
    assert e.value.code == ERR_INVALID_ARGUMENT
    bad[123, 7] = -1
    with pytest.raises(VgicpError):
        c.set_source_neighbors(20, bad)
    c.set_source_neighbors(20, prepared["s_nbr"])  # the handle is still usable
    c.calculate_source_covariances(O.REG_NONE)
    assert np.array_equal(c.get_source_covariances(), prepared["s_raw"])
    r = c.register(prepared["tgt"], prepared["src"], reg=O.REG_NORMALIZED_MIN_EIG)
    assert r.nr_iterations >= 0  # ran to the end with the raw covariances instead of failing on VGICP_ERR_UNSUPPORTED
    c.close()


def test_ndt_maps_are_kept_like_the_reference(pair02):
    """NDTCudaCore::create_{source,target}_voxelmap return early when the map exists (ndt_cuda.cu:123-141): a second create (or a
    second align) neither rebuilds the maps nor picks up a new resolution; set_*_cloud resets that cloud's map only."""
    from fast_gicp_b200.core import Core

    tgt, src = pair02
    c = Core(0)
    c.set_problem(2)
    c.set_resolution(1.0)
    c.set_target_cloud(tgt)
    c.set_source_cloud(src)
    c.ndt_create_voxelmaps()
    v1, n0 = c.num_voxels(), c.launch_count()
    c.set_resolution(0.5)
    c.ndt_create_voxelmaps()  # both maps exist: nothing happens
    assert c.num_voxels() == v1 and c.launch_count() == n0
    c.set_target_cloud(tgt)   # resets the target map: rebuilt with the resolution current now
    c.ndt_create_voxelmaps()
    assert c.num_voxels() > v1
    assert c.num_voxels() == O.VoxelMap(tgt, None, 0.5, accum_double=True).num_voxels
    c.close()


def _rbf_cloud():
    rng = np.random.default_rng(2)
    pts = (rng.normal(size=(1500, 3)) * [3.0, 3.0, 0.2]).astype(np.float32)
    pts[::7] += np.float32(40.0)  # a second sheet far from the origin: the padding points at the origin stay out of its range
    return pts


@pytest.mark.parametrize("method", [O.REG_NONE, O.REG_PLANE, O.REG_MIN_EIG, O.REG_FROBENIUS])
def test_rbf_covariances_bit_exact(method):
    """GPU_RBF_KERNEL mode, calculate_*_covariances_rbf (fast_vgicp_cuda.cu:205-219 -> covariance_estimation_rbf.cu:59-151 +
    covariance_regularization.cu): same 512-point block structure, zero padding, summation order and (double-evaluated) weight as the
    oracle restatement -> bit-for-bit; the GPU stores the symmetric part.  One point may differ by a double-rounding tie of exp."""
    from fast_gicp_b200.core import Core

    pts = _rbf_cloud()
    c = Core(0)
    for kw, md in ((0.5, 3.0), (0.25, 1.25)):
        c.set_kernel_params(kw, md)
        c.set_source_cloud(pts)
        c.calculate_source_covariances_rbf(method)
        got = c.get_source_covariances()
        raw = O.covariances_rbf(pts, kw, md)
        want = sym(raw if method == O.REG_NONE else O.regularize(raw, method)).astype(np.float32)
        bad = np.flatnonzero((got != want).any(axis=1))
        assert len(bad) <= 1, (method, kw, len(bad), np.abs(got - want).max())
        # target side: same kernel
        c.set_target_cloud(pts)
        c.calculate_target_covariances_rbf(method)
        assert np.array_equal(c.get_target_covariances(), got)
    c.close()


@pytest.mark.parametrize("method", [O.DIRECT1, O.DIRECT27])
def test_align_rbf_mode_matches_oracle(pair02, relative_pose, method):
    """Whole registration with NearestNeighborMethod::GPU_RBF_KERNEL (fast_vgicp_cuda_impl.hpp:96-108,125-140: RBF covariances for
    both clouds, PLANE) through the reference-facing class, against the oracle run the same way: same iterates, north-star pose
    tolerance, and the reference's own gate against data/relative.txt."""
    from fast_gicp_b200 import FastVGICPCuda
    from fast_gicp_b200.registration import NearestNeighborMethod

    tgt, src = pair02
    reg = FastVGICPCuda()
    reg.setResolution(1.0)
    reg.setNeighborSearchMethod(method, 0.0)
    reg.setNearestNeighborSearchMethod(NearestNeighborMethod.GPU_RBF_KERNEL)
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    reg.align()
    T = np.asarray(reg.getFinalTransformation(), dtype=np.float64)
    ref = O.register_f32(tgt, src, method=method, knn_method="rbf", kernel_width=0.5, max_dist=3.0, accum_double=True, symmetrize=True)
    assert reg.hasConverged() and ref.converged
    dt, dr = pose_error(ref.T, T)
    # getFinalTransformation() is the float image of the pose (pcl::Registration keeps Matrix4f): 1e-7 relative on a ~0.5 m translation
    assert dt < TRANS_TOL and dr < ROT_TOL, (dt, dr)
    gt_t, gt_r = pose_error(relative_pose, T)
    assert gt_t < 0.05 and gt_r < np.radians(1.0), (gt_t, gt_r)


# ----------------------------------------------------------------------------- getFitnessScore (SURVEY 8f-3)
def test_fitness_score_against_kdtree(prepared, relative_pose):
    """pcl::Registration::getFitnessScore(max_range): mean squared nearest-neighbour distance of the transformed source over the
    pairs with d^2 <= max_range (PCL compares the SQUARED distance with max_range)."""
    from scipy.spatial import cKDTree

    from fast_gicp_b200.core import Core

    c = Core(0)
    c.set_target_cloud(prepared["tgt"])
    c.set_source_cloud(prepared["src"])
    tree = cKDTree(prepared["tgt"].astype(np.float64))
    for T in (np.eye(4), relative_pose):
        Tf = T.astype(np.float32)
        p = (prepared["src"].astype(np.float32) @ Tf[:3, :3].T + Tf[:3, 3]).astype(np.float64)
        d, _ = tree.query(p, k=1)
        d2 = d * d
        assert abs(c.fitness_score(T) - d2.mean()) <= 1e-4 * d2.mean()
        for max_range in (0.05, 0.5):
            m = d2 <= max_range
            assert abs(c.fitness_score(T, max_range) - d2[m].mean()) <= 1e-3 * d2[m].mean()
    c.close()
