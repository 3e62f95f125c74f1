"""The float64 stage-1 and voxel references (cov_reference.py) against the CPU oracle, the comparator against deliberately wrong
variants, and the eig3_direct branches that the GPU stage-1 matrix (test_gpu_stage1_matrix.py) reaches.  CPU only.

The worst ratio |x - x_ref| / scale of every quantity, the rejection count of every wrong variant and the count of every branch
label are printed (outside pytest's capture) as the tests run."""
import numpy as np
import pytest

import oracle as O
import cov_reference as R

REGS = [(O.REG_MIN_EIG, "MIN_EIG"), (O.REG_PLANE, "PLANE"), (O.REG_FROBENIUS, "FROBENIUS")]


def report(capsys, text):
    with capsys.disabled():
        print(f"\n  [cov_reference] {text}", end="")


@pytest.fixture(scope="module")
def spectra():
    return R.spectrum_set()


@pytest.fixture(scope="module")
def knn_inputs():
    """{k: (pts, nbr, kind, the oracle's raw covariances)}: the hand-built neighbourhoods the GPU matrix uses."""
    out = {}
    for k in R.KNN_KS:
        pts, nbr, kind = R.knn_neighbourhoods(k)
        out[k] = (pts, nbr, kind, O.covariances(pts, nbr))
    return out


def _eig3_oracle(c9):
    ev, V = zip(*(O.eig3_direct(c) for c in c9))
    return np.array(ev), np.array(V)


# ---------------------------------------------------------------------------------------------------------------- reference vs oracle
def test_raw_knn_reference_matches_the_oracle(knn_inputs, capsys):
    worst = {}
    for k, (pts, nbr, kind, raw) in knn_inputs.items():
        ref, sc = R.raw_knn64(pts, nbr)
        r, bad = R.check(R.mat(raw), ref, sc, R.TAU_RAW)
        assert not len(bad), (k, kind[bad][:5], r[bad][:5])
        worst[k] = r.max()
    report(capsys, f"raw k-NN covariance: worst |x - x_ref| / ((k + 4) eps A) per k: " + ", ".join(f"k={k}: {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("method,name", REGS)
def test_regulariser_references_match_the_oracle(spectra, knn_inputs, method, name, capsys):
    worst = {}
    sets = [("spectra", spectra)] + [(f"k={k}", v[3]) for k, v in knn_inputs.items()]
    for what, raw in sets:
        for q, v in R.assert_regularised(method, raw, O.regularize(raw, method), what).items():
            worst[q] = max(worst.get(q, 0.0), v)
    report(capsys, f"{name}: worst ratio over {sum(len(s) for _, s in sets)} matrices: " + ", ".join(f"{q} {v:.3g}" for q, v in worst.items()))


@pytest.mark.parametrize("kw,md", [(0.5, 3.0), (0.25, 1.25)])
def test_rbf_reference_matches_the_oracle(kw, md, capsys):
    pts = R.lidar_scan(1500, seed=3)
    raw = O.covariances_rbf(pts, kw, md)
    q = np.unique(np.concatenate([np.arange(0, len(pts), 7), np.flatnonzero(R.in_range32(np.zeros(3, np.float32), pts, md))]))
    ref, sc = R.rbf64(pts, q, kw, md)
    r, bad = R.check(R.sym(raw[q]), ref, sc, R.TAU_RBF)
    assert not len(bad), (q[bad][:5], r[bad][:5])
    report(capsys, f"RBF ({kw}, {md}): worst ratio {r.max():.3g} over {len(q)} queries")


@pytest.mark.parametrize("res", [0.1, 0.5, 1.0])
def test_voxel_references_match_the_oracle(res, capsys):
    pts, cov = R.voxel_cloud(res)
    for ndt in (False, True):
        vm = O.VoxelMap(pts, None if ndt else cov, res, accum_double=True)
        ref = R.voxels64(pts, res, None if ndt else cov)
        ids = R.match_voxels(ref["coords"], vm.bucket_coord, vm.bucket_id)
        assert (ids >= 0).all() and np.array_equal(vm.vox_n[ids], ref["n"])
        n = ref["n"]
        assert all((n == m).sum() >= 20 for m in (1, 2, 3, 4)) and (n == 33).any() and n.max() >= 10000
        r = np.linalg.norm(ref["mean"], axis=1)
        assert all(((r > 0.99 * d) & (r < 1.01 * d)).sum() >= 5 for d in (1e3, 1e4))
        rm, bad = R.check(vm.vox_mean[ids][:, :, None], ref["mean"][:, :, None], ref["mean_scale"][:, :, None], R.TAU_VOXEL)
        assert not len(bad), ("mean", ndt, n[bad][:5])
        rc, bad = R.check(R.sym(vm.vox_cov[ids]), ref["cov"], ref["cov_scale"], R.TAU_VOXEL)
        assert not len(bad), ("cov", ndt, n[bad][:5], rc[bad][:5])
        report(capsys, f"{'NDT' if ndt else 'VGICP'} voxels at res {res}: {len(n)} voxels, worst ratio mean {rm.max():.3g}, covariance {rc.max():.3g}")


# ---------------------------------------------------------------------------------------------------------------- wrong variants
def assert_rejected(capsys, what, right, wrong):
    """right, wrong: (ratio, failing rows) of check(); the unmutated values pass, the mutated ones fail somewhere."""
    assert not len(right[1]), f"{what}: the unmutated values must pass ({len(right[1])} rows fail)"
    assert len(wrong[1]), f"{what}: the wrong variant passed"
    report(capsys, f"wrong variant rejected: {what} ({len(wrong[1])} of {len(wrong[0])} inputs)")


def test_plane_on_the_largest_eigenvector_is_rejected(spectra, capsys):
    p = R.plane64(spectra)
    det = np.flatnonzero(p["determined"])
    _, V = _eig3_oracle(spectra[det])
    v2 = V[:, :, 2].astype(np.float64)
    wrong = np.eye(3) - 0.999 * v2[:, :, None] * v2[:, None, :]
    right = R.check(R.sym(O.regularize(spectra[det], O.REG_PLANE)), p["ref"][det], p["scale"][det], R.TAU_PLANE)
    assert_rejected(capsys, "PLANE built on the eigenvector of lambda_max", right, R.check(wrong, p["ref"][det], p["scale"][det], R.TAU_PLANE))


def test_min_eig_clamped_relative_to_lambda_max_is_rejected(spectra, capsys):
    ev, V = _eig3_oracle(spectra)
    ev, V = ev.astype(np.float64), V.astype(np.float64)
    lam = np.maximum(1e-3 * ev.max(axis=1, keepdims=True), ev)
    wrong = np.einsum("nij,nj,njk->nik", V, lam, np.linalg.inv(V))
    ref, sc = R.min_eig64(spectra)
    right = R.check(R.sym(O.regularize(spectra, O.REG_MIN_EIG)), ref, sc, R.TAU_MIN_EIG)
    assert_rejected(capsys, "MIN_EIG clamped at 1e-3 lambda_max", right, R.check(wrong, ref, sc, R.TAU_MIN_EIG))


def test_frobenius_without_the_shift_is_rejected(spectra, capsys):
    C = R.lower(spectra)
    s = np.linalg.svd(C, compute_uv=False)
    ok = s[:, 2] > 1e-4 * s[:, 0]  # invertible without the shift: the wrong variant is finite there
    Ci = np.linalg.inv(C[ok])
    wrong = np.sqrt((Ci * Ci).sum(axis=(1, 2)))[:, None, None] * C[ok]
    ref, sc = R.frobenius64(spectra[ok])
    right = R.check(R.sym(O.regularize(spectra[ok], O.REG_FROBENIUS)), ref, sc, R.TAU_FROBENIUS)
    assert_rejected(capsys, "FROBENIUS without + 1e-3 I", right, R.check(wrong, ref, sc, R.TAU_FROBENIUS))


def test_raw_covariance_normalised_by_k_minus_1_is_rejected(knn_inputs, capsys):
    right_r, wrong_r, right_b, wrong_b = [], [], [], []
    for k, (pts, nbr, _, raw) in knn_inputs.items():
        if k < 2:
            continue
        ref, sc = R.raw_knn64(pts, nbr)
        r = R.check(R.mat(raw), ref, sc, R.TAU_RAW)
        w = R.check(R.mat(raw).astype(np.float64) * k / (k - 1), ref, sc, R.TAU_RAW)
        right_r.append(r[0]), right_b.append(r[1]), wrong_r.append(w[0]), wrong_b.append(w[1])
    assert_rejected(capsys, "raw covariance normalised by k - 1", (np.concatenate(right_r), np.concatenate(right_b)),
                    (np.concatenate(wrong_r), np.concatenate(wrong_b)))


def test_rbf_without_the_origin_padding_is_rejected(capsys):
    pts = R.lidar_scan(1500, seed=3)
    kw, md = 0.5, 3.0
    q = np.flatnonzero(R.in_range32(np.zeros(3, np.float32), pts, md))  # the queries the padding reaches
    assert len(q) >= 5
    ref, sc = R.rbf64(pts, q, kw, md)
    wrong, _ = R.rbf64(pts, q, kw, md, pad=False)
    right = R.check(R.sym(O.covariances_rbf(pts, kw, md)[q]), ref, sc, R.TAU_RBF)
    assert_rejected(capsys, "RBF without the origin padding", right, R.check(wrong, ref, sc, R.TAU_RBF))


def test_ndt_covariance_normalised_by_n_minus_1_is_rejected(capsys):
    pts, _ = R.voxel_cloud(0.5)
    ref = R.voxels64(pts, 0.5)
    vm = O.VoxelMap(pts, None, 0.5, accum_double=True)
    ids = R.match_voxels(ref["coords"], vm.bucket_coord, vm.bucket_id)
    n = ref["n"]
    sel = n >= 2
    raw = ref["raw"][sel] * (n[sel] / (n[sel] - 1))[:, None, None]
    wrong, _ = R.min_eig64(raw.transpose(0, 2, 1).reshape(-1, 9))
    right = R.check(R.sym(vm.vox_cov[ids][sel]), ref["cov"][sel], ref["cov_scale"][sel], R.TAU_VOXEL)
    assert_rejected(capsys, "NDT covariance normalised by n - 1", right, R.check(wrong, ref["cov"][sel], ref["cov_scale"][sel], R.TAU_VOXEL))


def test_vgicp_mean_without_the_last_point_is_rejected(capsys):
    pts, cov = R.voxel_cloud(0.5)
    ref = R.voxels64(pts, 0.5, cov)
    vm = O.VoxelMap(pts, cov, 0.5, accum_double=True)
    ids = R.match_voxels(ref["coords"], vm.bucket_coord, vm.bucket_id)
    n = ref["n"]
    last = np.full(len(n), -1)
    np.maximum.at(last, ref["inv"], np.arange(len(pts)))
    sel = n >= 2
    P = pts.astype(np.float64)
    wrong = (ref["mean"][sel] * n[sel, None] - P[last[sel]]) / (n[sel, None] - 1)
    right = R.check(vm.vox_mean[ids][sel][:, :, None], ref["mean"][sel][:, :, None], ref["mean_scale"][sel][:, :, None], R.TAU_VOXEL)
    assert_rejected(capsys, "VGICP voxel mean without the voxel's last point", right,
                    R.check(wrong[:, :, None], ref["mean"][sel][:, :, None], ref["mean_scale"][sel][:, :, None], R.TAU_VOXEL))


# ---------------------------------------------------------------------------------------------------------------- RBF paths
def test_sorted_rbf_clouds_reach_the_block_skip_and_the_padding(capsys):
    """The azimuth-ordered clouds of the GPU matrix, computed from the same float block boxes as the kernel: more than half of the
    (query, block) pairs are skipped, and in the padded cases some queries pick up weight from the origin padding and some do not."""
    pairs = skipped = 0
    lines = []
    reached = unreached = 0
    for n in R.RBF_NS:
        pts = R.lidar_scan(n, seed=n)
        nb = (n + R.RBF_BLOCK - 1) // R.RBF_BLOCK
        for kw, md in R.RBF_SETTINGS:
            frac, near = R.rbf_paths(pts, md)
            pairs += n * nb
            skipped += frac * n * nb
            if n % R.RBF_BLOCK:
                reached += near
                unreached += n - near
            lines.append(f"n={n} md={md}: skipped {frac:.2f}, padding reaches {near}")
    report(capsys, "sorted RBF clouds: " + "; ".join(lines) + f"; all: skipped {skipped / pairs:.3f} of {pairs} pairs")
    assert skipped / pairs > 0.5
    assert reached > 0 and unreached > 0


# ---------------------------------------------------------------------------------------------------------------- eig3 branches
def test_eig3_branches_reached_by_the_gpu_inputs(spectra, knn_inputs, capsys):
    """The restatement of eig3_direct's shift, scale and computeRoots reproduces the oracle's eigenvalues bit for bit; its branch
    labels, applied to the raw covariances the GPU matrix sends through the regularisers, reach every branch at least 20 times
    (counted as distinct matrices)."""
    counts = {lab: 0 for lab in R.EIG3_LABELS}
    for what, c9 in [("spectra", spectra)] + [(f"k={k}", v[3]) for k, v in knn_inputs.items()]:
        c9 = np.unique(c9, axis=0)
        ev, labels = R.eig3_branches(c9)
        ev_o, _ = _eig3_oracle(c9)
        assert np.array_equal(ev.view(np.int32), ev_o.astype(np.float32).view(np.int32)), what
        if what != "spectra":
            for lab, m in labels.items():
                counts[lab] += int(m.sum())
    report(capsys, "eig3_direct branches reached by the k-NN neighbourhoods: " + ", ".join(f"{lab}: {c}" for lab, c in counts.items()))
    assert all(c >= 20 for c in counts.values()), counts
