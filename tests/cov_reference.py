"""Float64 references of stage 1 (per-point covariances, their regularisers) and of the voxel Gaussians, in plain numpy, each with
the scale that the float computation's error is measured against; plus the inputs that test_cov_reference.py (CPU) and
test_gpu_stage1_matrix.py (GPU) share.

Every reference takes the float32 inputs the float code received and returns float64 results.  A comparison is per entry:
|x - x_ref| <= tau * scale, with scale derived below from the operations the float code performs and tau a constant calibrated on
the oracle (oracle/vgicp_oracle.c) and stated next to the comparator that uses it.  eps = 2^-23 (float32 machine epsilon), u = eps/2.

Raw k-NN covariance (k_covariance_knn, orc_covariances): the kernel sums S_rc = sum fma(p_r, p_c, S_rc) and s_r = sum p_r over the k
rows in float, then C_rc = fma(-mu_r, mu_c, S_rc / k) with mu = s / k.  Each running sum has an error <= k u sum|.| of its terms, the
divisions and the final fma one rounding each, and the error of mu_r enters through mu_c.  So
    |C - C_ref| <= (k + 4) eps * A,   A_rc = mean|p_r p_c| + mean|p_r| |mu_c| + |mu_r| mean|p_c|.
A is the cancellation scale of the one-pass formula: far from the origin (|p| = 1e4 m, spread 0.3 m) it is 1e8 times the covariance.
(The cross terms mean|p_r| |mu_c| bound the error the mean carries into mu_r mu_c; |mu_r mu_c| alone does not when p_c is non-zero
only where p_r is zero.)

Regularisers (regularize_cov + eig3_direct, orc_regularize) take the float32 raw covariance the kernel used (its lower triangle, as
selfadjointView<Lower> reads it), so their bounds are separate from the raw one.  lambda_0 <= lambda_1 <= lambda_2 are the float64
eigenvalues of that matrix, spread = lambda_2 - lambda_0, lmax = max(|lambda|).
  MIN_EIG  ref = V diag(max(1e-3, lambda)) V^T.  eig3_direct shifts by trace/3 and scales by max|s_ij| (the shift is subtracted
           again from the same float, so its rounding moves all eigenvalues alike), takes the cubic's roots by the trigonometric
           formula and rescales: each eigenvalue is good to about eps * lmax, except where two roots are close.  At a gap delta the
           roots come from q = a^3 - b^2, which cancels: the root error is eps * spread * min(spread / delta, eps^-1/2) (at a double
           root, sqrt(eps) * spread).  The clamp does not hide that error even for a pair of eigenvalues below 1e-3: on an exact
           line (0, 0, 30) the computed double root lands at sqrt(eps) * 30 = 0.01, above the clamp.  Eigenvector errors
           eps * spread / delta_ij rotate within a pair whose reconstructed values differ by delta_ij: eps * spread again.
           scale = eps * (max(lmax, 1e-3) + spread * min(spread / delta, eps^-1/2)), delta = the smaller of the two gaps.
  FROBENIUS ref = ||M^-1||_F M with M = C + 1e-3 I: two cofactor inversions, each with a relative error of about cond(M) eps, the
           second one amplifying the first's by cond(M) again.  scale = eps * cond(M)^2 * ||ref||_2.
  PLANE    ref = I - 0.999 n n^T, n the eigenvector of lambda_0.  n is determined to eps * spread / (lambda_1 - lambda_0) (the
           rounding of the shifted, scaled matrix is relative to the spread, the shift cancels), the rebuild V diag V^-1 adds a few
           eps: scale = eps * (1 + spread / (lambda_1 - lambda_0)) where lambda_1 - lambda_0 > 1e-3 spread.  Elsewhere the normal is
           not determined (lines, prolate sets, isotropic and zero covariances) and the result is held to what is: its eigenvalues are
           (1e-3, 1, 1), and its normal lies in the eigenspace of the small eigenvalues, |n . v_2| <= tau eps (1 + spread /
           (lambda_2 - lambda_1)) when that eigenspace is itself determined.

RBF covariance (k_covariance_rbf, orc_covariances_rbf): the kernel-weighted mean and covariance of the points within max_dist, the
cloud padded with points at the origin to a multiple of 512 (the reference's quirk: a padding point adds its weight to sum w and
nothing else).  Which points are within max_dist is decided on the float distance (dx dx + dy dy) + dz dz, as the kernel does: at
the boundary the two sides of the comparison are discontinuous, so the reference takes the same set and evaluates the rest in float64.
A weight carries about (2 + 2 kw md^2) eps (exp to ~1 ulp, the float distance to ~2 eps relative); a sum of m in-range terms over b
blocks is added sequentially (m within blocks, b partials): scale = (m + b + 8 + 2 kw md^2) eps * A with the weighted A of the raw case.

Voxel Gaussians (k_voxel_reduce, orc_voxelmap_build with double accumulation): the points of a voxel are summed in double and rounded
once.  VGICP: mean of the points, mean of the (packed, symmetric) point covariances; NDT: the population covariance, then MIN_EIG.
The float result is within 1 ulp (spacing of the float32 result) plus the double sum's own error n eps64 mean|term|, and for NDT the
one-pass (S - mu S^T) / n in double cancels like the raw case does in float: n eps64 (mean|p_r p_c| + |mu_r| mean|p_c|).  The NDT
result is compared after MIN_EIG: max(1e-3, .) is 1-Lipschitz, so the matrix function is 1-Lipschitz in the Frobenius norm and the
raw error passes through unamplified; scale = ||raw error||_F + TAU_MIN_EIG * the MIN_EIG scale.
"""
import math

import numpy as np

EPS32 = float(np.finfo(np.float32).eps)
EPS64 = float(np.finfo(np.float64).eps)
CLAMP = 1e-3        # covariance_regularization.cu: MIN_EIG clamp, FROBENIUS shift, PLANE small eigenvalue
RBF_BLOCK = 512     # covariance_estimation_rbf.cu: points per block, the cloud is padded to a multiple of it
PLANE_GAP = 1e-3    # PLANE: the normal counts as determined where lambda_1 - lambda_0 > PLANE_GAP * spread

REG_NONE, REG_MIN_EIG, REG_PLANE, REG_FROBENIUS = 0, 1, 3, 4  # RegularizationMethod (gicp_settings.hpp)

# The constants tau of the comparisons, calibrated on the CPU oracle (test_cov_reference.py prints the worst ratio of each): the
# worst ratio seen on 24 000 controlled spectra and on the hand-built neighbourhoods, with headroom.
TAU_RAW = 1.0        # worst seen 0.16: the (k + 4) eps bound is a worst-case sum of roundings
TAU_MIN_EIG = 8.0    # worst seen 2.4 (the 1e-3 of a clamped eigenvalue rebuilt through V diag V^-1)
TAU_FROBENIUS = 8.0  # worst seen 3.0
TAU_PLANE = 1e3      # worst seen 290 (determined normals next to a repeated top eigenvalue) and 350 (|n . v_2|)
TAU_RBF = 1.0        # worst seen 0.13: a worst-case sum of roundings, like the raw bound
TAU_VOXEL = 1.0      # worst seen 0.5 (the final rounding to float32 is half an ulp)


# ---------------------------------------------------------------------------------------------------------------- layouts
def mat(c9):
    """(N, 9) column-major 3x3 -> (N, 3, 3) float64 [row, col]."""
    return np.asarray(c9, dtype=np.float32).astype(np.float64).reshape(-1, 3, 3).transpose(0, 2, 1)


def lower(c9):
    """The symmetric matrices of the lower triangles of (N, 9) column-major 3x3s (what selfadjointView<Lower> reads), float64."""
    m = mat(c9)
    return np.tril(m) + np.swapaxes(np.tril(m, -1), 1, 2)


def sym(c9):
    """(M + M^T) / 2 in float64 -> (N, 3, 3): a stored result is compared through its symmetric part."""
    m = mat(c9)
    return 0.5 * (m + np.swapaxes(m, 1, 2))


def check(got, ref, scale, tau):
    """Per-entry |got - ref| <= tau * scale (scale broadcast against (N, 3, 3)) -> (ratio per matrix, failing matrices).
    ratio = max over entries of |got - ref| / scale; NaN or inf in got fails."""
    d = np.abs(np.asarray(got, dtype=np.float64) - ref)
    s = np.broadcast_to(np.asarray(scale, dtype=np.float64).reshape(np.shape(scale) + (1,) * (3 - np.ndim(scale))), d.shape)
    ok = d <= tau * s
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(s > 0, d / s, np.where(d > 0, np.inf, 0.0))
    r = np.where(np.isnan(d), np.inf, r)
    if not len(d):
        return np.zeros(0), np.zeros(0, dtype=np.int64)
    return r.reshape(len(d), -1).max(axis=1), np.flatnonzero(~ok.reshape(len(d), -1).all(axis=1))


# ---------------------------------------------------------------------------------------------------------------- raw k-NN
def raw_knn64(pts, nbr):
    """Two-pass float64 covariance of each row's neighbours, normalised by k -> (C (N, 3, 3), scale (N, 3, 3) = (k + 4) eps A)."""
    nbr = np.asarray(nbr, dtype=np.int64)
    k = nbr.shape[1]
    P = np.asarray(pts, dtype=np.float32).astype(np.float64)[nbr]  # (N, k, 3)
    mu = P.mean(axis=1)
    D = P - mu[:, None, :]
    C = np.einsum("nki,nkj->nij", D, D) / k
    aP = np.abs(P)
    am = aP.mean(axis=1)
    A = np.einsum("nki,nkj->nij", aP, aP) / k + am[:, :, None] * np.abs(mu)[:, None, :] + np.abs(mu)[:, :, None] * am[:, None, :]
    return C, (k + 4) * EPS32 * A


# ---------------------------------------------------------------------------------------------------------------- regularisers
def min_eig64(c9):
    """MIN_EIG of the lower triangles of c9 in float64 -> (ref (N, 3, 3), scale (N,))."""
    C = lower(c9)
    w, V = np.linalg.eigh(C)
    ref = np.einsum("nij,nj,nkj->nik", V, np.maximum(CLAMP, w), V)
    lmax = np.abs(w).max(axis=1)
    spread = w[:, 2] - w[:, 0]
    delta = np.minimum(w[:, 1] - w[:, 0], w[:, 2] - w[:, 1])
    with np.errstate(divide="ignore", invalid="ignore"):
        amp = np.where(delta > 0, np.minimum(spread / delta, EPS32 ** -0.5), EPS32 ** -0.5)
    amp = np.where(spread > 0, amp, 0.0)
    return ref, EPS32 * (np.maximum(lmax, CLAMP) + spread * amp)


def frobenius64(c9):
    """FROBENIUS of c9 in float64 -> (ref (N, 3, 3), scale (N,)).  Unlike the eigen-solver, the inversions read the whole matrix
    (an RBF covariance is symmetric only up to rounding); ref is the symmetric part, which is what the kernels store."""
    M = mat(c9) + CLAMP * np.eye(3)
    Mi = np.linalg.inv(M)
    ref = np.sqrt((Mi * Mi).sum(axis=(1, 2)))[:, None, None] * 0.5 * (M + np.swapaxes(M, 1, 2))
    s = np.linalg.svd(M, compute_uv=False)
    cond = s[:, 0] / s[:, 2]
    return ref, EPS32 * cond * cond * np.linalg.norm(ref, ord=2, axis=(1, 2))


def plane64(c9):
    """PLANE of the lower triangles of c9 in float64 -> dict(ref (N, 3, 3), scale (N,), determined (N,) bool, w, V).
    ref and scale apply where the normal is determined; plane_undetermined() checks the rest."""
    C = lower(c9)
    w, V = np.linalg.eigh(C)
    n = V[:, :, 0]
    ref = np.eye(3) - 0.999 * n[:, :, None] * n[:, None, :]
    spread = w[:, 2] - w[:, 0]
    gap = w[:, 1] - w[:, 0]
    lmax = np.abs(w).max(axis=1)
    determined = (gap > PLANE_GAP * spread) & (spread > 1e3 * EPS32 * lmax)
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = EPS32 * (1.0 + np.where(determined, spread / gap, 0.0))
    return dict(ref=ref, scale=scale, determined=determined, w=w, V=V)


PLANE_EIG_TOL = 1e-6  # |eigenvalues of a PLANE result - (1e-3, 1, 1)|: the rebuild V diag V^-1 of a near-orthonormal V in float


def plane_undetermined(got9, p):
    """For PLANE results whose normal is not determined: (max |eigenvalue - (1e-3, 1, 1)| per matrix, |n . v_2| / scale per matrix
    where v_2 is determined, else 0).  n = the result's eigenvector of its small eigenvalue."""
    G = sym(got9)
    gw, gV = np.linalg.eigh(G)
    eig_err = np.abs(gw - np.array([CLAMP, 1.0, 1.0])).max(axis=1)
    w = p["w"]
    spread, gap2 = w[:, 2] - w[:, 0], w[:, 2] - w[:, 1]
    v2_det = (gap2 > PLANE_GAP * spread) & (spread > 1e3 * EPS32 * np.abs(w).max(axis=1))
    dot = np.abs(np.einsum("ni,ni->n", gV[:, :, 0], p["V"][:, :, 2]))
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = EPS32 * (1.0 + spread / gap2)
    return eig_err, np.where(v2_det, dot / scale, 0.0)


def assert_regularised(method, raw9, got9, what=""):
    """got9 = regulariser `method` (MIN_EIG, PLANE or FROBENIUS) of the float32 raw covariances raw9, both (N, 9) column-major,
    against the float64 references -> {quantity: worst ratio}; raises naming the worst failing rows."""
    if method == REG_MIN_EIG:
        ref, sc = min_eig64(raw9)
        r, bad = check(sym(got9), ref, sc, TAU_MIN_EIG)
        out = {"MIN_EIG": r.max(initial=0.0)}
    elif method == REG_FROBENIUS:
        ref, sc = frobenius64(raw9)
        r, bad = check(sym(got9), ref, sc, TAU_FROBENIUS)
        out = {"FROBENIUS": r.max(initial=0.0)}
    elif method == REG_PLANE:
        p = plane64(raw9)
        det = p["determined"]
        r = np.zeros(len(det))
        r[det], b = check(sym(got9[det]), p["ref"][det], p["scale"][det], TAU_PLANE)
        und = np.flatnonzero(~det)
        e, nd = plane_undetermined(got9[und], {key: v[und] for key, v in p.items()})
        bad = np.union1d(np.flatnonzero(det)[b], und[~((e <= PLANE_EIG_TOL) & (nd <= TAU_PLANE))])
        out = {"PLANE": r.max(initial=0.0), "PLANE |n.v2|": nd.max(initial=0.0), "PLANE eigenvalues": e.max(initial=0.0)}
    else:
        raise ValueError(method)
    if len(bad):
        worst = bad[np.argsort(-r[bad])[:4]] if method != REG_PLANE else bad[:4]
        raise AssertionError(f"{what}: regulariser {method}: {len(bad)} of {len(raw9)} rows beyond the float64 bound, e.g. rows {worst.tolist()}: "
                             f"{np.linalg.eigvalsh(lower(raw9[worst])).tolist()}")
    return out


# ---------------------------------------------------------------------------------------------------------------- RBF
def rbf_padded(pts):
    """The float32 cloud padded with origin points to a multiple of RBF_BLOCK (covariance_estimation_rbf.cu:126-129)."""
    P = np.asarray(pts, dtype=np.float32)
    return np.vstack([P, np.zeros(((-len(P)) % RBF_BLOCK, 3), dtype=np.float32)])


def in_range32(x, ext, max_dist):
    """The kernel's float decision |x - p|^2 <= max_dist^2, spelled (dx dx + dy dy) + dz dz in float32."""
    d = np.float32(x)[None, :] - ext
    sq = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    md = np.float32(max_dist)
    return ~(sq > md * md)


def rbf64(pts, queries, kernel_width, max_dist, pad=True):
    """Kernel-weighted covariance of each query in float64 -> (C (Q, 3, 3), scale (Q, 3, 3)).  pad=False leaves the origin padding
    out (a wrong variant, for the comparator's own test)."""
    P32 = np.asarray(pts, dtype=np.float32)
    ext32 = rbf_padded(P32) if pad else P32
    ext = ext32.astype(np.float64)
    nblocks = (len(P32) + RBF_BLOCK - 1) // RBF_BLOCK
    kw = float(np.float32(kernel_width))
    out, scale = [], []
    for q in queries:
        inc = in_range32(P32[q], ext32, max_dist)
        p = ext[inc]
        d = p - P32[q].astype(np.float64)
        w = np.exp(-kw * (d * d).sum(axis=1))
        sw = w.sum()
        mu = (w @ p) / sw
        D = p - mu
        out.append((w[:, None] * D).T @ D / sw)
        ap = np.abs(p)
        am = (w @ ap) / sw
        A = (w[:, None] * ap).T @ ap / sw + am[:, None] * np.abs(mu)[None, :] + np.abs(mu)[:, None] * am[None, :]
        scale.append((len(p) + nblocks + 8 + 2 * kw * float(max_dist) ** 2) * EPS32 * A)
    return np.array(out).reshape(-1, 3, 3), np.array(scale).reshape(-1, 3, 3)


def rbf_paths(pts, max_dist):
    """What the sorted-cloud tests must show the kernel exercises, from the same float block boxes as k_rbf_block_boxes:
    (fraction of (query, block) pairs the box test skips, queries that pick up weight from the origin padding)."""
    ext = rbf_padded(pts)
    nb = len(ext) // RBF_BLOCK
    boxes = ext.reshape(nb, RBF_BLOCK, 3)
    lo, hi = boxes.min(axis=1), boxes.max(axis=1)
    x = np.asarray(pts, dtype=np.float32)
    md = np.float32(max_dist)
    zero = np.float32(0)
    dd = [np.maximum(np.maximum(lo[None, :, a] - x[:, None, a], x[:, None, a] - hi[None, :, a]), zero) for a in range(3)]
    need = ~((dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2] > md * md)
    padded = len(ext) > len(x)
    near = in_range32(np.zeros(3, np.float32), x, max_dist)  # symmetric: |x - 0|^2 in float is the same sum
    return 1.0 - need.mean(), int(near.sum()) if padded else 0


# ---------------------------------------------------------------------------------------------------------------- voxels
def voxel_coords32(pts, res):
    """calc_voxel_coord = floor(x / res - 0.5) in float32 (vector3_hash.cuh:35-38)."""
    return np.floor(np.asarray(pts, dtype=np.float32) / np.float32(res) - np.float32(0.5)).astype(np.int32)


def _ulp(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def voxels64(pts, res, cov9=None):
    """Voxel Gaussians in float64 -> dict(coords (V, 3), inv (N,) voxel of each point, n (V,), mean (V, 3), mean_scale (V, 3),
    cov (V, 3, 3), cov_scale (V, 3, 3) or (V,)).  cov9=None: NDT (two-pass population covariance, then MIN_EIG); else VGICP (the
    mean of the given covariances)."""
    P = np.asarray(pts, dtype=np.float32).astype(np.float64)
    coords, inv, n = np.unique(voxel_coords32(pts, res), axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    V = len(coords)
    bc = lambda x: np.bincount(inv, weights=x, minlength=V)  # noqa: E731
    mean = np.stack([bc(P[:, a]) for a in range(3)], axis=1) / n[:, None]
    amean = np.stack([bc(np.abs(P[:, a])) for a in range(3)], axis=1) / n[:, None]
    mean_scale = _ulp(mean) + n[:, None] * EPS64 * amean
    if cov9 is not None:
        Cp = sym(cov9).reshape(-1, 9)
        cov = np.stack([bc(Cp[:, j]) for j in range(9)], axis=1).reshape(-1, 3, 3) / n[:, None, None]
        acov = np.stack([bc(np.abs(Cp[:, j])) for j in range(9)], axis=1).reshape(-1, 3, 3) / n[:, None, None]
        return dict(coords=coords, inv=inv, n=n, mean=mean, mean_scale=mean_scale, cov=cov, cov_scale=_ulp(cov) + n[:, None, None] * EPS64 * acov)
    D = P - mean[inv]
    raw = np.stack([bc(D[:, r] * D[:, c]) for r in range(3) for c in range(3)], axis=1).reshape(-1, 3, 3) / n[:, None, None]
    app = np.stack([bc(np.abs(P[:, r] * P[:, c])) for r in range(3) for c in range(3)], axis=1).reshape(-1, 3, 3) / n[:, None, None]
    raw_err = _ulp(raw) + n[:, None, None] * EPS64 * (app + np.abs(mean)[:, :, None] * amean[:, None, :])
    ref, me_scale = min_eig64(raw.transpose(0, 2, 1).reshape(-1, 9))
    return dict(coords=coords, inv=inv, n=n, mean=mean, mean_scale=mean_scale, raw=raw, cov=ref,
                cov_scale=np.sqrt((raw_err ** 2).sum(axis=(1, 2))) + TAU_MIN_EIG * me_scale)


def match_voxels(coords, bucket_coord, bucket_id):
    """Voxel id of each reference coordinate in a built table (-1 when missing)."""
    occ = np.flatnonzero(bucket_id >= 0)
    ids = {tuple(int(v) for v in bucket_coord[b]): int(bucket_id[b]) for b in occ}
    return np.array([ids.get(tuple(int(v) for v in c), -1) for c in coords], dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------------- eig3 branches
EIG3_LABELS = ("scale == 0", "all-equal", "near-degenerate, k_is_2", "near-degenerate, !k_is_2", "general, k_is_2", "general, !k_is_2",
               "pivot i0 = 0", "pivot i0 = 1", "pivot i0 = 2", "pivot tie")


def eig3_branches(c9):
    """Float32 restatement of eig3_direct up to its branch decisions (shift, scale, computeRoots in the kernel's operation order,
    trig in double rounded once) -> (eigenvalues (N, 3) float32 as eig3_direct returns them, {label: bool (N,)}).  The labels
    read the shifted and scaled roots, which the returned eigenvalues no longer show; the pivot labels are those of the first
    extract_kernel call (the column of the most distinct eigenvalue)."""
    f = np.float32
    m = np.asarray(c9, dtype=np.float32).reshape(-1, 3, 3).transpose(0, 2, 1)  # [row, col]
    s00, s11, s22 = m[:, 0, 0].copy(), m[:, 1, 1].copy(), m[:, 2, 2].copy()
    s10, s20, s21 = m[:, 1, 0].copy(), m[:, 2, 0].copy(), m[:, 2, 1].copy()
    shift = ((s00 + s11) + s22) / f(3)
    s00, s11, s22 = s00 - shift, s11 - shift, s22 - shift
    scale = np.max(np.abs(np.stack([s00, s11, s22, s10, s20, s21])), axis=0)
    div = np.where(scale > 0, scale, f(1))
    s00, s11, s22, s10, s20, s21 = (np.where(scale > 0, v / div, v) for v in (s00, s11, s22, s10, s20, s21))
    inv3 = f(1) / f(3)
    c0 = (((s00 * s11) * s22 + ((f(2) * s10) * s20) * s21) - (s00 * s21) * s21 - (s11 * s20) * s20) - (s22 * s10) * s10
    c1 = ((((s00 * s11 - s10 * s10) + s00 * s22) - s20 * s20) + s11 * s22) - s21 * s21
    c2 = (s00 + s11) + s22
    c2o3 = c2 * inv3
    a3 = np.maximum((c2 * c2o3 - c1) * inv3, f(0))
    hb = f(0.5) * (c0 + c2o3 * ((f(2) * c2o3) * c2o3 - c1))
    q = np.maximum((a3 * a3) * a3 - hb * hb, f(0))
    rho = np.sqrt(a3)
    sq = np.sqrt(q)
    theta = np.array([math.atan2(float(a), float(b)) for a, b in zip(sq, hb)], dtype=np.float64).astype(np.float32) * inv3
    cos_t = np.array([math.cos(float(t)) for t in theta]).astype(np.float32)
    sin_t = np.array([math.sin(float(t)) for t in theta]).astype(np.float32)
    sqrt3 = np.sqrt(f(3))
    r0 = c2o3 - rho * (cos_t + sqrt3 * sin_t)
    r1 = c2o3 - rho * (cos_t - sqrt3 * sin_t)
    r2 = c2o3 + (f(2) * rho) * cos_t
    eps = f(1.1920929e-07)
    zero = scale == 0
    equal = ~zero & (r2 - r0 <= eps)
    rest = ~(zero | equal)
    d0, d1 = r2 - r1, r1 - r0
    k2 = d0 > d1
    near = np.where(k2, d1, d0) <= (f(2) * eps) * d1
    ek = np.where(k2, r2, r0)
    diag = np.abs(np.stack([s00 - ek, s11 - ek, s22 - ek], axis=1))
    i0 = np.zeros(len(diag), dtype=np.int64)
    best = diag[:, 0].copy()
    for i in (1, 2):
        up = diag[:, i] > best
        i0, best = np.where(up, i, i0), np.where(up, diag[:, i], best)
    tie = (diag == best[:, None]).sum(axis=1) > 1
    labels = {"scale == 0": zero, "all-equal": equal, "near-degenerate, k_is_2": rest & near & k2, "near-degenerate, !k_is_2": rest & near & ~k2,
              "general, k_is_2": rest & ~near & k2, "general, !k_is_2": rest & ~near & ~k2}
    for i in range(3):
        labels[f"pivot i0 = {i}"] = rest & (i0 == i)
    labels["pivot tie"] = rest & tie
    ev = np.stack([r0, r1, r2], axis=1) * scale[:, None] + shift[:, None]
    return ev.astype(np.float32), labels


# ---------------------------------------------------------------------------------------------------------------- inputs
KNN_KS = (1, 2, 3, 5, 20, 64)
KNN_KINDS = ("identical", "repeated", "line", "rotated line", "plane z", "rotated plane", "isotropic", "disk", "rotated disk", "prolate",
             "ring arc", "far 1e3", "far 1e4", "tiny")


def _rotation(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def _isotropic(k, rng):
    """k points whose float covariance is exactly a multiple of I: integer coordinates (every sum exact), so the division by k is
    the only rounding and, for k = 20, often leaves a diagonal that (3a)/3 does not give back (eig3_direct's all-equal branch)."""
    cube = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], dtype=np.float64)
    octa = np.vstack([np.eye(3), -np.eye(3)])
    if k == 20:
        a, b = rng.integers(1, 16, size=2)
        return np.vstack([a * cube, b * octa, b * octa])
    if k == 64:
        g = np.array([-3, -1, 1, 3], dtype=np.float64) * rng.integers(1, 8)
        return np.array([[x, y, z] for x in g for y in g for z in g])
    return np.vstack([octa] * 11)[:k] * rng.integers(1, 8)  # k < 6: no isotropic set; the first k of +-e_i


def _patch(kind, k, rng, nice):
    """k points of one hand-built neighbourhood."""
    R = _rotation(rng)
    c = rng.uniform(-30, 30, size=3)
    q = (lambda x: np.round(x * 64) / 64) if nice else (lambda x: x)  # nice: coordinates on a 1/64 grid, sums exact
    t = q(rng.uniform(-2, 2, size=k))
    u = q(rng.uniform(-2, 2, size=k))
    ang = 2 * np.pi * (np.arange(k) / k + rng.uniform())
    if kind == "identical":
        return np.tile(q(c), (k, 1))
    if kind == "repeated":  # drawn from three points with replacement: the row repeats indices
        return q(c + rng.normal(scale=0.5, size=(3, 3)))[rng.integers(0, 3, size=k)]
    if kind == "line":
        p = np.tile(q(c), (k, 1))
        p[:, rng.integers(3)] += t
        return p
    if kind == "rotated line":
        return c + np.outer(t, R[:, 0])
    if kind == "plane z":
        p = np.tile(q(c), (k, 1))
        p[:, 0] += t
        p[:, 1] += u
        return p
    if kind == "rotated plane":
        return c + np.outer(t, R[:, 0]) + np.outer(u, R[:, 1])
    if kind == "isotropic":  # nice: centred at the origin, so that the float covariance stays an exact multiple of I
        return _isotropic(k, rng) * 2.0 ** rng.integers(-6, 3) + (0.0 if nice else c)
    if kind in ("disk", "rotated disk"):  # a regular k-gon: lambda_1 = lambda_2 (k >= 3)
        r = rng.uniform(0.2, 2)
        p = np.stack([r * np.cos(ang), r * np.sin(ang), np.zeros(k)], axis=1)
        return c + (p @ R.T if kind == "rotated disk" else p)
    if kind == "prolate":  # two regular polygons at +-h along the axis: lambda_0 = lambda_1 (k even, k >= 6)
        r, h = rng.uniform(0.05, 0.3), rng.uniform(1, 3)
        half = np.arange(k) % 2
        a2 = 2 * np.pi * ((np.arange(k) // 2) / max(k // 2, 1) + rng.uniform())
        p = np.stack([r * np.cos(a2), r * np.sin(a2), np.where(half, h, -h)], axis=1)
        return c + p @ R.T
    if kind == "ring arc":  # consecutive returns of one lidar beam: range 5..40 m, 0.2 deg apart, constant height
        rr, el = rng.uniform(5, 40), rng.uniform(-0.3, 0.05)
        az = rng.uniform(0, 2 * np.pi) + np.radians(0.2) * np.arange(k)
        return np.stack([rr * np.cos(el) * np.cos(az), rr * np.cos(el) * np.sin(az), np.full(k, rr * np.sin(el))], axis=1)
    if kind in ("far 1e3", "far 1e4"):
        d = 1e3 if kind == "far 1e3" else 1e4
        v = rng.normal(size=3)
        return d * v / np.linalg.norm(v) + rng.normal(size=(k, 3)) * [0.3, 0.2, 0.1] @ R.T
    if kind == "tiny":  # 1e-3 m spread: every eigenvalue below the 1e-3 clamp
        return c + rng.normal(scale=1e-3, size=(k, 3)) @ R.T
    raise ValueError(kind)


def knn_neighbourhoods(k, patches=10, seed=0):
    """Hand-built k-point neighbourhoods of every kind -> (pts (n, 3) float32, nbr (n, k) int32, kind (n,) str).  Each patch's k points
    are consecutive in the cloud and the row of each is the patch, rotated to start at the point itself (so the rows of one
    patch add the same points in different orders)."""
    rng = np.random.default_rng(1000 * k + seed)
    pts, nbr, kind = [], [], []
    n = 0
    for kd in KNN_KINDS:
        for j in range(patches * 50 if (kd, k) == ("isotropic", 20) else patches):  # (about 1 in 6 (a, b) pairs takes the all-equal branch)
            p = _patch(kd, k, rng, nice=j % 2 == 0)
            idx = n + np.arange(k)
            pts.append(p)
            nbr.extend(np.roll(idx, -i) for i in range(k))
            kind.extend([kd] * k)
            n += k
    return np.vstack(pts).astype(np.float32), np.array(nbr, dtype=np.int32).reshape(-1, k), np.array(kind)


def spectrum_set(count=24000, seed=0):
    """Seeded 3x3 covariances with controlled spectra (column-major (count, 9) float32): eigenvalues 10^[-9, 0] times a scale
    10^[-4, 2], an eighth each with a repeated bottom pair, a repeated top pair, a zero eigenvalue and a triple; half rotated at
    random, a quarter axis-aligned (permuted diagonal), a quarter rotated about one coordinate axis."""
    rng = np.random.default_rng(seed)
    lam = np.sort(10.0 ** rng.uniform(-9, 0, size=(count, 3)), axis=1) * 10.0 ** rng.uniform(-4, 2, size=(count, 1))
    form = rng.integers(0, 8, size=count)
    lam[form == 0, 1] = lam[form == 0, 0]
    lam[form == 1, 1] = lam[form == 1, 2]
    lam[form == 2, 0] = 0.0
    lam[form == 3, :2] = lam[form == 3, 2:]
    out = np.empty((count, 3, 3))
    how = rng.integers(0, 4, size=count)
    for i in range(count):
        if how[i] < 2:
            R = _rotation(rng)
        elif how[i] == 2:
            R = np.eye(3)[rng.permutation(3)]
        else:
            a, ax = rng.uniform(0, 2 * np.pi), rng.integers(3)
            R = np.eye(3)
            i1, i2 = [j for j in range(3) if j != ax]
            R[i1, i1] = R[i2, i2] = np.cos(a)
            R[i1, i2], R[i2, i1] = -np.sin(a), np.sin(a)
        M = R @ np.diag(lam[i]) @ R.T
        out[i] = 0.5 * (M + M.T)
    return np.ascontiguousarray(out.astype(np.float32).transpose(0, 2, 1).reshape(count, 9))


RBF_NS = (1, 511, 512, 513, 4095, 4096, 4097, 4608, 20000)  # the block padding, the 8-block round boundary, several rounds
RBF_SETTINGS = ((0.5, 3.0), (0.25, 1.25))                   # (kernel_width, max_dist)


def lidar_scan(n, seed=0):
    """A lidar-like scan of n points in azimuth order (16 beams, ranges 0.8..40 m, a few returns near the sensor)."""
    rng = np.random.default_rng(seed)
    az = np.sort(rng.uniform(0, 2 * np.pi, size=n))
    el = np.radians(rng.integers(-15, 1, size=n) * 2.0)
    r = np.where(rng.uniform(size=n) < 0.05, rng.uniform(0.8, 2.5, size=n), rng.uniform(3, 40, size=n))
    r = np.minimum(r, 1.73 / np.maximum(np.sin(-el), 1e-3))  # beams below the horizon hit the ground at z = -1.73
    return np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], axis=1).astype(np.float32)


def voxel_cloud(res, seed=0):
    """A cloud whose voxels at resolution res hold exactly 1, 2, 3 and 4 points, collinear and coplanar points, 33 points, 10 000
    points, and sit at |p| = 1e3 and 1e4 m -> (pts (n, 3) float32, covariances (n, 9) float32: symmetric, positive definite)."""
    rng = np.random.default_rng(seed)
    blocks = []

    def put(cell, u):  # points at fractions u in [0.1, 0.9] of voxel `cell` (voxel c spans [(c + 0.5) res, (c + 1.5) res))
        blocks.append((np.asarray(cell, dtype=np.float64) + 0.5 + u) * res)

    base = np.stack(np.unravel_index(rng.choice(80 ** 3, size=400, replace=False), (80, 80, 80)), axis=1) - 40  # distinct cells
    for j, cell in enumerate(base):
        m = (1, 2, 3, 4)[j % 4] if j < 240 else None
        if m is not None:
            put(cell, rng.uniform(0.1, 0.9, size=(m, 3)))
        elif j < 280:  # collinear
            t = rng.uniform(0.1, 0.9, size=(12, 1))
            put(cell, np.hstack([t, np.full_like(t, 0.3), np.full_like(t, 0.6)]) if j % 2 else 0.1 + 0.8 * t * [1.0, 0.5, 0.25])
        elif j < 320:  # coplanar
            u = rng.uniform(0.1, 0.9, size=(15, 2))
            put(cell, np.hstack([u, np.full((15, 1), 0.45)]))
        else:
            put(cell, rng.uniform(0.1, 0.9, size=(rng.integers(5, 40), 3)))
    put((60, 60, 60), rng.uniform(0.1, 0.9, size=(33, 3)))
    put((-60, 60, 0), rng.uniform(0.1, 0.9, size=(10000, 3)))
    for d in (1e3, 1e4):
        for j in range(8):
            v = rng.normal(size=3)
            put(np.floor(d * v / np.linalg.norm(v) / res), rng.uniform(0.1, 0.9, size=(1 + j, 3)))
    pts = np.vstack(blocks).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]  # voxels interleaved in point order
    L = rng.normal(size=(len(pts), 3, 3)) * 0.1
    C = (L @ L.transpose(0, 2, 1) + 1e-3 * np.eye(3)).astype(np.float32)
    C = 0.5 * (C + C.transpose(0, 2, 1))
    return pts, np.ascontiguousarray(C.reshape(-1, 9))
