"""Float64 reference of one evaluation (update_correspondences(T_lin) + compute_error(T_eval, H, b)), in plain numpy.

Restated from the definitions of the VGICP and NDT derivative sums, not from any implementation of them.  Per correspondence
(source point a, voxel B) of the list `pairs` (found under T_lin):

    M = (C_B + R_lin C_A R_lin^T)^-1,   e = mu_B - T_eval a,   s = e^T M e,   J = [skew(T_eval a) | -I]
    VGICP:  w = sqrt(n_B); voxels with n_B <= 0 are skipped when H is wanted
    NDT:    w = res^2 / (res^2 + |e|^2); voxels with n_B <= 6 are skipped (C_A = 0 for point-to-distribution)
    err += w rho(s),   H += w rho'(s) J^T M J,   b += w rho'(s) J^T M e

with rho the robust kind (VGICP only; identity when None):
    HUBER          rho = s (s <= d2), 2 sqrt(d2 s) - d2 (else)       rho' = 1, sqrt(d2 / s)
    CAUCHY         rho = d2 ln(1 + s / d2)                           rho' = d2 / (d2 + s)
    GEMAN_MCCLURE  rho = s d2 / (d2 + s)                             rho' = (d2 / (d2 + s))^2
d2 = delta^2.  The poses are rounded to float32 first: that is the pose the evaluation receives.

Every one of the 43 results (err, the 36 entries of H, the 6 of b) also comes with A, the float64 sum of the absolute values of its
per-correspondence terms.  A float computation of the same sum has an error of a few float32 roundings per term, so A is the scale
an entry's tolerance is taken against: a per-entry check |x - x_ref| <= tau A + 1e-12 max(A) holds small entries (the
rotation-translation coupling, b near the optimum) to their own size, not to a fraction of the largest entry.
"""
import numpy as np

KINDS = ("NONE", "HUBER", "CAUCHY", "GEMAN_MCCLURE")
_CHUNK = 1 << 18


def _pose64(T):
    return np.asarray(T, dtype=np.float64).astype(np.float32).astype(np.float64)


def _mat(c9):
    """(N, 9) column-major 3x3 -> (N, 3, 3) float64."""
    return np.asarray(c9, dtype=np.float32).astype(np.float64).reshape(-1, 3, 3).transpose(0, 2, 1)


def rho64(kind, s, d2):
    """(rho(s), rho'(s)) in float64 for a robust kind name (None / "NONE": the plain sum)."""
    if kind in (None, "NONE"):
        return s, np.ones_like(s)
    if kind == "HUBER":
        big = s > d2
        ss = np.where(big, s, d2)
        return np.where(big, 2.0 * np.sqrt(d2 * ss) - d2, s), np.where(big, np.sqrt(d2 / ss), 1.0)
    q = d2 / (d2 + s)
    if kind == "CAUCHY":
        return d2 * np.log1p(s / d2), q
    if kind == "GEMAN_MCCLURE":
        return q * s, q * q
    raise ValueError(f"unknown robust kind {kind!r}")


def eval64_kinds(vox_mean, vox_cov, vox_n, src, src_cov, pairs, T_lin, T_eval, want_H, kinds=(None,), delta=1.0, ndt=False, res=1.0):
    """eval64 for several robust kinds from one pass over the correspondences -> {kind: (err, H, b, A)}."""
    Tl, Te = _pose64(T_lin), _pose64(T_eval)
    Rl = Tl[:3, :3]
    d2 = float(delta) * float(delta)
    vox_n = np.asarray(vox_n)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    mu = np.asarray(vox_mean, dtype=np.float32).astype(np.float64)
    src = np.asarray(src, dtype=np.float32).astype(np.float64)
    acc = {k: [np.zeros(43), np.zeros(43)] for k in kinds}  # kind -> [sums, sums of |terms|]
    for c0 in range(0, len(pairs), _CHUNK):
        ia, iv = pairs[c0:c0 + _CHUNK, 0], pairs[c0:c0 + _CHUNK, 1]
        n = vox_n[iv]
        keep = n > 6 if ndt else (n > 0 if want_H else np.ones(len(iv), dtype=bool))
        ia, iv, n = ia[keep], iv[keep], n[keep]
        S = _mat(vox_cov[iv])
        if src_cov is not None:
            S = S + Rl @ _mat(src_cov[ia]) @ Rl.T
        M = _inv3(S)  # M[i][j]: (K,) arrays
        p = src[ia] @ Te[:3, :3].T + Te[:3, 3]  # T_eval a
        e = mu[iv] - p
        Me = [M[i][0] * e[:, 0] + M[i][1] * e[:, 1] + M[i][2] * e[:, 2] for i in range(3)]
        s = e[:, 0] * Me[0] + e[:, 1] * Me[1] + e[:, 2] * Me[2]
        w = res * res / (res * res + (e * e).sum(axis=1)) if ndt else np.sqrt(n.astype(np.float64))
        if want_H:
            # J = [P | -I], P = skew(p), P^T = -P:  J^T M J = [[P^T M P, P M], [-M P, M]],  J^T M e = [P^T M e; -M e]
            z = np.zeros(len(ia))
            P = [[z, -p[:, 2], p[:, 1]], [p[:, 2], z, -p[:, 0]], [-p[:, 1], p[:, 0], z]]
            MP = [[M[i][0] * P[0][j] + M[i][1] * P[1][j] + M[i][2] * P[2][j] for j in range(3)] for i in range(3)]
            PtM = [[P[0][i] * M[0][j] + P[1][i] * M[1][j] + P[2][i] * M[2][j] for j in range(3)] for i in range(3)]
            h = [[None] * 6 for _ in range(6)]
            for i in range(3):
                for j in range(3):
                    h[i][j] = P[0][i] * MP[0][j] + P[1][i] * MP[1][j] + P[2][i] * MP[2][j]
                    h[i][3 + j] = -PtM[i][j]
                    h[3 + i][j] = -MP[i][j]
                    h[3 + i][3 + j] = M[i][j]
            g = [P[0][i] * Me[0] + P[1][i] * Me[1] + P[2][i] * Me[2] for i in range(3)] + [-Me[i] for i in range(3)]
            raw = np.stack([h[i][j] for i in range(6) for j in range(6)] + g, axis=1)
        for k in kinds:
            r, dr = rho64(None if ndt else k, s, d2)
            v, a = acc[k]
            t = w * r
            v[0] += t.sum()
            a[0] += np.abs(t).sum()
            if want_H:
                wd = w * dr  # >= 0: |wd raw| = wd |raw|
                v[1:] += wd @ raw
                a[1:] += wd @ np.abs(raw)
    out = {}
    for k, (v, a) in acc.items():
        out[k] = (v[0], v[1:37].reshape(6, 6).copy() if want_H else None, v[37:].copy() if want_H else None, a if want_H else a[:1].copy())
    return out


def _inv3(S):
    """Inverse of each (K, 3, 3) matrix by cofactors in float64 -> nested lists of (K,) arrays."""
    a = [[S[:, i, j] for j in range(3)] for i in range(3)]
    c = [[a[(j + 1) % 3][(i + 1) % 3] * a[(j + 2) % 3][(i + 2) % 3] - a[(j + 1) % 3][(i + 2) % 3] * a[(j + 2) % 3][(i + 1) % 3] for j in range(3)] for i in range(3)]
    det = a[0][0] * c[0][0] + a[0][1] * c[1][0] + a[0][2] * c[2][0]
    return [[c[i][j] / det for j in range(3)] for i in range(3)]


def eval64(vox_mean, vox_cov, vox_n, src, src_cov, pairs, T_lin, T_eval, want_H, robust=None, delta=1.0, ndt=False, res=1.0):
    """One evaluation in float64 -> (err, H (6,6) | None, b (6,) | None, A).

    vox_mean (V,3), vox_cov (V,9 column-major), vox_n (V,): the target voxel Gaussians; src (N,3), src_cov (N,9 column-major, or
    None for NDT point-to-distribution); pairs (K,2) = (source index, voxel id), the list found under T_lin.  A: (43,) = the float64
    sums of |per-correspondence term| of [err, H (row-major), b] when want_H, else (1,) for err."""
    return eval64_kinds(vox_mean, vox_cov, vox_n, src, src_cov, pairs, T_lin, T_eval, want_H, (robust,), delta, ndt, res)[robust]


def pack(err, H=None, b=None):
    """[err, H (row-major), b] as one vector (err alone when H is None)."""
    if H is None:
        return np.array([float(err)])
    return np.concatenate([[float(err)], np.asarray(H, dtype=np.float64).reshape(36), np.asarray(b, dtype=np.float64).reshape(6)])


def excess(got, ref, tau):
    """Per-entry check of got = (err, H, b) against ref = eval64's (err, H, b, A): returns (worst |x - x_ref| / A, failing entries).
    An entry fails when |x - x_ref| > tau A + 1e-12 max(A)."""
    A = ref[3]
    x, x0 = pack(*got[:3]), pack(*ref[:3])
    assert x.shape == A.shape, (x.shape, A.shape)
    d = np.abs(x - x0)
    bad = np.flatnonzero(~(d <= tau * A + 1e-12 * A.max()))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(A > 0, d / A, np.where(d > 0, np.inf, 0.0))
    return float(r.max()), bad


def entry_name(j):
    """Name of entry j of pack()'s layout, for failure messages."""
    return "err" if j == 0 else (f"H[{(j - 1) // 6},{(j - 1) % 6}]" if j < 37 else f"b[{j - 37}]")


def assert_close(got, ref, tau, what=""):
    """excess() with every failing entry named; returns the worst ratio."""
    worst, bad = excess(got, ref, tau)
    if len(bad):
        x, x0 = pack(*got[:3]), pack(*ref[:3])
        detail = ", ".join(f"{entry_name(j)}: {x[j]:.9g} vs {x0[j]:.9g} (A {ref[3][j]:.3g}, ratio {abs(x[j] - x0[j]) / max(ref[3][j], 1e-300):.3g})" for j in bad[:8])
        raise AssertionError(f"{what}: {len(bad)} entries beyond tau={tau:g}: {detail}")
    return worst
