"""Float64 reference of one continuous-time evaluation (vgicp_compute_error_ct) and of the 12 x 12 system built from it, in
plain numpy.  Restated from the model in include/vgicp_b200.h, not from the implementation.

Per correspondence (source point i, voxel B) of the list `pairs` (found with the points deskewed by xi_lin under T_lin), with
q_i the point deskewed by xi_eval and s_i its time offset:

    M = (C_B + R_lin C_i R_lin^T)^-1,   p = T_eval q_i,   e = mu_B - p,   J = [skew(p) | -I],   w = sqrt(n_B)
    err += w rho,   H0 += w rho' J^T M J,   H1 += s_i (..),   H2 += s_i^2 (..),   b0 += w rho' J^T M e,   b1 += s_i (..)

and, with K = [[R, 0], [[t]x R, R]] of T_eval,  H = [[H0, H1 K], [K^T H1, K^T H2 K]],  b = [b0; K^T b1].  Every entry also comes
with A, the float64 sum of |per-correspondence term| propagated through |K|: the scale of eval_reference's tau A tolerance.
"""
import numpy as np

from eval_reference import _inv3, _mat, rho64

_CHUNK = 1 << 17


def skew(v):
    """(K, 3) -> (K, 3, 3)."""
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1), np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def ct_sums(vox_mean, vox_cov, vox_n, q_eval, src_cov, s, pairs, T_lin, T_eval, robust=None, delta=1.0):
    """-> dict of the six sums (err, H0, H1, H2 (6,6), b0, b1 (6,)) and their |term| sums (keys with "A_").  q_eval (N,3): the
    source points at xi_eval (float64 or float32); s (N,): their time offsets; T_lin, T_eval used as given (round them to float32
    first to model the device)."""
    Tl, Te = np.asarray(T_lin, dtype=np.float64), np.asarray(T_eval, dtype=np.float64)
    Rl = Tl[:3, :3]
    d2 = float(delta) * float(delta)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    mu = np.asarray(vox_mean, dtype=np.float32).astype(np.float64)
    q = np.asarray(q_eval).astype(np.float64)
    s = np.asarray(s).astype(np.float64)
    vox_n = np.asarray(vox_n)
    out = {k: 0.0 for k in ("err", "A_err")}
    for k in ("H0", "H1", "H2", "A_H0", "A_H1", "A_H2"):
        out[k] = np.zeros((6, 6))
    for k in ("b0", "b1", "A_b0", "A_b1"):
        out[k] = np.zeros(6)
    for c0 in range(0, len(pairs), _CHUNK):
        ia, iv = pairs[c0:c0 + _CHUNK, 0], pairs[c0:c0 + _CHUNK, 1]
        keep = vox_n[iv] > 0
        ia, iv = ia[keep], iv[keep]
        S = _mat(vox_cov[iv]) + Rl @ _mat(src_cov[ia]) @ Rl.T
        Mi = _inv3(S)
        M = np.stack([np.stack([Mi[i][j] for j in range(3)], 1) for i in range(3)], 1)
        p = q[ia] @ Te[:3, :3].T + Te[:3, 3]
        e = mu[iv] - p
        J = np.concatenate([skew(p), -np.broadcast_to(np.eye(3), (len(p), 3, 3))], axis=2)
        Me = np.einsum("kab,kb->ka", M, e)
        sm = np.einsum("ka,ka->k", e, Me)
        w = np.sqrt(vox_n[iv].astype(np.float64))
        r, dr = rho64(robust, sm, d2)
        wd = w * dr
        G = np.einsum("kai,kab,kbj->kij", J, M, J)
        g = np.einsum("kai,ka->ki", J, Me)
        si = s[ia]
        out["err"] += float((w * r).sum())
        out["A_err"] += float(np.abs(w * r).sum())
        for k, f in (("0", np.ones_like(si)), ("1", si), ("2", si * si)):
            out["H" + k] += np.einsum("k,kij->ij", wd * f, G)
            out["A_H" + k] += np.einsum("k,kij->ij", wd * np.abs(f), np.abs(G))
            if k != "2":
                out["b" + k] += np.einsum("k,ki->i", wd * f, g)
                out["A_b" + k] += np.einsum("k,ki->i", wd * np.abs(f), np.abs(g))
    return out


def K_of(T):
    """K = [[R, 0], [[t]x R, R]] of the 4x4 T (as given)."""
    T = np.asarray(T, dtype=np.float64)
    R, t = T[:3, :3], T[:3, 3]
    K = np.zeros((6, 6))
    K[:3, :3] = R
    K[3:, 3:] = R
    K[3:, :3] = skew(t[None])[0] @ R
    return K


def system12(sums, T):
    """-> (err, H (12,12), b (12,), A (157,)) from ct_sums' dict and the pose the sums were taken at.  A is laid out like pack()."""
    K = K_of(T)
    aK = np.abs(K)
    H = np.block([[sums["H0"], sums["H1"] @ K], [K.T @ sums["H1"], K.T @ sums["H2"] @ K]])
    b = np.concatenate([sums["b0"], K.T @ sums["b1"]])
    AH = np.block([[sums["A_H0"], sums["A_H1"] @ aK], [aK.T @ sums["A_H1"], aK.T @ sums["A_H2"] @ aK]])
    Ab = np.concatenate([sums["A_b0"], aK.T @ sums["A_b1"]])
    return sums["err"], H, b, np.concatenate([[sums["A_err"]], AH.reshape(144), Ab])


def pack(err, H=None, b=None):
    if H is None:
        return np.array([float(err)])
    return np.concatenate([[float(err)], np.asarray(H, dtype=np.float64).reshape(144), np.asarray(b, dtype=np.float64).reshape(12)])


def assert_close(got, ref, tau, what=""):
    """Entry by entry: |x - x_ref| <= tau A + 1e-12 max(A) (eval_reference's scheme over the 157 entries); returns the worst ratio."""
    A = ref[3] if got[1] is not None else ref[3][:1]
    x, x0 = pack(*got[:3]), pack(*ref[:3]) if got[1] is not None else pack(ref[0])
    d = np.abs(x - x0)
    bad = np.flatnonzero(~(d <= tau * A + 1e-12 * A.max()))
    if len(bad):
        name = lambda j: "err" if j == 0 else (f"H[{(j - 1) // 12},{(j - 1) % 12}]" if j < 145 else f"b[{j - 145}]")  # noqa: E731
        raise AssertionError(f"{what}: {len(bad)} entries beyond tau={tau:g}: " + ", ".join(f"{name(j)}: {x[j]:.9g} vs {x0[j]:.9g} (A {A[j]:.3g})" for j in bad[:8]))
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.max(np.where(A > 0, d / A, 0.0)))
