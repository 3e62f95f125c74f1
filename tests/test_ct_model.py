"""Continuous-time registration (vgicp_compute_error_ct / vgicp_align_ct) on the CPU: the float64 model of tests/ct_reference.py
against explicit 12-column Jacobians, finite differences and eval64, and a numpy CT-LM over the oracle's correspondences that
registers the motion-distorted scan of test_deskew_model, which plain registration cannot.  tests/test_gpu_ct.py holds the
device to this model."""
import numpy as np

import oracle as O
from conftest import pose_error
from ct_reference import K_of, ct_sums, skew, system12
from eval_reference import eval64
from test_deskew_model import EFFECT_TWIST, deskew_f32, distorted_pair, syn

F = np.float32


def _f32pose(T):
    return np.asarray(T, dtype=np.float64).astype(np.float32).astype(np.float64)


def problem(seed=42):
    """The distorted pair of test_deskew_model with the oracle's PLANE covariances and voxel map."""
    tgt, src, ts, T = distorted_pair(seed)
    tc = O.estimate_covariances(tgt, 20, O.REG_PLANE)
    sc = O.estimate_covariances(src, 20, O.REG_PLANE)
    vm = O.VoxelMap(tgt, tc, 1.0, accum_double=True)
    return vm, src, sc, ts, T


def model_eval(vm, src, sc, times, offs, T_lin, xi_lin, T_eval, xi_eval, robust=None):
    """The device's evaluation, modelled: float32 deskew, the oracle's lookup under float poses, float64 sums."""
    q_lin = deskew_f32(src, times, xi_lin, 0.0)
    q_eval = deskew_f32(src, times, xi_eval, 0.0)
    pairs = O.find_correspondences(vm, q_lin, T_lin, offs)
    s = np.asarray(times, dtype=np.float32)
    sums = ct_sums(vm.vox_mean, vm.vox_cov, vm.vox_n, q_eval, sc, s, pairs, _f32pose(T_lin), _f32pose(T_eval), robust)
    return system12(sums, _f32pose(T_eval)), pairs


def test_factorised_system_equals_explicit_jacobians():
    vm, src, sc, ts, T = problem()
    offs = O.offsets(O.DIRECT7)
    xi = np.array([0.05, -0.03, np.radians(20.0), 9.0, 0.4, -0.2])
    Tl = _f32pose(T)
    q = deskew_f32(src, ts, xi, 0.0)
    pairs = O.find_correspondences(vm, q, Tl, offs)
    for robust in (None, "CAUCHY"):
        err, H, b, _ = system12(ct_sums(vm.vox_mean, vm.vox_cov, vm.vox_n, q, sc, ts, pairs, Tl, Tl, robust), Tl)
        # explicit: J12 = [J, s J K] per correspondence
        K = K_of(Tl)
        ia, iv = pairs[:, 0].astype(np.int64), pairs[:, 1].astype(np.int64)
        keep = vm.vox_n[iv] > 0
        ia, iv = ia[keep], iv[keep]
        R = Tl[:3, :3]
        S = vm.vox_cov[iv].astype(np.float64).reshape(-1, 3, 3).transpose(0, 2, 1) + R @ sc[ia].astype(np.float64).reshape(-1, 3, 3).transpose(0, 2, 1) @ R.T
        M = np.linalg.inv(S)
        p = q[ia].astype(np.float64) @ R.T + Tl[:3, 3]
        e = vm.vox_mean[iv].astype(np.float64) - p
        J = np.concatenate([skew(p), -np.broadcast_to(np.eye(3), (len(p), 3, 3))], axis=2)
        J12 = np.concatenate([J, ts[ia].astype(np.float64)[:, None, None] * (J @ K)], axis=2)
        sm = np.einsum("ka,kab,kb->k", e, M, e)
        from eval_reference import rho64

        r, dr = rho64(robust, sm, 1.0)
        wd = np.sqrt(vm.vox_n[iv].astype(np.float64)) * dr
        H_ex = np.einsum("k,kai,kab,kbj->ij", wd, J12, M, J12)
        b_ex = np.einsum("k,kai,kab,kb->i", wd, J12, M, e)
        assert np.max(np.abs(H - H_ex)) <= 1e-12 * np.max(np.abs(H_ex))
        assert np.max(np.abs(b - b_ex)) <= 1e-12 * np.max(np.abs(b_ex))
        assert abs(err - float((np.sqrt(vm.vox_n[iv].astype(np.float64)) * r).sum())) <= 1e-12 * abs(err)


def _err64(vm, src, sc, ts, pairs, Tl, T, xi):
    """err in float64 at fixed correspondences, the points moved by Exp(s xi) in float64 (no rounding anywhere)."""
    E = syn.se3_exp_batch(ts.astype(np.float64)[:, None] * np.asarray(xi)[None, :])
    q = np.einsum("nij,nj->ni", E[:, :3, :3], src.astype(np.float64)) + E[:, :3, 3]
    return ct_sums(vm.vox_mean, vm.vox_cov, vm.vox_n, q, sc, ts, pairs, Tl, T)["err"], q


def test_b_is_half_the_gradient_of_err():
    """At xi = 0 the linearisation is exact: 2 b equals a central difference of err to 1e-6.  At 20 deg/s over the 0.1 s sweep the
    twist block carries the J_l(s xi) ~ I approximation: its relative error stays within |s omega| / 2 = 1.75 % (0.1 s at 20 deg/s)."""
    vm, src, sc, ts, T = problem()
    offs = O.offsets(O.DIRECT7)
    pairs = O.find_correspondences(vm, src, T, offs)
    for xi, tol_xi in ((np.zeros(6), 1e-6), (np.array([0.0, 0.0, np.radians(20.0), 10.0, 0.0, 0.0]), 0.0175)):
        err, q = _err64(vm, src, sc, ts, pairs, T, T, xi)
        sums = ct_sums(vm.vox_mean, vm.vox_cov, vm.vox_n, q, sc, ts, pairs, T, T)
        _, H, b, _ = system12(sums, T)
        g = np.zeros(12)
        for j in range(12):
            h = 1e-6
            d = np.zeros(12)
            d[j] = h
            ep = _err64(vm, src, sc, ts, pairs, T, O.se3_exp(d[:6]) @ T, xi + d[6:])[0]
            em = _err64(vm, src, sc, ts, pairs, T, O.se3_exp(-d[:6]) @ T, xi - d[6:])[0]
            g[j] = (ep - em) / (2 * h)
        assert np.linalg.norm(2 * b[:6] - g[:6]) <= 1e-6 * np.linalg.norm(g[:6]), (2 * b[:6], g[:6])
        rel = np.linalg.norm(2 * b[6:] - g[6:]) / np.linalg.norm(g[6:])
        print(f"xi = {xi}: twist-block gradient relative error {rel:.3g}")
        assert rel <= tol_xi, rel


def test_zero_time_offsets_reduce_to_eval64():
    vm, src, sc, ts, T = problem()
    offs = O.offsets(O.DIRECT7)
    Tl = T @ O.se3_exp(np.array([0.001, -0.002, 0.003, 0.02, -0.01, 0.03]))
    pairs = O.find_correspondences(vm, src, Tl, offs)
    zero = np.zeros(len(src), dtype=np.float32)
    for robust in (None, "HUBER"):
        sums = ct_sums(vm.vox_mean, vm.vox_cov, vm.vox_n, src, sc, zero, pairs, _f32pose(Tl), _f32pose(T), robust)
        ref = eval64(vm.vox_mean, vm.vox_cov, vm.vox_n, src, sc, pairs, Tl, T, True, robust=robust)
        assert abs(sums["err"] - ref[0]) <= 1e-12 * abs(ref[0])
        assert np.max(np.abs(sums["H0"] - ref[1])) <= 1e-12 * np.max(np.abs(ref[1]))
        assert np.max(np.abs(sums["b0"] - ref[2])) <= 1e-12 * np.max(np.abs(ref[1]))
        assert not sums["H1"].any() and not sums["H2"].any() and not sums["b1"].any()


def ct_lm(vm, src, sc, ts, offs, guess, xi_guess, xi0, W, params=None):
    """vgicp_align_ct's LM in numpy over the model evaluation -> (T, xi, iterations, converged)."""
    p = dict(max_iterations=64, rotation_epsilon=2e-3, transformation_epsilon=5e-4, lm_max_iterations=10, lm_init_lambda_factor=1e-9)
    S = float(np.max(np.abs(ts)))
    T, xi = np.asarray(guess, dtype=np.float64).copy(), np.asarray(xi_guess, dtype=np.float64).copy()
    lam, converged = -1.0, False

    def small(d):
        D = O.se3_exp(d)
        return max(np.max(np.abs(D[:3, :3] - np.eye(3))) / p["rotation_epsilon"], np.max(np.abs(D[:3, 3])) / p["transformation_epsilon"]) < 1.0

    for it in range(p["max_iterations"]):
        (err, H, b, _), pairs = model_eval(vm, src, sc, ts, offs, T, xi, T, xi)
        y0 = err + float(W @ (xi - xi0) ** 2)
        H = H + np.diag(np.concatenate([np.zeros(6), W]))
        b = b + np.concatenate([np.zeros(6), W * (xi - xi0)])
        if lam < 0:
            lam = p["lm_init_lambda_factor"] * np.max(np.abs(np.diag(H)))
        nu, step = 2.0, None
        for j in range(p["lm_max_iterations"]):
            d = np.linalg.solve(H + lam * np.eye(12), -b)
            T2, xi2 = O.se3_exp(d[:6]) @ T, xi + d[6:]
            done = small(d[:6]) and small(S * d[6:])
            if np.linalg.norm(xi2[:3]) * S <= np.pi / 2:
                q = deskew_f32(src, ts, xi2, 0.0)
                e2 = ct_sums(vm.vox_mean, vm.vox_cov, vm.vox_n, q, sc, ts, pairs, _f32pose(T), _f32pose(T2))["err"] + float(W @ (xi2 - xi0) ** 2)
                rho = (y0 - e2) / float(d @ (lam * d - b))
            else:
                rho = -1.0
            if rho >= 0:
                T, xi = T2, xi2
                lam *= max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3)
                step = d
                break
            if done:
                step = d
                break
            lam, nu = lam * nu, 2 * nu
        if step is None:
            return T, xi, it, False
        if small(step[:6]) and small(S * step[6:]):
            return T, xi, it, True
    return T, xi, p["max_iterations"], converged


def twist_error(xi, truth):
    """(|omega - omega_true| [deg/s], |v - v_true| [m/s])"""
    return float(np.degrees(np.linalg.norm(xi[:3] - truth[:3]))), float(np.linalg.norm(xi[3:] - truth[3:]))


def test_ct_lm_registers_the_distorted_scan():
    """Plain registration misses the 0.05 m / 1 deg gate on this scan (0.240 m / 0.55 deg, test_deskew_model); the CT-LM meets it
    from the raw scan and recovers the sweep's twist."""
    vm, src, sc, ts, T = problem()
    offs = O.offsets(O.DIRECT7)
    Tc, xi, it, conv = ct_lm(vm, src, sc, ts, offs, np.eye(4), np.zeros(6), np.zeros(6), np.full(6, 1e-6))
    t, r = pose_error(T, Tc)
    tw = twist_error(xi, EFFECT_TWIST)
    print(f"CT-LM: {it} iterations, converged {conv}, pose error {t:.4f} m / {np.degrees(r):.4f} deg, twist error {tw[0]:.3f} deg/s / {tw[1]:.4f} m/s, xi {xi}")
    assert conv and t < 0.05 and r < np.radians(1.0), (t, np.degrees(r))
