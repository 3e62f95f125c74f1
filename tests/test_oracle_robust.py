"""CPU checks of the robust-kernel checker (oracle_robust): its err, H and b against a float64 restatement of the definition,
b against a finite difference of err, NONE against the plain oracle bit for bit, and the contamination scenario that motivates
robust kernels (a moving-object cluster that pulls plain VGICP off the reference gate)."""
import numpy as np
import pytest

import oracle as O
import oracle_robust as R
from conftest import pose_error

KINDS = ["NONE", "HUBER", "CAUCHY", "GEMAN_MCCLURE"]
ROBUST = KINDS[1:]
GATE_T, GATE_R = 0.05, np.radians(1.0)  # the reference test's gate (gicp_test.cpp)


def contaminate(src, seed=1, frac=0.3, shift=0.8):
    """A stand-in for a moving object: the `frac` of source points nearest one seeded random source point, duplicated and
    shifted by `shift` m in x, appended to the source."""
    rng = np.random.default_rng(seed)
    c = src[rng.integers(len(src))]
    idx = np.argsort(((src - c) ** 2).sum(1))[: int(frac * len(src))]
    moved = src[idx].copy()
    moved[:, 0] += shift
    return np.concatenate([src, moved]).astype(np.float32)


@pytest.fixture(scope="module")
def problem(pair01):
    R.build()
    tgt, src = pair01
    tc = O.estimate_covariances(tgt)
    sc = O.estimate_covariances(src)
    return O.VoxelMap(tgt, tc, 1.0), src, sc


def rho64(kind, d2, s):
    if kind == "NONE":
        return s, np.ones_like(s)
    if kind == "HUBER":
        big = s > d2
        ss = np.where(big, s, 1.0)
        return np.where(big, 2.0 * np.sqrt(d2 * ss) - d2, s), np.where(big, np.sqrt(d2 / ss), 1.0)
    q = d2 / (d2 + s)
    if kind == "CAUCHY":
        return d2 * np.log1p(s / d2), q
    return d2 * s / (d2 + s), q * q


def skew(p):
    z = np.zeros(len(p))
    return np.stack([np.stack([z, -p[:, 2], p[:, 1]], 1), np.stack([p[:, 2], z, -p[:, 0]], 1), np.stack([-p[:, 1], p[:, 0], z], 1)], 1)


def restated(vmap, src, sc, pairs, T_lin, T_eval, kind, scale):
    """float64 err, H, b of the definition over a fixed correspondence list"""
    d2 = float(R.scale_sq(scale))
    ia, iv = pairs[:, 0], pairs[:, 1]
    n = vmap.vox_n[iv].astype(np.float64)
    keep = n > 0
    ia, iv, n = ia[keep], iv[keep], n[keep]
    a = src[ia].astype(np.float64)
    CA = sc[ia].reshape(-1, 3, 3).transpose(0, 2, 1).astype(np.float64)  # column-major rows
    CB = vmap.vox_cov[iv].reshape(-1, 3, 3).transpose(0, 2, 1).astype(np.float64)
    Rl = T_lin[:3, :3].astype(np.float32).astype(np.float64)
    p = a @ T_eval[:3, :3].T + T_eval[:3, 3]
    M = np.linalg.inv(CB + Rl @ CA @ Rl.T)
    e = vmap.vox_mean[iv].astype(np.float64) - p
    Me = np.einsum("nij,nj->ni", M, e)
    s = np.einsum("ni,ni->n", e, Me)
    r, dr = rho64(kind, d2, s)
    w = np.sqrt(n)
    J = np.concatenate([skew(p), -np.broadcast_to(np.eye(3), (len(p), 3, 3))], 2)  # [skew(p) | -I]
    wd = (w * dr)[:, None, None]
    H = np.einsum("nki,nkl,nlj->ij", J, wd * M, J)
    b = np.einsum("nki,nk->i", J, (w * dr)[:, None] * Me)
    return float((w * r).sum()), H, b


def test_rho_matches_the_definition():
    s = np.concatenate([np.zeros(1), np.logspace(-6, 4, 400)]).astype(np.float32)
    for kind in KINDS:
        for scale in (0.5, 1.0, 3.0):
            r, d = R.rho(kind, scale, s)
            r64, d64 = rho64(kind, float(R.scale_sq(scale)), s.astype(np.float64))
            np.testing.assert_allclose(r, r64, rtol=4e-7, atol=0, err_msg=kind)
            np.testing.assert_allclose(d, d64, rtol=4e-7, atol=0, err_msg=kind)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("at", ["identity", "relative"])
def test_robust_sums_match_float64_restatement(problem, relative_pose, kind, at):
    vmap, src, sc = problem
    T = np.eye(4) if at == "identity" else relative_pose
    offs = O.offsets(O.DIRECT7)
    pairs = O.find_correspondences(vmap, src, T, offs)
    e, H, b, nc = R.evaluate(vmap, src, sc, offs, T, T, robust=kind, robust_scale=1.0)
    assert nc == len(pairs)
    e64, H64, b64 = restated(vmap, src, sc, pairs, T, T, kind, 1.0)
    assert abs(e - e64) <= 2e-5 * abs(e64)
    assert np.abs(H - H64).max() <= 2e-5 * np.abs(H64).max()
    assert np.abs(b - b64).max() <= 2e-4 * np.abs(b64).max()


@pytest.mark.parametrize("kind", KINDS)
def test_b_is_half_the_gradient_of_err(problem, relative_pose, kind):
    """b = 1/2 d err / d xi (left perturbation exp(xi) T, the optimiser's update) at fixed correspondences and linearisation
    pose: a rho' that does not belong to rho fails this."""
    vmap, src, sc = problem
    T_lin = relative_pose
    T0 = O.se3_exp(np.array([0.01, -0.005, 0.008, 0.05, -0.04, 0.03])) @ T_lin  # off the minimum: a gradient to compare
    pairs = O.find_correspondences(vmap, src, T_lin, O.offsets(O.DIRECT1))
    _, _, b = R.derivatives(vmap, src, sc, pairs, T_lin, T0, robust=kind, robust_scale=1.0)
    g = np.zeros(6)
    for k in range(6):
        h = 1e-3
        dx = np.zeros(6)
        dx[k] = h
        ep = R.derivatives(vmap, src, sc, pairs, T_lin, O.se3_exp(dx) @ T0, want_H=False, robust=kind, robust_scale=1.0)[0]
        em = R.derivatives(vmap, src, sc, pairs, T_lin, O.se3_exp(-dx) @ T0, want_H=False, robust=kind, robust_scale=1.0)[0]
        g[k] = (ep - em) / (2 * h)
    np.testing.assert_allclose(b, 0.5 * g, rtol=0, atol=5e-3 * np.abs(b).max())


def test_none_is_bit_identical_to_the_plain_oracle(problem, relative_pose):
    vmap, src, sc = problem
    for method in (O.DIRECT1, O.DIRECT7, O.DIRECT27):
        offs = O.offsets(method)
        for T in (np.eye(4), relative_pose):
            for want_H in (True, False):
                a = O.evaluate(vmap, src, sc, offs, T, T, want_H=want_H)
                r = R.evaluate(vmap, src, sc, offs, T, T, want_H=want_H, robust="NONE", robust_scale=7.0)
                assert a[0] == r[0] and a[3] == r[3]
                assert np.array_equal(a[1], r[1]) and np.array_equal(a[2], r[2])
        a = O.align_f32(vmap, src, sc, offs)
        r = R.align_f32(vmap, src, sc, offs, robust="NONE")
        assert np.array_equal(a.T, r.T) and np.array_equal(a.H, r.H)
        assert (a.iterations, a.converged, a.n_linearize, a.n_error) == (r.iterations, r.converged, r.n_linearize, r.n_error)


@pytest.fixture(scope="module")
def contaminated(problem, pair01):
    vmap, _, _ = problem
    s = contaminate(pair01[1])
    return vmap, s, O.estimate_covariances(s)


def test_contamination_defeats_plain_vgicp(contaminated, relative_pose):
    vmap, s, sc = contaminated
    r = R.align_f32(vmap, s, sc, O.offsets(O.DIRECT1), robust="NONE")
    dt, dr = pose_error(relative_pose, r.T)
    assert dt > GATE_T, (dt, np.degrees(dr))  # 0.077 m / 0.83 deg


@pytest.mark.parametrize("kind", ROBUST)
def test_robust_kernels_pass_the_gate_on_contaminated_source(contaminated, relative_pose, kind):
    vmap, s, sc = contaminated
    r = R.align_f32(vmap, s, sc, O.offsets(O.DIRECT1), robust=kind, robust_scale=1.0)
    dt, dr = pose_error(relative_pose, r.T)
    assert r.converged
    assert dt < GATE_T and dr < GATE_R, (kind, dt, np.degrees(dr))
