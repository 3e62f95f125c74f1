"""Motion compensation (vgicp_deskew_source) on the CPU: the numpy float32 restatement of the recipe in include/vgicp_b200.h,
the series it uses, twist_from_motion, the motion-distorted scan generator, and the effect of deskewing on a registration with
the CPU oracle.  tests/test_gpu_deskew.py checks the device against deskew_f32 byte for byte."""
import importlib.util
import math
import os

import numpy as np
import pytest

import oracle as O
from conftest import pose_error

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _module(name, rel):
    """Load a package module without the package __init__ (which needs the CUDA library)."""
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


syn = _module("_synthetic", "fast_gicp_b200/synthetic.py")
core = _module("_core", "fast_gicp_b200/core.py")

# ------------------------------------------------------------------------------------------------------------ numpy model
# Horner coefficients of include/vgicp_b200.h, highest power first
A_COEF = [F("1.6059044e-10"), F("-2.5052108e-08"), F("2.7557319e-06"), F("-0.0001984127"), F("0.008333334"), F("-0.16666667"), F("1.0")]
B_COEF = [F("-2.0876756e-09"), F("2.755732e-07"), F("-2.4801588e-05"), F("0.0013888889"), F("-0.041666668"), F("0.5")]
C_COEF = [F("-1.6059044e-10"), F("2.5052108e-08"), F("-2.7557319e-06"), F("0.0001984127"), F("-0.008333334"), F("0.16666667")]


def horner(coef, q):
    h = np.full_like(q, coef[0])
    for c in coef[1:]:
        h = h * q + c
    return h


def deskew_f32(pts, times, twist, t_ref=0.0):
    """vgicp_deskew_source restated in numpy float32, operation for operation."""
    p = np.asarray(pts, dtype=np.float32)[:, :3]
    tau = F(t_ref)
    xi = np.asarray(twist, dtype=np.float64).astype(np.float32)
    s = np.asarray(times, dtype=np.float32) - tau
    w = [s * xi[j] for j in range(3)]
    u = [s * xi[3 + j] for j in range(3)]
    q = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    A, B, C = horner(A_COEF, q), horner(B_COEF, q), horner(C_COEF, q)
    z = np.zeros_like(s)
    K = [[z, -w[2], w[1]], [w[2], z, -w[0]], [-w[1], w[0], z]]
    out = np.empty_like(p)
    for j in range(3):
        R, V = [], []
        for k in range(3):
            d = F(1) if j == k else F(0)
            k2 = w[j] * w[k] - q if j == k else w[j] * w[k]
            R.append((d + A * K[j][k]) + B * k2)
            V.append((d + B * K[j][k]) + C * k2)
        out[:, j] = ((R[0] * p[:, 0] + R[1] * p[:, 1]) + R[2] * p[:, 2]) + ((V[0] * u[0] + V[1] * u[1]) + V[2] * u[2])
    return out


def random_twist(rng, max_theta, span):
    """A twist whose rotation over |t - t_ref| <= span is at most max_theta, with up to 30 m/s of translation."""
    w = rng.normal(size=3)
    w *= rng.uniform(0.0, max_theta / span) / np.linalg.norm(w)
    return np.concatenate([w, rng.uniform(-30.0, 30.0, size=3)])


# ------------------------------------------------------------------------------------------------------------ series
def test_series_within_two_ulp_of_closed_forms():
    theta = np.linspace(0.0, np.pi / 2, 100001)
    q = (theta * theta).astype(np.float32)
    qd = q.astype(np.float64)
    th = np.sqrt(qd)
    with np.errstate(divide="ignore", invalid="ignore"):
        ref_a = np.where(th > 0, np.sin(th) / th, 1.0)
        ref_b = np.where(th > 0, 2.0 * np.sin(0.5 * th) ** 2 / qd, 0.5)  # (1 - cos) / theta^2 without the cancellation
        # (theta - sin) / theta^3 cancels for small theta: below 0.1 the float64 series (exact there) stands in
        ser_c = sum((-1) ** k * qd ** k / math.factorial(2 * k + 3) for k in range(12))
        ref_c = np.where(th > 0.1, (th - np.sin(th)) / (qd * th), ser_c)
    for coef, ref in ((A_COEF, ref_a), (B_COEF, ref_b), (C_COEF, ref_c)):
        got = horner(coef, q).astype(np.float64)
        ulp = np.spacing(ref.astype(np.float32)).astype(np.float64)
        assert np.max(np.abs(got - ref) / ulp) <= 2.0


def test_restatement_matches_se3_exp_in_double():
    rng = np.random.default_rng(3)
    n = 4000
    for trial in range(8):
        span = 0.1
        xi = random_twist(rng, np.pi / 2 if trial == 0 else rng.uniform(0.0, np.pi / 2), span)
        t_ref = rng.uniform(0.0, 0.1)
        times = (t_ref + rng.uniform(-span, span, size=n)).astype(np.float32)
        times[0] = F(t_ref + span)  # reach the edge
        pts = rng.uniform(-100.0, 100.0, size=(n, 3)).astype(np.float32)
        got = deskew_f32(pts, times, xi, t_ref).astype(np.float64)
        s = times.astype(np.float64) - np.float64(F(t_ref))
        ref = np.empty((n, 3))
        for i in range(n):
            T = O.se3_exp(s[i] * xi.astype(np.float32).astype(np.float64))
            ref[i] = T[:3, :3] @ pts[i].astype(np.float64) + T[:3, 3]
        bound = 1e-6 * (np.linalg.norm(pts, axis=1) + np.abs(s) * np.linalg.norm(xi[3:]))
        assert np.all(np.linalg.norm(got - ref, axis=1) <= bound)


def test_zero_twist_returns_the_points():
    rng = np.random.default_rng(5)
    pts = rng.uniform(-100.0, 100.0, size=(1000, 3)).astype(np.float32)
    pts[:5] = 0.0
    times = rng.uniform(0.0, 0.1, size=1000).astype(np.float32)
    out = deskew_f32(pts, times, np.zeros(6), 0.05)
    assert np.array_equal(out, pts)  # == treats -0 as 0: only the sign of a zero may differ


# ------------------------------------------------------------------------------------------------------------ twist_from_motion
def test_twist_from_motion_round_trips_through_se3_exp():
    rng = np.random.default_rng(11)
    for trial in range(200):
        w = rng.normal(size=3)
        angle = [0.0, 1e-9, 1e-5, 1e-3][trial] if trial < 4 else rng.uniform(0.0, np.pi - 0.1)
        w *= angle / np.linalg.norm(w)
        xi = np.concatenate([w, rng.uniform(-5.0, 5.0, size=3)])
        dt = rng.uniform(0.05, 0.2)
        T = O.se3_exp(xi)
        got = core.twist_from_motion(T, dt)
        assert np.max(np.abs(O.se3_exp(got * dt) - T)) < 1e-12
        assert np.max(np.abs(got * dt - xi)) < 1e-9


# ------------------------------------------------------------------------------------------------------------ generator
def test_distorted_scan_with_zero_twist_is_scan():
    world = syn._make_world(np.random.default_rng(7))
    T = np.eye(4)
    T[:3, 3] = [3.0, 1.0, 0.2]
    ref = syn.scan(world, 16, 600, T, np.random.default_rng(5))
    got, times = syn.distorted_scan(world, 16, 600, T, np.zeros(6), 0.1, np.random.default_rng(5))
    assert got.tobytes() == ref.tobytes()
    assert times.dtype == np.float32 and len(times) == len(got) and times.min() >= 0.0 and times.max() < 0.1


def test_distorted_scan_deskewed_lies_on_the_world():
    world = syn._make_world(np.random.default_rng(7))
    yaw = np.radians(30.0)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
    T[:3, 3] = [3.0, 1.0, 0.2]
    xi = np.array([0.01, -0.02, np.radians(40.0), 15.0, 0.5, 0.1])
    pts, times = syn.distorted_scan(world, 32, 1000, T, xi, 0.1, np.random.default_rng(5), noise=0.0)
    E = syn.se3_exp_batch(times.astype(np.float64)[:, None] * xi[None, :])
    p0 = np.einsum("nij,nj->ni", E[:, :3, :3], pts.astype(np.float64)) + E[:, :3, 3]
    pw = p0 @ T[:3, :3].T + T[:3, 3]
    dist = np.abs(pw[:, 2] + 1.73)
    for lo, hi in world:
        inside = np.all((pw >= lo - 1e-3) & (pw <= hi + 1e-3), axis=1)
        face = np.min(np.abs(np.concatenate([pw - lo, pw - hi], axis=1)), axis=1)
        dist = np.where(inside, np.minimum(dist, face), dist)
    assert dist.max() < 1e-4
    # and the distortion is real: the raw points, taken as if fired at t = 0, miss the surfaces by far more
    raw = pts.astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    assert np.abs(raw - pw).max() > 1.0


def test_downsample_with_values_keeps_voxel_downsample_points():
    rng = np.random.default_rng(2)
    pts = rng.uniform(-5.0, 5.0, size=(5000, 3)).astype(np.float32)
    vals = rng.uniform(0.0, 0.1, size=5000).astype(np.float32)
    p, v = syn.voxel_downsample_values(pts, vals, 0.5)
    assert p.tobytes() == syn.voxel_downsample(pts, 0.5).tobytes()
    assert v.dtype == np.float32 and len(v) == len(p) and v.min() >= 0.0 and v.max() <= 0.1


# ------------------------------------------------------------------------------------------------------------ effect
# A car at 10 m/s turning at 20 deg/s (an urban turn), a 10 Hz sweep: 1 m and 2 deg of motion inside one scan.
EFFECT_TWIST = np.array([0.0, 0.0, np.radians(20.0), 10.0, 0.0, 0.0])
EFFECT_POSE = (0.8, 0.05, 0.7)


def distorted_pair(seed=42):
    """(clean target scanned at the origin, distorted source, its timestamps, pose of the source sensor at t = 0)."""
    world = syn._make_world(np.random.default_rng(seed))
    tgt = syn.voxel_downsample(syn.scan(world, 64, 2083, np.eye(4), np.random.default_rng(seed)), 0.25)
    yaw = np.radians(EFFECT_POSE[2])
    T = np.eye(4)
    T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
    T[:3, 3] = [EFFECT_POSE[0], EFFECT_POSE[1], 0.0]
    pts, times = syn.distorted_scan(world, 64, 2083, T, EFFECT_TWIST, 0.1, np.random.default_rng(seed + 1))
    src, ts = syn.voxel_downsample_values(pts, times, 0.25)
    return tgt, src, ts, T


def test_deskew_brings_a_distorted_scan_within_the_gate():
    """Oracle (DIRECT7, PLANE): raw 0.240 m / 0.55 deg from the truth, deskewed with the true twist 0.0009 m / 0.007 deg."""
    tgt, src, ts, T = distorted_pair()
    raw = O.register_f32(tgt, src, method=O.DIRECT7, accum_double=True)
    fixed = O.register_f32(tgt, deskew_f32(src, ts, EFFECT_TWIST, 0.0), method=O.DIRECT7, accum_double=True)
    t0, r0 = pose_error(T, raw.T)
    t1, r1 = pose_error(T, fixed.T)
    assert not (t0 < 0.05 and r0 < np.radians(1.0)), (t0, np.degrees(r0))
    assert fixed.converged and t1 < 0.05 and r1 < np.radians(1.0), (t1, np.degrees(r1))
    assert t0 > 0.2 and t1 < 0.002, (t0, t1)
