#!/usr/bin/env python3
"""Motion-compensated scan-to-map odometry: drift without deskew, with a constant-velocity deskew and with the true twist, and
the cost of the device deskew (vgicp_deskew_source) against the host route it replaces.

    python scripts/bench_deskew.py [--frames 30] [--repeats 5] [--device 0]

A seeded synthetic sequence on the arc of scripts/bench_local_map.py (one world, 0.8 m and 2 degrees per frame at 10 Hz: 8 m/s
and 20 deg/s, a constant body twist).  Every scan is distorted (fast_gicp_b200/synthetic.py distorted_scan: each azimuth column
fired at its own time of the 0.1 s sweep from its own pose), then downsampled at 0.25 m with the timestamps averaged per voxel.
The vehicle is already moving when the sequence starts and the motion of the frame before the first is known: it seeds the
guess extrapolation and the constant-velocity twist.  The first scan, loaded as the source, deskewed as in its arm and swapped into
the target, is the initial map.  Each frame, in each arm: set the scan, deskew it to the start of the sweep (or not), k-NN PLANE covariances (k = 20), register
against the local map (DIRECT7; the guess extrapolates the last motion), append it at the pose found and crop the map (radius
60 m, 150 k points).  Arms:
  none       no deskew;
  const_vel  twist = log(T_{k-2}^-1 T_{k-1}) / 0.1 s from the last two estimated poses;
  true       the generator's twist (an upper bound).
Drift at the last frame against the ground truth and the translation error of every frame are reported per arm.

Cost: per frame, the device route (set_source_cloud of the raw scan + vgicp_deskew_source) against the host route (the same
deskew in numpy float64, then set_source_cloud of the result), both ending in a device synchronisation; the routes alternate for
`repeats` passes over the sequence and the median per frame is reported.  The card's name, power limit and SM clock are read in
the same run.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_local_map import drift, new_core  # noqa: E402
from bench_multi_hypothesis import card_info  # noqa: E402

PERIOD = 0.1  # s, a 10 Hz sweep
TWIST = np.array([0.0, 0.0, np.radians(20.0), 8.0, 0.0, 0.0])  # 0.8 m and 2 degrees per frame


def sequence(frames, seed):
    from fast_gicp_b200 import synthetic as syn

    world = syn._make_world(np.random.default_rng(seed))
    poses = syn.se3_exp_batch(PERIOD * np.arange(frames)[:, None] * TWIST[None, :])
    scans = []
    for k in range(frames):
        pts, times = syn.distorted_scan(world, 64, 2083, poses[k], TWIST, PERIOD, np.random.default_rng(seed * 1000 + k))
        scans.append(syn.voxel_downsample_values(pts, times, 0.25))
    return poses, scans


def syn_exp(xi):
    from fast_gicp_b200 import synthetic as syn

    return syn.se3_exp_batch(xi)[0]


def host_deskew(pts, times, twist):
    """The host route: Exp(t_i twist) p_i per point in numpy float64."""
    from fast_gicp_b200 import synthetic as syn

    E = syn.se3_exp_batch(times.astype(np.float64)[:, None] * np.asarray(twist)[None, :])
    return (np.einsum("nij,nj->ni", E[:, :3, :3], pts.astype(np.float64)) + E[:, :3, 3]).astype(np.float32)


def odometry(c, scans, poses, arm, radius, cap):
    """One arm over the sequence -> (last pose, per-frame translation error against the ground truth [m])."""
    from fast_gicp_b200.core import REG_PLANE, pose_from_c, twist_from_motion

    # the vehicle is already moving when the sequence starts, and the motion of the frame before it is known (it seeds the guess
    # extrapolation and the constant-velocity twist)
    prev, cur = np.linalg.inv(syn_exp(PERIOD * TWIST)), np.eye(4)

    def load(pts, times):
        c.set_source_cloud(pts)
        if arm == "true":
            c.deskew_source(times, TWIST, 0.0)
        elif arm == "const_vel":
            c.deskew_source(times, twist_from_motion(np.linalg.inv(prev) @ cur, PERIOD), 0.0)
        c.find_source_neighbors(20)
        c.calculate_source_covariances(REG_PLANE)

    load(*scans[0])  # the first scan becomes the map: loaded as the source so that it is deskewed on the device, then swapped
    c.swap_source_and_target()
    c.create_target_voxelmap()
    errors = []
    for k in range(1, len(scans)):
        load(*scans[k])
        T = pose_from_c(c.align(cur @ np.linalg.inv(prev) @ cur).T)
        c.append_source_to_target(T)
        c.crop_target(T[:3, 3], radius, cap)
        prev, cur = cur, T
        errors.append(round(float(np.linalg.norm(T[:3, 3] - poses[k][:3, 3])), 4))
    return cur, errors


def cost_pass(c, scans, route):
    out = []
    for pts, times in scans[1:]:
        t0 = time.perf_counter()
        if route == "device":
            c.set_source_cloud(pts)
            c.deskew_source(times, TWIST, 0.0)
        else:
            c.set_source_cloud(host_deskew(pts, times, TWIST))
        c.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--radius", type=float, default=60.0)
    ap.add_argument("--cap", type=int, default=150000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    t_start = time.perf_counter()

    def log(msg):
        print("[bench_deskew %7.1fs] %s" % (time.perf_counter() - t_start, msg), file=sys.stderr, flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_deskew needs a CUDA device (an H100); there is no CPU measurement")
    poses, scans = sequence(a.frames, a.seed)
    log(f"{len(scans)} scans, {int(np.mean([len(s[0]) for s in scans]))} points each on average")
    rec = {"gpu": card_info(a.device), "twist": TWIST.tolist(), "period_s": PERIOD, "radius_m": a.radius, "cap_points": a.cap}
    for arm in ("none", "const_vel", "true"):
        c = new_core(a.device)
        T, errors = odometry(c, scans, poses, arm, a.radius, a.cap)
        rec[f"drift_{arm}"] = drift(poses[-1], T)
        rec[f"translation_error_per_frame_{arm}"] = errors
        c.close()
        log(f"{arm}: {rec[f'drift_{arm}']}")
    # the device result equals the float32 restatement; the host route differs from it in the last bits (float64), so only the
    # costs are compared here
    dev_c, host_c = new_core(a.device), new_core(a.device)
    cost_pass(dev_c, scans, "device")  # warm-up
    cost_pass(host_c, scans, "host")
    passes = {"device": [], "host": []}
    for rep in range(a.repeats):
        for route, c in (("device", dev_c), ("host", host_c)) if rep % 2 == 0 else (("host", host_c), ("device", dev_c)):
            passes[route].append(cost_pass(c, scans, route))
    for route in ("device", "host"):
        per_frame = np.median(np.array(passes[route]), axis=0)
        rec[f"{route}_load_and_deskew_ms_mean"] = round(float(per_frame.mean()), 3)
    # the deskew call alone (set_source_cloud outside the clock)
    alone = []
    for rep in range(a.repeats):
        for pts, times in scans[1:]:
            dev_c.set_source_cloud(pts)
            dev_c.synchronize()
            t0 = time.perf_counter()
            dev_c.deskew_source(times, TWIST, 0.0)
            dev_c.synchronize()
            alone.append((time.perf_counter() - t0) * 1e3)
    rec["device_deskew_call_ms_median"] = round(float(np.median(alone)), 3)
    host_only = []
    for pts, times in scans[1:]:
        t0 = time.perf_counter()
        host_deskew(pts, times, TWIST)
        host_only.append((time.perf_counter() - t0) * 1e3)
    rec["host_deskew_numpy_ms_median"] = round(float(np.median(host_only)), 3)
    print(json.dumps({"deskew": rec}), flush=True)


if __name__ == "__main__":
    main()
