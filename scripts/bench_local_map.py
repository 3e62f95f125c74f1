#!/usr/bin/env python3
"""Scan-to-map odometry benchmark: map maintenance on the device (vgicp_append_source_to_target + vgicp_crop_target) against
the host route (read back the source covariances, rotate, concatenate and crop on the host, upload the whole map again).

    python scripts/bench_local_map.py [--frames 30] [--repeats 3] [--device 0]

A seeded synthetic sequence (fast_gicp_b200/synthetic.py: one world, a 64-beam scan every 0.8 m along an arc turning 2 degrees
per frame, 0.25 m voxel downsample).  Each frame: register the new scan against the local map (DIRECT7, PLANE k-NN
covariances, k = 20; the guess extrapolates the last motion), then append it at the pose found and keep the newest points
within the radius, at most the cap.  Both arms run on their own handle; before any timing, every frame's align result must be
byte-identical between them.  The arms then alternate for `repeats` passes over the sequence; per frame the median of the
host clock around map maintenance and around registration (both end in a device synchronisation) is reported, with the map
size.  Drift at the last frame against the ground truth is reported for scan-to-map and for plain scan-to-scan (the
previous scan as the target); it is not a gate.  The card's name, power limit and SM clock are read in the same run.
Prints one JSON line; writes nothing.
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

from bench_multi_hypothesis import card_info  # noqa: E402


def sequence(frames, seed):
    from fast_gicp_b200 import synthetic as syn

    world = syn._make_world(np.random.default_rng(seed))
    poses, scans = [], []
    xy = np.zeros(2)
    for k in range(frames):
        yaw = np.radians(2.0 * k)
        T = np.eye(4)
        T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
        T[:2, 3] = xy
        xy = xy + 0.8 * np.array([np.cos(yaw), np.sin(yaw)])
        poses.append(T)
        scans.append(syn.voxel_downsample(syn.scan(world, 64, 2083, T, np.random.default_rng(seed * 1000 + k)), 0.25))
    return poses, scans


def rotate_covariances(T, cov9):
    """R C R^T in IEEE float32 in the order include/vgicp_b200.h documents for vgicp_append_source_to_target."""
    R = np.asarray(T, dtype=np.float64)[:3, :3].astype(np.float32)
    C = np.asarray(cov9, dtype=np.float32).reshape(-1, 3, 3)
    M = np.empty_like(C)
    N = np.empty_like(C)
    for i in range(3):
        for k in range(3):
            M[:, i, k] = (R[i, 0] * C[:, 0, k] + R[i, 1] * C[:, 1, k]) + R[i, 2] * C[:, 2, k]
    for i in range(3):
        for j in range(3):
            N[:, i, j] = (M[:, i, 0] * R[j, 0] + M[:, i, 1] * R[j, 1]) + M[:, i, 2] * R[j, 2]
    S = np.empty_like(N)
    for i in range(3):
        for j in range(3):
            S[:, i, j] = N[:, i, i] if i == j else np.float32(0.5) * (N[:, i, j] + N[:, j, i])
    return S.reshape(-1, 9)


def crop_indices(pts, center, radius, cap):
    c = np.asarray(center, dtype=np.float64).astype(np.float32)
    d = pts - c
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = np.flatnonzero(d2 <= np.float32(radius * radius))
    return keep[len(keep) - cap:] if cap and len(keep) > cap else keep


def new_core(dev):
    from fast_gicp_b200.core import Core

    c = Core(dev)
    c.set_resolution(1.0)
    c.set_neighbor_search_method("DIRECT7")
    return c


def load_source(c, pts):
    from fast_gicp_b200.core import REG_PLANE

    c.set_source_cloud(pts)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(REG_PLANE)


def run(c, scans, arm, radius, cap):
    """One pass over the sequence on handle c -> per frame (align result bytes, T, maintenance ms, registration ms, map size)."""
    from fast_gicp_b200.core import REG_PLANE, pose_from_c

    c.set_target_cloud(scans[0])
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.synchronize()
    P, S = (scans[0].copy(), c.get_target_covariances()) if arm == "host" else (None, None)
    prev, cur = np.eye(4), np.eye(4)
    out = []
    for k in range(1, len(scans)):
        guess = cur @ np.linalg.inv(prev) @ cur
        t0 = time.perf_counter()
        load_source(c, scans[k])
        r = c.align(guess)  # (ends in a device synchronisation)
        t1 = time.perf_counter()
        T = pose_from_c(r.T)
        if arm == "device":
            c.append_source_to_target(T)
            c.crop_target(T[:3, 3], radius, cap)
            n = c.num_target_points()
        else:
            P = np.vstack([P, c.transform_source(T)])
            S = np.vstack([S, rotate_covariances(T, c.get_source_covariances())])
            keep = crop_indices(P, T[:3, 3], radius, cap)
            P, S = P[keep], S[keep]
            c.set_target_cloud(P)
            c.set_target_covariances(S)
            c.create_target_voxelmap()
            n = len(P)
        c.synchronize()
        t2 = time.perf_counter()
        out.append((bytes(r), T, (t2 - t1) * 1e3, (t1 - t0) * 1e3, n))
        prev, cur = cur, T
    return out


def scan_to_scan(c, scans):
    from fast_gicp_b200.core import pose_from_c

    prev_rel, T = np.eye(4), np.eye(4)
    for k in range(1, len(scans)):
        r = c.register(scans[k - 1], scans[k], guess=prev_rel)
        prev_rel = pose_from_c(r.T)
        T = T @ prev_rel
    return T


def drift(T_gt, T):
    d = np.linalg.inv(T_gt) @ T
    ang = np.degrees(np.arccos(np.clip((np.trace(d[:3, :3]) - 1.0) / 2.0, -1.0, 1.0)))
    return {"translation_m": round(float(np.linalg.norm(d[:3, 3])), 4), "rotation_deg": round(float(ang), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--radius", type=float, default=60.0)
    ap.add_argument("--cap", type=int, default=150000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    t_start = time.perf_counter()

    def log(msg):
        print("[bench_local_map %7.1fs] %s" % (time.perf_counter() - t_start, msg), file=sys.stderr, flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_local_map needs a CUDA device (an H100); there is no CPU measurement")
    poses, scans = sequence(a.frames, a.seed)
    log(f"{len(scans)} scans, {int(np.mean([len(s) for s in scans]))} points each on average")
    dev_c, host_c = new_core(a.device), new_core(a.device)
    # equality before timing (this pass also warms both handles up)
    ref_dev = run(dev_c, scans, "device", a.radius, a.cap)
    ref_host = run(host_c, scans, "host", a.radius, a.cap)
    for k, (x, y) in enumerate(zip(ref_dev, ref_host)):
        if x[0] != y[0] or x[4] != y[4]:
            raise SystemExit(f"frame {k + 1}: the device and host routes differ")
    log("device and host routes: byte-identical align results on every frame")
    passes = {"device": [], "host": []}
    for rep in range(a.repeats):
        for arm, c in (("device", dev_c), ("host", host_c)) if rep % 2 == 0 else (("host", host_c), ("device", dev_c)):
            passes[arm].append(run(c, scans, arm, a.radius, a.cap))
    frames = []
    for k in range(len(scans) - 1):
        row = {"frame": k + 1, "map_points": ref_dev[k][4]}
        for arm in ("device", "host"):
            row[f"{arm}_maintain_ms"] = round(float(np.median([p[k][2] for p in passes[arm]])), 3)
            row[f"{arm}_register_ms"] = round(float(np.median([p[k][3] for p in passes[arm]])), 3)
        frames.append(row)
    steady = frames[len(frames) // 2:]
    summary = {arm: {"maintain_ms_mean": round(float(np.mean([f[f"{arm}_maintain_ms"] for f in steady])), 3),
                     "register_ms_mean": round(float(np.mean([f[f"{arm}_register_ms"] for f in steady])), 3)} for arm in ("device", "host")}
    s2s = scan_to_scan(new_core(a.device), scans)
    rec = {"gpu": card_info(a.device), "frames": frames, "second_half_mean": summary, "radius_m": a.radius, "cap_points": a.cap,
           "drift_scan_to_map": drift(poses[-1], ref_dev[-1][1]), "drift_scan_to_scan": drift(poses[-1], s2s)}
    print(json.dumps({"local_map": rec}), flush=True)


if __name__ == "__main__":
    main()
