#!/usr/bin/env python3
"""Voxel-capped local map: scan-to-map odometry with the map thinned to at most M points per cell (vgicp_thin_target) against
today's route, a point cap that keeps the newest points (vgicp_crop_target's max_points).

    python scripts/bench_thin_map.py [--frames 30] [--repeats 3] [--leaf 0.5] [--max-per-voxel 4] [--stop 0] [--drive-back]

The sequence is scripts/bench_local_map.py's (the same world, scans and seed: 64-beam scans every 0.8 m along an arc, 0.25 m
downsample).  --stop K inserts K stationary frames (the same pose, fresh range noise) in the middle of the sequence;
--drive-back appends the way back over the start (the poses in reverse order, fresh range noise).  Each frame: register the new
scan against the map (DIRECT7, PLANE k-NN covariances, k = 20; the guess extrapolates the last motion), then maintain the map.
Arms, each on its own handle:
  cap        append + crop to the radius with the point cap (default 150 k points);
  thin       append + thin (leaf, M) + crop to the radius without a cap;
  host_thin  the thinned route on the host (synthetic.thin_indices and the crop's float32 test on numpy arrays, then the map
             uploaded again): used only as the equality check.
Before any timing, the thin and host_thin arms must give byte-identical align results and map sizes on every frame.  The cap and
thin arms then alternate for `repeats` passes; per frame the median of the host clock around append, thin, crop and registration
(each ends in a device synchronisation) is reported with the map size.  Drift at the last frame against the ground truth is
reported for both arms.  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line; writes nothing.
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

from bench_local_map import crop_indices, drift, load_source, new_core, rotate_covariances, sequence  # noqa: E402
from bench_multi_hypothesis import card_info  # noqa: E402


def frames_for(frames, seed, stop, drive_back):
    """bench_local_map's sequence, with `stop` stationary frames inserted at its middle and, optionally, the way back."""
    from fast_gicp_b200 import synthetic as syn

    poses, scans = sequence(frames, seed)
    if not stop and not drive_back:
        return poses, scans
    world = syn._make_world(np.random.default_rng(seed))
    extra = iter(range(frames, 10 * frames + stop))  # noise seeds past the sequence's own

    def fresh(T):
        return syn.voxel_downsample(syn.scan(world, 64, 2083, T, np.random.default_rng(seed * 1000 + next(extra))), 0.25)

    mid = frames // 2
    P, S = list(poses[:mid + 1]), list(scans[:mid + 1])
    for _ in range(stop):
        P.append(poses[mid])
        S.append(fresh(poses[mid]))
    P += poses[mid + 1:]
    S += scans[mid + 1:]
    if drive_back:
        for T in poses[-2::-1]:
            P.append(T)
            S.append(fresh(T))
    return P, S


def run(c, scans, arm, a):
    """One pass over the sequence on handle c -> per frame (align result bytes, T, append, thin, crop, registration ms, map size)."""
    from fast_gicp_b200.core import REG_PLANE, pose_from_c
    from fast_gicp_b200.synthetic import thin_indices

    c.set_target_cloud(scans[0])
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.synchronize()
    P, S = (scans[0].copy(), c.get_target_covariances()) if arm == "host_thin" else (None, None)
    prev, cur = np.eye(4), np.eye(4)
    out = []

    def clock(f):
        t0 = time.perf_counter()
        f()
        c.synchronize()
        return (time.perf_counter() - t0) * 1e3

    for k in range(1, len(scans)):
        guess = cur @ np.linalg.inv(prev) @ cur
        t0 = time.perf_counter()
        load_source(c, scans[k])
        r = c.align(guess)  # (ends in a device synchronisation)
        t_reg = (time.perf_counter() - t0) * 1e3
        T = pose_from_c(r.T)
        t_app = t_thin = t_crop = 0.0
        if arm == "host_thin":
            P = np.vstack([P, c.transform_source(T)])
            S = np.vstack([S, rotate_covariances(T, c.get_source_covariances())])
            keep = thin_indices(P, a.leaf, a.max_per_voxel)
            P, S = P[keep], S[keep]
            keep = crop_indices(P, T[:3, 3], a.radius, 0)
            P, S = P[keep], S[keep]
            c.set_target_cloud(P)
            c.set_target_covariances(S)
            c.create_target_voxelmap()
            c.synchronize()
            n = len(P)
        else:
            t_app = clock(lambda: c.append_source_to_target(T))
            if arm == "thin":
                t_thin = clock(lambda: c.thin_target(a.leaf, a.max_per_voxel))
            t_crop = clock(lambda: c.crop_target(T[:3, 3], a.radius, a.cap if arm == "cap" else 0))
            n = c.num_target_points()
        out.append((bytes(r), T, t_app, t_thin, t_crop, t_reg, n))
        prev, cur = cur, T
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--radius", type=float, default=60.0)
    ap.add_argument("--cap", type=int, default=150000)
    ap.add_argument("--leaf", type=float, default=0.5)
    ap.add_argument("--max-per-voxel", type=int, default=4)
    ap.add_argument("--stop", type=int, default=0, help="stationary frames inserted in the middle of the sequence")
    ap.add_argument("--drive-back", action="store_true", help="append the way back over the start")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    t_start = time.perf_counter()

    def log(msg):
        print("[bench_thin_map %7.1fs] %s" % (time.perf_counter() - t_start, msg), file=sys.stderr, flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_thin_map needs a CUDA device (an H100); there is no CPU measurement")
    poses, scans = frames_for(a.frames, a.seed, a.stop, a.drive_back)
    log(f"{len(scans)} scans, {int(np.mean([len(s) for s in scans]))} points each on average")
    handles = {arm: new_core(a.device) for arm in ("cap", "thin", "host_thin")}
    # equality before timing (this pass also warms the handles up)
    ref = {arm: run(handles[arm], scans, arm, a) for arm in ("cap", "thin", "host_thin")}
    for k, (x, y) in enumerate(zip(ref["thin"], ref["host_thin"])):
        if x[0] != y[0] or x[6] != y[6]:
            raise SystemExit(f"frame {k + 1}: the device and host thinned routes differ")
    log("thinned route, device and host: byte-identical align results and map sizes on every frame")
    passes = {"cap": [], "thin": []}
    for rep in range(a.repeats):
        for arm in ("cap", "thin") if rep % 2 == 0 else ("thin", "cap"):
            passes[arm].append(run(handles[arm], scans, arm, a))
    steps = ("append_ms", "thin_ms", "crop_ms", "register_ms")
    frames = []
    for k in range(len(scans) - 1):
        row = {"frame": k + 1}
        for arm in ("cap", "thin"):
            row[f"{arm}_map_points"] = ref[arm][k][6]
            for j, name in enumerate(steps):
                if arm == "cap" and name == "thin_ms":
                    continue
                row[f"{arm}_{name}"] = round(float(np.median([p[k][2 + j] for p in passes[arm]])), 3)
        frames.append(row)
    steady = frames[len(frames) // 2:]
    summary = {}
    for arm in ("cap", "thin"):
        names = [s for s in steps if not (arm == "cap" and s == "thin_ms")]
        summary[arm] = {f"{s}_mean": round(float(np.mean([f[f"{arm}_{s}"] for f in steady])), 3) for s in names}
        summary[arm]["maintain_ms_mean"] = round(float(np.mean([sum(f[f"{arm}_{s}"] for s in names if s != "register_ms") for f in steady])), 3)
        summary[arm]["map_points_mean"] = int(np.mean([f[f"{arm}_map_points"] for f in steady]))
    rec = {"gpu": card_info(a.device), "frames": frames, "second_half_mean": summary, "radius_m": a.radius, "cap_points": a.cap, "leaf_m": a.leaf,
           "max_points_per_voxel": a.max_per_voxel, "stationary_frames": a.stop, "drive_back": a.drive_back,
           "drift_cap": drift(poses[-1], ref["cap"][-1][1]), "drift_thin": drift(poses[-1], ref["thin"][-1][1])}
    print(json.dumps({"thin_map": rec}), flush=True)


if __name__ == "__main__":
    main()
