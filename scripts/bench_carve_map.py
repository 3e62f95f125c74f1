#!/usr/bin/env python3
"""Dynamic objects in the local map: scan-to-map odometry past moving vehicles, with the map carved by each registered scan
(vgicp_carve_target) against today's route, which only appends, thins and crops.

    python scripts/bench_carve_map.py [--frames 30] [--repeats 3] [--leaf 0.5] [--max-per-voxel 4] [--radius 60]

The sequence is scripts/bench_thin_map.py's (the same path, seed and 64-beam scans every 0.8 m, 0.25 m downsample) with two
4 x 2 x 1.5 m vehicles (synthetic.moving_object_sequence): one overtaking in the lane to the left at twice the sensor's speed
from 8 m ahead, one oncoming in the lane to the right from 50 m ahead.  Static boxes the vehicles would drive through are taken
out of the world.  Each frame: register the new scan against the map (DIRECT7, PLANE k-NN covariances, k = 20; the guess
extrapolates the last motion), then maintain the map.  Arms, each on its own handle:
  thin        append + thin (leaf, M) + crop to the radius;
  carve       carve with the library's defaults, then as thin;
  host_carve  the carved route on the host (synthetic.carve_indices, thin_indices and the crop's float32 test on numpy arrays,
              the map uploaded again): the equality check, and the per-point labels (vehicle or static, frame) that the ghost
              counts come from.  A host copy of the thin arm gives its labels the same way.
Before any timing, the carve and host_carve arms must give byte-identical align results and map sizes on every frame, and the
thin arm's host copy its map sizes.  The thin and carve arms then alternate for `repeats` passes; per frame the median of the
host clock around each step (each ends in a device synchronisation) is reported with the map size, the vehicle points older than
one frame left in the map ("ghosts") and the static points carved so far.  Drift at the last frame is reported for both arms.  The
card's name, power limit and SM clock are read in the same run.  Prints one JSON line; writes nothing.
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

from bench_local_map import crop_indices, drift, load_source, new_core, rotate_covariances  # noqa: E402
from bench_multi_hypothesis import card_info  # noqa: E402

MOVERS = ((3.5, 8.0, 2.0), (-3.5, 50.0, -1.0))


def run(c, scans, boxes, arm, a):
    """One pass over the sequence on handle c -> per frame (align bytes, T, carve, append, thin, crop, registration ms, map size,
    ghosts, static points carved so far); the last two only on the host arms (labels), else -1."""
    from fast_gicp_b200.core import REG_PLANE, carve_params, pose_from_c
    from fast_gicp_b200.synthetic import carve_indices, in_boxes, thin_indices

    params = carve_params()
    c.set_target_cloud(scans[0])
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.synchronize()
    host = arm.startswith("host")
    if host:
        P, S = scans[0].copy(), c.get_target_covariances()
        box, frame = in_boxes(P, boxes[0]), np.zeros(len(P), dtype=np.int64)
    static_carved = 0
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
        t_carve = t_app = t_thin = t_crop = 0.0
        ghosts = -1
        if host:
            if arm == "host_carve":
                keep = carve_indices(P, scans[k], T, params)
                static_carved += int((~box).sum() - (~box[keep]).sum())
                P, S, box, frame = P[keep], S[keep], box[keep], frame[keep]
            Q = c.transform_source(T)
            P, S = np.vstack([P, Q]), np.vstack([S, rotate_covariances(T, c.get_source_covariances())])
            box, frame = np.r_[box, in_boxes(Q, boxes[k])], np.r_[frame, np.full(len(Q), k)]
            for keep in (thin_indices(P, a.leaf, a.max_per_voxel), None):
                keep = crop_indices(P, T[:3, 3], a.radius, 0) if keep is None else keep
                P, S, box, frame = P[keep], S[keep], box[keep], frame[keep]
            c.set_target_cloud(P)
            c.set_target_covariances(S)
            c.create_target_voxelmap()
            c.synchronize()
            n = len(P)
            ghosts = int((box & (frame < k - 1)).sum())
        else:
            if arm == "carve":
                t_carve = clock(lambda: c.carve_target(T))
            t_app = clock(lambda: c.append_source_to_target(T))
            t_thin = clock(lambda: c.thin_target(a.leaf, a.max_per_voxel))
            t_crop = clock(lambda: c.crop_target(T[:3, 3], a.radius, 0))
            n = c.num_target_points()
        out.append((bytes(r), T, t_carve, t_app, t_thin, t_crop, t_reg, n, ghosts, static_carved if host else -1))
        prev, cur = cur, T
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--radius", type=float, default=60.0)
    ap.add_argument("--leaf", type=float, default=0.5)
    ap.add_argument("--max-per-voxel", type=int, default=4)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    t_start = time.perf_counter()

    def log(msg):
        print("[bench_carve_map %7.1fs] %s" % (time.perf_counter() - t_start, msg), file=sys.stderr, flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_carve_map needs a CUDA device (an H100); there is no CPU measurement")
    from fast_gicp_b200.synthetic import moving_object_sequence

    poses, scans, boxes = moving_object_sequence(a.frames, a.seed, movers=MOVERS)
    log(f"{len(scans)} scans, {int(np.mean([len(s) for s in scans]))} points each on average")
    arms = ("thin", "carve", "host_thin", "host_carve")
    handles = {arm: new_core(a.device) for arm in arms}
    # equality before timing (this pass also warms the handles up)
    ref = {arm: run(handles[arm], scans, boxes, arm, a) for arm in arms}
    for k in range(len(scans) - 1):
        x, y = ref["carve"][k], ref["host_carve"][k]
        if x[0] != y[0] or x[7] != y[7]:
            raise SystemExit(f"frame {k + 1}: the device and host carved routes differ")
        if ref["thin"][k][0] != ref["host_thin"][k][0] or ref["thin"][k][7] != ref["host_thin"][k][7]:
            raise SystemExit(f"frame {k + 1}: the device and host thinned routes differ")
    log("device and host routes: byte-identical align results and map sizes on every frame")
    passes = {"thin": [], "carve": []}
    for rep in range(a.repeats):
        for arm in ("thin", "carve") if rep % 2 == 0 else ("carve", "thin"):
            passes[arm].append(run(handles[arm], scans, boxes, arm, a))
    steps = ("carve_ms", "append_ms", "thin_ms", "crop_ms", "register_ms")
    frames = []
    for k in range(len(scans) - 1):
        row = {"frame": k + 1}
        for arm in ("thin", "carve"):
            row[f"{arm}_map_points"] = ref[arm][k][7]
            row[f"{arm}_ghost_points"] = ref["host_" + arm][k][8]
            for j, name in enumerate(steps):
                if arm == "thin" and name == "carve_ms":
                    continue
                row[f"{arm}_{name}"] = round(float(np.median([p[k][2 + j] for p in passes[arm]])), 3)
        row["carve_static_removed_total"] = ref["host_carve"][k][9]
        frames.append(row)
    steady = frames[len(frames) // 2:]
    summary = {}
    for arm in ("thin", "carve"):
        names = [s for s in steps if not (arm == "thin" and s == "carve_ms")]
        summary[arm] = {f"{s}_mean": round(float(np.mean([f[f"{arm}_{s}"] for f in steady])), 3) for s in names}
        summary[arm]["maintain_ms_mean"] = round(float(np.mean([sum(f[f"{arm}_{s}"] for s in names if s != "register_ms") for f in steady])), 3)
        summary[arm]["map_points_mean"] = int(np.mean([f[f"{arm}_map_points"] for f in steady]))
        summary[arm]["ghost_points_last"] = frames[-1][f"{arm}_ghost_points"]
    rec = {"gpu": card_info(a.device), "frames": frames, "second_half_mean": summary, "radius_m": a.radius, "leaf_m": a.leaf, "max_points_per_voxel": a.max_per_voxel,
           "movers": MOVERS, "static_points_carved": frames[-1]["carve_static_removed_total"], "drift_thin": drift(poses[-1], ref["thin"][-1][1]),
           "drift_carve": drift(poses[-1], ref["carve"][-1][1])}
    print(json.dumps({"carve_map": rec}), flush=True)


if __name__ == "__main__":
    main()
