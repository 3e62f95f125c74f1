#!/usr/bin/env python3
"""Multi-source alignment benchmark: vgicp_align_sources against a loop of set_source_cloud + find_source_neighbors +
calculate_source_covariances + vgicp_align over the same B sources, on the same handle.

    python scripts/bench_align_sources.py [--sources 1,4,16,64] [--warmup 2] [--steps 5] [--device 0] [--no-large]

Sources: scans of one synthetic world (fast_gicp_b200.synthetic.scan, 64 beams) from sensor poses spread over a few metres and
degrees, voxel-downsampled to about 17 k points; each guess is the true pose with a seeded jitter.  Maps of the same world: a 64-beam
scan from the origin downsampled to about 17 k points (DIRECT27, resolution 1.0), and the 1 M-point 128-beam kitti_like_pair
target (DIRECT1, resolution 0.5).  Per map and B the two arms must return identical results (pose, Hessian, counters) before
anything is timed; they are then timed alternately, each call ending in a device sync.  Stage-1 time (unpack, k-NN, covariances) and
optimiser time (evaluation kernels) come from vgicp_get_profile in one profiled call of each arm: only the optimiser is batched.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line; writes nothing.
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

SEED = 44  # the world of kitti_like_pair(seed=44), so that the large map and the sources see the same boxes


def yaw_pose(x, y, yaw_deg):
    T = np.eye(4)
    a = np.radians(yaw_deg)
    T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    T[:2, 3] = [x, y]
    return T


def make_sources(B_max, note):
    """B_max scans (sensor frame) of the world from nearby poses, downsampled to about 17 k points, and their jittered guesses."""
    from fast_gicp_b200 import synthetic as S

    world = S._make_world(np.random.default_rng(SEED))
    rng = np.random.default_rng(7)
    poses = [yaw_pose(*rng.uniform(-3.0, 3.0, size=2), rng.uniform(-10.0, 10.0)) for _ in range(B_max)]
    raw = [S.scan(world, 64, 2083, T, np.random.default_rng(100 + i)) for i, T in enumerate(poses)]
    leaf = min((0.2, 0.25, 0.3, 0.35, 0.4, 0.5), key=lambda l: abs(len(S.voxel_downsample(raw[0], l)) - 17000))
    srcs = [S.voxel_downsample(r, leaf) for r in raw]
    guesses = np.stack([T @ yaw_pose(*rng.uniform(-0.2, 0.2, size=2), rng.uniform(-1.0, 1.0)) for T in poses])
    note("%d sources, leaf %.2f m, %d..%d points" % (B_max, leaf, min(map(len, srcs)), max(map(len, srcs))))
    return world, srcs, guesses, leaf


def arm_sources(c, S, G):
    return c.align_sources(S, G)


def arm_loop(c, S, G):
    out = []
    for s, g in zip(S, G):
        c.set_source_cloud(s)
        c.find_source_neighbors(20)
        c.calculate_source_covariances()
        out.append(c.align(g))
    return out


def profiled(c, fn, S, G):
    """GPU time per part of one call from vgicp_get_profile: stage 1 (unpack, k-NN, covariances) and the optimiser's evaluations."""
    c.set_profiling(True)
    fn(c, S, G)
    pr = c.get_profile()
    c.set_profiling(False)
    return {"stage1_gpu_ms": pr["unpack_points"][0] + pr["knn"][0] + pr["covariance"][0], "optimizer_gpu_ms": pr["linearize"][0] + pr["compute_error"][0],
            "stage1_launches": int(pr["unpack_points"][1] + pr["knn"][1] + pr["covariance"][1]),
            "evaluation_launches": int(pr["linearize"][1] + pr["compute_error"][1])}


def record(device, maps, srcs, guesses, Bs, W, K, note):
    from fast_gicp_b200.core import REG_PLANE, Core

    rec = {"card": card_info(device), "protocol": "per map and B: %d warm-up + %d timed calls of each arm, alternating; host clock around each "
                                                  "call, which ends in a device sync; GPU times per part from one profiled call of each arm" % (W, K)}
    for name, tgt, res, method in maps:
        c = Core(device)
        c.set_resolution(res)
        c.set_neighbor_search_method(method)
        c.set_target_cloud(tgt)
        c.find_target_neighbors(20)
        c.calculate_target_covariances(REG_PLANE)
        c.create_target_voxelmap()
        rows = []
        for B in Bs:
            S, G = srcs[:B], guesses[:B]
            a, b = arm_sources(c, S, G), arm_loop(c, S, G)
            for i, (x, y) in enumerate(zip(a, b)):  # identical poses, Hessians and counters, or no timing
                if bytes(x) != bytes(y):
                    raise SystemExit("%s B=%d: align_sources differs from the loop for source %d" % (name, B, i))
            p_src, p_loop = profiled(c, arm_sources, S, G), profiled(c, arm_loop, S, G)
            t_src, t_loop = [], []
            for j in range(W + K):
                c.synchronize()
                t0 = time.perf_counter()
                arm_sources(c, S, G)
                c.synchronize()
                t1 = time.perf_counter()
                arm_loop(c, S, G)
                c.synchronize()
                t2 = time.perf_counter()
                if j >= W:
                    t_src.append(1e3 * (t1 - t0))
                    t_loop.append(1e3 * (t2 - t1))
            ms_s, ms_l = float(np.median(t_src)), float(np.median(t_loop))
            rows.append({"B": B, "align_sources_ms": ms_s, "loop_ms": ms_l, "speedup": ms_l / ms_s, "registrations_per_s_sources": B / (ms_s * 1e-3),
                         "registrations_per_s_loop": B / (ms_l * 1e-3), "profile_sources": p_src, "profile_loop": p_loop,
                         "converged": int(sum(r.converged for r in a)), "identical_to_loop": True})
            note("%s B=%d: %.2f ms vs %.2f ms (stage 1 GPU %.2f / %.2f ms, optimiser GPU %.2f / %.2f ms)" % (
                name, B, ms_s, ms_l, p_src["stage1_gpu_ms"], p_loop["stage1_gpu_ms"], p_src["optimizer_gpu_ms"], p_loop["optimizer_gpu_ms"]))
        c.close()
        rec[name] = {"n_target": len(tgt), "method": method, "res": res, "n_source_min": int(min(map(len, srcs))), "n_source_max": int(max(map(len, srcs))),
                     "rows": rows}
    rec["card_after"] = card_info(device)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", default="1,4,16,64", help="comma-separated B values")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--no-large", action="store_true", help="skip the 1 M-point map")
    args = ap.parse_args()
    from fast_gicp_b200 import synthetic as S

    t0 = time.perf_counter()

    def note(msg):
        print("[bench_align_sources %7.1fs] %s" % (time.perf_counter() - t0, msg), file=sys.stderr, flush=True)

    Bs = [int(x) for x in args.sources.split(",") if x.strip()]
    world, srcs, guesses, leaf = make_sources(max(Bs), note)
    small = S.voxel_downsample(S.scan(world, 64, 2083, np.eye(4), np.random.default_rng(SEED)), leaf)
    maps = [("map17k", small, 1.0, "DIRECT27")]
    if not args.no_large:
        big, _, _ = S.kitti_like_pair(beams=128, az_steps=8192, seed=SEED, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
        maps.append(("map1m", big, 0.5, "DIRECT1"))
    note("maps: %s" % ", ".join("%s %d points" % (m[0], len(m[1])) for m in maps))
    rec = record(args.device, maps, srcs, guesses, Bs, args.warmup, args.steps, note)
    print(json.dumps({"align_sources": rec}), flush=True)


if __name__ == "__main__":
    main()
