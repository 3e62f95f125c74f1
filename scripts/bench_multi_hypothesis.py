#!/usr/bin/env python3
"""Multi-hypothesis alignment benchmark: vgicp_align_multi against a loop of vgicp_align over the same B initial guesses.

    python scripts/bench_multi_hypothesis.py [--hypotheses 1,8,32,128] [--warmup 3] [--steps 10] [--device 0]

One pair, source and target prepared once, B guesses: a +-40 deg yaw sweep around the ground truth with a seeded translation jitter
(most converge to the truth, some do not).  Per B the two arms are timed alternately after warm-up, each call ending in a device sync;
identical results (pose, Hessian, counters) are asserted before any timing.  Pairs: the 17 k-point C2 fixture pair (DIRECT27, PLANE,
k = 20) at every B, and the 1 M-point C4 pair (DIRECT1 = the bulk-copy streaming kernel, DIRECT27) at B in {1, 8}.  The card's name,
power limit and SM clock are read in the same run.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info(local_rank):
    """Name, power limit and SM clock of the card, read in the same run as the numbers they qualify."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(local_rank), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def multi_hypothesis_guesses(T_gt, B, seed):
    """B initial guesses: a yaw sweep of +-40 deg around the ground truth plus a seeded translation jitter of up to 0.75 m."""
    rng = np.random.default_rng(seed)
    yaws = np.linspace(-np.radians(40.0), np.radians(40.0), B) if B > 1 else np.zeros(1)
    G = []
    for yaw in yaws:
        D = np.eye(4)
        D[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
        D[:3, 3] = rng.uniform(-0.75, 0.75, size=3)
        G.append(D @ T_gt)
    return np.stack(G)


def multi_hypothesis_record(local_rank, pairs, W, K, note):
    """vgicp_align_multi against a loop of vgicp_align over the same guesses on the same handle (source and target prepared once),
    timed alternately in the same run with a device sync inside each timed window.  Both arms must return identical results."""
    from fast_gicp_b200.core import REG_PLANE, Core

    rec = {"card": card_info(local_rank), "protocol": "per B: %d warm-up + %d timed calls of each arm, alternating; host clock around each call, "
                                                      "which ends in a device sync" % (W, K)}
    for name, tgt, src, T_gt, res, methods, bs in pairs:
        for method in methods:
            c = Core(local_rank)
            c.set_resolution(res)
            c.set_neighbor_search_method(method)
            c.set_target_cloud(tgt)
            c.find_target_neighbors(20)
            c.calculate_target_covariances(REG_PLANE)
            c.create_target_voxelmap()
            c.set_source_cloud(src)
            c.find_source_neighbors(20)
            c.calculate_source_covariances(REG_PLANE)
            rows = []
            for B in bs:
                G = multi_hypothesis_guesses(T_gt, B, seed=B)
                multi = c.align_multi(G)
                loop = [c.align(g) for g in G]
                for i, (a, b) in enumerate(zip(multi, loop)):  # identical poses, Hessians and counters, or no timing
                    if bytes(a) != bytes(b):
                        raise SystemExit("%s %s B=%d: align_multi differs from align for guess %d" % (name, method, B, i))
                c.set_profiling(True)
                c.align_multi(G)
                pr = c.get_profile()
                c.set_profiling(False)
                launches_multi = pr["linearize"][1] + pr["compute_error"][1]
                t_multi, t_loop = [], []
                for j in range(W + K):
                    c.synchronize()
                    t0 = time.perf_counter()
                    c.align_multi(G)
                    c.synchronize()
                    t1 = time.perf_counter()
                    for g in G:
                        c.align(g)
                    c.synchronize()
                    t2 = time.perf_counter()
                    if j >= W:
                        t_multi.append(1e3 * (t1 - t0))
                        t_loop.append(1e3 * (t2 - t1))
                ms_m, ms_l = float(np.median(t_multi)), float(np.median(t_loop))
                rows.append({"B": B, "align_multi_ms": ms_m, "align_loop_ms": ms_l, "speedup": ms_l / ms_m,
                             "hypotheses_per_s_multi": B / (ms_m * 1e-3), "hypotheses_per_s_loop": B / (ms_l * 1e-3),
                             "launches_multi": int(launches_multi), "evaluations_loop": int(sum(r.n_linearize + r.n_compute_error for r in loop)),
                             "rounds": int(max(1 + r.n_compute_error for r in multi)), "converged": int(sum(r.converged for r in multi)),
                             "identical_to_loop": True})
                note("multi-hypothesis %s %s B=%d: %.2f ms vs %.2f ms" % (name, method, B, ms_m, ms_l))
            c.close()
            rec["%s_%s" % (name, method)] = {"n_target": len(tgt), "n_source": len(src), "res": res, "rows": rows}
    rec["card_after"] = card_info(local_rank)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hypotheses", default="1,8,32,128", help="comma-separated B values for the C2 pair")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--no-c4", action="store_true", help="skip the 1M-point pair")
    args = ap.parse_args()
    from fast_gicp_b200.synthetic import kitti_like_pair

    t0 = time.perf_counter()

    def note(msg):
        print("[bench_multi_hypothesis %7.1fs] %s" % (time.perf_counter() - t0, msg), file=sys.stderr, flush=True)

    Bs = [int(x) for x in args.hypotheses.split(",") if x.strip()]
    d = np.load(os.path.join(ROOT, "tests", "golden", "pair_0p1.npz"))
    T_c2 = np.loadtxt(os.path.join(ROOT, "tests", "golden", "relative.txt"))
    pairs = [("c2", np.ascontiguousarray(d["target"], dtype=np.float32), np.ascontiguousarray(d["source"], dtype=np.float32), T_c2, 1.0, ["DIRECT27"], Bs)]
    if not args.no_c4:
        c4t, c4s, T_c4 = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
        pairs.append(("c4", c4t, c4s, T_c4, 0.5, ["DIRECT1", "DIRECT27"], [1, 8]))
    rec = multi_hypothesis_record(args.device, pairs, args.warmup, args.steps, note)
    print(json.dumps({"multi_hypothesis": rec}), flush=True)


if __name__ == "__main__":
    main()
