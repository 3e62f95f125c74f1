#!/usr/bin/env python3
"""Robust-kernel benchmark: the cost of vgicp_set_robust_kernel's kinds against NONE.

    python scripts/bench_robust.py [--warmup 3] [--steps 20] [--device 0] [--no-c4]

C2 (the 17 k-point fixture pair, PLANE, k = 20) with DIRECT27 and DIRECT1: the whole registration (vgicp_register: k-NN,
covariances, voxel map, LM from identity), host clock around each call, which ends in a device sync.  C4 (the 1 M-point synthetic
pair, resolution 0.5) with DIRECT1 (the bulk-copy streaming kernel) and DIRECT27: one evaluation kernel (H, b, err at the ground
truth), timed with the library's CUDA-event profiling.  The arms (NONE, HUBER, CAUCHY, GEMAN_MCCLURE, scale 1) alternate inside every
step on one handle.  Before any timing, every configuration checks that NONE set after the other kinds returns the same bytes as a
fresh handle.  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line; writes nothing.
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

KINDS = ["NONE", "HUBER", "CAUCHY", "GEMAN_MCCLURE"]


def prepared(dev, tgt, src, method, res):
    from fast_gicp_b200.core import REG_PLANE, Core

    c = Core(dev)
    c.set_resolution(res)
    c.set_neighbor_search_method(method)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(REG_PLANE)
    return c


def outputs(c, T):
    """bytes of what a registration and an evaluation return"""
    r = c.align()
    c.update_correspondences(T)
    e, H, b = c.compute_error(T, True)
    return bytes(r) + np.float64(e).tobytes() + H.tobytes() + b.tobytes()


def check_none_restores(dev, tgt, src, method, res, T):
    fresh = prepared(dev, tgt, src, method, res)
    used = prepared(dev, tgt, src, method, res)
    want = outputs(fresh, T)
    for k in KINDS[1:]:
        used.set_robust_kernel(k, 1.0)
        outputs(used, T)
    used.set_robust_kernel("NONE")
    same = outputs(used, T) == want
    fresh.close()
    used.close()
    if not same:
        raise SystemExit("%s res %.2f: NONE after a robust kind differs from a fresh handle" % (method, res))


def registration_record(dev, tgt, src, method, T, W, K, note):
    from fast_gicp_b200.core import REG_PLANE, Core

    c = Core(dev)
    c.set_neighbor_search_method(method)
    t = {k: [] for k in KINDS}
    iters = {}
    for j in range(W + K):
        for k in KINDS:
            c.set_robust_kernel(k, 1.0)
            c.synchronize()
            t0 = time.perf_counter()
            r = c.register(tgt, src, k=20, reg=REG_PLANE)
            c.synchronize()
            if j >= W:
                t[k].append(1e3 * (time.perf_counter() - t0))
            iters[k] = (int(r.nr_iterations), int(r.n_linearize), int(r.n_compute_error))
    c.close()
    rows = {k: {"ms_median": float(np.median(v)), "ms_min": float(np.min(v)), "iterations_linearize_error": iters[k]} for k, v in t.items()}
    note("C2 %s registration: %s" % (method, ", ".join("%s %.3f ms" % (k, rows[k]["ms_median"]) for k in KINDS)))
    return rows


def evaluation_record(dev, tgt, src, method, res, T, W, K, note):
    c = prepared(dev, tgt, src, method, res)
    c.update_correspondences(T)
    c.compute_error(T, True)
    t = {k: [] for k in KINDS}
    for j in range(W + K):
        for k in KINDS:
            c.set_robust_kernel(k, 1.0)
            c.set_profiling(True)  # (resets the counters)
            c.compute_error(T, True)
            ms, n = c.get_profile()["linearize"]
            c.set_profiling(False)
            if j >= W:
                t[k].append(ms / max(n, 1))
    c.close()
    rows = {k: {"kernel_ms_median": float(np.median(v)), "kernel_ms_min": float(np.min(v))} for k, v in t.items()}
    note("C4 %s evaluation kernel: %s" % (method, ", ".join("%s %.4f ms" % (k, rows[k]["kernel_ms_median"]) for k in KINDS)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--no-c4", action="store_true", help="skip the 1M-point pair")
    args = ap.parse_args()
    from fast_gicp_b200.synthetic import kitti_like_pair

    t0 = time.perf_counter()

    def note(msg):
        print("[bench_robust %7.1fs] %s" % (time.perf_counter() - t0, msg), file=sys.stderr, flush=True)

    d = np.load(os.path.join(ROOT, "tests", "golden", "pair_0p1.npz"))
    c2t, c2s = np.ascontiguousarray(d["target"], dtype=np.float32), np.ascontiguousarray(d["source"], dtype=np.float32)
    T_c2 = np.loadtxt(os.path.join(ROOT, "tests", "golden", "relative.txt"))
    rec = {"card": card_info(args.device), "protocol": "%d warm-up + %d timed steps; the four arms alternate inside every step on one handle" % (args.warmup, args.steps)}
    for method in ("DIRECT27", "DIRECT1"):
        check_none_restores(args.device, c2t, c2s, method, 1.0, T_c2)
        rec["c2_%s_registration" % method] = registration_record(args.device, c2t, c2s, method, T_c2, args.warmup, args.steps, note)
    if not args.no_c4:
        c4t, c4s, T_c4 = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
        for method in ("DIRECT1", "DIRECT27"):
            check_none_restores(args.device, c4t, c4s, method, 0.5, T_c4)
            rec["c4_%s_evaluation" % method] = evaluation_record(args.device, c4t, c4s, method, 0.5, T_c4, args.warmup, args.steps, note)
    rec["none_after_robust_identical_to_fresh_handle"] = True
    rec["card_after"] = card_info(args.device)
    print(json.dumps({"robust_kernels": rec}), flush=True)


if __name__ == "__main__":
    main()
