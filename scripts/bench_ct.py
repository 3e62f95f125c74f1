#!/usr/bin/env python3
"""Continuous-time scan-to-map odometry: the three arms of scripts/bench_deskew.py plus a `ct` arm, and the cost of the
continuous-time evaluation against the plain one.

    python scripts/bench_ct.py [--frames 30] [--repeats 5] [--weight 1e-3] [--device 0]

Sequence and the arms none / const_vel / true: bench_deskew.py's, imported (30 frames at 8 m/s and 20 deg/s, every scan distorted
over its 0.1 s sweep).  The ct arm, each frame: set the raw scan and its timestamps, k-NN PLANE covariances, vgicp_align_ct from
the extrapolated pose with the twist guess and prior mean both the previous frame's estimated twist (weights --weight), then deskew
the scan with the estimated twist, recompute its covariances, append it at the pose found and crop the map.  The motion of the
frame before the first is known, as in the other arms: it seeds the first twist and deskews the first scan.  Drift at the last
frame and the translation error of every frame are reported for all four arms.

Costs, with the card's name, power limit and SM clock read in the same run:
  per frame of the ct arm, vgicp_align_ct against vgicp_align on the same handle state (host clock around calls that end in a
  device synchronisation, the two alternating in order frame by frame; medians);
  the evaluation kernel: compute_error_ct against compute_error, both linearising at the same pose, at a 17 k-point scan and at a
  1 M-point cloud, DIRECT1, DIRECT27 and DIRECT_RADIUS 1.5 (the generic offset list), kernel time from CUDA events around each
  launch (vgicp_set_profiling), medians of `repeats` alternating blocks of 50 launches.  Plain DIRECT1 at 1 M points is the
  streaming kernel; the continuous-time evaluation runs the compacted one there.
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

from bench_deskew import PERIOD, TWIST, odometry, sequence, syn_exp  # noqa: E402
from bench_local_map import drift, new_core  # noqa: E402
from bench_multi_hypothesis import card_info  # noqa: E402


def odometry_ct(c, scans, poses, radius, cap, weight):
    """The ct arm -> (last pose, per-frame translation error [m], per-frame twist estimates, align_ct ms, align ms)."""
    from fast_gicp_b200.core import REG_PLANE, pose_from_c, twist_from_motion

    prev, cur = np.linalg.inv(syn_exp(PERIOD * TWIST)), np.eye(4)
    xi = twist_from_motion(np.linalg.inv(prev) @ cur, PERIOD)
    W = np.full(6, weight)

    def covs():
        c.find_source_neighbors(20)
        c.calculate_source_covariances(REG_PLANE)

    c.set_source_cloud(scans[0][0])
    c.deskew_source(scans[0][1], xi, 0.0)
    covs()
    c.swap_source_and_target()
    c.create_target_voxelmap()
    errors, twists, t_ct, t_plain = [], [], [], []
    for k in range(1, len(scans)):
        pts, times = scans[k]
        c.set_source_cloud(pts)
        c.set_source_timestamps(times, 0.0)
        covs()
        guess = cur @ np.linalg.inv(prev) @ cur
        c.synchronize()
        for which in (("ct", "plain") if k % 2 else ("plain", "ct")):
            t0 = time.perf_counter()
            if which == "ct":
                res = c.align_ct(guess, xi, xi, W)
            else:
                c.align(guess)
            c.synchronize()
            (t_ct if which == "ct" else t_plain).append((time.perf_counter() - t0) * 1e3)
        T, xi = pose_from_c(res.T), np.array(res.twist)
        c.deskew_source(times, xi, 0.0)
        covs()
        c.append_source_to_target(T)
        c.crop_target(T[:3, 3], radius, cap)
        prev, cur = cur, T
        errors.append(round(float(np.linalg.norm(T[:3, 3] - poses[k][:3, 3])), 4))
        twists.append([round(float(v), 4) for v in xi])
    return cur, errors, twists, t_ct, t_plain


def kernel_costs(c, n_pts, repeats, methods):
    """{method: (plain kernel ms, ct kernel ms)} at the handle's current source, medians of alternating blocks."""
    rng = np.random.default_rng(3)
    c.set_source_timestamps(rng.uniform(0.0, 0.1, size=n_pts).astype(np.float32), 0.0)
    T, xi = np.eye(4), np.array([0.0, 0.0, 0.35, 8.0, 0.0, 0.0])
    out = {}
    for name, (m, r) in methods.items():
        c.set_neighbor_search_method(m, r)
        for _ in range(5):  # warm-up
            c.update_correspondences(T)
            c.compute_error(T, True)
            c.compute_error_ct(T, xi, T, xi, True)
        per = {"plain": [], "ct": []}
        for rep in range(repeats):
            for which in (("plain", "ct") if rep % 2 == 0 else ("ct", "plain")):
                c.set_profiling(True)
                c.update_correspondences(T)
                for _ in range(50):
                    if which == "plain":
                        c.compute_error(T, True)
                    else:
                        c.compute_error_ct(T, xi, T, xi, True)
                ms, cnt = c.get_profile()["linearize"]  # (CUDA events around every evaluation launch with H)
                per[which].append(ms / max(cnt, 1))
                c.set_profiling(False)
        out[name] = {"plain_kernel_ms": round(float(np.median(per["plain"])), 4), "ct_kernel_ms": round(float(np.median(per["ct"])), 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--radius", type=float, default=60.0)
    ap.add_argument("--cap", type=int, default=150000)
    ap.add_argument("--weight", type=float, default=1e-3)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    t_start = time.perf_counter()

    def log(msg):
        print("[bench_ct %7.1fs] %s" % (time.perf_counter() - t_start, msg), file=sys.stderr, flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_ct needs a CUDA device (an H100); there is no CPU measurement")
    from fast_gicp_b200.core import REG_PLANE
    from fast_gicp_b200.synthetic import kitti_like_pair

    poses, scans = sequence(a.frames, a.seed)
    log(f"{len(scans)} scans, {int(np.mean([len(s[0]) for s in scans]))} points each on average")
    rec = {"gpu": card_info(a.device), "twist": TWIST.tolist(), "period_s": PERIOD, "radius_m": a.radius, "cap_points": a.cap, "prior_weight": a.weight}
    for arm in ("none", "const_vel", "true"):
        c = new_core(a.device)
        T, errors = odometry(c, scans, poses, arm, a.radius, a.cap)
        rec[f"drift_{arm}"] = drift(poses[-1], T)
        rec[f"translation_error_per_frame_{arm}"] = errors
        c.close()
        log(f"{arm}: {rec[f'drift_{arm}']}")
    c = new_core(a.device)
    T, errors, twists, t_ct, t_plain = odometry_ct(c, scans, poses, a.radius, a.cap, a.weight)
    c.close()
    rec["drift_ct"] = drift(poses[-1], T)
    rec["translation_error_per_frame_ct"] = errors
    rec["twist_per_frame_ct"] = twists
    rec["align_ct_ms_median"] = round(float(np.median(t_ct)), 3)
    rec["align_ms_median_same_frames"] = round(float(np.median(t_plain)), 3)
    log(f"ct: {rec['drift_ct']}, align_ct {rec['align_ct_ms_median']} ms vs align {rec['align_ms_median_same_frames']} ms")

    methods = {"DIRECT1": ("DIRECT1", -1.0), "DIRECT27": ("DIRECT27", -1.0), "DIRECT_RADIUS_1.5": ("DIRECT_RADIUS", 1.5)}
    # 17 k points: the last scan of the sequence against the first
    c = new_core(a.device)
    for which, pts in (("target", scans[0][0]), ("source", scans[-1][0])):
        getattr(c, f"set_{which}_cloud")(pts)
        getattr(c, f"find_{which}_neighbors")(20)
        getattr(c, f"calculate_{which}_covariances")(REG_PLANE)
    c.create_target_voxelmap()
    rec["kernel_17k"] = {"n_source": len(scans[-1][0]), **kernel_costs(c, len(scans[-1][0]), a.repeats, methods)}
    c.close()
    log(f"17k: {rec['kernel_17k']}")
    tgt, src, _ = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0)
    rng = np.random.default_rng(44)
    tgt, src = tgt[rng.permutation(len(tgt))[:1_000_000]], src[rng.permutation(len(src))[:1_000_000]]
    c = new_core(a.device)
    c.set_resolution(0.5)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(REG_PLANE)
    rec["kernel_1M"] = {"n_source": len(src), "resolution": 0.5, **kernel_costs(c, len(src), a.repeats, methods)}
    c.close()
    log(f"1M: {rec['kernel_1M']}")
    print(json.dumps({"ct": rec}), flush=True)


if __name__ == "__main__":
    main()
