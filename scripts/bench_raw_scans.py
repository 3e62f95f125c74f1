#!/usr/bin/env python3
"""Raw timestamped scans into the registration without a host round trip: the cost of the device front end against the host
routes it replaces, and continuous-time odometry driven by it.

    python scripts/bench_raw_scans.py [--frames 30] [--repeats 5] [--weight 1e-3] [--device 0]

Sequence: scripts/bench_deskew.py's (30 frames at 8 m/s and 20 deg/s, every scan distorted over its 0.1 s sweep; same world, poses
and noise seeds), but each raw distorted scan (64 x 2083 rays) is kept as 32-byte PointXYZIT-like records -- x y z, intensity (a
synthetic return strength), time, ring, padding -- instead of being downsampled on the host.

Cost per frame, four routes from the raw records to a source cloud with one timestamp per point, each ending in a device
synchronisation, host clock, the routes alternating in order for `repeats` passes; medians per frame, then their median:
  device  one upload of the records, InputPrep.approximate_voxel_grid_fields at 0.25 m (time and intensity averaged per voxel),
          set_source_cloud_device and set_source_timestamps_device reading the prep output in place;
  exact   the same with InputPrep.voxel_grid, the exact grid (pcl::VoxelGrid) on the device, instead of the approximate one;
  numpy   synthetic.voxel_downsample_values (the exact-grid numpy downsample bench_deskew.py / bench_ct.py use), then
          set_source_cloud and set_source_timestamps;
  serial  the serial C filter with fields (oracle_fields: the same approximate grid, standing in for PCL on the host), then
          the same host calls.
Odometry: bench_ct.py's ct arm driven by each device front end, the approximate and the exact grid -- per frame upload + prep,
device cloud and timestamps, k-NN PLANE covariances, align_ct from the extrapolated pose (twist guess and prior mean: the previous
estimate, weights --weight), deskew_source_stored with the estimated twist, covariances, append, crop.  Their drifts after the last
frame are reported, not gated against bench_ct.py's: the numpy downsample there divides by the leaf in float64 sums, so even the
exact grid's point set differs from it in the last bits.  The device route is also split into its upload, the filter with fields,
the xyz-only filter (vgicp_prep_approximate_voxel_grid on the same device records) and the exact grid with fields.  Filter only,
device in and device out: the exact grid on a raw sweep with fields, on a 1 M-point unfiltered kitti_like_pair cloud (x y z) and
on 1 M points in one voxel with fields (the worst case: one in-order sum), CUDA events around `repeats` windows of 10 calls each
after a warm-up.  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line; writes nothing.
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

from bench_deskew import PERIOD, TWIST, syn_exp  # noqa: E402
from bench_local_map import drift, new_core  # noqa: E402
from bench_multi_hypothesis import card_info  # noqa: E402

LEAF = 0.25
RECORD = np.dtype([("x", np.float32), ("y", np.float32), ("z", np.float32), ("intensity", np.float32), ("time", np.float32), ("ring", np.float32),
                   ("pad", np.float32, 2)])
FIELDS = [4, 3]  # float columns of the record averaged per voxel: time (first, so that it sits at float 3 of the output), intensity
STRIDE = 4 * (3 + len(FIELDS))  # bytes per output record


def raw_sequence(frames, seed):
    """bench_deskew.sequence's poses and raw distorted scans, as (n, 8) float32 views of 32-byte records."""
    from fast_gicp_b200 import synthetic as syn

    world = syn._make_world(np.random.default_rng(seed))
    poses = syn.se3_exp_batch(PERIOD * np.arange(frames)[:, None] * TWIST[None, :])
    scans = []
    for k in range(frames):
        pts, times = syn.distorted_scan(world, 64, 2083, poses[k], TWIST, PERIOD, np.random.default_rng(seed * 1000 + k))
        rec = np.zeros(len(pts), dtype=RECORD)
        rec["x"], rec["y"], rec["z"], rec["time"] = pts[:, 0], pts[:, 1], pts[:, 2], times
        rec["intensity"] = (200.0 / (1.0 + np.linalg.norm(pts, axis=1))).astype(np.float32)
        rec["ring"] = (k % 64)
        scans.append(rec.view(np.float32).reshape(len(rec), 8))
    return poses, scans


def device_load(c, prep, raw, exact=False):
    """One upload, the filter with fields on the device (the approximate grid, or the exact one), the source and its timestamps
    read in place -> the prep output (kept alive by the caller until the next synchronisation)."""
    import torch

    d = torch.from_numpy(raw).cuda()
    out = prep.voxel_grid(d, LEAF, FIELDS) if exact else prep.approximate_voxel_grid_fields(d, LEAF, FIELDS)
    m = out.shape[0]
    c.set_cloud_device("source", out.data_ptr(), m, STRIDE)
    c.set_source_timestamps_device(out.data_ptr() + 12, m, STRIDE, 0.0)
    return out


def host_load(c, raw, route):
    import oracle_fields as OF
    from fast_gicp_b200 import synthetic as syn

    if route == "numpy":
        pts, times = syn.voxel_downsample_values(np.ascontiguousarray(raw[:, :3]), raw[:, 4], LEAF)
    else:
        out = OF.approximate_voxel_grid_fields(raw, LEAF, FIELDS)
        pts, times = out[:, :3], out[:, 3]
    c.set_source_cloud(np.ascontiguousarray(pts))
    c.set_source_timestamps(np.ascontiguousarray(times), 0.0)
    return len(pts)


def cost_pass(c, prep, scans, route):
    out, sizes = [], []
    for raw in scans[1:]:
        t0 = time.perf_counter()
        if route in ("device", "exact"):
            keep = device_load(c, prep, raw, route == "exact")
            m = keep.shape[0]
        else:
            m = host_load(c, raw, route)
        c.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
        sizes.append(m)
    return out, sizes


def breakdown(prep, scans, repeats):
    """Medians per call over the sequence: the upload of the raw records, the filter with fields and the xyz-only filter on the
    uploaded records (device in, device out), host clock around calls that end in a synchronisation."""
    import ctypes as C

    import torch

    up, fields, xyz, exact = [], [], [], []
    for _ in range(repeats):
        for raw in scans[1:]:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            d = torch.from_numpy(raw).cuda()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            prep.approximate_voxel_grid_fields(d, LEAF, FIELDS)
            t2 = time.perf_counter()
            out = torch.empty((len(raw), 3), dtype=torch.float32, device="cuda")
            m = C.c_size_t(0)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            rc = prep._lib.vgicp_prep_approximate_voxel_grid(prep._h, d.data_ptr(), len(raw), raw.strides[0], 1, C.c_float(LEAF), 0, out.data_ptr(), len(raw), 1, C.byref(m))
            t4 = time.perf_counter()
            assert rc == 0
            prep.voxel_grid(d, LEAF, FIELDS)
            exact.append((time.perf_counter() - t4) * 1e3)
            up.append((t1 - t0) * 1e3)
            fields.append((t2 - t1) * 1e3)
            xyz.append((t4 - t3) * 1e3)
    return {"upload_ms_median": round(float(np.median(up)), 3), "prep_fields_ms_median": round(float(np.median(fields)), 3),
            "prep_xyz_only_ms_median": round(float(np.median(xyz)), 3), "prep_exact_fields_ms_median": round(float(np.median(exact)), 3)}


def exact_filter_only(prep, scans, repeats):
    """The exact grid alone, device in and device out, at three sizes: ms per call (median over `repeats` windows of 10 calls,
    CUDA events; every call ends in the library's own synchronisation)."""
    import torch

    from fast_gicp_b200 import synthetic as syn

    big, _, _ = syn.kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
    rng = np.random.default_rng(5)
    one = np.zeros((1_000_000, 8), np.float32)
    one[:, :3] = rng.uniform(0.01, 0.24, (len(one), 3))
    one[:, 3:5] = rng.uniform(0.0, 100.0, (len(one), 2))
    cases = {"sweep_fields": (scans[1], FIELDS), "kitti_1m_xyz": (np.ascontiguousarray(big, dtype=np.float32), []), "one_voxel_1m_fields": (one, FIELDS)}
    rec = {}
    for name, (raw, fields) in cases.items():
        d = torch.from_numpy(raw).cuda()
        out = prep.voxel_grid(d, LEAF, fields)
        for _ in range(3):
            prep.voxel_grid(d, LEAF, fields)
        times = []
        for _ in range(repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                prep.voxel_grid(d, LEAF, fields)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) / 10)
        rec[name] = {"points": len(raw), "fields": len(fields), "voxels": int(out.shape[0]), "ms_median": round(float(np.median(times)), 3)}
    return rec


def odometry_device(c, prep, scans, poses, radius, cap, weight, exact=False):
    """bench_ct.odometry_ct with the device front end (the exact grid when `exact`) -> (last pose, per-frame translation error [m], per-frame twists)."""
    from fast_gicp_b200.core import REG_PLANE, pose_from_c, twist_from_motion

    prev, cur = np.linalg.inv(syn_exp(PERIOD * TWIST)), np.eye(4)
    xi = twist_from_motion(np.linalg.inv(prev) @ cur, PERIOD)
    W = np.full(6, weight)

    def covs():
        c.find_source_neighbors(20)
        c.calculate_source_covariances(REG_PLANE)

    keep = device_load(c, prep, scans[0], exact)
    c.deskew_source_stored(xi)
    covs()
    c.swap_source_and_target()
    c.create_target_voxelmap()
    c.synchronize()
    errors, twists = [], []
    for k in range(1, len(scans)):
        keep = device_load(c, prep, scans[k], exact)
        covs()
        res = c.align_ct(cur @ np.linalg.inv(prev) @ cur, xi, xi, W)
        T, xi = pose_from_c(res.T), np.array(res.twist)
        c.deskew_source_stored(xi)
        covs()
        c.append_source_to_target(T)
        c.crop_target(T[:3, 3], radius, cap)
        c.synchronize()
        del keep
        prev, cur = cur, T
        errors.append(round(float(np.linalg.norm(T[:3, 3] - poses[k][:3, 3])), 4))
        twists.append([round(float(v), 4) for v in xi])
    return cur, errors, twists


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
        print("[bench_raw_scans %7.1fs] %s" % (time.perf_counter() - t_start, msg), file=sys.stderr, flush=True)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_raw_scans needs a CUDA device (an H100); there is no CPU measurement")
    torch.cuda.set_device(a.device)
    from fast_gicp_b200.prep import InputPrep

    poses, scans = raw_sequence(a.frames, a.seed)
    prep = InputPrep(a.device)
    rec = {"gpu": card_info(a.device), "leaf_m": LEAF, "record_bytes": RECORD.itemsize, "raw_points_per_scan_mean": int(np.mean([len(s) for s in scans])),
           "twist": TWIST.tolist(), "period_s": PERIOD}
    log(f"{len(scans)} raw scans, {rec['raw_points_per_scan_mean']} points each on average")
    routes = ("device", "exact", "numpy", "serial")
    cores = {r: new_core(a.device) for r in routes}
    sizes = {}
    for r in routes:  # warm-up
        sizes[r] = cost_pass(cores[r], prep, scans, r)[1]
    passes = {r: [] for r in routes}
    for rep in range(a.repeats):
        order = routes[rep % len(routes):] + routes[:rep % len(routes)]
        for r in order if rep % 2 == 0 else order[::-1]:
            passes[r].append(cost_pass(cores[r], prep, scans, r)[0])
    for r in routes:
        per_frame = np.median(np.array(passes[r]), axis=0)
        rec[f"{r}_raw_to_source_ms_median"] = round(float(np.median(per_frame)), 3)
        rec[f"{r}_points_per_scan_mean"] = int(np.mean(sizes[r]))
        cores[r].close()
    rec["device_breakdown"] = breakdown(prep, scans, a.repeats)
    log({k: v for k, v in rec.items() if k.endswith("_ms_median")})
    log(rec["device_breakdown"])
    rec["exact_filter_only"] = exact_filter_only(prep, scans, a.repeats)
    log(rec["exact_filter_only"])
    for arm, exact in (("device_front_end", False), ("exact_front_end", True)):
        c = new_core(a.device)
        T, errors, twists = odometry_device(c, prep, scans, poses, a.radius, a.cap, a.weight, exact)
        c.close()
        rec[f"drift_ct_{arm}"] = drift(poses[-1], T)
        rec[f"translation_error_per_frame_ct_{arm}"] = errors
        rec[f"twist_per_frame_ct_{arm}"] = twists
        log(f"ct with the {arm.replace('_', ' ')}: {rec[f'drift_ct_{arm}']}")
    rec["frames"] = a.frames
    prep.close()
    print(json.dumps({"raw_scans": rec}), flush=True)


if __name__ == "__main__":
    main()
