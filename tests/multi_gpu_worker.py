"""Worker of tests/test_multi_gpu.py and scripts/bench_c4_sharded.py: one process per GPU, source sharded across ranks,
linear system exchanged inside the evaluation kernel over NVLink peer mailboxes.  Prints one JSON line per rank."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist

    from fast_gicp_b200 import distributed as D
    from fast_gicp_b200.core import REG_PLANE, Core, pose_from_c

    rank, world, local = D.env_rank_world()
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")  # host transport for the 64-byte IPC handles only
    workload = sys.argv[1] if len(sys.argv) > 1 else "pair02"
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if workload == "pair02":
        d = np.load(os.path.join(ROOT, "tests", "golden", "pair_0p2.npz"))
        tgt, src, res, method = d["target"], d["source"], 1.0, "DIRECT27"
    else:
        from fast_gicp_b200.synthetic import kitti_like_pair

        tgt, src, _ = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
        res, method = 0.5, os.environ.get("VGICP_C4_METHOD", "DIRECT27")  # DIRECT1: the bandwidth-bound configuration (DESIGN.md 4)

    def prepare(c):
        c.set_resolution(res)
        c.set_neighbor_search_method(method)
        c.set_target_cloud(tgt)
        c.find_target_neighbors(20)
        c.calculate_target_covariances(REG_PLANE)
        c.create_target_voxelmap()
        c.set_source_cloud(src)
        c.find_source_neighbors(20)
        c.calculate_source_covariances(REG_PLANE)

    c = Core(local)
    prepare(c)  # stage 1 + 2 replicated on every rank (only stage 3 is sharded here)
    # reference values on the unsharded handle
    T = np.eye(4)
    T[:3, 3] = [0.3, 0.05, 0.0]
    e_full, H_full, b_full = c.linearize(T)
    full = c.align()

    # exchange IPC handles, shard the source
    lo, hi = D.setup_source_sharding(c, len(src))

    e_sh, H_sh, b_sh = c.linearize(T)
    err_only, _, _ = c.compute_error(T, want_H=False)
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    for _ in range(reps):
        c.compute_error(T, want_H=True)
    torch.cuda.synchronize()
    ms_eval = 1e3 * (time.perf_counter() - t0) / reps
    dist.barrier()
    sharded = c.align()
    # stage 1 sharded as well: a fresh handle whose k-NN queries and covariances are split over the ranks and exchanged by peer stores
    c2 = Core(local)
    c2.set_resolution(res)
    c2.set_neighbor_search_method(method)
    lo2, hi2 = D.setup_source_sharding(c2, len(src), max_points=max(len(src), len(tgt)))
    torch.cuda.synchronize()
    dist.barrier()
    t1 = time.perf_counter()
    c2.set_target_cloud(tgt)
    c2.find_target_neighbors(20)
    c2.calculate_target_covariances(REG_PLANE)
    c2.create_target_voxelmap()
    c2.set_source_cloud(src)
    c2.find_source_neighbors(20)
    c2.calculate_source_covariances(REG_PLANE)
    full_sharded = c2.align()
    ms_full_sharded = 1e3 * (time.perf_counter() - t1)
    cov_equal = bool(np.array_equal(c2.get_source_covariances(), c.get_source_covariances()) and np.array_equal(c2.get_target_covariances(), c.get_target_covariances()))
    # host-supplied neighbour rows after a k-NN search of a smaller cloud: the covariances must not follow that search's order.
    # B is the target scaled, so that covariances left over from the run above differ from B's
    tgt_b = (tgt * np.float32(1.01)).astype(np.float32)
    c3 = Core(local)
    c3.set_target_cloud(tgt_b)
    c3.find_target_neighbors(20)
    c3.calculate_target_covariances(REG_PLANE)
    c2.set_target_cloud(tgt_b[: len(tgt_b) // 2])
    c2.find_target_neighbors(20)
    c2.set_target_cloud(tgt_b)
    c2.set_target_neighbors(20, c3.get_target_neighbors())
    c2.calculate_target_covariances(REG_PLANE)
    given_rows_cov_equal = bool(np.array_equal(c2.get_target_covariances(), c3.get_target_covariances()))
    c3.close()
    err2 = c2.comm_error()
    dist.barrier()
    c2.comm_shutdown()
    c2.close()
    out = {
        "rank": rank, "world": world, "shard": [lo, hi], "comm_error": c.comm_error(),
        "H_rel_diff_vs_full": float(np.abs(H_sh - H_full).max() / np.abs(H_full).max()),
        "b_rel_diff_vs_full": float(np.abs(b_sh - b_full).max() / np.abs(b_full).max()),
        "err_rel_diff_vs_full": float(abs(e_sh - e_full) / abs(e_full)), "err_only_rel": float(abs(err_only - e_full) / abs(e_full)),
        "H_sum": float(H_sh.sum()), "b": [float(x) for x in b_sh], "err": float(e_sh),
        "T": [float(x) for x in pose_from_c(sharded.T).reshape(-1)], "T_full": [float(x) for x in pose_from_c(full.T).reshape(-1)],
        "iters": [int(sharded.nr_iterations), int(full.nr_iterations)], "converged": bool(sharded.converged), "ms_per_evaluation": ms_eval,
        "stage1_sharded_covariances_equal": cov_equal, "stage1_sharded_T": [float(x) for x in pose_from_c(full_sharded.T).reshape(-1)],
        "stage1_sharded_iters": int(full_sharded.nr_iterations), "stage1_sharded_comm_error": err2, "ms_registration_stage1_sharded": ms_full_sharded,
        "given_rows_covariances_equal": given_rows_cov_equal,
    }
    print(json.dumps(out), flush=True)
    dist.barrier()
    c.comm_shutdown()
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
