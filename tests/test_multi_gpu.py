"""Source sharding across GPUs (SURVEY.md 8e): needs >= 2 GPUs, skipped otherwise."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_workers(world, args=(), timeout=600):
    port = _free_port()
    procs = []
    for rank in range(world):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "multi_gpu_worker.py"), *args], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    outs = [p.communicate(timeout=timeout) for p in procs]
    res = []
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0, e[-3000:]
        res.append(json.loads(o.strip().splitlines()[-1]))
    return res


@pytest.mark.gpu
def test_sharded_evaluation_matches_single_gpu():
    import torch

    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else 4
    res = run_workers(world)
    for r in res:
        assert r["comm_error"] == 0
        # the exchanged system equals the unsharded one up to the float rounding of the per-warp partial sums (sharding changes
        # which points share a warp; block and rank level sums are double)
        assert r["H_rel_diff_vs_full"] < 1e-6 and r["b_rel_diff_vs_full"] < 1e-5 and r["err_rel_diff_vs_full"] < 1e-6 and r["err_only_rel"] < 1e-6
        assert r["converged"] and r["iters"][0] == r["iters"][1]
        assert np.abs(np.array(r["T"]) - np.array(r["T_full"])).max() < 1e-6
        # stage 1 sharded too: the exchanged covariances are the unsharded ones bit for bit, so the registration walks the same iterates
        assert r["stage1_sharded_comm_error"] == 0 and r["stage1_sharded_covariances_equal"]
        assert r["stage1_sharded_T"] == r["T"] and r["stage1_sharded_iters"] == r["iters"][0]
        # neighbour rows given by the host after a k-NN search of a smaller cloud: unsharded covariances, bit for bit
        assert r["given_rows_covariances_equal"]
    # every rank holds bit-identical sums (same doubles added in rank order)
    for r in res[1:]:
        assert r["H_sum"] == res[0]["H_sum"] and r["b"] == res[0]["b"] and r["err"] == res[0]["err"] and r["T"] == res[0]["T"]
    assert sorted(tuple(r["shard"]) for r in res)[0][0] == 0
