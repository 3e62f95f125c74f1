"""Worker of tests/test_gpu_multi_hypothesis.py::test_communicator_handle_is_unsupported: one process per GPU joins a two-rank
source-sharding communicator, then checks that vgicp_align_multi and vgicp_evaluate_poses refuse the handle without launching."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist

    from fast_gicp_b200 import distributed as D
    from fast_gicp_b200.core import ERR_UNSUPPORTED, REG_PLANE, AlignResult, Core

    rank, world, local = D.env_rank_world()
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    d = np.load(os.path.join(ROOT, "tests", "golden", "pair_0p2.npz"))
    tgt, src = d["target"], d["source"]
    c = Core(local)
    c.set_neighbor_search_method("DIRECT7")
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(REG_PLANE)
    D.setup_source_sharding(c, len(src))
    G = np.tile(np.eye(4).reshape(16), 2)
    res = (AlignResult * 2)()
    err = np.zeros(2)
    n0 = c.launch_count()
    dp = G.ctypes.data_as(C.POINTER(C.c_double))
    rc = (c._lib.vgicp_align_multi(c._h, dp, 2, None, res), c._lib.vgicp_evaluate_poses(c._h, dp, 2, err.ctypes.data_as(C.POINTER(C.c_double)), None, None, None))
    assert rc == (ERR_UNSUPPORTED, ERR_UNSUPPORTED), rc
    assert c.launch_count() == n0
    dist.barrier()
    c.comm_shutdown()
    c.close()
    dist.destroy_process_group()
    print("unsupported ok", flush=True)


if __name__ == "__main__":
    main()
