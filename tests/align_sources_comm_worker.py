"""Worker of tests/test_gpu_align_sources.py::test_communicator_handle_is_unsupported: one process per GPU joins a two-rank
source-sharding communicator, then checks that vgicp_align_sources refuses the handle without launching."""
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
    S = [src, src[::2].copy()]
    xyz = (C.c_void_p * 2)(*[s.ctypes.data for s in S])
    n = (C.c_size_t * 2)(*[len(s) for s in S])
    res = (AlignResult * 2)()
    n0 = c.launch_count()
    rc = c._lib.vgicp_align_sources(c._h, xyz, n, 12, 0, 20, REG_PLANE, None, 2, None, res)
    assert rc == ERR_UNSUPPORTED, rc
    assert c.launch_count() == n0
    dist.barrier()
    c.comm_shutdown()
    c.close()
    dist.destroy_process_group()
    print("unsupported ok", flush=True)


if __name__ == "__main__":
    main()
