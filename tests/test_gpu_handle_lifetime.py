"""Destroying a handle frees what it holds in every state, including the resources it creates lazily: each case creates a handle,
brings it into a state that holds such a resource, destroys it, and repeats.  Afterwards a fresh handle registers the golden pair
bit for bit as the first one did."""
import os

import numpy as np
import pytest

from fast_gicp_b200.core import REG_PLANE, Core, pose_from_c

pytestmark = pytest.mark.gpu

CYCLES = 3


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


@pytest.fixture(scope="module")
def golden():
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "pair_0p2.npz"))
    return np.ascontiguousarray(d["target"][:, :3], np.float32), np.ascontiguousarray(d["source"][:, :3], np.float32)


def _registration(tgt, src):
    c = Core(0)
    c.set_neighbor_search_method("DIRECT7")
    r = c.register(tgt, src)
    out = (np.asarray(r.T).tobytes(), np.asarray(r.H).tobytes(), r.nr_iterations, r.converged, r.n_linearize, r.n_compute_error)
    c.close()
    return out


def _prepared(tgt, src):
    c = Core(0)
    c.set_neighbor_search_method("DIRECT7")
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()
    c.set_source_cloud(src)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(REG_PLANE)
    return c


def _times(n):
    return np.linspace(0.0, 0.1, n, dtype=np.float32)


def multi_pose(torch, tgt, src):
    c = _prepared(tgt, src)
    c.align_multi(np.stack([np.eye(4)] * 3))
    return c


def multi_source(torch, tgt, src):
    c = _prepared(tgt, src)
    c.align_sources([src, src[::2].copy()])
    return c


def deskew(torch, tgt, src):
    c = _prepared(tgt, src)
    c.deskew_source(_times(len(src)), [0.0, 0.0, 0.35, 8.0, 0.0, 0.0], 0.05)
    return c


def ct_channel(torch, tgt, src):
    c = _prepared(tgt, src)
    c.set_source_timestamps(_times(len(src)), 0.05)
    c.compute_error_ct(np.eye(4), np.zeros(6), np.eye(4), np.zeros(6))
    return c


def profiling_pending(torch, tgt, src):
    c = _prepared(tgt, src)
    c.set_profiling(True)
    c.align()  # (the events stay pending: get_profile is never called)
    return c


def stage1_graph(torch, tgt, src):
    c = Core(0)
    c.set_neighbor_search_method("DIRECT7")
    dt, ds = torch.from_numpy(tgt).cuda(), torch.from_numpy(src).cuda()
    for _ in range(3):  # eager, captured, replayed
        c.register_raw(dt.data_ptr(), dt.shape[0], ds.data_ptr(), ds.shape[0], 12, True, 20, REG_PLANE)
    return c


def voxelmap_pending(torch, tgt, src):
    c = Core(0)
    c.set_target_cloud(tgt)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(REG_PLANE)
    c.create_target_voxelmap()  # (finished only by the next call that needs the map)
    return c


def thin_and_carve(torch, tgt, src):
    c = Core(0)
    c.set_neighbor_search_method("DIRECT7")
    r = c.register(tgt, src)
    c.carve_target(pose_from_c(r.T))
    c.thin_target(0.5, 2)
    return c


def prep_exact_grid(torch, tgt, src):
    from fast_gicp_b200.prep import InputPrep

    p = InputPrep(0)
    p.voxel_grid(torch.from_numpy(tgt).cuda(), 0.25, (), 2)
    return p


STATES = [multi_pose, multi_source, deskew, ct_channel, profiling_pending, stage1_graph, voxelmap_pending, thin_and_carve, prep_exact_grid]


@pytest.mark.parametrize("state", STATES, ids=[s.__name__ for s in STATES])
def test_destroy_in_state(torch, golden, state):
    tgt, src = golden
    first = _registration(tgt, src)
    for _ in range(CYCLES):
        state(torch, tgt, src).close()
    assert _registration(tgt, src) == first
