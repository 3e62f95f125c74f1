"""What a change to one of a handle's inputs invalidates: one table of (operation) -> which facts of a fully prepared VGICP handle
are still there.  Each fact is read through its getter and is either present or refused with BAD_STATE.  The timestamps are read
last, by a stored deskew with a zero twist, because that changes the source."""
import numpy as np
import pytest

import oracle as O
from test_gpu_multi_hypothesis import setup

pytestmark = pytest.mark.gpu

FACTS = ("source_neighbors", "source_covariances", "target_neighbors", "target_covariances", "voxel_map", "linearisation", "timestamps")


def _times(n):
    return np.linspace(0.0, 0.1, n, dtype=np.float32)


def _pair(pair02):
    return pair02[0][::4].copy(), pair02[1][::4].copy()


def _prepared(tgt, src):
    from fast_gicp_b200.core import Core

    c = setup(Core(0), tgt, src, method=O.DIRECT7)
    c.set_source_timestamps(_times(len(src)), 0.0)
    c.update_correspondences(np.eye(4))
    return c


def _read(c):
    """'+' per fact that its getter returns, 'B' per fact it refuses with BAD_STATE (any other error fails the test)."""
    from fast_gicp_b200.core import ERR_BAD_STATE, VgicpError

    reads = (c.get_source_neighbors, c.get_source_covariances, c.get_target_neighbors, c.get_target_covariances, c.num_voxels,
             lambda: c.compute_error(np.eye(4), want_H=False), lambda: c.deskew_source_stored(np.zeros(6)))
    out = ""
    for read in reads:
        try:
            read()
            out += "+"
        except VgicpError as e:
            assert e.code == ERR_BAD_STATE, str(e)
            out += "B"
    return out


def _device(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _apply(c, op, tgt, src, torch):
    src2, tgt2 = src[::2].copy(), tgt[::2].copy()
    if op == "set_source_cloud":
        c.set_source_cloud(src2)
    elif op == "set_source_cloud_device":
        d = _device(torch, src2)
        c.set_cloud_device("source", d.data_ptr(), len(src2), 12)
        c.synchronize()
    elif op == "set_target_cloud":
        c.set_target_cloud(tgt2)
    elif op == "set_target_cloud_device":
        d = _device(torch, tgt2)
        c.set_cloud_device("target", d.data_ptr(), len(tgt2), 12)
        c.synchronize()
    elif op == "register":
        c.register(tgt, src)
    elif op == "set_source_neighbors":
        c.set_source_neighbors(20, c.get_source_neighbors())
    elif op == "set_target_neighbors":
        c.set_target_neighbors(20, c.get_target_neighbors())
    elif op == "find_source_neighbors":
        c.find_source_neighbors(20)
    elif op == "find_target_neighbors":
        c.find_target_neighbors(20)
    elif op == "calculate_source_covariances":
        c.calculate_source_covariances(O.REG_PLANE)
    elif op == "calculate_target_covariances":
        c.calculate_target_covariances(O.REG_PLANE)
    elif op == "calculate_source_covariances_rbf":
        c.calculate_source_covariances_rbf(O.REG_PLANE)
    elif op == "calculate_target_covariances_rbf":
        c.calculate_target_covariances_rbf(O.REG_PLANE)
    elif op == "set_source_covariances":
        c.set_source_covariances(c.get_source_covariances())
    elif op == "set_target_covariances":
        c.set_target_covariances(c.get_target_covariances())
    elif op == "deskew_source":
        c.deskew_source(_times(len(src)), np.zeros(6), 0.0)
    elif op == "deskew_source_stored":
        c.deskew_source_stored(np.zeros(6))
    elif op == "append_source_to_target":
        c.append_source_to_target(np.eye(4))
    elif op == "crop_target":
        c.crop_target(np.zeros(3), float("inf"), len(tgt) // 2)
    elif op == "thin_target":
        c.thin_target(0.5, 4)
    elif op == "swap_source_and_target":
        c.swap_source_and_target()
    elif op == "comm_export_arena":
        c.comm_export_arena(max(len(tgt), len(src)))
    elif op == "set_problem_ndt":
        c.set_problem(1)
    elif op == "set_problem_same":
        c.set_problem(0)
    else:
        raise ValueError(op)


# per operation, the facts in FACTS order after it: + present, B BAD_STATE
TABLE = {
    "set_source_cloud":                 "BB+++BB",
    "set_source_cloud_device":          "BB+++BB",
    "set_target_cloud":                 "++BBBB+",
    "set_target_cloud_device":          "++BBBB+",
    "register":                         "++++++B",
    "set_source_neighbors":             "+++++++",
    "set_target_neighbors":             "+++++++",
    "find_source_neighbors":            "+++++++",
    "find_target_neighbors":            "+++++++",
    "calculate_source_covariances":     "+++++++",
    "calculate_target_covariances":     "+++++++",
    "calculate_source_covariances_rbf": "+++++++",
    "calculate_target_covariances_rbf": "+++++++",
    "set_source_covariances":           "+++++++",
    "set_target_covariances":           "++++BB+",
    "deskew_source":                    "BB+++B+",
    "deskew_source_stored":             "BB+++B+",
    "append_source_to_target":          "++B++++",
    "crop_target":                      "++B++++",
    "thin_target":                      "++B++++",
    "swap_source_and_target":           "++++++B",
    "comm_export_arena":                "+B+BBB+",
    "set_problem_ndt":                  "+++++B+",
    "set_problem_same":                 "+++++++",
}


@pytest.fixture(scope="module")
def torch():
    import torch as t

    assert t.cuda.is_available()
    return t


def test_prepared_handle_has_every_fact(pair02):
    tgt, src = _pair(pair02)
    c = _prepared(tgt, src)
    try:
        assert _read(c) == "+" * len(FACTS)
    finally:
        c.close()


@pytest.mark.parametrize("op", list(TABLE))
def test_operation_leaves(pair02, torch, op):
    tgt, src = _pair(pair02)
    c = _prepared(tgt, src)
    try:
        _apply(c, op, tgt, src, torch)
        got = _read(c)
        assert got == TABLE[op], f"{op}: facts {dict(zip(FACTS, got))}, expected {dict(zip(FACTS, TABLE[op]))}"
    finally:
        c.close()


def _ndt_voxels(tgt, src):
    from fast_gicp_b200.core import Core

    c = Core(0)
    try:
        c.set_resolution(1.0)
        c.set_problem(1)
        c.set_target_cloud(tgt)
        c.set_source_cloud(src)
        return c.num_voxels()
    finally:
        c.close()


@pytest.mark.parametrize("op", ["set_target_cloud", "append_source_to_target", "crop_target"])
def test_ndt_map_follows_the_target(pair02, op):
    """The NDT target map, built before the change, is rebuilt from the target as it is after it.  Append and crop refuse under
    NDT: they run under VGICP, between two set_problem(1)."""
    tgt, src = _pair(pair02)
    c = _prepared(tgt, src)
    try:
        c.set_problem(1)
        before = c.num_voxels()
        if op == "set_target_cloud":
            after_tgt = tgt[: len(tgt) // 2].copy()
            c.set_target_cloud(after_tgt)
        else:
            c.set_problem(0)
            if op == "append_source_to_target":
                after_tgt = np.concatenate([tgt, src])
                c.append_source_to_target(np.eye(4))
            else:
                after_tgt = tgt[-(len(tgt) // 2):].copy()
                c.crop_target(np.zeros(3), float("inf"), len(tgt) // 2)
            c.set_problem(1)
        expect = _ndt_voxels(after_tgt, src)
        assert expect != before
        assert c.num_voxels() == expect
    finally:
        c.close()


def test_register_eager_capture_replay_leave_one_table(pair02, torch):
    """vgicp_register on resident clouds runs stage 1 eagerly, then captures it, then replays the graph: the handle's state after
    each of the three runs is the same."""
    from fast_gicp_b200.core import Core

    tgt, src = _pair(pair02)
    dt, ds = _device(torch, tgt), _device(torch, src)
    c = Core(0)
    try:
        c.set_resolution(1.0)
        c.set_neighbor_search_method(O.DIRECT7)
        for run in ("eager", "capture", "replay"):
            c.register_raw(dt.data_ptr(), len(tgt), ds.data_ptr(), len(src), 12, True, 20, O.REG_PLANE)
            assert _read(c) == TABLE["register"], run
    finally:
        c.close()
