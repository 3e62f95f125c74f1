"""Which precondition an evaluating entry point refuses first: one table of (entry point x handle state) -> status.  Every
refusal must leave the launch count where it was.  The states combine missing inputs with settings that make a call
unsupported, so that a check moved ahead of another one changes a status here."""
import numpy as np
import pytest

import oracle as O
from test_gpu_multi_hypothesis import setup

pytestmark = pytest.mark.gpu

TWIST_BEYOND_SERIES = np.array([0.0, 0.0, 20.0, 0.0, 0.0, 0.0])  # 20 rad/s over a 0.1 s sweep: more than pi/2


def _source_only(c, src, covariances):
    c.set_source_cloud(src)
    if covariances:
        c.find_source_neighbors(20)
        c.calculate_source_covariances(O.REG_PLANE)


def _ndt(c, tgt, src, target=True):
    """(Keeps the default neighbour search: the correspondence getter must find its offset table on the device without a
    set_neighbor_search_method call.)"""
    c.set_problem(1)
    c.set_source_cloud(src)
    if target:
        c.set_target_cloud(tgt)


def _times(src):
    return np.linspace(0.0, 0.1, len(src), dtype=np.float32)


def build_state(c, state, tgt, src):
    if state == "fresh":
        return
    if state == "source_without_covariances":
        _source_only(c, src, False)
    elif state == "covariances_without_map":
        _source_only(c, src, True)
    elif state == "map_without_update_correspondences":
        setup(c, tgt, src, method=O.DIRECT7)
    elif state == "ndt_robust_without_target":  # the robust kind is refused before the missing target
        _ndt(c, tgt, src, target=False)
        c.set_robust_kernel("HUBER", 1.0)
    elif state == "ndt_without_target":
        _ndt(c, tgt, src, target=False)
    elif state == "ct_without_timestamps":
        setup(c, tgt, src, method=O.DIRECT7)
        c.update_correspondences(np.eye(4))
    elif state == "ct_under_ndt":
        _ndt(c, tgt, src)
        c.set_source_timestamps(_times(src), 0.0)
        c.update_correspondences(np.eye(4))
    elif state == "ct_source_sharding_without_timestamps":  # sharding is refused before the missing timestamps
        setup(c, tgt, src, method=O.DIRECT7)
        c.update_correspondences(np.eye(4))
        c.set_source_shard(0, len(src) // 2)
    elif state == "ct_twist_beyond_series":
        setup(c, tgt, src, method=O.DIRECT7)
        c.set_source_timestamps(_times(src), 0.0)
        c.update_correspondences(np.eye(4))
    else:
        raise ValueError(state)


def call(c, entry, state):
    xi = TWIST_BEYOND_SERIES if state == "ct_twist_beyond_series" else np.zeros(6)
    I, G = np.eye(4), np.stack([np.eye(4)] * 2)
    if entry == "compute_error":
        c.compute_error(I, True)
    elif entry == "align":
        c.align(I)
    elif entry == "align_multi":
        c.align_multi(G)
    elif entry == "evaluate_poses":
        c.evaluate_poses(G, want_H=True)
    elif entry == "compute_error_ct":
        c.compute_error_ct(I, xi, I, xi, True)
    elif entry == "align_ct":
        c.align_ct(I, twist_guess=xi)
    elif entry == "update_correspondences":
        c.update_correspondences(I)
    elif entry == "get_voxel_correspondences":
        c.get_voxel_correspondences()
    else:
        raise ValueError(entry)


ENTRIES = ("compute_error", "align", "align_multi", "evaluate_poses", "compute_error_ct", "align_ct", "update_correspondences",
           "get_voxel_correspondences")
# per state, the status of each entry point in ENTRIES order: . OK, B BAD_STATE, U UNSUPPORTED, I INVALID_ARGUMENT
TABLE = {
    "fresh":                                 "BBBBBBBB",
    "source_without_covariances":            "BBBBBBBB",
    "covariances_without_map":               "BBBBBBBB",
    "map_without_update_correspondences":    "B...BB.B",
    "ndt_robust_without_target":             "UUUUUUBB",
    "ndt_without_target":                    "BBBBUUBB",
    "ct_without_timestamps":                 "....BB..",
    "ct_under_ndt":                          "....UU..",
    "ct_source_sharding_without_timestamps": "....UU..",
    "ct_twist_beyond_series":                "....II..",
}
CASES = [(e, s, TABLE[s][i]) for s in TABLE for i, e in enumerate(ENTRIES)]


@pytest.mark.parametrize("entry,state,expect", CASES, ids=[f"{e}-{s}" for e, s, _ in CASES])
def test_refusal_order(pair02, entry, state, expect):
    from fast_gicp_b200.core import ERR_BAD_STATE, ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, OK, Core, VgicpError

    code = {".": OK, "B": ERR_BAD_STATE, "U": ERR_UNSUPPORTED, "I": ERR_INVALID_ARGUMENT}[expect]
    tgt, src = pair02[0][::4].copy(), pair02[1][::4].copy()
    c = Core(0)
    try:
        build_state(c, state, tgt, src)
        n0 = c.launch_count()
        got = OK
        try:
            call(c, entry, state)
        except VgicpError as e:
            got = e.code
        assert got == code, f"{entry} in state {state}: status {got}, expected {code}"
        if got != OK:
            assert c.launch_count() == n0, f"{entry} in state {state}: the refusal launched a kernel"
    finally:
        c.close()
