"""The float64 evaluation reference (eval_reference.eval64) against the float CPU oracle, and the per-entry comparator against
deliberately wrong sums.  CPU only: these pin the reference that test_gpu_eval_matrix.py holds every evaluation kernel to."""
import numpy as np
import pytest

import oracle as O
import oracle_robust as R
from conftest import random_pose
from eval_reference import KINDS, eval64, eval64_kinds, excess

# The float oracle forms every per-correspondence term in float32 and sums in double, so it differs from eval64 by a few float
# roundings per term, with random signs; measured on pair_0p2 with PLANE covariances: at most 4.2e-6 A.
TAU = 1e-5
# The loosest per-entry tolerance the GPU matrix uses (PLANE covariances and NDT against eval64): the mutations must fail even there.
TAU_LOOSE = 1e-4
METHODS = [(O.DIRECT1, -1.0), (O.DIRECT7, -1.0), (O.DIRECT27, -1.0), (O.DIRECT_RADIUS, 1.5)]


@pytest.fixture(scope="module")
def plane(pair02):
    R.build()
    tgt, src = pair02
    t_cov = O.symmetrized(O.regularize(O.covariances(tgt, O.knn(tgt, 20)), O.REG_PLANE))
    s_cov = O.symmetrized(O.regularize(O.covariances(src, O.knn(src, 20)), O.REG_PLANE))
    return dict(src=src, s_cov=s_cov, vm=O.VoxelMap(tgt, t_cov, 1.0, accum_double=True))


def pose_pairs(relative_pose, seed):
    """(T_lin, T_eval) with T_eval != T_lin: at the identity and near the ground truth."""
    rng = np.random.default_rng(seed)
    return [(T, T @ random_pose(rng, 0.01, 0.1)) for T in (np.eye(4), relative_pose)]


def ref64(vm, src, s_cov, pairs, Tl, Te, want_H=True, **kw):
    return eval64(vm.vox_mean, vm.vox_cov, vm.vox_n, src, s_cov, pairs, Tl, Te, want_H, **kw)


@pytest.mark.parametrize("method,radius", METHODS)
def test_eval64_matches_the_float_oracle(plane, relative_pose, method, radius):
    vm, src, s_cov = plane["vm"], plane["src"], plane["s_cov"]
    offs = O.offsets(method, radius)
    for Tl, Te in pose_pairs(relative_pose, method):
        pairs = O.find_correspondences(vm, src, Tl, offs)
        for want_H in (True, False):
            refs = eval64_kinds(vm.vox_mean, vm.vox_cov, vm.vox_n, src, s_cov, pairs, Tl, Te, want_H, kinds=KINDS)
            for kind in KINDS:
                got = R.evaluate(vm, src, s_cov, offs, Tl, Te, want_H, robust=kind, robust_scale=1.0)
                if want_H and kind == "NONE":  # the plain oracle and the robust one with NONE are the same sums
                    plain = O.evaluate(vm, src, s_cov, offs, Tl, Te, True)
                    assert plain[3] == got[3] == len(pairs)
                    worst, bad = excess(plain, refs[kind], TAU)
                    assert not len(bad), (kind, bad, worst)
                worst, bad = excess(got if want_H else (got[0], None, None), refs[kind], TAU)
                assert not len(bad), (kind, want_H, bad, worst)


@pytest.mark.parametrize("mode", [O.P2D, O.D2D])
@pytest.mark.parametrize("method,radius", METHODS)
def test_eval64_matches_the_ndt_oracle(pair02, relative_pose, mode, method, radius):
    tgt, src = pair02
    tm = O.VoxelMap(tgt, None, 1.0, accum_double=True)
    if mode == O.D2D:
        sm = O.VoxelMap(src, None, 1.0, accum_double=True)
        s_pts, s_cov = sm.vox_mean, sm.vox_cov
    else:
        s_pts, s_cov = src, None
    offs = O.offsets(method, radius)
    for Tl, Te in pose_pairs(relative_pose, 10 + method):
        pairs = O.find_correspondences(tm, s_pts, Tl, offs)
        for want_H in (True, False):
            ref = ref64(tm, s_pts, s_cov, pairs, Tl, Te, want_H, ndt=True, res=1.0)
            got = O.evaluate_ndt(tm, s_pts, s_cov, offs, Tl, Te, want_H)
            worst, bad = excess(got if want_H else (got[0], None, None), ref, TAU)
            assert not len(bad), (want_H, bad, worst)


# ---- the comparator is not vacuous: each wrong input is rejected at TAU_LOOSE, and the same sums without the mutation pass at TAU

def assert_mutation_caught(right, wrong, ref):
    worst, bad = excess(right, ref, TAU)
    assert not len(bad), ("the unmutated sums must pass", bad, worst)
    _, bad = excess(wrong, ref, TAU_LOOSE)
    assert len(bad), "the mutated sums passed the per-entry check"


@pytest.fixture(scope="module")
def case(plane, relative_pose):
    (Tl, Te), = pose_pairs(relative_pose, 99)[1:]
    offs = O.offsets(O.DIRECT7)
    pairs = O.find_correspondences(plane["vm"], plane["src"], Tl, offs)
    return dict(plane, Tl=Tl, Te=Te, offs=offs, pairs=pairs, ref=ref64(plane["vm"], plane["src"], plane["s_cov"], pairs, Tl, Te))


def test_dropping_one_offset_is_caught(case):
    vm, src, s_cov, Tl, Te = case["vm"], case["src"], case["s_cov"], case["Tl"], case["Te"]
    right = O.evaluate(vm, src, s_cov, case["offs"], Tl, Te, True)
    wrong = O.evaluate(vm, src, s_cov, case["offs"][:-1], Tl, Te, True)  # the correspondences of offset (0, 0, -1) lost
    assert wrong[3] < right[3]
    assert_mutation_caught(right, wrong, case["ref"])


def test_evaluation_rotation_in_place_of_the_linearisation_rotation_is_caught(case):
    vm, src, s_cov, Tl, Te, pairs = case["vm"], case["src"], case["s_cov"], case["Tl"], case["Te"], case["pairs"]
    right = R.derivatives(vm, src, s_cov, pairs, Tl, Te)
    wrong = R.derivatives(vm, src, s_cov, pairs, Te, Te)  # R_eval C_A R_eval^T over the correspondences of T_lin
    assert_mutation_caught(right, wrong, case["ref"])


def test_one_flipped_sign_in_b_is_caught(case):
    vm, src, s_cov, Tl, Te = case["vm"], case["src"], case["s_cov"], case["Tl"], case["Te"]
    right = O.evaluate(vm, src, s_cov, case["offs"], Tl, Te, True)
    A_b = case["ref"][3][37:]
    j = int(np.argmin(np.abs(right[2]) / A_b))  # the entry of b smallest against its own scale: the hardest one to catch
    b = right[2].copy()
    b[j] = -b[j]
    assert_mutation_caught(right, (right[0], right[1], b), case["ref"])


def test_unit_weights_in_place_of_sqrt_n_are_caught(case):
    vm, src, s_cov, Tl, Te, pairs = case["vm"], case["src"], case["s_cov"], case["Tl"], case["Te"], case["pairs"]
    assert vm.vox_n.max() > 1
    right = O.evaluate(vm, src, s_cov, case["offs"], Tl, Te, True)
    wrong = eval64(vm.vox_mean, vm.vox_cov, np.ones_like(vm.vox_n), src, s_cov, pairs, Tl, Te, True)  # w = 1
    assert_mutation_caught(right, wrong, case["ref"])


def test_cauchy_without_its_derivative_is_caught(case):
    vm, src, s_cov, Tl, Te, pairs = case["vm"], case["src"], case["s_cov"], case["Tl"], case["Te"], case["pairs"]
    ref = ref64(vm, src, s_cov, pairs, Tl, Te, robust="CAUCHY")
    right = R.evaluate(vm, src, s_cov, case["offs"], Tl, Te, True, robust="CAUCHY")
    plain = O.evaluate(vm, src, s_cov, case["offs"], Tl, Te, True)
    wrong = (right[0], plain[1], plain[2])  # err = sum w rho(s), but H and b weighted by w instead of w rho'(s)
    assert_mutation_caught(right, wrong, ref)
