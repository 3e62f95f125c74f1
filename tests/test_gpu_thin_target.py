"""Voxel-capped local map: vgicp_thin_target keeps at most M target points per cell, the oldest.

Handle A is thinned on the device; a fresh handle B is given the expected arrays directly (set_target_cloud with the kept points,
set_target_covariances with their 3x3s, create_target_voxelmap).  Both must then hold the same bytes and evaluate identically.
The kept rows come from synthetic.thin_indices, the numpy restatement of the rule in include/vgicp_b200.h."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from test_gpu_local_map import (INC, LIB, _assert_same_evaluations, _assert_same_map, _core, _load_source_knn, _load_target_arrays, _load_target_knn, _map_state, _res_tuple,
                                _sequence, _target_points, crop_indices, rotate_covariances)

pytestmark = pytest.mark.gpu


def thin_indices(pts, leaf, M):
    from fast_gicp_b200.synthetic import thin_indices as f

    return f(pts, leaf, M)


def _random_cov9(rng, n):
    A = rng.normal(scale=0.1, size=(n, 3, 3))
    C = A @ A.transpose(0, 2, 1) + 0.01 * np.eye(3)
    return C.reshape(n, 9).astype(np.float32)


def _with_arrays(P, S, src, src_cov, res=1.0):
    c = _core(res=res)
    _load_target_arrays(c, P, S)
    c.set_source_cloud(src)
    c.set_source_covariances(src_cov)
    return c


def _source_for(P, rng, m=400):
    idx = rng.choice(len(P), size=min(m, len(P)), replace=False)
    src = (P[idx] + rng.normal(scale=0.05, size=(len(idx), 3))).astype(np.float32)
    return src, _random_cov9(rng, len(src))


def _check_thin(a, P, S, src, src_cov, leaf, M, poses=None, res=1.0):
    """Thin A on the device; compare everything with a fresh handle given the expected arrays."""
    keep = thin_indices(P, leaf, M)
    a.thin_target(leaf, M)
    assert a.num_target_points() == len(keep)
    b = _with_arrays(P[keep], S[keep], src, src_cov, res=res)
    assert np.array_equal(_target_points(a), P[keep]) and np.array_equal(_target_points(b), P[keep])
    assert a.get_target_covariances().tobytes() == S[keep].tobytes() == b.get_target_covariances().tobytes()
    _assert_same_map(a, b)
    if poses is None:
        poses = [np.eye(4), np.array([[1, 0, 0, 0.05], [0, 1, 0, -0.03], [0, 0, 1, 0.02], [0, 0, 0, 1]], dtype=np.float64)]
    _assert_same_evaluations(a, b, poses)
    b.close()
    return keep


def _cloud(n, seed, leaf=0.5, per_cell=5.0):
    """n points in a cube sized for about per_cell points per cell of `leaf`, around a negative offset, plus exact duplicates."""
    rng = np.random.default_rng(seed)
    side = max(leaf, leaf * (n / per_cell) ** (1.0 / 3.0))
    P = rng.uniform(-side / 2 - 3.3, side / 2 - 3.3, size=(n, 3)).astype(np.float32)
    if n > 4:
        P[n // 2:n // 2 + n // 8] = P[:n // 8]  # exact duplicates later in the array
    if n > 100:
        P[-40:] = P[1]  # one crowded cell, beyond every M < 40
    return P, _random_cov9(rng, n), rng


# ------------------------------------------------------------------------------------------------------------ sizes x M
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 2047, 2048, 2049])
@pytest.mark.parametrize("M", [1, 2, 20, "n"])
def test_thin_equals_fresh_upload(n, M):
    P, S, rng = _cloud(n, seed=n)
    M = n if M == "n" else M
    src, sc = _source_for(P, rng)
    a = _with_arrays(P, S, src, sc)
    keep = _check_thin(a, P, S, src, sc, 0.5, M)
    assert len(keep) == n if M >= n else len(keep) < n
    a.close()


def test_thin_after_append_of_the_fixture_pair(pair02, relative_pose):
    tgt, src = pair02
    a = _core()
    _load_target_knn(a, tgt)
    _load_source_knn(a, src)
    P = np.vstack([tgt, a.transform_source(relative_pose)])
    S = np.vstack([a.get_target_covariances(), rotate_covariances(relative_pose, a.get_source_covariances())])
    a.append_source_to_target(relative_pose)
    keep = thin_indices(P, 0.5, 2)
    assert 0 < len(keep) < len(P)
    a.thin_target(0.5, 2)
    b = _core()
    _load_target_arrays(b, P[keep], S[keep])
    _load_source_knn(b, src)
    assert np.array_equal(_target_points(a), P[keep])
    assert a.get_target_covariances().tobytes() == S[keep].tobytes()
    _assert_same_map(a, b)
    vm = O.VoxelMap(P[keep], S[keep], 1.0, accum_double=True)
    assert a.num_voxels() == vm.num_voxels
    assert np.array_equal(a.get_voxel_means(), vm.vox_mean) and np.array_equal(a.get_voxel_covs(), vm.vox_cov)
    rng = np.random.default_rng(3)
    from conftest import random_pose

    poses = [np.asarray(relative_pose, dtype=np.float64), np.eye(4)] + [relative_pose @ random_pose(rng, np.radians(3), 0.3) for _ in range(2)]
    _assert_same_evaluations(a, b, poses)


@pytest.mark.parametrize("n", [150_000, 1_000_000])
def test_thin_large_maps(n):
    rng = np.random.default_rng(n)
    if n == 1_000_000:
        from fast_gicp_b200.synthetic import kitti_like_pair

        P, _, _ = kitti_like_pair(beams=128, az_steps=8192, seed=44, pose=(0.5, 0.0, 1.0), downsample=0.0, max_points=1_000_000)
        P = np.ascontiguousarray(P[:n])
    else:
        P, _, rng = _cloud(n, seed=5, leaf=0.5, per_cell=3.0)
    S = _random_cov9(rng, len(P))
    src, sc = _source_for(P, rng, m=5000)
    a = _with_arrays(P, S, src, sc)
    keep = _check_thin(a, P, S, src, sc, 0.5, 4)
    assert len(keep) < len(P)
    a.close()


# ------------------------------------------------------------------------------------------------------------ key widths
def _box_cloud(width, n=3000, seed=0):
    """Points at leaf 1.0 whose cells span exactly `width` key bits (bits(max - min) summed over the axes), with repeated cells."""
    bx = min(22, width)
    by = min(21, width - bx)
    bz = width - bx - by
    assert bz <= 22
    rng = np.random.default_rng(seed)
    cols = []
    for b in (bx, by, bz):
        span = (1 << b) - 1
        base = -(span // 2) - 1 if b else 7
        vals = np.unique(np.array([0, 1 if span else 0, span // 2, span], dtype=np.int64)) + base
        frac = rng.choice([0.25, 0.5, 0.75], size=n)
        cols.append(rng.choice(vals, size=n).astype(np.float64) + frac)
    P = np.stack(cols, axis=1).astype(np.float32)
    assert np.array_equal(np.floor(P.astype(np.float64)), np.floor(np.stack(cols, axis=1)))  # exact in float32
    return P, _random_cov9(rng, n), rng


@pytest.mark.parametrize("width", [0, 1, 9, 10, 18, 27, 36, 45, 54, 63, 64])
def test_key_widths(width):
    P, S, rng = _box_cloud(width, seed=width)
    src, sc = _source_for(P, rng, m=200)
    a = _with_arrays(P, S, src, sc)
    keep = _check_thin(a, P, S, src, sc, 1.0, 2, poses=[np.eye(4)])
    assert len(keep) < len(P)
    if width == 0:
        assert keep.tolist() == [0, 1]
    a.close()


def test_tiny_leaf_over_a_wide_extent():
    rng = np.random.default_rng(21)
    P = rng.uniform(-100, 100, size=(5000, 3)).astype(np.float32)
    P = np.vstack([P, P[:1500], P[:700]])  # cells of 1, 2 and 3 points at leaf 1e-3 (54-bit keys)
    S = _random_cov9(rng, len(P))
    src, sc = _source_for(P, rng)
    a = _with_arrays(P, S, src, sc)
    keep = _check_thin(a, P, S, src, sc, 1e-3, 2, poses=[np.eye(4)])
    assert len(keep) == 5000 + 1500
    a.close()


def test_key_of_65_bits_is_refused():
    from fast_gicp_b200 import core as K

    P, S, rng = _box_cloud(65, seed=65)
    src, sc = _source_for(P, rng, m=200)
    a = _with_arrays(P, S, src, sc)
    before = _snapshot(a)
    l0 = a.launch_count()
    assert a._lib.vgicp_thin_target(a._h, 1.0, 2) == K.ERR_INVALID_ARGUMENT
    assert a.launch_count() == l0 + 1  # the box pass only
    _assert_unchanged(a, before)
    a.close()


# ------------------------------------------------------------------------------------------------------------ refusals
def _snapshot(c, with_eval=True):
    out = dict(n=c.num_target_points(), pts=_target_points(c).tobytes(), cov=c.get_target_covariances().tobytes(), map=_map_state(c))
    if with_eval:
        c.update_correspondences(np.eye(4))
        e, H, b = c.compute_error(np.eye(4))
        out["eval"] = (e, H.tobytes(), b.tobytes())
    return out


def _assert_unchanged(c, before, with_eval=True):
    after = _snapshot(c, with_eval)
    assert after["n"] == before["n"] and after["pts"] == before["pts"] and after["cov"] == before["cov"]
    for k in before["map"]:
        assert np.asarray(before["map"][k]).tobytes() == np.asarray(after["map"][k]).tobytes(), k  # (bytes: NaN means compare equal)
    if with_eval:
        assert after["eval"] == before["eval"]


def test_refusals_change_nothing():
    from fast_gicp_b200 import core as K

    P, S, rng = _cloud(3000, seed=1)
    src, sc = _source_for(P, rng)
    a = _with_arrays(P, S, src, sc)
    lib, h = a._lib, a._h
    before = _snapshot(a)
    l0 = a.launch_count()
    # argument checks: nothing launched
    for leaf in (float("nan"), float("inf"), -float("inf"), 0.0, -0.5, 1e-300, 1e-39, 1e39):
        assert lib.vgicp_thin_target(h, leaf, 2) == K.ERR_INVALID_ARGUMENT, leaf
    for M in (0, -1, -(1 << 31)):
        assert lib.vgicp_thin_target(h, 0.5, M) == K.ERR_INVALID_ARGUMENT, M
    for problem in (1, 2):
        a.set_problem(problem)
        assert lib.vgicp_thin_target(h, 0.5, 2) == K.ERR_UNSUPPORTED
    a.set_problem(0)
    a.set_stage1_sharding(1)
    assert lib.vgicp_thin_target(h, 0.5, 2) == K.ERR_UNSUPPORTED
    a.set_stage1_sharding(0)
    assert a.launch_count() == l0
    # found by the box pass: a cell outside the int range, a key wider than 64 bits
    assert lib.vgicp_thin_target(h, 1e-10, 2) == K.ERR_INVALID_ARGUMENT
    assert lib.vgicp_thin_target(h, 1e-6, 2) == K.ERR_INVALID_ARGUMENT
    assert a.launch_count() == l0 + 2
    with pytest.raises(K.VgicpError) as e:
        a.thin_target(0.5, 0)
    assert e.value.code == K.ERR_INVALID_ARGUMENT
    _assert_unchanged(a, before)
    # the handle still thins correctly afterwards
    _check_thin(a, P, S, src, sc, 0.5, 3)
    a.close()


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_point_is_refused(bad):
    from fast_gicp_b200 import core as K

    P, S, rng = _cloud(2000, seed=2)
    P[1234, 1] = bad
    a = _core()
    _load_target_arrays(a, P, S)
    before = _snapshot(a, with_eval=False)
    l0 = a.launch_count()
    assert a._lib.vgicp_thin_target(a._h, 0.5, 2) == K.ERR_INVALID_ARGUMENT
    assert a.launch_count() == l0 + 1
    _assert_unchanged(a, before, with_eval=False)
    a.close()


def test_missing_target_or_covariances():
    from fast_gicp_b200 import core as K

    P, _, _ = _cloud(500, seed=3)
    for setup in ("no target", "target without covariances"):
        c = _core()
        if setup != "no target":
            c.set_target_cloud(P)
        l0 = c.launch_count()
        assert c._lib.vgicp_thin_target(c._h, 0.5, 2) == K.ERR_BAD_STATE, setup
        assert c.launch_count() == l0
        c.close()


# ------------------------------------------------------------------------------------------------------------ settings
def test_robust_kernel_and_first_resolution_survive():
    P, S, rng = _cloud(4000, seed=4)
    src, sc = _source_for(P, rng)
    a = _with_arrays(P, S, src, sc)
    a.set_robust_kernel("CAUCHY", 1.0)
    a.set_resolution(0.5)  # the map keeps the resolution it was first created with
    keep = thin_indices(P, 0.5, 2)
    a.thin_target(0.5, 2)
    b = _with_arrays(P[keep], S[keep], src, sc, res=1.0)
    b.set_robust_kernel("CAUCHY", 1.0)
    plain = _with_arrays(P[keep], S[keep], src, sc, res=1.0)
    _assert_same_map(a, b)
    T0 = np.eye(4)
    for c in (a, b, plain):
        c.update_correspondences(T0)
    ea, eb, ep = a.compute_error(T0), b.compute_error(T0), plain.compute_error(T0)
    assert ea[0] == eb[0] and ea[1].tobytes() == eb[1].tobytes()
    assert ea[0] != ep[0]
    assert a.num_voxels() == O.VoxelMap(P[keep], S[keep], 1.0, accum_double=True).num_voxels
    for c in (a, b, plain):
        c.close()


# ------------------------------------------------------------------------------------------------------------ sequence
def test_append_thin_crop_sequence_device_equals_host():
    from fast_gicp_b200.core import pose_from_c

    _, scans = _sequence(30)
    leaf, M, radius = 0.5, 4, 40.0
    a, b = _core(), _core()
    _load_target_knn(a, scans[0])
    _load_target_knn(b, scans[0])
    P, S = scans[0].copy(), b.get_target_covariances()
    T = np.eye(4)
    for k in range(1, len(scans)):
        _load_source_knn(a, scans[k])
        _load_source_knn(b, scans[k])
        ra, rb = a.align(T), b.align(T)
        assert _res_tuple(ra) == _res_tuple(rb), k
        T = pose_from_c(ra.T)
        a.append_source_to_target(T)
        a.thin_target(leaf, M)
        a.crop_target(T[:3, 3], radius, 0)
        P = np.vstack([P, b.transform_source(T)])
        S = np.vstack([S, rotate_covariances(T, b.get_source_covariances())])
        keep = thin_indices(P, leaf, M)
        P, S = P[keep], S[keep]
        keep = crop_indices(P, T[:3, 3], radius, 0)
        P, S = P[keep], S[keep]
        _load_target_arrays(b, P, S)
        assert a.num_target_points() == len(P), k
        assert a.get_target_covariances().tobytes() == S.tobytes(), k


# ------------------------------------------------------------------------------------------------------------ surfaces
def _python_mirror_loop(scans):
    from fast_gicp_b200 import FastVGICPCuda

    reg = FastVGICPCuda()
    reg.setNeighborSearchMethod("DIRECT7")
    reg.setInputTarget(scans[0])
    out = []
    for k in (1, 2, 3):
        reg.setInputSource(scans[k])
        out.append(reg.align(reg.getFinalTransformation()))
        assert reg.hasConverged()
        reg.appendSourceToTarget(reg.getFinalTransformation())
        reg.thinTarget(0.5, 2)
        reg.cropTarget(out[-1][:3, 3].astype(np.float64), 40.0, 0)
    reg.setInputSource(scans[4])
    out.append(reg.align(reg.getFinalTransformation()))
    return reg, out


def test_python_mirror_loop_matches_core():
    from fast_gicp_b200.core import pose_from_c

    _, scans = _sequence(5)
    reg, out = _python_mirror_loop(scans)
    a = _core()
    _load_target_knn(a, scans[0])
    T = np.eye(4, dtype=np.float32)
    for k in (1, 2, 3, 4):
        _load_source_knn(a, scans[k])
        T = pose_from_c(a.align(T.astype(np.float64), reg._params()).T).astype(np.float32)
        assert np.array_equal(T, out[k - 1]), k
        if k < 4:
            a.append_source_to_target(T.astype(np.float64))
            a.thin_target(0.5, 2)
            a.crop_target(T[:3, 3].astype(np.float64), 40.0, 0)
    assert a.num_target_points() == reg.vgicp_cuda_.num_target_points()


def test_pygicp_loop_matches_python_mirror():
    if LIB not in sys.path:
        sys.path.insert(0, LIB)
    import pygicp

    _, scans = _sequence(5)
    _, want = _python_mirror_loop(scans)
    reg = pygicp.FastVGICPCuda()
    reg.set_neighbor_search_method("DIRECT7", 1.5)
    reg.set_input_target(scans[0].astype(np.float64))
    got = []
    for k in (1, 2, 3):
        reg.set_input_source(scans[k].astype(np.float64))
        got.append(reg.align(reg.get_final_transformation()))
        reg.append_source_to_target(reg.get_final_transformation())
        reg.thin_target(0.5, 2)
        reg.crop_target(got[-1][:3, 3].astype(np.float64), 40.0, 0)
    reg.set_input_source(scans[4].astype(np.float64))
    got.append(reg.align(reg.get_final_transformation()))
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


CPP_LOOP = r"""
#include <cstdio>
#include <vector>
#include <fast_gicp_b200/fast_vgicp_cuda.hpp>
using Cloud = pcl::PointCloud<pcl::PointXYZ>;
static Cloud::Ptr load(const char* path, int n) {
  auto c = pcl::make_shared<Cloud>();
  c->resize(n);
  std::vector<float> xyz(3 * (size_t)n);
  FILE* f = std::fopen(path, "rb");
  if (!f || std::fread(xyz.data(), sizeof(float), xyz.size(), f) != xyz.size()) return nullptr;
  std::fclose(f);
  for (int i = 0; i < n; i++) { c->at(i).x = xyz[3 * i]; c->at(i).y = xyz[3 * i + 1]; c->at(i).z = xyz[3 * i + 2]; }
  return c;
}
int main(int argc, char** argv) {
  std::vector<Cloud::Ptr> scans;
  for (int k = 0; k < 5; k++) scans.push_back(load(argv[1 + 2 * k], std::atoi(argv[2 + 2 * k])));
  fast_gicp::FastVGICPCuda<pcl::PointXYZ, pcl::PointXYZ> reg;
  reg.setNeighborSearchMethod(fast_gicp::NeighborSearchMethod::DIRECT7);
  reg.setInputTarget(scans[0]);
  Cloud aligned;
  for (int k = 1; k < 5; k++) {
    reg.setInputSource(scans[k]);
    reg.align(aligned, reg.getFinalTransformation());
    Eigen::Matrix4f T = reg.getFinalTransformation();
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) std::printf("%.9g ", T(r, c));
    std::printf("\n");
    if (k < 4) {
      reg.appendSourceToTarget(T);
      reg.thinTarget(0.5, 2);
      const double c[3] = {T(0, 3), T(1, 3), T(2, 3)};
      reg.cropTarget(c, 40.0, 0);
    }
  }
  return 0;
}
"""


def test_cpp_mirror_loop_matches_python_mirror(tmp_path):
    _, scans = _sequence(5)
    _, want = _python_mirror_loop(scans)
    src = tmp_path / "loop.cpp"
    src.write_text(CPP_LOOP)
    exe = tmp_path / "loop"
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([gxx, "-std=c++17", "-O2", str(src), "-o", str(exe), "-I", INC, "-L", LIB, "-Wl,-rpath," + LIB, "-lvgicp_b200"])
    args = []
    for k, s in enumerate(scans):
        (tmp_path / f"s{k}.bin").write_bytes(np.ascontiguousarray(s, dtype=np.float32).tobytes())
        args += [str(tmp_path / f"s{k}.bin"), str(len(s))]
    out = subprocess.run([str(exe)] + args, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.split("\n")
    for k in range(4):
        got = np.array([float(x) for x in lines[k].split()], dtype=np.float32).reshape(4, 4)
        assert np.array_equal(got, want[k]), k

