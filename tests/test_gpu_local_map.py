"""Local map for scan-to-map odometry: vgicp_append_source_to_target and vgicp_crop_target.

Handle A is changed on the device; a fresh handle B is given the expected arrays directly (set_target_cloud with the points,
set_target_covariances with the 3x3s, create_target_voxelmap).  Both must then hold the same bytes and evaluate identically.
The expected arrays come from numpy float32 restatements of the recipes in include/vgicp_b200.h."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle as O
from conftest import random_pose

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fast_gicp_b200", "lib")
INC = os.path.join(ROOT, "fast_gicp_b200", "cpp", "include")

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ numpy models
def rotate_covariances(T, cov9):
    """R C R^T in IEEE float32 in the header's order; returns (n, 9) stored the way set_covariances stores a 3x3."""
    R = np.asarray(T, dtype=np.float64)[:3, :3].astype(np.float32)
    C = np.asarray(cov9, dtype=np.float32).reshape(-1, 3, 3)  # symmetric: row- and column-major alike
    M = np.empty_like(C)
    N = np.empty_like(C)
    for i in range(3):
        for k in range(3):
            M[:, i, k] = (R[i, 0] * C[:, 0, k] + R[i, 1] * C[:, 1, k]) + R[i, 2] * C[:, 2, k]
    for i in range(3):
        for j in range(3):
            N[:, i, j] = (M[:, i, 0] * R[j, 0] + M[:, i, 1] * R[j, 1]) + M[:, i, 2] * R[j, 2]
    S = np.empty_like(N)
    for i in range(3):
        for j in range(3):
            S[:, i, j] = N[:, i, i] if i == j else np.float32(0.5) * (N[:, i, j] + N[:, j, i])
    return S.reshape(-1, 9)


def crop_indices(pts, center, radius, max_points):
    """Indices kept by vgicp_crop_target: the float32 radius test, then the last max_points passing indices."""
    c = np.asarray(center, dtype=np.float64).astype(np.float32)
    d = np.asarray(pts, dtype=np.float32) - c
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    keep = np.flatnonzero(d2 <= np.float32(radius * radius))
    if max_points and len(keep) > max_points:
        keep = keep[len(keep) - max_points:]
    return keep


# ------------------------------------------------------------------------------------------------------------ helpers
def _core(method="DIRECT7", res=1.0):
    from fast_gicp_b200.core import Core

    c = Core(0)
    c.set_resolution(res)
    c.set_neighbor_search_method(method, 1.5)
    return c


def _load_target_knn(c, pts):
    c.set_target_cloud(pts)
    c.find_target_neighbors(20)
    c.calculate_target_covariances(O.REG_PLANE)
    c.create_target_voxelmap()


def _load_source_knn(c, pts):
    c.set_source_cloud(pts)
    c.find_source_neighbors(20)
    c.calculate_source_covariances(O.REG_PLANE)


def _load_target_arrays(c, pts, cov9):
    c.set_target_cloud(pts)
    c.set_target_covariances(cov9)
    c.create_target_voxelmap()


def _target_points(c):
    """The target's points, read back through swap + transform_source(identity) (exact up to the sign of zero)."""
    c.swap_source_and_target()
    p = c.transform_source(np.eye(4))
    c.swap_source_and_target()
    return p


def _map_state(c):
    coords, ids = c.get_voxel_buckets()
    return dict(num_buckets=c.num_buckets(), num_voxels=c.num_voxels(), coords=coords, ids=ids, n=c.get_voxel_num_points(), mean=c.get_voxel_means(),
                cov=c.get_voxel_covs())


def _assert_same_map(a, b):
    ma, mb = _map_state(a), _map_state(b)
    assert ma["num_buckets"] == mb["num_buckets"] and ma["num_voxels"] == mb["num_voxels"]
    for k in ("coords", "ids", "n", "mean", "cov"):
        assert ma[k].tobytes() == mb[k].tobytes(), k


def _res_tuple(r):
    return (bytes(r.T), bytes(r.H), r.nr_iterations, r.converged, r.n_linearize, r.n_compute_error, r.lm_failed)


def _assert_same_evaluations(a, b, poses):
    for T in poses:
        a.update_correspondences(T)
        b.update_correspondences(T)
        ea, Ha, ba = a.compute_error(T)
        eb, Hb, bb = b.compute_error(T)
        assert ea == eb and Ha.tobytes() == Hb.tobytes() and ba.tobytes() == bb.tobytes()
    assert _res_tuple(a.align(poses[0])) == _res_tuple(b.align(poses[0]))
    ma, mb = a.align_multi(np.stack(poses)), b.align_multi(np.stack(poses))
    assert [_res_tuple(r) for r in ma] == [_res_tuple(r) for r in mb]
    for want_H in (False, True):
        ra, rb = a.evaluate_poses(np.stack(poses), want_H), b.evaluate_poses(np.stack(poses), want_H)
        for x, y in zip(ra, rb):
            assert (x is None and y is None) or x.tobytes() == y.tobytes()


@pytest.fixture
def appended(pair02, relative_pose):
    """A with the 0.2 m pair loaded (PLANE k-NN covariances) and the expected arrays of an append at relative.txt."""
    tgt, src = pair02

    def make(T):
        a = _core()
        _load_target_knn(a, tgt)
        _load_source_knn(a, src)
        P = np.vstack([tgt, a.transform_source(T)])
        S = np.vstack([a.get_target_covariances(), rotate_covariances(T, a.get_source_covariances())])
        return a, P, S

    return make


def _fresh_with(P, S, src, res=1.0):
    b = _core(res=res)
    _load_target_arrays(b, P, S)
    _load_source_knn(b, src)
    return b


# ------------------------------------------------------------------------------------------------------------ append
@pytest.mark.parametrize("which", ["relative", "random"])
def test_append_equals_concatenation(appended, pair02, relative_pose, which):
    tgt, src = pair02
    T = relative_pose if which == "relative" else random_pose(np.random.default_rng(11), np.radians(20), 3.0)
    a, P, S = appended(T)
    a.append_source_to_target(T)
    b = _fresh_with(P, S, src)
    assert a.num_target_points() == len(tgt) + len(src)
    assert np.array_equal(_target_points(a), P) and np.array_equal(_target_points(b), P)
    assert a.get_target_covariances().tobytes() == S.tobytes() == b.get_target_covariances().tobytes()
    _assert_same_map(a, b)
    vm = O.VoxelMap(P, S, 1.0, accum_double=True)
    coords, ids = a.get_voxel_buckets()
    assert a.num_buckets() == vm.num_buckets and a.num_voxels() == vm.num_voxels
    assert np.array_equal(ids, vm.bucket_id) and np.array_equal(coords, vm.bucket_coord)
    assert np.array_equal(a.get_voxel_num_points(), vm.vox_n)
    assert np.array_equal(a.get_voxel_means(), vm.vox_mean) and np.array_equal(a.get_voxel_covs(), vm.vox_cov)
    rng = np.random.default_rng(3)
    poses = [np.asarray(relative_pose, dtype=np.float64), np.eye(4)] + [relative_pose @ random_pose(rng, np.radians(3), 0.3) for _ in range(3)]
    _assert_same_evaluations(a, b, poses)
    # the merged map has no neighbour rows; k-NN covariances of it can still be computed
    from fast_gicp_b200.core import VgicpError

    with pytest.raises(VgicpError) as e:
        a.get_target_neighbors()
    assert e.value.code == 2
    a.find_target_neighbors(20)
    a.calculate_target_covariances(O.REG_PLANE)
    a.create_target_voxelmap()
    assert a.num_voxels() > 0


# ------------------------------------------------------------------------------------------------------------ crop
@pytest.mark.parametrize("center,radius,max_points", [((2.0, -20.0, 0.5), 18.0, 0), ((0.0, 0.0, 0.0), float("inf"), 6000), ((2.0, -20.0, 0.5), 25.0, 7000),
                                                      ((0.0, 0.0, 0.0), float("inf"), 0)])
def test_crop_against_numpy_model(appended, pair02, relative_pose, center, radius, max_points):
    tgt, src = pair02
    a, P, S = appended(relative_pose)
    a.append_source_to_target(relative_pose)
    before = _map_state(a)
    a.crop_target(center, radius, max_points)
    keep = crop_indices(P, center, radius, max_points)
    if radius == float("inf") and max_points == 0:
        assert len(keep) == len(P)
        after = _map_state(a)
        for k in before:
            assert np.array_equal(before[k], after[k]), k
    else:
        assert 0 < len(keep) < len(P)
    assert a.num_target_points() == len(keep)
    b = _fresh_with(P[keep], S[keep], src)
    assert np.array_equal(_target_points(a), P[keep])
    assert a.get_target_covariances().tobytes() == S[keep].tobytes()
    _assert_same_map(a, b)
    _assert_same_evaluations(a, b, [np.asarray(relative_pose, dtype=np.float64), np.eye(4)])


def test_crop_to_zero_is_refused_and_changes_nothing(appended, pair02, relative_pose):
    from fast_gicp_b200.core import ERR_INVALID_ARGUMENT, VgicpError

    a, P, S = appended(relative_pose)
    a.append_source_to_target(relative_pose)
    before = _map_state(a)
    a.update_correspondences(relative_pose)
    e0 = a.compute_error(relative_pose)
    launches = a.launch_count()
    with pytest.raises(VgicpError) as e:
        a.crop_target((1e4, 1e4, 0.0), 5.0, 0)
    assert e.value.code == ERR_INVALID_ARGUMENT
    assert a.launch_count() == launches + 1  # the counting pass only
    assert a.num_target_points() == len(P)
    after = _map_state(a)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    assert a.get_target_covariances().tobytes() == S.tobytes()
    e1 = a.compute_error(relative_pose)
    assert e0[0] == e1[0] and e0[1].tobytes() == e1[1].tobytes()


# ------------------------------------------------------------------------------------------------------------ sequence
def _sequence(n_frames, seed=4):
    from fast_gicp_b200 import synthetic as syn

    rng = np.random.default_rng(seed)
    world = syn._make_world(rng)
    poses, scans = [], []
    xy = np.zeros(2)
    for k in range(n_frames):  # 0.8 m steps along an arc turning 2.5 degrees per frame
        yaw = np.radians(2.5 * k)
        T = np.eye(4)
        T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
        T[:2, 3] = xy
        xy = xy + 0.8 * np.array([np.cos(yaw), np.sin(yaw)])
        poses.append(T)
        scans.append(syn.voxel_downsample(syn.scan(world, 32, 1024, T, np.random.default_rng(seed * 100 + k)), 0.5))
    return poses, scans


def test_scan_to_map_sequence_device_equals_host():
    from fast_gicp_b200.core import pose_from_c

    _, scans = _sequence(8)
    radius, cap = 40.0, 12000
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
        a.crop_target(T[:3, 3], radius, cap)
        P = np.vstack([P, b.transform_source(T)])
        S = np.vstack([S, rotate_covariances(T, b.get_source_covariances())])
        keep = crop_indices(P, T[:3, 3], radius, cap)
        P, S = P[keep], S[keep]
        _load_target_arrays(b, P, S)
        assert a.num_target_points() == len(P) <= cap
        assert a.get_target_covariances().tobytes() == S.tobytes()


# ------------------------------------------------------------------------------------------------------------ interactions
def test_set_target_cloud_after_append_is_a_fresh_state(appended, pair02, relative_pose):
    tgt, src = pair02
    a, _, _ = appended(relative_pose)
    a.append_source_to_target(relative_pose)
    _load_target_knn(a, src)
    b = _core()
    _load_target_knn(b, src)
    _load_source_knn(b, src)
    _assert_same_map(a, b)
    assert a.num_target_points() == len(src)
    _assert_same_evaluations(a, b, [np.asarray(relative_pose, dtype=np.float64), np.eye(4)])


def test_swap_after_append(appended, pair02, relative_pose):
    tgt, src = pair02
    a, P, S = appended(relative_pose)
    a.append_source_to_target(relative_pose)
    b = _fresh_with(P, S, src)
    a.swap_source_and_target()
    b.swap_source_and_target()
    assert a.num_source_points() == b.num_source_points() == len(P)
    assert a.transform_source(np.eye(4)).tobytes() == b.transform_source(np.eye(4)).tobytes()
    _assert_same_map(a, b)
    Tinv = np.linalg.inv(relative_pose)
    _assert_same_evaluations(a, b, [Tinv, np.eye(4)])


def test_robust_kernel_survives_append(appended, pair02, relative_pose):
    tgt, src = pair02
    a, P, S = appended(relative_pose)
    a.set_robust_kernel("CAUCHY", 1.0)
    a.append_source_to_target(relative_pose)
    b = _fresh_with(P, S, src)
    b.set_robust_kernel("CAUCHY", 1.0)
    plain = _fresh_with(P, S, src)
    T0 = np.asarray(relative_pose, dtype=np.float64)
    for c in (a, b, plain):
        c.update_correspondences(T0)
    ea, eb, ep = a.compute_error(T0), b.compute_error(T0), plain.compute_error(T0)
    assert ea[0] == eb[0] and ea[1].tobytes() == eb[1].tobytes()
    assert ea[0] != ep[0]


def test_append_keeps_the_first_map_resolution(appended, pair02, relative_pose):
    tgt, src = pair02
    a, P, S = appended(relative_pose)
    a.set_resolution(0.5)
    a.append_source_to_target(relative_pose)
    b = _fresh_with(P, S, src, res=1.0)
    _assert_same_map(a, b)
    assert a.num_voxels() == O.VoxelMap(P, S, 1.0, accum_double=True).num_voxels


# ------------------------------------------------------------------------------------------------------------ errors
def test_errors_return_before_any_launch(appended, pair02, relative_pose):
    from fast_gicp_b200 import core as K

    tgt, src = pair02
    a, P, S = appended(relative_pose)
    lib, h = a._lib, a._h
    T = K.pose_to_c(relative_pose)
    c3 = np.zeros(3)
    dp = lambda x: x.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    launches = a.launch_count()
    n0 = a.num_target_points()

    def crop(center, radius, cap=0):
        return lib.vgicp_crop_target(h, center, float(radius), cap)

    assert lib.vgicp_append_source_to_target(h, None) == K.ERR_INVALID_ARGUMENT
    for bad in (np.nan, np.inf):
        Tb = T.copy()
        Tb[5] = bad
        assert lib.vgicp_append_source_to_target(h, dp(Tb)) == K.ERR_INVALID_ARGUMENT
    assert crop(None, 10.0) == K.ERR_INVALID_ARGUMENT
    assert crop(dp(c3), float("nan")) == K.ERR_INVALID_ARGUMENT
    assert crop(dp(c3), -1.0) == K.ERR_INVALID_ARGUMENT
    for problem in (1, 2):
        a.set_problem(problem)
        assert lib.vgicp_append_source_to_target(h, dp(T)) == K.ERR_UNSUPPORTED
        assert crop(dp(c3), 10.0) == K.ERR_UNSUPPORTED
    a.set_problem(0)
    a.set_stage1_sharding(1)
    assert lib.vgicp_append_source_to_target(h, dp(T)) == K.ERR_UNSUPPORTED
    assert crop(dp(c3), 10.0) == K.ERR_UNSUPPORTED
    a.set_stage1_sharding(0)
    assert a.launch_count() == launches and a.num_target_points() == n0
    # missing points or covariances
    for setup in ("no source", "source without covariances", "target without covariances", "no target"):
        c = _core()
        if setup != "no target":
            c.set_target_cloud(tgt)
            if setup != "target without covariances":
                c.find_target_neighbors(20)
                c.calculate_target_covariances(O.REG_PLANE)
        if setup != "no source":
            c.set_source_cloud(src)
            if setup != "source without covariances":
                c.find_source_neighbors(20)
                c.calculate_source_covariances(O.REG_PLANE)
        l0 = c.launch_count()
        assert c._lib.vgicp_append_source_to_target(c._h, dp(T)) == K.ERR_BAD_STATE, setup
        if setup in ("target without covariances", "no target"):
            assert c._lib.vgicp_crop_target(c._h, dp(c3), 10.0, 0) == K.ERR_BAD_STATE, setup
        assert c.launch_count() == l0
        c.close()


def test_append_beyond_the_cloud_limit():
    """A merged target above 2^31 / 64 points (what set_target_cloud accepts) is refused before anything is launched."""
    from fast_gicp_b200 import core as K

    half = ((1 << 31) // 64) // 2 + 1
    pts = np.zeros((half, 3), dtype=np.float32)
    cov = np.zeros((half, 9), dtype=np.float32)
    c = _core()
    c.set_target_cloud(pts)
    c.set_target_covariances(cov)
    c.set_source_cloud(pts)
    c.set_source_covariances(cov)
    l0 = c.launch_count()
    T = K.pose_to_c(np.eye(4))
    assert c._lib.vgicp_append_source_to_target(c._h, T.ctypes.data_as(ctypes.POINTER(ctypes.c_double))) == K.ERR_INVALID_ARGUMENT
    assert c.launch_count() == l0 and c.num_target_points() == half
    c.close()


# ------------------------------------------------------------------------------------------------------------ surfaces
def _python_mirror_loop(scans):
    from fast_gicp_b200 import FastVGICPCuda

    reg = FastVGICPCuda()
    reg.setNeighborSearchMethod("DIRECT7")
    reg.setInputTarget(scans[0])
    out = []
    for k in (1, 2):
        reg.setInputSource(scans[k])
        out.append(reg.align(reg.getFinalTransformation()))
        assert reg.hasConverged()
        reg.appendSourceToTarget(reg.getFinalTransformation())
    reg.cropTarget(out[-1][:3, 3].astype(np.float64), 40.0, 9000)
    reg.setInputSource(scans[3])
    out.append(reg.align(reg.getFinalTransformation()))
    return reg, out


def test_python_mirror_loop_and_reload():
    _, scans = _sequence(4)
    reg, out = _python_mirror_loop(scans)
    c = reg.vgicp_cuda_
    assert c.num_target_points() <= 9000
    reg.setInputTarget(scans[0])  # the device map is not scans[0] any more: this reloads it
    assert c.num_target_points() == len(scans[0])
    # the same loop spelled on the core
    from fast_gicp_b200.core import pose_from_c

    a = _core()
    _load_target_knn(a, scans[0])
    T = np.eye(4, dtype=np.float32)
    for k in (1, 2, 3):
        _load_source_knn(a, scans[k])
        T = pose_from_c(a.align(T.astype(np.float64), reg._params()).T).astype(np.float32)
        assert np.array_equal(T, out[k - 1]), k
        if k < 3:
            a.append_source_to_target(T.astype(np.float64))
        if k == 2:
            a.crop_target(T[:3, 3].astype(np.float64), 40.0, 9000)


def test_pygicp_loop_matches_python_mirror():
    if LIB not in sys.path:
        sys.path.insert(0, LIB)
    import pygicp

    _, scans = _sequence(4)
    _, want = _python_mirror_loop(scans)
    reg = pygicp.FastVGICPCuda()
    reg.set_neighbor_search_method("DIRECT7", 1.5)
    reg.set_input_target(scans[0].astype(np.float64))
    got = []
    for k in (1, 2):
        reg.set_input_source(scans[k].astype(np.float64))
        got.append(reg.align(reg.get_final_transformation()))
        reg.append_source_to_target(reg.get_final_transformation())
    reg.crop_target(got[-1][:3, 3].astype(np.float64), 40.0, 9000)
    reg.set_input_source(scans[3].astype(np.float64))
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
  for (int k = 0; k < 4; k++) scans.push_back(load(argv[1 + 2 * k], std::atoi(argv[2 + 2 * k])));
  fast_gicp::FastVGICPCuda<pcl::PointXYZ, pcl::PointXYZ> reg;
  reg.setNeighborSearchMethod(fast_gicp::NeighborSearchMethod::DIRECT7);
  reg.setInputTarget(scans[0]);
  Cloud aligned;
  for (int k = 1; k < 4; k++) {
    if (k == 3) {
      Eigen::Matrix4f T = reg.getFinalTransformation();
      const double c[3] = {T(0, 3), T(1, 3), T(2, 3)};
      reg.cropTarget(c, 40.0, 9000);
    }
    reg.setInputSource(scans[k]);
    reg.align(aligned, reg.getFinalTransformation());
    Eigen::Matrix4f T = reg.getFinalTransformation();
    for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) std::printf("%.9g ", T(r, c));
    std::printf("\n");
    if (k < 3) reg.appendSourceToTarget(T);
  }
  reg.setInputTarget(scans[0]);
  size_t n = 0;
  vgicp_get_num_target_points(reg.handle(), &n);
  std::printf("%zu\n", n);
  return 0;
}
"""


def test_cpp_mirror_loop_matches_python_mirror(tmp_path):
    _, scans = _sequence(4)
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
    for k in range(3):
        got = np.array([float(x) for x in lines[k].split()], dtype=np.float32).reshape(4, 4)
        assert np.array_equal(got, want[k]), k
    assert int(lines[3]) == len(scans[0])
