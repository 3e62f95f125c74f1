"""Dynamic objects in the local map: vgicp_carve_target removes the target points the registered scan sees through.

Handle A is carved on the device; a fresh handle B is given the expected arrays directly (set_target_cloud with the kept points,
set_target_covariances with their 3x3s, create_target_voxelmap).  Both must then hold the same bytes and evaluate identically.
The kept rows come from synthetic.carve_indices, the numpy restatement of the rule in include/vgicp_b200.h."""
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_handle_state import _pair, _prepared, _read
from test_gpu_local_map import (INC, LIB, _assert_same_evaluations, _assert_same_map, _core, _load_source_knn, _load_target_arrays, _load_target_knn, _res_tuple,
                                _target_points, crop_indices, rotate_covariances)
from test_gpu_thin_target import _assert_unchanged, _random_cov9, _snapshot

pytestmark = pytest.mark.gpu


def carve_indices(target, source, T, params):
    from fast_gicp_b200.synthetic import carve_indices as f

    return f(target, source, T, params)


def carve_params(**kw):
    from fast_gicp_b200.core import carve_params as f

    return f(**kw)


def _pose(rng):
    yaw = rng.uniform(-np.pi, np.pi)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
    T[:3, 3] = rng.uniform(-5, 5, size=3) * [1, 1, 0.1]
    return T


def _scene(n, seed, n_src=20000):
    """(map P (n, 3), its covariances, scan (sensor frame), T, rng): half the map lies along the scan's rays, pulled towards the
    sensor or pushed past the return (so that both outcomes occur), the other half is spread over the scene."""
    rng = np.random.default_rng(seed)
    T = _pose(rng)
    src = (rng.normal(size=(n_src, 3)) * [20.0, 20.0, 1.5]).astype(np.float32)
    k = n // 2
    Q = src[rng.integers(0, n_src, k)].astype(np.float64) * rng.uniform(0.3, 1.5, size=(k, 1))
    U = rng.uniform(-40.0, 40.0, size=(n - k, 3)) * [1.0, 1.0, 0.08]
    P = np.vstack([Q @ T[:3, :3].T + T[:3, 3], U + T[:3, 3]]).astype(np.float32)
    P = np.ascontiguousarray(P[rng.permutation(n)])
    return P, _random_cov9(rng, n), src, T, rng


def _with(P, S, src, src_cov=None):
    c = _core()
    _load_target_arrays(c, P, S)
    c.set_source_cloud(src)
    if src_cov is not None:
        c.set_source_covariances(src_cov)
    return c


def _check_carve(P, S, src, T, params, evaluate=True):
    """Carve A on the device; compare with the model and with a fresh handle given the expected arrays."""
    from fast_gicp_b200 import core as K

    keep = carve_indices(P, src, T, params)
    sc = _random_cov9(np.random.default_rng(len(src)), len(src)) if evaluate else None
    a = _with(P, S, src, sc)
    if len(keep) == 0:
        before = _snapshot(a, with_eval=False)
        with pytest.raises(K.VgicpError) as e:
            a.carve_target(T, **params)
        assert e.value.code == K.ERR_INVALID_ARGUMENT
        _assert_unchanged(a, before, with_eval=False)
        a.close()
        return keep
    removed = a.carve_target(T, **params)
    assert removed == len(P) - len(keep)
    assert a.num_target_points() == len(keep)
    b = _with(P[keep], S[keep], src, sc)
    assert np.array_equal(_target_points(a), P[keep])
    assert a.get_target_covariances().tobytes() == S[keep].tobytes() == b.get_target_covariances().tobytes()
    _assert_same_map(a, b)
    if evaluate:
        dT = np.eye(4)
        dT[:3, 3] = [0.05, -0.03, 0.02]
        _assert_same_evaluations(a, b, [T, T @ dT])
    a.close()
    b.close()
    return keep


# ------------------------------------------------------------------------------------------------------------ sizes
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 2047, 2048, 2049, 150_000, 1_000_000])
def test_carve_equals_fresh_upload(n):
    P, S, src, T, _ = _scene(n, seed=n)
    keep = _check_carve(P, S, src, T, carve_params())
    if n > 1000:
        assert 0 < len(keep) < n


def _ring(n=500, r=20.0):
    """n returns at range r around the sensor, at elevation 0"""
    az = np.linspace(-np.pi, np.pi, n, endpoint=False)
    return np.stack([r * np.cos(az), r * np.sin(az), np.zeros(n)], axis=1).astype(np.float32)


def test_single_point_kept_and_removed():
    S = _random_cov9(np.random.default_rng(0), 1)
    src = _ring()
    assert len(_check_carve(np.float32([[40.0, 0.0, 0.0]]), S, src, np.eye(4), carve_params())) == 1
    assert len(_check_carve(np.float32([[5.0, 0.0, 0.0]]), S, src, np.eye(4), carve_params())) == 0  # refused: it would leave no points


# ------------------------------------------------------------------------------------------------------------ images x windows
@pytest.mark.parametrize("window", [0, 1, 2])
@pytest.mark.parametrize("image", [(1, 1), (1021, 37), (1024, 64), (4096, 4096)])
def test_image_sizes_and_windows(image, window):
    P, S, src, T, _ = _scene(20000, seed=image[0] + window)
    keep = _check_carve(P, S, src, T, carve_params(width=image[0], height=image[1], window=window), evaluate=window == 1)
    assert 0 < len(keep) <= len(P)
    if image != (1, 1):  # (one pixel: r_min is the nearest return of the whole scan)
        assert len(keep) < len(P)


def test_duplicated_and_non_finite_source_rows():
    P, S, src, T, rng = _scene(30000, seed=8)
    clean = carve_indices(P, src, T, carve_params())
    dup = np.vstack([src, src[::3], src[:100]])
    assert np.array_equal(_check_carve(P, S, dup, T, carve_params()), clean)
    bad = src.copy()
    rows = rng.choice(len(bad), 300, replace=False)
    bad[rows[:100], 0] = np.nan
    bad[rows[100:200], 1] = np.inf
    bad[rows[200:], 2] = -np.inf
    bad[rows[:10]] = 0.0  # |x| + |y| == 0: no pixel either
    keep = _check_carve(P, S, bad, T, carve_params(), evaluate=False)
    assert 0 < len(keep) < len(P)


# ------------------------------------------------------------------------------------------------------------ refusals
def test_refusals_change_nothing():
    import ctypes as C

    from fast_gicp_b200 import core as K

    P, S, src, T, _ = _scene(5000, seed=1)
    a = _with(P, S, src, _random_cov9(np.random.default_rng(1), len(src)))
    lib, h = a._lib, a._h
    before = _snapshot(a)
    l0 = a.launch_count()

    def rc(T=T, **kw):
        p = K.CarveParams(**carve_params(**kw))
        return lib.vgicp_carve_target(h, K._dp(K.pose_to_c(T)), C.byref(p), None)

    assert lib.vgicp_carve_target(h, None, C.byref(K.CarveParams(**carve_params())), None) == K.ERR_INVALID_ARGUMENT
    assert lib.vgicp_carve_target(h, K._dp(K.pose_to_c(T)), None, None) == K.ERR_INVALID_ARGUMENT
    for bad in (np.nan, np.inf):
        Tb = T.copy()
        Tb[1, 3] = bad
        assert rc(T=Tb) == K.ERR_INVALID_ARGUMENT
    hp = np.pi / 2
    for kw in (dict(width=0), dict(height=0), dict(width=-1), dict(width=4097, height=4096), dict(width=1 << 24, height=2), dict(elevation_min=0.1, elevation_max=0.1),
               dict(elevation_min=0.2, elevation_max=0.1), dict(elevation_min=-hp), dict(elevation_max=hp), dict(elevation_min=np.nan), dict(elevation_max=np.inf),
               dict(window=-1), dict(window=9), dict(margin=-0.1), dict(margin=np.nan), dict(margin=np.inf), dict(margin=1e39), dict(margin_rel=-0.01),
               dict(margin_rel=1.0), dict(margin_rel=np.nan)):
        assert rc(**kw) == K.ERR_INVALID_ARGUMENT, kw
    for problem in (1, 2):
        a.set_problem(problem)
        assert rc() == K.ERR_UNSUPPORTED
    a.set_problem(0)
    a.set_stage1_sharding(1)
    assert rc() == K.ERR_UNSUPPORTED
    a.set_stage1_sharding(0)
    assert a.launch_count() == l0
    _assert_unchanged(a, before)
    # a carve that would leave no points: refused after the rank, target and map as they were
    ring = _ring()
    allin = _with(ring * np.float32(0.25), S[:500], ring)
    before = _snapshot(allin, with_eval=False)
    with pytest.raises(K.VgicpError) as e:
        allin.carve_target(np.eye(4))
    assert e.value.code == K.ERR_INVALID_ARGUMENT
    _assert_unchanged(allin, before, with_eval=False)
    allin.close()
    # the handle still carves correctly afterwards
    keep = carve_indices(P, src, T, carve_params())
    assert a.carve_target(T) == len(P) - len(keep)
    assert np.array_equal(_target_points(a), P[keep])
    a.close()


def test_missing_source_target_or_covariances():
    from fast_gicp_b200 import core as K

    P, S, src, T, _ = _scene(500, seed=3)
    for setup in ("no source", "empty source", "no target", "target without covariances"):
        c = _core()
        if setup in ("no source", "empty source"):
            _load_target_arrays(c, P, S)
            if setup == "empty source":
                c.set_source_cloud(np.zeros((0, 3), dtype=np.float32))
        else:
            c.set_source_cloud(src)
            if setup != "no target":
                c.set_target_cloud(P)
        l0 = c.launch_count()
        with pytest.raises(K.VgicpError) as e:
            c.carve_target(T)
        assert e.value.code == K.ERR_BAD_STATE, setup
        assert c.launch_count() == l0
        c.close()


def test_handle_state_after_a_carve(pair02):
    tgt, src = _pair(pair02)
    c = _prepared(tgt, src)
    try:
        removed = c.carve_target(np.eye(4))
        assert 0 < removed < len(tgt)
        assert _read(c) == "++B++++"
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------------------ sequence
def test_moving_object_odometry_device_equals_host():
    """align, carve, append, thin, crop on the device against the host route (the models, then the map uploaded again)."""
    from fast_gicp_b200 import synthetic as syn
    from fast_gicp_b200.core import pose_from_c

    _, scans, _ = syn.moving_object_sequence(12, 7, beams=32, az_steps=1024)
    params, leaf, M, radius = carve_params(), 0.5, 4, 40.0
    a, b = _core(), _core()
    _load_target_knn(a, scans[0])
    _load_target_knn(b, scans[0])
    P, S = scans[0].copy(), b.get_target_covariances()
    T = np.eye(4)
    total = 0
    for k in range(1, len(scans)):
        _load_source_knn(a, scans[k])
        _load_source_knn(b, scans[k])
        ra, rb = a.align(T), b.align(T)
        assert _res_tuple(ra) == _res_tuple(rb), k
        T = pose_from_c(ra.T)
        removed = a.carve_target(T)
        a.append_source_to_target(T)
        a.thin_target(leaf, M)
        a.crop_target(T[:3, 3], radius, 0)
        keep = carve_indices(P, scans[k], T, params)
        assert removed == len(P) - len(keep), k
        total += removed
        P, S = P[keep], S[keep]
        P = np.vstack([P, b.transform_source(T)])
        S = np.vstack([S, rotate_covariances(T, b.get_source_covariances())])
        keep = syn.thin_indices(P, leaf, M)
        P, S = P[keep], S[keep]
        keep = crop_indices(P, T[:3, 3], radius, 0)
        P, S = P[keep], S[keep]
        _load_target_arrays(b, P, S)
        assert a.num_target_points() == len(P), k
        assert a.get_target_covariances().tobytes() == S.tobytes(), k
    assert total > 0
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------------------ surfaces
def _scans(n):
    from fast_gicp_b200 import synthetic as syn

    return syn.moving_object_sequence(n, 7, beams=32, az_steps=1024)[1]


def _python_mirror_loop(scans):
    from fast_gicp_b200 import FastVGICPCuda

    reg = FastVGICPCuda()
    reg.setNeighborSearchMethod("DIRECT7")
    reg.setInputTarget(scans[0])
    out, removed = [], []
    for k in (1, 2, 3):
        reg.setInputSource(scans[k])
        out.append(reg.align(reg.getFinalTransformation()))
        removed.append(reg.carveTarget(reg.getFinalTransformation()))
        reg.appendSourceToTarget(reg.getFinalTransformation())
    reg.setInputSource(scans[4])
    out.append(reg.align(reg.getFinalTransformation()))
    return out, removed


def test_python_mirror_and_pygicp_match_core():
    from fast_gicp_b200.core import pose_from_c

    scans = _scans(5)
    out, removed = _python_mirror_loop(scans)
    assert sum(removed) > 0
    a = _core()
    _load_target_knn(a, scans[0])
    T = np.eye(4, dtype=np.float32)
    from fast_gicp_b200 import FastVGICPCuda

    params = FastVGICPCuda()._params()
    for k in (1, 2, 3, 4):
        _load_source_knn(a, scans[k])
        T = pose_from_c(a.align(T.astype(np.float64), params).T).astype(np.float32)
        assert np.array_equal(T, out[k - 1]), k
        if k < 4:
            assert a.carve_target(T.astype(np.float64)) == removed[k - 1], k
            a.append_source_to_target(T.astype(np.float64))
    if LIB not in sys.path:
        sys.path.insert(0, LIB)
    import pygicp

    reg = pygicp.FastVGICPCuda()
    reg.set_neighbor_search_method("DIRECT7", 1.5)
    reg.set_input_target(scans[0].astype(np.float64))
    for k in (1, 2, 3, 4):
        reg.set_input_source(scans[k].astype(np.float64))
        got = reg.align(reg.get_final_transformation())
        assert np.array_equal(got, out[k - 1]), k
        if k < 4:
            assert reg.carve_target(reg.get_final_transformation()) == removed[k - 1], k
            reg.append_source_to_target(reg.get_final_transformation())


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
    if (k < 4) {
      std::printf("%zu", reg.carveTarget(T));
      reg.appendSourceToTarget(T);
    }
    std::printf("\n");
  }
  return 0;
}
"""


def test_cpp_mirror_matches_python_mirror(tmp_path):
    scans = _scans(5)
    want, removed = _python_mirror_loop(scans)
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
        vals = lines[k].split()
        got = np.array([float(x) for x in vals[:16]], dtype=np.float32).reshape(4, 4)
        assert np.array_equal(got, want[k]), k
        if k < 3:
            assert int(vals[16]) == removed[k], k
