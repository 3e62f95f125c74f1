#!/bin/bash
# compute-sanitizer passes over the hot path: memcheck + racecheck + synccheck on one full registration per neighbour mode,
# on both k-NN search paths, and on all four users of the shared block rank (voxel ids, crop and thinning, both voxel grids).
# memcheck also reports every allocation left at exit and every failing CUDA call; the driver ends by destroying a handle in each
# state that holds a lazily created resource, and empties torch's cache so that only the libraries' own allocations remain.
# One log per tool, written by the loop at the end into the directory given as the first argument.
set -u
cat > /tmp/san_driver.py <<'PY'
import sys, numpy as np
sys.path.insert(0, ".")
from fast_gicp_b200.core import Core
d = np.load("tests/golden/pair_0p2.npz")
tgt, src = d["target"][::3].copy(), d["source"][::3].copy()
for method, hint, vindex, spec in (("DIRECT27", 0, 0, 1), ("DIRECT7", 1, 0, 1), ("DIRECT1", 0, 1, 0), ("DIRECT_RADIUS", 1, 1, 1),
                                   ("DIRECT27", 0, 1, 0)):
    c = Core(0)
    c.set_neighbor_search_method(method, 1.5)
    c.set_execution_hint(hint)
    c.set_voxel_index(vindex); c.set_speculation(spec)
    r = c.register(tgt, src)
    c.calculate_source_covariances_rbf(3)
    print(method, "converged", bool(r.converged), "fitness", c.fitness_score(np.eye(4)))
    c.close()
# a cloud below 256 points: every query takes the block-cooperative scan of the whole cloud (k <= 32 and the wide k > 32 kernels)
c = Core(0)
for k in (20, 64):
    c.set_source_cloud(src[:200]); c.find_source_neighbors(k)
    print("small cloud k", k, "rows", c.get_source_neighbors().shape)
c.close()
# a far outlier: the voxel bounding box no longer fits the direct-mapped index, the k-NN grid's levels are all coarse there and the deferred (block-cooperative) search takes the queries
c = Core(0)
c.set_neighbor_search_method("DIRECT27")
far = np.vstack([tgt, np.array([[3.0e6, -2.0e6, 1.0e6]], dtype=np.float32)])
r = c.register(far, src)
print("outlier", "converged", bool(r.converged))
c.close()
# DIRECT1 on a cloud above the streaming threshold: k_linearize_stream (bulk copies into shared memory, mbarriers), 1M-class sort path
from fast_gicp_b200.synthetic import kitti_like_pair
bt, bs, _ = kitti_like_pair(beams=48, az_steps=2083, seed=5, pose=(0.4, 0.05, 0.5), downsample=0.0)
c = Core(0)
c.set_resolution(0.5); c.set_neighbor_search_method("DIRECT1")
r = c.register(bt, bs)
print("stream", len(bs), "converged", bool(r.converged))
c.close()
# local map: carve it with the registered source (range image, atomicMin, window test), append the source (the target's arrays
# grow with a device copy), thin it (cell box, u64 keys and sort, keep mask), crop it (block rank, compaction)
c = Core(0)
c.set_neighbor_search_method("DIRECT7")
r = c.register(tgt, src)
from fast_gicp_b200.core import pose_from_c
print("carved", c.carve_target(pose_from_c(r.T), window=2))
c.append_source_to_target(pose_from_c(r.T))
c.thin_target(0.5, 2)
c.crop_target((0.0, 0.0, 0.0), 30.0, len(tgt))
r = c.align(pose_from_c(r.T))
print("local map", c.num_target_points(), "converged", bool(r.converged))
c.close()
# motion compensation: timestamps read out of a 32-byte point struct, the source deskewed in place, covariances recomputed
c = Core(0)
c.set_neighbor_search_method("DIRECT7")
cloud = np.zeros(len(src), dtype=np.dtype({"names": ["xyz", "time"], "formats": [("<f4", 3), "<f4"], "offsets": [0, 16], "itemsize": 32}))
cloud["xyz"], cloud["time"] = src[:, :3], np.linspace(0.0, 0.1, len(src), dtype=np.float32)
c.set_target_cloud(tgt); c.find_target_neighbors(20); c.calculate_target_covariances(3); c.create_target_voxelmap()
c.set_source_cloud(src)
c.deskew_source(cloud["time"], [0.0, 0.0, 0.35, 8.0, 0.0, 0.0], 0.05)
c.find_source_neighbors(20); c.calculate_source_covariances(3)
r = c.align()
print("deskew", c.num_source_points(), "converged", bool(r.converged))
# continuous time: the timestamps kept by the deskew, the pose and the residual twist estimated together (k_linearize_ct), both hints
for hint, method in ((0, "DIRECT7"), (1, "DIRECT_RADIUS")):
    c.set_execution_hint(hint); c.set_neighbor_search_method(method, 1.5)
    c.set_source_timestamps(cloud["time"], 0.05)
    r = c.align_ct(np.eye(4), np.zeros(6), np.zeros(6), np.full(6, 1e-3))
    print("ct", method, "converged", bool(r.converged), "twist", list(r.twist))
c.close()
# timestamped scans on the device: the voxel grid with fields (k_prep_walk / scatter / tail with F = 2, input and output on the
# device), the source and its timestamps read in place from its output (k_gather_times), the stored deskew, continuous time
import torch
from fast_gicp_b200.prep import InputPrep
p = InputPrep(0)
rec = np.zeros((len(src), 8), dtype=np.float32)
rec[:, :3], rec[:, 3], rec[:, 4] = src[:, :3], 50.0, np.linspace(0.0, 0.1, len(src), dtype=np.float32)
out = p.approximate_voxel_grid_fields(torch.from_numpy(rec).cuda(), 0.25, [4, 3], True)
m = out.shape[0]
c = Core(0)
c.set_neighbor_search_method("DIRECT7")
c.set_target_cloud(tgt); c.find_target_neighbors(20); c.calculate_target_covariances(3); c.create_target_voxelmap()
c.set_cloud_device("source", out.data_ptr(), m, 20)
c.set_source_timestamps_device(out.data_ptr() + 12, m, 20, 0.05)
c.deskew_source_stored([0.0, 0.0, 0.35, 8.0, 0.0, 0.0])
c.find_source_neighbors(20); c.calculate_source_covariances(3)
r = c.align_ct(np.eye(4), np.zeros(6), np.zeros(6), np.full(6, 1e-3))
print("raw scan", m, "points, ct converged", bool(r.converged))
# the exact voxel grid with fields and a minimum count (k_grid_box, k_grid_keys and the sort, k_grid_heads, k_grid_centroids)
g = p.voxel_grid(torch.from_numpy(rec).cuda(), 0.25, [4, 3], 2)
print("voxel grid", g.shape[0], "voxels of >= 2 points")
c.close(); p.close()
# NDT D2D through the same evaluation kernels
c = Core(0)
c.set_problem(2); c.set_neighbor_search_method("DIRECT7")
c.set_target_cloud(tgt); c.set_source_cloud(src); c.ndt_create_voxelmaps()
r = c.align()
print("ndt d2d", "converged", bool(r.converged))
c.close()
# stage 1, RBF covariances: k_covariance_rbf shares its staged tiles and per-lane partials across a __syncthreads per round of eight
# blocks; one point (511 padding points), one round plus a padded block, and several rounds with a partial last one
c = Core(0)
for n in (1, 513, 4097):
    c.set_source_cloud(np.ascontiguousarray(d["target"][:n])); c.calculate_source_covariances_rbf(3)
    print("rbf", n, "finite", bool(np.isfinite(c.get_source_covariances()).all()))
c.close()
# handle lifetime: every state with a lazily created resource (multi-pose, multi-source, deskew, CT, profiling, stage-1 graph,
# pending voxel map, thin and carve, the exact grid), destroyed there
sys.path.insert(0, "tests")
from test_gpu_handle_lifetime import STATES
t32, s32 = np.ascontiguousarray(tgt[:, :3], np.float32), np.ascontiguousarray(src[:, :3], np.float32)
for state in STATES:
    state(torch, t32, s32).close()
    print("lifetime", state.__name__, "closed")
torch.cuda.empty_cache()
PY
out=${1:-/tmp/vgicp_sanitizer}  # the directory the logs go to (first argument)
mkdir -p "$out"
for tool in memcheck racecheck synccheck; do
  extra=""
  [ $tool = memcheck ] && extra="--leak-check full --report-api-errors all"
  log="$out/sanitizer_$tool.log"
  timeout 900 compute-sanitizer --tool $tool $extra --print-limit 20 python /tmp/san_driver.py > "$log" 2>&1
  echo "== $tool: $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' "$log" | tail -1)"
done
