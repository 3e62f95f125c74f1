"""The host model of vgicp_carve_target (synthetic.carve_indices): against an independent float64 restatement of the rule, on
hand-built scenes, under the invariances the rule promises, and on a drive past a moving vehicle with the full map maintenance
(carve, append, thin, crop).  CPU only."""
import math

import numpy as np
import pytest

from fast_gicp_b200 import synthetic as syn

BASE = dict(width=1024, height=64, elevation_min=math.radians(-25.0), elevation_max=math.radians(3.0), window=1, margin=0.3, margin_rel=0.02)


def params(**kw):
    p = dict(BASE)
    p.update(kw)
    return p


def removed_set(target, source, T, p):
    keep = syn.carve_indices(target, source, T, p)
    return np.setdiff1d(np.arange(len(target)), keep)


# ------------------------------------------------------------------------------------------------------------ float64 restatement
def pixel64(x, y, z, p):
    """(row, col, u, a * W / 4, r) in float64, or None without a pixel."""
    if not (math.isfinite(x) and math.isfinite(y) and math.isfinite(z)) or abs(x) + abs(y) == 0:
        return None
    q = abs(y) / (abs(x) + abs(y))
    a = (q if x >= 0 else 2 - q) if y >= 0 else (2 + q if x < 0 else 4 - q)
    t_lo, t_hi = math.tan(p["elevation_min"]), math.tan(p["elevation_max"])
    u = (z / math.hypot(x, y) - t_lo) * (p["height"] / (t_hi - t_lo))
    if not (0 <= u < p["height"]):
        return None
    aw = a * p["width"] / 4
    return int(math.floor(u)), int(math.floor(aw)) % p["width"], u, aw, math.sqrt(x * x + y * y + z * z)


def near_boundary(px, tol=1e-4):
    _, _, u, aw, _ = px
    return min(u - math.floor(u), math.ceil(u) - u) < tol or min(aw - math.floor(aw), math.ceil(aw) - aw) < tol


def model64(target, source, T, p, tol=1e-4):
    """Removed flags in float64 (a dict image, a loop over the window) and the rows too close to a bin edge or to the threshold
    for float32 and float64 to agree."""
    img = {}
    for x, y, z in np.asarray(source, dtype=np.float64):
        px = pixel64(x, y, z, p)
        if px:
            key = (px[0], px[1])
            img[key] = min(img.get(key, math.inf), px[4])
    R, t = np.asarray(T, dtype=np.float64)[:3, :3], np.asarray(T, dtype=np.float64)[:3, 3]
    S = (np.asarray(target, dtype=np.float64) - t) @ R
    removed, unsure = np.zeros(len(S), dtype=bool), np.zeros(len(S), dtype=bool)
    w, H, W = p["window"], p["height"], p["width"]
    for i, (x, y, z) in enumerate(S):
        px = pixel64(x, y, z, p)
        if px is None:
            continue
        unsure[i] = near_boundary(px, tol)
        rows = [rr for rr in range(px[0] - w, px[0] + w + 1) if 0 <= rr < H]
        vals = [img[(rr, (px[1] + dc) % W)] for rr in rows for dc in range(-w, w + 1) if (rr, (px[1] + dc) % W) in img]
        if vals:
            r_min = min(vals)
            thr = r_min - (p["margin"] + p["margin_rel"] * r_min)
            removed[i] = px[4] < thr
            unsure[i] |= abs(px[4] - thr) < tol
    return removed, unsure


def _random_pose(rng):
    yaw = rng.uniform(-np.pi, np.pi)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
    T[:3, 3] = rng.uniform(-3, 3, size=3)
    return T


@pytest.mark.parametrize("seed,window,width,height", [(0, 1, 1024, 64), (1, 0, 360, 32), (2, 2, 97, 13), (3, 1, 1, 1), (4, 3, 2048, 128)])
def test_against_float64(seed, window, width, height):
    rng = np.random.default_rng(seed)
    p = params(window=window, width=width, height=height, elevation_min=-0.5, elevation_max=0.2)
    src = rng.normal(size=(3000, 3)) * [20.0, 20.0, 2.0]
    src = src[[not (px and near_boundary(px)) for px in (pixel64(*s, p) for s in src)]].astype(np.float32)  # source rows clear of bin edges
    T = _random_pose(rng)
    # map points: the source's points placed by T, pulled towards the sensor or pushed away, plus a uniform cloud
    Q = src[rng.choice(len(src), 2000)].astype(np.float64) * rng.uniform(0.3, 1.5, size=(2000, 1))
    tgt = np.vstack([Q @ T[:3, :3].T + T[:3, 3], rng.uniform(-40, 40, size=(2000, 3)) * [1, 1, 0.1]]).astype(np.float32)
    removed, unsure = model64(tgt, src, T, p)
    got = np.zeros(len(tgt), dtype=bool)
    got[removed_set(tgt, src, T, p)] = True
    assert unsure.mean() < 0.05
    assert np.array_equal(got[~unsure], removed[~unsure])
    if width * height > 1:
        assert 20 < removed.sum() < len(tgt) - 100


# ------------------------------------------------------------------------------------------------------------ hand-built scenes
SMALL = params(width=8, height=4, elevation_min=math.radians(-30.0), elevation_max=math.radians(30.0), window=0, margin=0.3, margin_rel=0.0)
I4 = np.eye(4)


def carve(tgt, src, p=SMALL, T=I4):
    return syn.carve_indices(np.asarray(tgt, dtype=np.float32), np.asarray(src, dtype=np.float32), T, p).tolist()


def test_in_front_behind_and_on_the_surface():
    src = [[10.0, 0.0, 0.0]]
    tgt = [[5.0, 0.0, 0.0], [12.0, 0.0, 0.0], [10.0, 0.0, 0.0], [9.75, 0.0, 0.0], [9.65, 0.0, 0.0]]
    assert carve(tgt, src) == [1, 2, 3]  # 5 m and 9.65 m lie more than 0.3 m in front; 9.75 m lies within the margin
    assert carve(tgt, src, params(**{**SMALL, "margin_rel": 0.5})) == [0, 1, 2, 3, 4]  # thr = 10 - (0.3 + 5) = 4.7


def test_the_nearest_return_of_a_pixel_counts():
    src = [[10.0, 0.0, 0.0], [6.0, 0.1, 0.0], [20.0, 0.1, 0.0]]
    assert carve([[5.0, 0.0, 0.0], [5.8, 0.0, 0.0]], src) == [1]


def test_empty_pixels_and_windows_keep_the_point():
    src = [[10.0, 0.0, 0.0]]  # col 0, one row
    tgt = [[0.0, 5.0, 0.0], [-5.0, 0.0, 0.0], [5.0, 0.0, 2.0]]  # col 2, col 4, another row: empty
    assert carve(tgt, src) == [0, 1, 2]
    assert carve(tgt, src, params(**{**SMALL, "window": 1})) == [0, 1, 2]  # the windows do not reach col 0's row 1 ... 2
    assert carve([[1.0, 0.0, 0.0]], np.zeros((0, 3))) == [0]


def test_points_outside_the_vertical_field_of_view_are_kept():
    src = [[10.0, 0.0, 0.0], [10.0, 0.0, 20.0], [10.0, 0.0, -20.0]]  # only the first has a pixel
    tgt = [[5.0, 0.0, 10.0], [5.0, 0.0, -10.0], [2.0, 0.0, 0.0]]
    assert carve(tgt, src) == [0, 1]
    assert carve(tgt, src, params(**{**SMALL, "window": 3})) == [0, 1]


def test_column_wraps():
    src = [[10.0, -0.1, 0.0]]  # a = 4 - q: column W - 1
    ok, row, col, _ = syn._carve_pixels(np.float32(src), 8, 4, np.float32(2.0), np.float32(math.tan(math.radians(-30))),
                                        np.float32(4 / (2 * math.tan(math.radians(30)))))
    assert ok[0] and col[0] == 7
    tgt = [[5.0, 0.1, 0.0]]  # column 0
    assert carve(tgt, src) == [0]
    assert carve(tgt, src, params(**{**SMALL, "window": 1})) == []
    assert carve(src, tgt, params(**{**SMALL, "window": 1})) == [0]  # the surface is now in column 0 and the map point behind it
    assert carve([[5.0, -0.1, 0.0]], [[10.0, 0.1, 0.0]], params(**{**SMALL, "window": 1})) == []  # and the other way round


def test_axes_signed_zero_and_diagonals():
    p = SMALL
    e_lo = np.float32(math.tan(p["elevation_min"]))
    inv_de = np.float32(p["height"] / (math.tan(p["elevation_max"]) - math.tan(p["elevation_min"])))
    pts = np.float32([[5, 5, 0], [-5, 5, 0], [-5, -5, 0], [5, -5, 0], [5, 0, 0], [5, -0.0, 0], [-5, 0, 0], [-5, -0.0, 0], [0, 5, 0], [0, -5, 0], [-0.0, 5, 0],
                      [0, 0, 1], [-0.0, -0.0, 1], [0, 0, 0]])
    ok, _, col, _ = syn._carve_pixels(pts, 8, 4, np.float32(2.0), e_lo, inv_de)
    assert ok.tolist() == [True] * 11 + [False] * 3
    assert col[:11].tolist() == [1, 3, 5, 7, 0, 0, 4, 4, 2, 6, 2]  # a = 0.5, 1.5, 2.5, 3.5; y = -0 counts as y >= 0
    # x = y = 0 has no pixel: neither as a return nor as a map point
    assert carve([[0.0, 0.0, 3.0], [5.0, 0.0, 0.0]], [[0.0, 0.0, 9.0], [10.0, 0.0, 0.0]]) == [0]
    assert carve([[5.0, -0.0, 0.0]], [[10.0, 0.0, 0.0]]) == []


def test_window_zero_against_two():
    src = [[0.0, 10.0, 0.0]]  # column 2
    tgt = [[5.0, 0.0, 0.0]]  # column 0
    assert carve(tgt, src) == [0]
    assert carve(tgt, src, params(**{**SMALL, "window": 1})) == [0]
    assert carve(tgt, src, params(**{**SMALL, "window": 2})) == []


def test_non_finite_rows():
    src = [[10.0, 0.0, 0.0], [np.nan, 0.0, 0.0], [np.inf, 1.0, 0.0], [1.0, -np.inf, 0.0]]
    tgt = [[5.0, 0.0, 0.0], [np.nan, 0.0, 0.0], [np.inf, 0.0, 0.0], [0.0, 0.0, -np.inf]]
    assert carve(tgt, src) == [1, 2, 3]


def test_pose_places_the_scan():
    T = np.eye(4)
    T[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]  # 90 degrees about z
    T[:3, 3] = [100.0, -50.0, 1.0]
    src = [[10.0, 0.0, 0.0]]  # in the map: (100, -40, 1)
    assert carve([[100.0, -45.0, 1.0], [100.0, -35.0, 1.0], [105.0, -50.0, 1.0]], src, T=T) == [1, 2]


# ------------------------------------------------------------------------------------------------------------ invariances
@pytest.fixture(scope="module")
def scene():
    rng = np.random.default_rng(5)
    poses, scans, _ = syn.moving_object_sequence(3, 11, beams=32, az_steps=1024)
    P = np.vstack([(s.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32) for T, s in zip(poses[:2], scans[:2])])
    return P, scans[2], poses[2], rng


def test_source_order_and_duplicates_do_not_matter(scene):
    P, src, T, rng = scene
    p = params()
    base = syn.carve_indices(P, src, T, p)
    assert 0 < len(base) < len(P)
    assert np.array_equal(syn.carve_indices(P, src[rng.permutation(len(src))], T, p), base)
    assert np.array_equal(syn.carve_indices(P, np.vstack([src, src[::3], src[:50]]), T, p), base)


def test_more_returns_in_measured_pixels_only_shrink_the_removed_set(scene):
    """Returns added in pixels that already hold one can only lower r_min, hence the threshold: the removed set shrinks.  (A
    return in an empty window can remove a point: it is new evidence, not a lower range.)"""
    P, src, T, rng = scene
    p = params()
    ok0, row0, col0, _ = syn._carve_pixels(src, p["width"], p["height"], np.float32(256.0), np.float32(math.tan(p["elevation_min"])),
                                           np.float32(p["height"] / (math.tan(p["elevation_max"]) - math.tan(p["elevation_min"]))))
    measured = set((row0[ok0] * p["width"] + col0[ok0]).tolist())
    extra = (src[rng.choice(len(src), 3000)] * rng.uniform(0.3, 1.2, size=(3000, 1))).astype(np.float32)
    ok, row, col, _ = syn._carve_pixels(extra, p["width"], p["height"], np.float32(256.0), np.float32(math.tan(p["elevation_min"])),
                                        np.float32(p["height"] / (math.tan(p["elevation_max"]) - math.tan(p["elevation_min"]))))
    extra = extra[ok & np.isin(row * p["width"] + col, list(measured))]
    assert len(extra) > 1000
    fewer = removed_set(P, src, T, p)
    more = removed_set(P, np.vstack([src, extra]), T, p)
    assert len(more) < len(fewer)
    assert np.all(np.isin(more, fewer))


# ------------------------------------------------------------------------------------------------------------ functional
def _placed(T, s):
    return (s.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


def maintenance_loop(poses, scans, boxes, p, leaf=0.5, M=4, radius=60.0):
    """carve (p, or none when None), append, thin, crop with the ground-truth poses on the host models.  -> (box points older than
    one frame left in the map at the last frame, static points carved over the sequence, final map size)"""
    from test_gpu_local_map import crop_indices

    P = _placed(poses[0], scans[0])
    box, frame = syn.in_boxes(P, boxes[0]), np.zeros(len(P), dtype=np.int64)
    static_carved = 0
    for k in range(1, len(scans)):
        if p is not None:
            keep = syn.carve_indices(P, scans[k], poses[k], p)
            static_carved += int((~box).sum() - (~box[keep]).sum())
            P, box, frame = P[keep], box[keep], frame[keep]
        Q = _placed(poses[k], scans[k])
        P, box, frame = np.vstack([P, Q]), np.r_[box, syn.in_boxes(Q, boxes[k])], np.r_[frame, np.full(len(Q), k)]
        for keep in (syn.thin_indices(P, leaf, M), None):
            keep = crop_indices(P, poses[k][:3, 3], radius, 0) if keep is None else keep
            P, box, frame = P[keep], box[keep], frame[keep]
    return int((box & (frame < len(scans) - 2)).sum()), static_carved, len(P)


def test_moving_vehicle_leaves_no_trail():
    """Ground-truth drive of 20 frames (64 beams, the defaults' sensor) past a vehicle overtaking in the next lane; seeded, exact
    models, so the counts are fixed: 2705 vehicle points older than one frame stay in the map without carving, 8 with the
    library's defaults, which remove 1968 static points (distant ground that the scan grazes) over the 19 carves."""
    from fast_gicp_b200.core import carve_params

    poses, scans, boxes = syn.moving_object_sequence(20, 7)
    ghosts0, _, _ = maintenance_loop(poses, scans, boxes, None)
    ghosts, static_carved, n = maintenance_loop(poses, scans, boxes, carve_params())
    assert ghosts0 > 2000
    assert ghosts <= 20
    assert static_carved <= 2500
    assert n > 100000


def test_moving_object_sequence_keeps_the_static_scans():
    """Without movers the sequence is scripts/bench_local_map.py's: the same world, path and noise seeds, the same bytes."""
    poses, scans, boxes = syn.moving_object_sequence(3, 7, movers=(), beams=16, az_steps=256)
    world = syn._make_world(np.random.default_rng(7))
    for k, (T, s) in enumerate(zip(poses, scans)):
        assert boxes[k] == []
        assert np.array_equal(s, syn.voxel_downsample(syn.scan(world, 16, 256, T, np.random.default_rng(7000 + k)), 0.25))
    assert np.allclose(poses[2][:2, 3], [0.8 + 0.8 * np.cos(np.radians(2.0)), 0.8 * np.sin(np.radians(2.0))])


def test_null_handle_and_params_are_refused():
    import ctypes as C

    from fast_gicp_b200 import core

    lib = core.load_library()
    p = core.CarveParams(**core.carve_params())
    T = core.pose_to_c(np.eye(4))
    assert lib.vgicp_carve_target(None, core._dp(T), C.byref(p), None) == core.ERR_INVALID_ARGUMENT
    assert core.carve_params() == {"width": 1024, "height": 64, "elevation_min": -25.0 * math.pi / 180.0, "elevation_max": 3.0 * math.pi / 180.0, "window": 1,
                                   "margin": 0.3, "margin_rel": 0.02}
