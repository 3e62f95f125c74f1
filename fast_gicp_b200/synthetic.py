"""Synthetic KITTI-shaped scans (SURVEY.md 8d, configs C3/C4): a spinning multi-beam lidar over a ground plane and
axis-aligned boxes, range noise, optional voxel-grid downsample.  Pure numpy (input generation, not part of the hot path).
"""
import numpy as np


def _ray_box(o, d, lo, hi):
    """Slab test for rays o + t d (o (3,), d (R,3)) against the box [lo, hi]; returns t (inf when missed)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0 = (lo - o) * inv
        t1 = (hi - o) * inv
    tmin = np.minimum(t0, t1).max(axis=1)
    tmax = np.maximum(t0, t1).min(axis=1)
    hit = (tmax >= np.maximum(tmin, 0.0)) & (tmin > 0.0)
    return np.where(hit, tmin, np.inf)


def _make_world(rng, n_boxes=40):
    boxes = []
    while len(boxes) < n_boxes:
        c = rng.uniform(-80, 80, size=2)
        if np.hypot(*c) < 12.0:
            continue
        wl = rng.uniform(2, 20, size=2)
        h = rng.uniform(2, 12)
        boxes.append((np.array([c[0] - wl[0] / 2, c[1] - wl[1] / 2, -1.73]), np.array([c[0] + wl[0] / 2, c[1] + wl[1] / 2, -1.73 + h])))
    return boxes


def scan(world, beams, az_steps, sensor_pose, noise_rng, max_range=120.0, noise=0.02):
    """One revolution seen from `sensor_pose` (4x4, sensor -> world); returns points in the SENSOR frame, float32."""
    el = np.radians(np.linspace(-24.8, 2.0, beams))
    az = np.linspace(-np.pi, np.pi, az_steps, endpoint=False)
    ce, se = np.cos(el)[:, None], np.sin(el)[:, None]
    d_s = np.stack([ce * np.cos(az)[None, :], ce * np.sin(az)[None, :], np.broadcast_to(se, (beams, az_steps))], axis=-1).reshape(-1, 3)
    R, o = sensor_pose[:3, :3], sensor_pose[:3, 3]
    d = d_s @ R.T
    t = np.full(len(d), np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = (-1.73 - o[2]) / d[:, 2]  # ground plane z = -1.73
    t = np.where((tg > 0) & np.isfinite(tg), tg, t)
    for lo, hi in world:
        t = np.minimum(t, _ray_box(o, d, lo, hi))
    ok = np.isfinite(t) & (t < max_range) & (t > 1.0)
    r = t[ok] + noise_rng.normal(0.0, noise, size=int(ok.sum()))
    return (d_s[ok] * r[:, None]).astype(np.float32)


def voxel_downsample(pts, leaf):
    """Exact centroid voxel grid (pcl::VoxelGrid-like), output ordered by voxel index."""
    if leaf <= 0:
        return pts
    ijk = np.floor(pts / np.float32(leaf)).astype(np.int64)
    ijk -= ijk.min(axis=0)
    dims = ijk.max(axis=0) + 1
    idx = ijk[:, 0] + dims[0] * (ijk[:, 1] + dims[1] * ijk[:, 2])
    order = np.argsort(idx, kind="stable")
    idx_s = idx[order]
    starts = np.flatnonzero(np.r_[True, idx_s[1:] != idx_s[:-1]])
    sums = np.add.reduceat(pts[order].astype(np.float64), starts, axis=0)
    counts = np.diff(np.r_[starts, len(idx_s)])[:, None]
    return (sums / counts).astype(np.float32)


def se3_exp_batch(xi):
    """Exp of rotation-first twists xi (m, 6) -> (m, 4, 4), float64; the formula of se3_exp in csrc/lsq_math.hpp, vectorised.
    A zero twist gives the identity exactly."""
    xi = np.asarray(xi, dtype=np.float64).reshape(-1, 6)
    w, v = xi[:, :3], xi[:, 3:]
    th2 = (w * w).sum(axis=1)
    th = np.sqrt(th2)
    small = th2 < 1e-10
    with np.errstate(divide="ignore", invalid="ignore"):
        imag = np.where(small, 0.5 - th2 / 48.0 + th2 * th2 / 3840.0, np.sin(0.5 * th) / th)
        real = np.where(small, 1.0 - th2 / 8.0 + th2 * th2 / 384.0, np.cos(0.5 * th))
        c1 = np.where(small, 0.0, (1.0 - np.cos(th)) / th2)
        c2 = np.where(small, 0.0, (th - np.sin(th)) / (th2 * th))
    qx, qy, qz = (imag[:, None] * w).T
    tx, ty, tz = 2.0 * qx, 2.0 * qy, 2.0 * qz
    twx, twy, twz = tx * real, ty * real, tz * real
    txx, txy, txz, tyy, tyz, tzz = tx * qx, ty * qx, tz * qx, ty * qy, tz * qy, tz * qz
    T = np.zeros((len(xi), 4, 4))
    T[:, 0, 0], T[:, 0, 1], T[:, 0, 2] = 1.0 - (tyy + tzz), txy - twz, txz + twy
    T[:, 1, 0], T[:, 1, 1], T[:, 1, 2] = txy + twz, 1.0 - (txx + tzz), tyz - twx
    T[:, 2, 0], T[:, 2, 1], T[:, 2, 2] = txz - twy, tyz + twx, 1.0 - (txx + tyy)
    Om = np.zeros((len(xi), 3, 3))
    Om[:, 0, 1], Om[:, 0, 2], Om[:, 1, 2] = -w[:, 2], w[:, 1], -w[:, 0]
    Om[:, 1, 0], Om[:, 2, 0], Om[:, 2, 1] = w[:, 2], -w[:, 1], w[:, 0]
    V = np.eye(3)[None] + c1[:, None, None] * Om + c2[:, None, None] * (Om @ Om)
    V = np.where(small[:, None, None], T[:, :3, :3], V)
    T[:, :3, 3] = np.einsum("nij,nj->ni", V, v)
    T[:, 3, 3] = 1.0
    return T


def distorted_scan(world, beams, az_steps, start_pose, twist, period, noise_rng, max_range=120.0, noise=0.02):
    """One revolution of a sensor that moves while it spins: azimuth column a is fired at t_a = period * a / az_steps from the
    pose start_pose @ Exp(t_a twist) (twist = rotation-first [omega, v] per second in the sensor frame at t = 0).  Returns
    (points, times): each point in the sensor frame of its own firing time (float32), and that time (float32).  With a zero
    twist the points are scan(world, beams, az_steps, start_pose, ...)'s bytes."""
    el = np.radians(np.linspace(-24.8, 2.0, beams))
    az = np.linspace(-np.pi, np.pi, az_steps, endpoint=False)
    ce, se = np.cos(el)[:, None], np.sin(el)[:, None]
    d_s = np.stack([ce * np.cos(az)[None, :], ce * np.sin(az)[None, :], np.broadcast_to(se, (beams, az_steps))], axis=-1).reshape(-1, 3)
    t_col = period * np.arange(az_steps) / az_steps
    dT = se3_exp_batch(t_col[:, None] * np.asarray(twist, dtype=np.float64)[None, :])  # sensor at t_a in the sensor frame at 0
    col = np.tile(np.arange(az_steps), beams)
    R, o = start_pose[:3, :3], start_pose[:3, 3]
    d = np.einsum("nij,nj->ni", dT[col, :3, :3], d_s) @ R.T
    o = dT[col, :3, 3] @ R.T + o
    t = np.full(len(d), np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = (-1.73 - o[:, 2]) / d[:, 2]  # ground plane z = -1.73
    t = np.where((tg > 0) & np.isfinite(tg), tg, t)
    for lo, hi in world:
        t = np.minimum(t, _ray_box(o, d, lo, hi))
    ok = np.isfinite(t) & (t < max_range) & (t > 1.0)
    r = t[ok] + noise_rng.normal(0.0, noise, size=int(ok.sum()))
    return (d_s[ok] * r[:, None]).astype(np.float32), t_col[col[ok]].astype(np.float32)


def voxel_downsample_values(pts, values, leaf):
    """voxel_downsample that also averages a per-point value channel (e.g. timestamps) over each voxel -> (points, values);
    the points are voxel_downsample(pts, leaf)'s."""
    values = np.asarray(values, dtype=np.float32)
    if leaf <= 0:
        return pts, values
    ijk = np.floor(pts / np.float32(leaf)).astype(np.int64)
    ijk -= ijk.min(axis=0)
    dims = ijk.max(axis=0) + 1
    idx = ijk[:, 0] + dims[0] * (ijk[:, 1] + dims[1] * ijk[:, 2])
    order = np.argsort(idx, kind="stable")
    idx_s = idx[order]
    starts = np.flatnonzero(np.r_[True, idx_s[1:] != idx_s[:-1]])
    sums = np.add.reduceat(pts[order].astype(np.float64), starts, axis=0)
    vsums = np.add.reduceat(values[order].astype(np.float64), starts)
    counts = np.diff(np.r_[starts, len(idx_s)])
    return (sums / counts[:, None]).astype(np.float32), (vsums / counts).astype(np.float32)


def thin_indices(pts, leaf, M):
    """Rows vgicp_thin_target keeps, ascending: row i is kept iff fewer than M earlier rows share its cell, with the header's
    cells c = floor(p * (1 / (float)leaf)) in float32 (one multiplication per axis)."""
    p = np.asarray(pts, dtype=np.float32).reshape(-1, 3)
    inv = np.float32(1.0) / np.float32(leaf)
    cells = np.floor(p * inv).astype(np.int64)
    _, group = np.unique(cells, axis=0, return_inverse=True)
    group = group.reshape(-1)
    order = np.argsort(group, kind="stable")  # rows of one cell contiguous, in array order
    g = group[order]
    starts = np.flatnonzero(np.r_[True, g[1:] != g[:-1]])
    rank = np.arange(len(g)) - np.repeat(starts, np.diff(np.r_[starts, len(g)]))  # earlier rows of the same cell
    return np.sort(order[rank < M])


def _carve_pixels(p, W, H, wq, e_lo, inv_de):
    """vgicp_carve_target's pixel and range of float32 sensor-frame points (n, 3) -> (has_pixel, row, col, r)."""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(all="ignore"):
        s = np.abs(x) + np.abs(y)
        q = np.abs(y) / s
        a = np.where(y >= 0, np.where(x >= 0, q, np.float32(2) - q), np.where(x < 0, np.float32(2) + q, np.float32(4) - q))
        xy = x * x + y * y
        u = (z / np.sqrt(xy) - e_lo) * inv_de
        ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & (s != 0) & (u >= 0) & (u < np.float32(H))
        col = np.where(ok, np.floor(a * wq), 0).astype(np.int64)
        row = np.where(ok, np.floor(u), 0).astype(np.int64)
        r = np.sqrt(xy + z * z)
    col[col == W] = 0
    return ok, row, col, r


def carve_indices(target, source, T, params):
    """Rows vgicp_carve_target keeps, ascending, with the header's float32 rule: the source (the scan in its sensor frame) fills a
    height x width image with its least range per pixel; target row i, taken into the sensor frame by Ti = [R^T | -R^T t] (formed
    in double, cast once), is removed iff it has a pixel, a non-empty pixel lies within `window` rows and columns of it, and its
    range r < r_min - (margin + margin_rel * r_min).  params: a dict with the keys of vgicp_carve_params (core.carve_params)."""
    import math

    W, H, w = int(params["width"]), int(params["height"]), int(params["window"])
    wq = np.float32(W) * np.float32(0.25)
    t_lo, t_hi = math.tan(params["elevation_min"]), math.tan(params["elevation_max"])
    e_lo, inv_de = np.float32(t_lo), np.float32(H / (t_hi - t_lo))
    margin, margin_rel = np.float32(params["margin"]), np.float32(params["margin_rel"])
    empty = np.uint32(0xFFFFFFFF)
    img = np.full(W * H, empty, dtype=np.uint32)
    ok, row, col, r = _carve_pixels(np.asarray(source, dtype=np.float32).reshape(-1, 3), W, H, wq, e_lo, inv_de)
    np.minimum.at(img, row[ok] * W + col[ok], r[ok].view(np.uint32))  # r >= 0: the bit order is the numeric order
    Tm = np.asarray(T, dtype=np.float64)
    Ti = np.empty((3, 4), dtype=np.float32)
    for j in range(3):
        for k in range(3):
            Ti[j, k] = Tm[k, j]
        Ti[j, 3] = -((float(Tm[0, j]) * float(Tm[0, 3]) + float(Tm[1, j]) * float(Tm[1, 3])) + float(Tm[2, j]) * float(Tm[2, 3]))
    m = np.asarray(target, dtype=np.float32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        s = np.stack([((Ti[j, 0] * m[:, 0] + Ti[j, 1] * m[:, 1]) + Ti[j, 2] * m[:, 2]) + Ti[j, 3] for j in range(3)], axis=1)
    ok, row, col, r = _carve_pixels(s, W, H, wq, e_lo, inv_de)
    best = np.full(len(m), empty, dtype=np.uint32)
    for dr in range(-w, w + 1):
        rr = row + dr
        inside = (rr >= 0) & (rr < H)
        for dc in range(-w, w + 1):
            v = img[np.clip(rr, 0, H - 1) * W + (col + dc) % W]
            best = np.minimum(best, np.where(inside, v, empty))
    r_min = best.view(np.float32)
    with np.errstate(all="ignore"):
        removed = ok & (best != empty) & (r < r_min - (margin + margin_rel * r_min))
    return np.flatnonzero(~removed)


def in_boxes(pts, boxes, pad=(0.3, 0.3, 0.1)):
    """Points (n, 3) inside any of the axis-aligned boxes [(lo, hi), ...] grown by pad per axis."""
    p = np.asarray(pts, dtype=np.float64)
    out = np.zeros(len(p), dtype=bool)
    for lo, hi in boxes:
        out |= np.all((p >= np.asarray(lo) - pad) & (p <= np.asarray(hi) + pad), axis=1)
    return out


def _path_point(s, step, turn_deg):
    """Point and heading at arc length s along the path of 0.8 m-style steps whose heading turns turn_deg per step."""
    k = int(s // step)
    xy = np.zeros(2)
    for i in range(k):
        yaw = np.radians(turn_deg * i)
        xy = xy + step * np.array([np.cos(yaw), np.sin(yaw)])
    yaw = np.radians(turn_deg * k)
    return xy + (s - k * step) * np.array([np.cos(yaw), np.sin(yaw)]), yaw


DEFAULT_MOVERS = ((3.5, 8.0, 2.0),)  # (lane offset to the left in m, start ahead in m, speed over the sensor's)


def moving_object_sequence(frames, seed, movers=DEFAULT_MOVERS, beams=64, az_steps=2083, downsample=0.25, step=0.8, turn_deg=2.0, size=(4.0, 2.0, 1.5)):
    """A drive past moving vehicles -> (poses, scans, boxes): the sensor moves `step` m per frame along an arc turning turn_deg
    per frame through _make_world(seed)'s world (scripts/bench_local_map.py's sequence: the same path and noise seeds); each mover
    is a size[0] x size[1] x size[2] m axis-aligned box 0.2 m above the ground that follows the same path, offset to the left and
    `ahead` m ahead at frame 0, at `speed` times the sensor's speed.  Static boxes that any mover's positions come within 1 m of
    are removed from the world, so that no vehicle drives through a building.  boxes[k]: the movers' (lo, hi) at frame k, in the
    world frame (in_boxes labels the points they produced).  scans[k] is in the sensor frame of poses[k]."""
    world = _make_world(np.random.default_rng(seed))
    boxes = []
    for k in range(frames):
        fb = []
        for lane, ahead, speed in movers:
            xy, yaw = _path_point(ahead + speed * step * k, step, turn_deg)
            c = xy + lane * np.array([-np.sin(yaw), np.cos(yaw)])
            lo = np.array([c[0] - size[0] / 2, c[1] - size[1] / 2, -1.53])
            fb.append((lo, lo + np.array([size[0], size[1], size[2]])))
        boxes.append(fb)
    every = [b for fb in boxes for b in fb]
    world = [(lo, hi) for lo, hi in world if not any(np.all(lo - 1.0 <= mhi) and np.all(mlo - 1.0 <= hi) for mlo, mhi in every)]
    poses, scans = [], []
    xy = np.zeros(2)
    for k in range(frames):
        yaw = np.radians(turn_deg * k)
        T = np.eye(4)
        T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
        T[:2, 3] = xy
        xy = xy + step * np.array([np.cos(yaw), np.sin(yaw)])
        poses.append(T)
        scans.append(voxel_downsample(scan(world + boxes[k], beams, az_steps, T, np.random.default_rng(seed * 1000 + k)), downsample))
    return poses, scans, boxes


def kitti_like_pair(beams=64, az_steps=2083, seed=42, pose=(0.8, 0.05, 0.7), downsample=0.25, max_points=None):
    """(target, source, T_gt): target scanned at the origin, source from a sensor moved by pose=(tx, ty, yaw_deg).
    T_gt maps source-frame points into the target frame (what registration should recover)."""
    rng = np.random.default_rng(seed)
    world = _make_world(rng)
    T = np.eye(4)
    yaw = np.radians(pose[2])
    T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
    T[:3, 3] = [pose[0], pose[1], 0.0]
    tgt = scan(world, beams, az_steps, np.eye(4), np.random.default_rng(seed))
    src = scan(world, beams, az_steps, T, np.random.default_rng(seed + 1))
    if max_points:
        tgt, src = tgt[:max_points], src[:max_points]
    return voxel_downsample(tgt, downsample), voxel_downsample(src, downsample), T
