"""Depth frames and constructed clouds for the neighbour-search tests of dnr_dn_normals (tests/test_gpu_normals_search.py
runs them on the device, tests/test_normals_search_cpu.py checks the oracle and the mirror on them).  Every case is
generated from a seed.  A frame case is (depth [h,w] f32, (fx, fy, cx, cy), c2w OpenCV, query pixels or None for every
distinct position); a cloud case is (points [N,3] f64, k, query rows or None)."""
from __future__ import annotations

import numpy as np

from oracle import normals_ref as R

K = 200
FULL_W, FULL_H = 1920, 1440


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return rz @ ry @ rx


def pose(ax=0.3, ay=-0.5, az=0.2, t=(3.7, -2.4, 5.1)):
    c2w = np.eye(4)
    c2w[:3, :3] = _rot(ax, ay, az)
    c2w[:3, 3] = t
    return c2w


def room_depth(w, h, hole_share, seed=0, foreground=True):
    """A 0.4-6 m room frame (a ramp of planes with a ripple), a box 0.8 m away in front of it (depth discontinuities) and
    hole_share of the pixels zeroed in blobs."""
    g = np.random.default_rng(seed)
    u, v = np.meshgrid(np.arange(w) / w, np.arange(h) / h)
    z = 0.4 + 5.6 * u ** 2 + 0.3 * np.sin(v * 6) + 0.05 * np.sin(u * 40) * v
    if foreground:
        z = np.where((abs(u - 0.3) < 0.12) & (abs(v - 0.6) < 0.15), 0.8 + 0.1 * v, z)
    holes = np.zeros((h, w), bool)
    r0 = max(2, min(w, h) // 60)
    while holes.mean() < hole_share:
        cx, cy, r = g.integers(0, w), g.integers(0, h), g.integers(r0, 8 * r0)
        holes |= ((u * w - cx) ** 2 + (v * h - cy) ** 2) < r * r
    return np.where(holes, 0, z).astype(np.float32)


def exact_holes(w, h, count, seed):
    d = room_depth(w, h, 0.0, seed)
    flat = d.reshape(-1)
    flat[np.random.default_rng(seed).choice(flat.size, count, replace=False)] = 0
    return d


def lattice_depth(w, h):
    """Dyadic depths constant on 64-pixel blocks: with fx = fy = 1024 and cx, cy on pixel corners the camera coordinates
    are exact, and so are the world points under an identity rotation and a dyadic translation."""
    u, v = np.meshgrid(np.arange(w) // 64, np.arange(h) // 64)
    return (1.0 + ((u + 2 * v) % 8) / 16.0).astype(np.float32)


def distant_depth(w, h, seed=0):
    """The room with five pixels 10^5 m away: the grid stretches, so the fine cells hold hundreds of points."""
    d = room_depth(w, h, 0.02, seed)
    g = np.random.default_rng(seed + 1)
    d[g.integers(0, h, 5), g.integers(0, w, 5)] = 1e5
    return d


def frames(full=True):
    """{name: (depth, intrinsics, c2w)}; full: the capture-resolution frames too."""
    out = {"room_256": (room_depth(256, 192, 0.05, 1), (180.0, 180.0, 128.0, 96.0), pose())}
    if not full:
        return out
    W, H = FULL_W, FULL_H
    intr = (1400.0, 1400.0, W / 2, H / 2)
    out["room_2pct"] = (room_depth(W, H, 0.02, 2), intr, pose())
    out["room_40pct"] = (room_depth(W, H, 0.40, 3), intr, pose(-0.7, 0.4, 1.1, (-6.5, 3.25, 1.75)))
    out["resized_5x"] = (_resized(1280, 960), (900.0, 900.0, 640.0, 480.0), pose(0.1, 0.2, -0.3, (2.0, 4.0, -3.0)))
    c2w = np.eye(4)
    c2w[:3, 3] = (3.5, -1.25, 2.0)
    out["lattice"] = (lattice_depth(W, H), (1024.0, 1024.0, W / 2, H / 2), c2w)
    for m in (K - 1, K, K + 1):
        out[f"holes_{m}"] = (exact_holes(W, H, m, 10 + m), intr, pose())
    out["distant"] = (distant_depth(W, H, 4), intr, pose(0.2, 0.1, 0.0, (1.0, 1.0, 1.0)))
    return out


def _resized(w, h):
    from dn_splatter_b200.depth_normals import resize_nearest

    return resize_nearest(room_depth(256, 192, 0.1, 5), w, h)


def frame_queries(depth, pts, n_random=6000, per_stratum=2000, seed=0):
    """Stratified query pixels of a frame: border rows and columns, pixels next to holes, depth discontinuities, the
    camera centre, the points nearest each bounding-box face and random pixels (about 12 k at 1920 x 1440)."""
    g = np.random.default_rng(seed)
    h, w = depth.shape
    idx = np.arange(h * w).reshape(h, w)
    pick = lambda a, m: g.choice(a, min(m, len(a)), replace=False) if len(a) else a  # noqa: E731
    border = np.r_[idx[0], idx[-1], idx[:, 0], idx[:, -1]]
    hole = depth == 0
    near = np.zeros_like(hole)
    near[1:] |= hole[:-1]
    near[:-1] |= hole[1:]
    near[:, 1:] |= hole[:, :-1]
    near[:, :-1] |= hole[:, 1:]
    dz = np.zeros(depth.shape, np.float32)
    dz[:, 1:] = np.maximum(dz[:, 1:], abs(np.diff(depth, axis=1)))
    dz[1:] = np.maximum(dz[1:], abs(np.diff(depth, axis=0)))
    disc = (dz > 0.1) & ~hole & ~near
    faces = np.concatenate([np.argsort(s * pts[:, a])[:100] for a in range(3) for s in (1, -1)])
    q = [pick(border, per_stratum), pick(idx[near & ~hole], per_stratum), pick(idx[disc], per_stratum), idx[hole][:1], faces,
         pick(np.arange(h * w), n_random)]
    return np.unique(np.concatenate(q).astype(np.int64))


def clouds():
    """{name: (points, k, queries or None)} of constructed search geometries."""
    g = np.random.default_rng(11)
    out = {}
    # Morton discontinuity: queries beside the x = 1/2 plane of a uniform cube, whose Morton neighbours lie far away
    cube = g.uniform(0, 1, (20000, 3))
    out["morton_discontinuity"] = (cube, 30, np.flatnonzero(abs(cube[:, 0] - 0.5) < 2e-3))
    # R above the extent: the level rule stops at 2^21 cells
    a = g.uniform(0, 0.01, (10, 3))
    b = 1 - g.uniform(0, 0.01, (500, 3))
    out["level_clamped"] = (np.r_[a, b], K, None)
    # the k-th position split among its copies
    base = g.uniform(0, 1, (600, 3))
    rep = g.integers(1, 7, 600)
    out["split"] = (np.repeat(base, rep, axis=0)[g.permutation(rep.sum())], 30, None)
    # distinct positions whose squared distances are subnormal or underflow to 0 (spacing 10^-163 .. 2 10^-161)
    sub = np.unique(g.integers(0, 200, (1500, 3)), axis=0) * 1e-163
    out["subnormal"] = (g.permutation(sub), 30, None)
    # -0.0 / +0.0: a plane through the origin with signed zeros, each position also present with the other sign
    pl = np.c_[g.integers(-20, 21, (800, 2)) * 0.05, np.zeros(800)]
    pl[g.random(800) < 0.5, 2] = -0.0
    pl[pl[:, 0] == 0, 0] = -0.0
    flip = pl[:200].copy()
    flip[:, 2] = np.where(np.signbit(flip[:, 2]), 0.0, -0.0)
    out["signed_zero"] = (np.r_[pl, flip], 30, None)
    # a narrow cloud 10^4 away from the origin
    out["offset_1e4"] = (np.c_[g.uniform(0, 1e-2, (3000, 2)), 1e-4 * g.normal(size=3000)] + 1e4, K, None)
    # a dyadic line on cell boundaries: q - R lands exactly on a cell face, which only the 2^-40 margin crosses
    out["margin"] = (np.c_[np.arange(1025) / 8.0, np.zeros((1025, 2))], 30, None)
    return out
