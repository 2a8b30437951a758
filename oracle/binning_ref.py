"""ORACLE (test infrastructure, NOT product code): the tile binning of csrc/binning.cu (dnr_bin_scan + dnr_bin_sort) as a
contract on (Gaussian, list) pairs, in numpy on the CPU; the reference of tests/test_gpu_binning.py.

The lists are kept per list tile of `ts` = 16 << list_shift pixels.  What the binning owes the rasterizer:

  * `list_box`: the lists a Gaussian may appear in, the float32 box of dnr_tile_box / list_box at edge `ts`;
  * `needed`: the pairs the raster can composite.  The raster composites a Gaussian only at pixel centres inside its
    16 px gsplat tile box (dnr_in_tile_box) and only where op * exp(-sigma) >= 1/255.  The reference asks that in fp64,
    from the float32 conic and opacity the kernels see, with a margin of 1e-4 for the raster's fp32 / ex2.approx
    evaluation (the binning itself keeps a margin of 0.1 sigma, DNR_CULL_MARGIN).  The exponent is concave, so its
    maximum over the rectangle of pixel centres (image x list x tile box) is at the centre when the centre lies inside
    and otherwise on an edge, where it is a 1-D parabola: `min_sigma` evaluates that in closed form.  That continuous
    rectangle contains every pixel centre, so `needed` is a superset of the discrete contract; `needed_discrete` checks
    a pair against the pixel centres themselves, and a pair the binning drops is a finding only when it fails there too;
  * `expected_lists`: with DNR_FLAG_EXACT_LISTS, every list of the box, each list ordered by (depth key as uint32,
    Gaussian index): gsplat's isect_tiles;
  * `truncated`: what a capacity below the count keeps.  emit_kernel writes the pairs in emission order (Gaussians by
    (depth key, index), each Gaussian's lists row-major, ascending in x) and drops those of rank >= cap; the stable sort
    by list id then keeps each list in emission order.

Nothing here evaluates the kernel's own float expressions except `list_box`, whose integers the contract is stated in.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
ALPHA_MIN = 1.0 / 255.0
RASTER_MARGIN = 1e-4  # relative, on the alpha threshold: the raster's fp32 power and ex2.approx
TILE = 16


def lists_xy(width: int, height: int, ts: int):
    return -(-width // ts), -(-height // ts)


def list_box(means2d, radii, ts: int, lists_x: int, lists_y: int):
    """(x0, y0, x1, y1) int64 [N]: lists [x0, x1) x [y0, y1) at edge `ts`, all zero where radius <= 0.  float32
    radius * (1/ts) and mean * (1/ts), floor / ceil, clamped to [0, lists]."""
    m = np.asarray(means2d, dtype=F32).reshape(-1, 2)
    rad = np.asarray(radii).reshape(-1)
    inv = F32(1.0 / ts)
    r = rad.astype(F32) * inv
    tcx, tcy = m[:, 0] * inv, m[:, 1] * inv
    with np.errstate(invalid="ignore"):
        x0 = np.clip(np.floor(tcx - r), 0, lists_x)
        y0 = np.clip(np.floor(tcy - r), 0, lists_y)
        x1 = np.clip(np.ceil(tcx + r), 0, lists_x)
        y1 = np.clip(np.ceil(tcy + r), 0, lists_y)
    vis = rad > 0
    return tuple(np.where(vis, v, 0).astype(np.int64) for v in (x0, y0, x1, y1))


def box_pairs(means2d, radii, ts: int, lists_x: int, lists_y: int):
    """Every (Gaussian, list) of the list boxes, Gaussian by Gaussian in index order, each box row-major ascending in
    x: (gid int64 [P], list id int64 [P])."""
    x0, y0, x1, y1 = list_box(means2d, radii, ts, lists_x, lists_y)
    nx, ny = x1 - x0, y1 - y0
    cnt = nx * ny
    gid = np.repeat(np.arange(cnt.size, dtype=np.int64), cnt)
    local = np.arange(gid.size, dtype=np.int64) - (np.cumsum(cnt) - cnt)[gid]
    w = np.maximum(nx[gid], 1)
    return gid, (y0[gid] + local // w) * lists_x + x0[gid] + local % w


def pair_rects(means2d, radii, gid, lid, ts: int, width: int, height: int):
    """Pixel index rectangles [px0, px1) x [py0, py1) of each pair: image x list x the Gaussian's 16 px tile box."""
    lx_n, ly_n = lists_xy(width, height, ts)
    tx_n, ty_n = lists_xy(width, height, TILE)
    tx0, ty0, tx1, ty1 = list_box(means2d, radii, TILE, tx_n, ty_n)
    lx, ly = lid % lx_n, lid // lx_n
    px0 = np.maximum(TILE * tx0[gid], ts * lx)
    px1 = np.minimum(np.minimum(TILE * tx1[gid], ts * lx + ts), width)
    py0 = np.maximum(TILE * ty0[gid], ts * ly)
    py1 = np.minimum(np.minimum(TILE * ty1[gid], ts * ly + ts), height)
    return px0, px1, py0, py1


def _sigma(A, B, C, dx, dy):
    return 0.5 * (A * dx * dx + C * dy * dy) + B * dx * dy


def min_sigma(means2d, conics, gid, rects):
    """fp64 minimum of sigma over the continuous rectangle of pixel centres of each pair (+inf where it is empty)."""
    m = np.asarray(means2d, dtype=F32).astype(np.float64).reshape(-1, 2)[gid]
    con = np.asarray(conics, dtype=F32).astype(np.float64).reshape(-1, 3)[gid]
    A, B, C = con[:, 0], con[:, 1], con[:, 2]
    if not bool(((A > 0) & (C > 0) & (A * C - B * B > 0)).all()):
        raise ValueError("min_sigma: a conic is not positive definite")
    px0, px1, py0, py1 = rects
    empty = (px1 <= px0) | (py1 <= py0)
    d0, d1 = px0 + 0.5 - m[:, 0], px1 - 0.5 - m[:, 0]  # dx = pixel centre - mean over the rectangle
    e0, e1 = py0 + 0.5 - m[:, 1], py1 - 0.5 - m[:, 1]
    with np.errstate(invalid="ignore"):
        best = np.full(gid.size, np.inf)
        for d in (d0, d1):  # vertical edges: the parabola in dy has its minimum at -B dx / C
            e = np.clip(-B * d / C, e0, e1)
            best = np.minimum(best, _sigma(A, B, C, d, e))
        for e in (e0, e1):
            d = np.clip(-B * e / A, d0, d1)
            best = np.minimum(best, _sigma(A, B, C, d, e))
    inside = (d0 <= 0) & (d1 >= 0) & (e0 <= 0) & (e1 >= 0)
    best = np.where(inside, 0.0, best)
    return np.where(empty, np.inf, best)


def reaches(opac, sigma):
    """op * exp(-sigma) >= (1/255) (1 - 1e-4), in fp64."""
    return np.asarray(opac, dtype=np.float64) * np.exp(-sigma) >= ALPHA_MIN * (1.0 - RASTER_MARGIN)


def needed(means2d, conics, opac, radii, ts: int, width: int, height: int):
    """(gid, list id) of the pairs the raster can composite (continuous form), in box_pairs order."""
    lx_n, ly_n = lists_xy(width, height, ts)
    gid, lid = box_pairs(means2d, radii, ts, lx_n, ly_n)
    if gid.size == 0:
        return gid, lid
    rects = pair_rects(means2d, radii, gid, lid, ts, width, height)
    op = np.asarray(opac, dtype=F32).astype(np.float64).reshape(-1)[gid]
    keep = reaches(op, min_sigma(means2d, conics, gid, rects))
    return gid[keep], lid[keep]


def needed_discrete(means2d, conics, opac, radii, gid, lid, ts: int, width: int, height: int):
    """bool [P]: some pixel centre of the pair's rectangle passes the alpha test (brute force, for a few pairs)."""
    rects = pair_rects(means2d, radii, gid, lid, ts, width, height)
    m = np.asarray(means2d, dtype=F32).astype(np.float64).reshape(-1, 2)
    con = np.asarray(conics, dtype=F32).astype(np.float64).reshape(-1, 3)
    op = np.asarray(opac, dtype=F32).astype(np.float64).reshape(-1)
    out = np.zeros(gid.size, dtype=bool)
    for k, g in enumerate(gid):
        px0, px1, py0, py1 = (int(r[k]) for r in rects)
        if px1 <= px0 or py1 <= py0:
            continue
        dx = np.arange(px0, px1, dtype=np.float64) + 0.5 - m[g, 0]
        dy = np.arange(py0, py1, dtype=np.float64) + 0.5 - m[g, 1]
        s = _sigma(con[g, 0], con[g, 1], con[g, 2], dx[None, :], dy[:, None])
        out[k] = bool(reaches(op[g], s.min()))
    return out


def _lists(gid, lid, depth_keys, n_lists):
    k = np.asarray(depth_keys).reshape(-1).view(np.uint32)
    order = np.lexsort((gid, k[gid], lid))
    counts = np.bincount(lid, minlength=n_lists)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return gid[order].astype(np.int32), offsets


def expected_lists(means2d, radii, depth_keys, ts: int, width: int, height: int):
    """The exact route: (flatten_ids int32 [I], offsets int64 [n_lists + 1]), every list of every box, each list
    ordered by (depth key as uint32, Gaussian index); Gaussians with radius 0 are left out."""
    lx_n, ly_n = lists_xy(width, height, ts)
    gid, lid = box_pairs(means2d, radii, ts, lx_n, ly_n)
    return _lists(gid, lid, depth_keys, lx_n * ly_n)


def pairs_of(flatten_ids, offsets):
    """(gid, list id) int64 of a list layout."""
    offsets = np.asarray(offsets, dtype=np.int64)
    lid = np.repeat(np.arange(offsets.size - 1, dtype=np.int64), np.diff(offsets))
    return np.asarray(flatten_ids, dtype=np.int64)[: lid.size], lid


def emission_rank(gid, lid, depth_keys):
    """int64 [P]: the position of each pair in emit_kernel's write order."""
    k = np.asarray(depth_keys).reshape(-1).view(np.uint32)
    order = np.lexsort((lid, gid, k[gid]))
    rank = np.empty(gid.size, dtype=np.int64)
    rank[order] = np.arange(gid.size, dtype=np.int64)
    return rank


def truncated(flatten_ids, offsets, depth_keys, cap: int):
    """The capacity rule on a complete list layout: the pairs of emission rank < cap, each list in its own order."""
    gid, lid = pairs_of(flatten_ids, offsets)
    keep = emission_rank(gid, lid, depth_keys) < cap
    return _lists(gid[keep], lid[keep], depth_keys, np.asarray(offsets).size - 1)
