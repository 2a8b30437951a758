"""fp64 numpy restatement of the reference's scripts/depth_normal_consistency.py (DepthNormalConsistency) and
scripts/depth_to_normal.py (DepthToNormal), and of the Open3D call they make.

Quirks kept (each pinned by tests/golden/dn_depth_normals.npz):
- depth files: a PNG read as 16 bit and a .npy (channel 0 of a 3-D array) are both multiplied by 0.001, then cast to f32;
- the camera coordinates (u + 0.5 - cx) * d / fx are formed in f32 (numpy's weak Python scalars), then `@ inv(R) + t` in
  f64, so every depth-0 pixel lands exactly on the camera centre and joins the cloud;
- a normal is negated where (p - t) . n > 0;
- DepthNormalConsistency decodes the mono normal as 2 m - 1 (dsine: then diag(1, -1, -1)), tests degrees > angle_treshold
  and names its outputs with png -> jpg; DepthToNormal decodes (m - 0.5) * 2, takes the angle between the *encoded*
  vectors (n + 1) / 2 and m * 0.5 + 0.5, tests > 10 and keeps the frame's own file name.

Open3D's PointCloud.estimate_normals(KDTreeSearchParamKNN(k)) with fast_normal_computation=True [EXT, restated from
Open3D's EstimateNormals.cpp, not installed here]: the min(k, N) nearest points of each point, itself included; fewer than
3 -> identity covariance; else E[x x^T] - E[x] E[x]^T from fp64 cumulants summed in neighbour order and divided by the
count; FastEigen3x3 (Geometric Tools' robust symmetric solver); a zero vector becomes (0, 0, 1).  nanoflann's order among
equidistant points cannot be reproduced; this project's tie rule: distinct positions in (squared distance, smallest point
index) order, all copies of a position before the next.  Squared distances are ((dx dx + dy dy) + dz dz) with
d = p - q, as the kernel computes them.
"""
from __future__ import annotations

import math

import numpy as np

SCALE_FACTOR = 0.001
OPENGL_TO_OPENCV = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])


def backproject(depth: np.ndarray, fx, fy, cx, cy, w: int, h: int, c2w: np.ndarray):
    """(world points [h*w,3] f64, camera coordinates [h*w,3] f32) exactly as the scripts' backproject forms them."""
    coords = np.stack(np.meshgrid(np.arange(w), np.arange(h), indexing="xy"), axis=-1) + 0.5
    coords = coords.reshape(-1, 2).astype(np.float32)
    d = depth.reshape(-1, 1)
    cam = np.zeros([w, h, 3], dtype=np.float32).reshape(-1, 3)
    cam[:, 0] = (coords[:, 0] - cx) * d[:, 0] / fx
    cam[:, 1] = (coords[:, 1] - cy) * d[:, 0] / fy
    cam[:, 2] = d[:, 0]
    return cam @ np.linalg.inv(c2w[..., :3, :3]) + c2w[..., :3, 3], cam


def unique_positions(points: np.ndarray):
    """(positions [U,3], smallest index [U], multiplicity [U], position of each point [N]); -0.0 equals +0.0."""
    p = np.asarray(points, np.float64) + 0.0
    uniq, first, inv, counts = np.unique(p, axis=0, return_index=True, return_inverse=True, return_counts=True)
    return uniq, first, counts, inv.reshape(-1)


def sq_dist(q: np.ndarray, pts: np.ndarray) -> np.ndarray:
    d = pts - q
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn(points: np.ndarray, k: int, queries=None):
    """Per query point (default: every point), the neighbour positions' smallest indices, one entry per copy taken, in
    the tie rule's order: a list of int arrays of length min(k, N)."""
    uniq, first, counts, inv = unique_positions(points)
    n = len(points)
    kk = min(k, n)
    qs = range(n) if queries is None else queries
    cache, out = {}, []
    for i in qs:
        u = inv[i]
        if u not in cache:
            d2 = sq_dist(uniq[u], uniq)
            order = np.lexsort((first, d2))
            cache[u] = _cut(first[order], counts[order], kk)
        out.append(cache[u])
    return out


def _cut(order_first, order_counts, kk, split=True):
    """The neighbour list of positions already in key order: copies until kk, the last position's split."""
    c = np.cumsum(order_counts)
    last = int(np.searchsorted(c, kk))
    take = order_counts[: last + 1].copy()
    if split:
        take[-1] -= c[last] - kk
    return np.repeat(order_first[: last + 1], take)


def knn_fast(points: np.ndarray, k: int, queries):
    """knn(points, k, queries) under the same tie rule, fast at millions of points: the min(kk, U) nearest positions of a
    cKDTree give the kk-th squared distance; a ball query at a slightly inflated radius (the tree rounds its own
    distances) closes the set, whose d2 are recomputed exactly, ordered by (d2, smallest index) and cut at kk."""
    from scipy.spatial import cKDTree

    uniq, first, counts, inv = unique_positions(points)
    kk = min(k, len(points))
    qu = inv[np.asarray(queries, np.int64)]
    us, back = np.unique(qu, return_inverse=True)
    tree = cKDTree(uniq)
    m = min(kk, len(uniq))
    _, idx = tree.query(uniq[us], k=m, workers=-1)
    idx = idx.reshape(len(us), m)
    d2 = sq_dist(uniq[us][:, None, :], uniq[idx])
    o = np.lexsort((first[idx], d2), axis=-1)
    d2s = np.take_along_axis(d2, o, 1)
    cum = np.cumsum(np.take_along_axis(counts[idx], o, 1), axis=1)
    kth = d2s[np.arange(len(us)), np.argmax(cum >= kk, axis=1)]
    balls = tree.query_ball_point(uniq[us], np.sqrt(kth) * (1 + 2.0 ** -20) + 2.0 ** -500, workers=-1)
    res = []
    for i, b in enumerate(balls):
        b = np.asarray(b, np.int64)
        e = sq_dist(uniq[us[i]], uniq[b])
        oo = np.lexsort((first[b], e))
        assert counts[b].sum() >= kk
        res.append(_cut(first[b][oo], counts[b][oo], kk))
    return [res[j] for j in back]


# ---- numpy restatement of dnr_dn_normals' search geometry (csrc/normals.cu) ----
MORTON_BITS = 21
CAP = 768  # candidate buffer entries per warp; the kernel compacts before a 32-entry push batch when more than CAP - 32
R_MARGIN = 1.0 + 2.0 ** -40
R_FLOOR = 2.0 ** -510  # a k-th d2 that underflowed below 2^-1022 says only that the true distance is below 2^-511

# Plausible kernel mistakes; search_mirror(..., slip=...) restates each (tests/test_normals_search_cpu.py shows every one
# changes some query's neighbour multiset or examined count on the GPU test's cases).
SEARCH_SLIPS = {
    "no_margin": "R is the rounded k-th distance, without the 2^-40 relative margin",
    "no_floor": "R is not floored, so a k-th d2 that underflowed to 0 or a subnormal gives a box of one cell",
    "cell_unclamped": "cell_of clamps at 0 (the u32 conversion saturates) but not at 2^21 - 1",
    "unweighted": "the selects count positions instead of points (multiplicities ignored)",
    "largest_index": "among equal squared distances the largest smallest-index wins",
    "no_split": "the k-th position contributes all its copies (rem ignored)",
    "window_twice": "window entries are pushed again when a cell range covers them",
}


def grid_of(points: np.ndarray):
    """(lo [3], cell) as estimate_normals sets them: the bounding box's low corner and its largest extent / 2^21."""
    p = np.asarray(points, np.float64)
    lo, hi = p.min(0), p.max(0)
    extent = float((hi - lo).max())
    return lo, (extent / (1 << MORTON_BITS) if extent > 0 else 1.0)


def _spread3(v):
    x = v.astype(np.uint64) & np.uint64(0x1FFFFF)
    for s, m in ((32, 0x1F00000000FFFF), (16, 0x1F0000FF0000FF), (8, 0x100F00F00F00F00F), (4, 0x10C30C30C30C30C3),
                 (2, 0x1249249249249249)):
        x = (x | (x << np.uint64(s))) & np.uint64(m)
    return x


def morton(cx, cy, cz):
    return _spread3(cx) | (_spread3(cy) << np.uint64(1)) | (_spread3(cz) << np.uint64(2))


def _floor_cell(x, lo, inv):
    return np.floor((x - lo) * inv)


def cell_of(x, lo, inv, clamp=True):
    c = np.maximum(_floor_cell(x, lo, inv), 0.0)
    if clamp:
        c = np.minimum(c, float((1 << MORTON_BITS) - 1))
    return c.astype(np.uint64)


def search_order(points: np.ndarray, lo, cell, slip=None):
    """The kernel's distinct positions in its order (Morton key, then x / y / z bits, then index, all stable):
    (upts [U,3], ukey [U] u64, umin [U], count [U], position of each point [N])."""
    p = np.asarray(points, np.float64) + 0.0
    inv = 1.0 / cell
    cl = slip != "cell_unclamped"
    key = morton(*(cell_of(p[:, a], lo[a], inv, cl) for a in range(3)))
    bits = p.view(np.uint64)
    order = np.lexsort((bits[:, 2], bits[:, 1], bits[:, 0], key))
    ps = p[order]
    head = np.r_[True, (ps[1:] != ps[:-1]).any(1)]
    ustart = np.flatnonzero(head)
    count = np.diff(np.r_[ustart, len(p)])
    pos = np.empty(len(p), np.int64)
    pos[order] = np.cumsum(head) - 1
    return ps[ustart], key[order[ustart]], order[ustart], count, pos


def _le(d2, tie, td2, ttie):
    return (d2 < td2) | ((d2 == td2) & (tie <= ttie))


def _kth(d2, tie, w, kk):
    """(d2, tie) of the kk-th point by weight in (d2, tie) order, over one row (1-D arrays)."""
    o = np.lexsort((tie, d2))
    i = int(np.argmax(np.cumsum(w[o]) >= kk))
    return d2[o[i]], tie[o[i]]


def search_mirror(points: np.ndarray, k: int, queries, lo=None, cell=None, slip=None, chunk_entries=1 << 23):
    """The search of dnr_dn_normals restated per query point.  Returns a dict of per-query arrays:
    nbrs (the neighbour multiset's smallest indices, in (d2, index) order), examined (the window's size plus the sizes of
    every scanned cell range, as the kernel counts them), shortcut (multiplicity >= kk), everything (the window is every
    position), level (-1 without a grid search), level_clamped (the level rule reached 21: R above the extent, one cell),
    box_clamped (the
    box [q - R, q + R] left the grid on some axis), compactions (mid-scan buffer compactions: the kernel's pushes
    simulated in their 32-entry batches)."""
    assert slip is None or slip in SEARCH_SLIPS, slip
    pts = np.asarray(points, np.float64)
    n = len(pts)
    if lo is None:
        lo, cell = grid_of(pts)
    lo = np.asarray(lo, np.float64)
    inv = 1.0 / cell
    kk = min(k, n)
    upts, ukey, umin, count, pos = search_order(pts, lo, cell, slip)
    U = len(upts)
    tie_of = (lambda f: -f.astype(np.int64)) if slip == "largest_index" else (lambda f: f.astype(np.int64))
    utie = tie_of(umin)
    wsel = np.ones(U, np.int64) if slip == "unweighted" else count.astype(np.int64)
    qu_all = pos[np.asarray(queries, np.int64)]
    us, back = np.unique(qu_all, return_inverse=True)
    nq = len(us)
    out = dict(examined=np.zeros(nq, np.int64), R=np.zeros(nq), split=np.zeros(nq, bool), shortcut=count[us] >= kk,
               everything=np.zeros(nq, bool),
               level=np.full(nq, -1), level_clamped=np.zeros(nq, bool), box_clamped=np.zeros(nq, bool),
               compactions=np.zeros(nq, np.int64))
    nbrs = [None] * nq
    # R: the search radius of a grid search; split: the kk-th point is one of several copies of its position

    def finish(i, d2, tie, w_cut, ucand):
        o = np.lexsort((tie, d2))
        f = umin[ucand[o]]
        if slip == "unweighted":  # the kk-th position by count; every copy of the earlier ones, rem = 1 for the last
            m = min(kk, len(o))
            nbrs[i] = np.r_[np.repeat(f[: m - 1], count[ucand[o[: m - 1]]]), f[m - 1: m]][:k] if m else f[:0]
        else:
            nbrs[i] = _cut(f, w_cut[o], kk, split=slip != "no_split")
        out["split"][i] = np.searchsorted(np.cumsum(w_cut[o]), kk) < len(o) and np.cumsum(w_cut[o])[
            np.searchsorted(np.cumsum(w_cut[o]), kk)] > kk

    for i in np.flatnonzero(out["shortcut"]):
        nbrs[i] = _cut(umin[us[i]: us[i] + 1], count[us[i]: us[i] + 1], kk, split=slip != "no_split")
        out["split"][i] = count[us[i]] > kk
    rest = np.flatnonzero(~out["shortcut"])
    win = np.arange(-kk, kk + 1)
    # queries in chunks bounded by the window entries (cell ranges are split further below)
    step = max(1, chunk_entries // (8 * (2 * kk + 1)))
    for c0 in range(0, len(rest), step):
        rows = rest[c0: c0 + step]
        u = us[rows]
        wlo, whi = np.maximum(u - kk, 0), np.minimum(u + kk + 1, U)
        j = u[:, None] + win[None, :]
        ok = (j >= wlo[:, None]) & (j < whi[:, None])
        jc = np.clip(j, 0, U - 1)
        q = upts[u]
        wd2 = np.where(ok, sq_dist(q[:, None, :], upts[jc]), np.inf)
        wtie = np.where(ok, utie[jc], np.iinfo(np.int64).max)
        ww = np.where(ok, wsel[jc], 0)
        out["examined"][rows] = whi - wlo
        every = (wlo == 0) & (whi == U)
        out["everything"][rows] = every
        o = np.lexsort((wtie, wd2), axis=-1)
        cum = np.cumsum(np.take_along_axis(ww, o, 1), axis=1)
        at = np.take_along_axis(o, np.argmax(cum >= kk, axis=1)[:, None], 1)[:, 0]
        td2 = wd2[np.arange(len(rows)), at]
        ttie = wtie[np.arange(len(rows)), at]
        R = np.sqrt(td2) * (1.0 if slip == "no_margin" else R_MARGIN)
        if slip != "no_floor":
            R = np.maximum(R, R_FLOOR)
        level = np.zeros(len(rows), np.int64)
        for l in range(MORTON_BITS):
            level += cell * float(1 << l) * 2 < R
        lclamp = level == MORTON_BITS
        cl = slip != "cell_unclamped"
        c_lo = np.stack([cell_of(q[:, a] - R, lo[a], inv, cl) for a in range(3)], 1) >> level[:, None].astype(np.uint64)
        c_hi = np.stack([cell_of(q[:, a] + R, lo[a], inv, cl) for a in range(3)], 1) >> level[:, None].astype(np.uint64)
        top = float((1 << MORTON_BITS) - 1)
        bclamp = ((_floor_cell(q - R[:, None], lo, inv) < 0) | (_floor_cell(q + R[:, None], lo, inv) > top)).any(1)
        nxyz = (c_hi.astype(np.int64) - c_lo.astype(np.int64) + 1)
        ncell = np.where(every, 0, nxyz.prod(1))
        grid = ~every
        out["level"][rows[grid]] = level[grid]
        out["R"][rows[grid]] = R[grid]
        out["level_clamped"][rows] = lclamp & grid
        out["box_clamped"][rows] = bclamp & grid
        mc = int(ncell.max()) if len(ncell) else 0
        cidx = np.arange(mc)[None, :]
        cvalid = cidx < ncell[:, None]
        nx, ny = nxyz[:, :1], nxyz[:, 1:2]
        cx = c_lo[:, :1].astype(np.int64) + cidx % nx
        cy = c_lo[:, 1:2].astype(np.int64) + (cidx // nx) % ny
        cz = c_lo[:, 2:3].astype(np.int64) + cidx // (nx * ny)
        sh = level[:, None].astype(np.uint64)
        k0 = morton(np.where(cvalid, cx, 0).astype(np.uint64) << sh, np.where(cvalid, cy, 0).astype(np.uint64) << sh,
                    np.where(cvalid, cz, 0).astype(np.uint64) << sh)
        s = np.searchsorted(ukey, k0, "left")
        e = np.searchsorted(ukey, k0 + (np.uint64(1) << (np.uint64(3) * sh)), "left")
        ln = np.where(cvalid, e - s, 0)
        out["examined"][rows] += ln.sum(1)
        # candidates, query by query in sub-chunks bounded by their entries
        tot = ln.sum(1)
        r0 = 0
        while r0 < len(rows):
            r1 = r0 + max(1, int(np.searchsorted(np.cumsum(tot[r0:]), chunk_entries, "right")))
            sl = slice(r0, r1)
            L = ln[sl].reshape(-1)
            starts = s[sl].reshape(-1)
            cid = np.repeat(np.arange(L.size), L)
            off = np.arange(L.sum()) - np.repeat(np.cumsum(L) - L, L)
            jj = starts[cid] + off
            qi = cid // mc
            inwin = (jj >= wlo[sl][qi]) & (jj < whi[sl][qi])
            d2 = sq_dist(q[sl][qi], upts[jj])
            keep = _le(d2, utie[jj], td2[sl][qi], ttie[sl][qi]) & ((~inwin) | (slip == "window_twice"))
            qs = np.searchsorted(qi, np.arange(r1 - r0 + 1))  # the entries of each query are contiguous
            # mid-scan compactions, where the pushes could overflow the buffer
            wkeep = _le(wd2[sl], wtie[sl], td2[sl, None], ttie[sl, None]) & ok[sl]
            bound = wkeep.sum(1) + np.bincount(qi[keep], minlength=r1 - r0)
            for b in np.flatnonzero((bound > CAP - 32) & grid[sl]):
                m = slice(qs[b], qs[b + 1])
                bb = np.cumsum(np.r_[0, -(-L[b * mc: (b + 1) * mc] // 32)])  # first batch ordinal of each cell
                batch = bb[cid[m] - b * mc] + off[m] // 32
                out["compactions"][rows[r0 + b]] = _compactions(
                    wd2[r0 + b][wkeep[b]], wtie[r0 + b][wkeep[b]], ww[r0 + b][wkeep[b]], d2[m], utie[jj[m]], wsel[jj[m]],
                    batch, keep[m], int(bb[-1]), td2[r0 + b], ttie[r0 + b], kk)
            for b in range(r1 - r0):
                m = slice(qs[b], qs[b + 1])
                km = keep[m]
                wm = ok[r0 + b]
                ucand = np.r_[j[r0 + b][wm], jj[m][km]]
                finish(rows[r0 + b], np.r_[wd2[r0 + b][wm], d2[m][km]], np.r_[wtie[r0 + b][wm], utie[jj[m][km]]],
                       count[ucand].astype(np.int64), ucand)
            r0 = r1
    out = {key: v[back] for key, v in out.items()}
    out["nbrs"] = [nbrs[b] for b in back]
    return out


def _compactions(bd2, btie, bw, d2, tie, w, batch, pushable, nbatch, td2, ttie, kk):
    """How many times the kernel's buffer is cut back mid-scan: before each 32-entry batch (nbatch of them) it compacts
    when it holds more than CAP - 32 entries; a batch pushes its entries whose key is <= the running k-th key."""
    cnt, comps, b0 = len(bd2), 0, 0
    buf = [bd2, btie, bw]
    d2, tie, w, batch = d2[pushable], tie[pushable], w[pushable], batch[pushable]
    while True:
        live = (batch >= b0) & _le(d2, tie, td2, ttie)
        per = np.bincount(batch[live] - b0, minlength=nbatch - b0)
        before = cnt + np.r_[0, np.cumsum(per)[:-1]]
        over = np.flatnonzero(before > CAP - 32)
        if not len(over):
            return comps
        b = b0 + int(over[0])
        took = live & (batch < b)
        buf = [np.r_[buf[0], d2[took]], np.r_[buf[1], tie[took]], np.r_[buf[2], w[took]]]
        td2, ttie = _kth(buf[0], buf[1], buf[2], kk)
        kept = _le(buf[0], buf[1], td2, ttie)
        buf = [a[kept] for a in buf]
        cnt, comps, b0 = len(buf[0]), comps + 1, b


def covariance(points: np.ndarray, nbr: np.ndarray) -> np.ndarray:
    """Open3D's ComputeCovariance over points[nbr] in order (sequential fp64 cumulants)."""
    if len(nbr) < 3:
        return np.eye(3)
    p = np.asarray(points, np.float64)[nbr]
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    cum = np.array([np.cumsum(v)[-1] for v in (x, y, z, x * x, x * y, x * z, y * y, y * z, z * z)]) / float(len(nbr))
    c = np.empty((3, 3))
    c[0, 0] = cum[3] - cum[0] * cum[0]
    c[1, 1] = cum[6] - cum[1] * cum[1]
    c[2, 2] = cum[8] - cum[2] * cum[2]
    c[0, 1] = c[1, 0] = cum[4] - cum[0] * cum[1]
    c[0, 2] = c[2, 0] = cum[5] - cum[0] * cum[2]
    c[1, 2] = c[2, 1] = cum[7] - cum[1] * cum[2]
    return c


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _eigvec0(A, e):
    r0 = (A[0][0] - e, A[0][1], A[0][2])
    r1 = (A[0][1], A[1][1] - e, A[1][2])
    r2 = (A[0][2], A[1][2], A[2][2] - e)
    c = [_cross(r0, r1), _cross(r0, r2), _cross(r1, r2)]
    d = [_dot(v, v) for v in c]
    imax, dmax = 0, d[0]
    if d[1] > dmax:
        imax, dmax = 1, d[1]
    if d[2] > dmax:
        imax = 2
    s = math.sqrt(d[imax])
    return tuple(v / s for v in c[imax])


def _eigvec1(A, e0, e1):
    if abs(e0[0]) > abs(e0[1]):
        il = 1 / math.sqrt(e0[0] * e0[0] + e0[2] * e0[2])
        U = (-e0[2] * il, 0.0, e0[0] * il)
    else:
        il = 1 / math.sqrt(e0[1] * e0[1] + e0[2] * e0[2])
        U = (0.0, e0[2] * il, -e0[1] * il)
    V = _cross(e0, U)
    AU = tuple(A[r][0] * U[0] + A[r][1] * U[1] + A[r][2] * U[2] for r in range(3))
    AV = tuple(A[r][0] * V[0] + A[r][1] * V[1] + A[r][2] * V[2] for r in range(3))
    m00 = U[0] * AU[0] + U[1] * AU[1] + U[2] * AU[2] - e1
    m01 = U[0] * AV[0] + U[1] * AV[1] + U[2] * AV[2]
    m11 = V[0] * AV[0] + V[1] * AV[1] + V[2] * AV[2] - e1
    a00, a01, a11 = abs(m00), abs(m01), abs(m11)
    if a00 >= a11:
        if max(a00, a01) > 0:
            if a00 >= a01:
                m01 /= m00
                m00 = 1 / math.sqrt(1 + m01 * m01)
                m01 *= m00
            else:
                m00 /= m01
                m01 = 1 / math.sqrt(1 + m00 * m00)
                m00 *= m01
            return tuple(m01 * U[i] - m00 * V[i] for i in range(3))
        return U
    if max(a11, a01) > 0:
        if a11 >= a01:
            m01 /= m11
            m11 = 1 / math.sqrt(1 + m01 * m01)
            m01 *= m11
        else:
            m11 /= m01
            m01 = 1 / math.sqrt(1 + m11 * m11)
            m11 *= m01
        return tuple(m11 * U[i] - m01 * V[i] for i in range(3))
    return U


def fast_eigen3x3(cov: np.ndarray, branch: list | None = None) -> np.ndarray:
    """Open3D's FastEigen3x3: the unit eigenvector of the smallest eigenvalue of a symmetric 3x3 (zero for a zero matrix).
    `branch`, if given, receives the name of the path taken."""
    C = [[float(cov[r][c]) for c in range(3)] for r in range(3)]
    mx = max(C[0][0], C[0][1], C[0][2], C[1][1], C[1][2], C[2][2])
    note = branch.append if branch is not None else (lambda _: None)
    if mx == 0:
        note("zero")
        return np.zeros(3)
    A = [[v / mx for v in row] for row in C]
    norm = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2]
    if norm > 0:
        q = (A[0][0] + A[1][1] + A[2][2]) / 3
        b00, b11, b22 = A[0][0] - q, A[1][1] - q, A[2][2] - q
        p = math.sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6)
        c00 = b11 * b22 - A[1][2] * A[1][2]
        c01 = A[0][1] * b22 - A[1][2] * A[0][2]
        c02 = A[0][1] * A[1][2] - b11 * A[0][2]
        det = (b00 * c00 - A[0][1] * c01 + A[0][2] * c02) / (p * p * p)
        half_det = min(max(det * 0.5, -1.0), 1.0)
        angle = math.acos(half_det) / 3.0
        beta2 = math.cos(angle) * 2
        beta0 = math.cos(angle + 2.09439510239319549) * 2
        beta1 = -(beta0 + beta2)
        ev = (q + p * beta0, q + p * beta1, q + p * beta2)
        if half_det >= 0:
            v2 = _eigvec0(A, ev[2])
            if ev[2] < ev[0] and ev[2] < ev[1]:
                note("pos/2")
                return np.array(v2)
            v1 = _eigvec1(A, v2, ev[1])
            if ev[1] < ev[0] and ev[1] < ev[2]:
                note("pos/1")
                return np.array(v1)
            note("pos/0")
            return np.array(_cross(v1, v2))
        v0 = _eigvec0(A, ev[0])
        if ev[0] < ev[1] and ev[0] < ev[2]:
            note("neg/0")
            return np.array(v0)
        v1 = _eigvec1(A, v0, ev[1])
        if ev[1] < ev[0] and ev[1] < ev[2]:
            note("neg/1")
            return np.array(v1)
        note("neg/2")
        return np.array(_cross(v0, v1))
    note("diagonal")
    if C[0][0] < C[1][1] and C[0][0] < C[2][2]:
        return np.array([1.0, 0.0, 0.0])
    if C[1][1] < C[0][0] and C[1][1] < C[2][2]:
        return np.array([0.0, 1.0, 0.0])
    return np.array([0.0, 0.0, 1.0])


def estimate_normals(points: np.ndarray, k: int = 200, nbrs=None):
    """(normals [N,3], covariances [N,3,3]) as Open3D's estimate_normals(KDTreeSearchParamKNN(k)) under the tie rule.
    nbrs: precomputed knn(points, k)."""
    pts = np.asarray(points, np.float64)
    nbrs = knn(pts, k) if nbrs is None else nbrs
    normals = np.empty((len(pts), 3))
    covs = np.empty((len(pts), 3, 3))
    done = {}
    for i, nb in enumerate(nbrs):
        key = (pts[i] + 0.0).tobytes()
        if key not in done:
            c = covariance(pts, nb)
            n = fast_eigen3x3(c)
            if np.linalg.norm(n) == 0.0:
                n = np.array([0.0, 0.0, 1.0])
            done[key] = (n, c)
        normals[i], covs[i] = done[key]
    return normals, covs


def orient(points: np.ndarray, normals: np.ndarray, center: np.ndarray) -> np.ndarray:
    n = normals.copy()
    flip = ((points - center.reshape(1, 3)) * n).sum(axis=-1) > 0
    n[flip] = -n[flip]
    return n


def angle_between(n1: np.ndarray, n2: np.ndarray) -> np.ndarray:
    """compute_angle_between_normals of the scripts ([..., 3] each)."""
    a = n1 / np.linalg.norm(n1, axis=-1, keepdims=True)
    b = n2 / np.linalg.norm(n2, axis=-1, keepdims=True)
    return np.degrees(np.arccos(np.clip(np.sum(a * b, axis=-1), -1.0, 1.0)))


def mono_rotation(c2w: np.ndarray) -> np.ndarray:
    return np.transpose(np.linalg.inv(c2w)[:3, :3])


def consistency(normals: np.ndarray, mono_u8: np.ndarray, c2w: np.ndarray, mode: str, threshold: float):
    """(degrees [N], mask [N] bool, normals image [N,3] u8) of one frame; mode "omnidata" / "dsine"
    (DepthNormalConsistency) or "depth_to_normal" (DepthToNormal, whose threshold is 10)."""
    R = mono_rotation(c2w)
    m = mono_u8.reshape(-1, 3) / 255.0
    enc = ((normals + 1) / 2 * 255).astype(np.uint8)
    if mode == "depth_to_normal":
        m = (m.T - 0.5) * 2
        m = (R @ m).T
        m = m / np.linalg.norm(m, axis=1, keepdims=True)
        deg = angle_between((normals + 1) / 2, m * 0.5 + 0.5)
    else:
        m = 2 * m - 1
        if mode == "dsine":
            m = m @ np.diag([1, -1, -1])
        m = (R @ m.T).T
        m = m / np.linalg.norm(m, axis=1, keepdims=True)
        deg = angle_between(normals, m)
    return deg, deg > threshold, enc
