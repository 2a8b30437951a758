"""The grid-hash k-NN of csrc/knn.cu mirrored step by step in numpy (same cell map with clamping, same shell walk, same
termination bound, same sorted top-K insertion, fp32 distances) and checked against sklearn — the library the
reference's knn_sk calls — on point sets with outliers, queries outside the grid, flat (2-D) sets and tiny sets."""
import math

import numpy as np
import pytest

from dn_splatter_b200.sugar import choose_grid


def grid_for(points):
    p = points.astype(np.float64)
    return choose_grid(p.min(0).tolist(), p.max(0).tolist(), p.mean(0).tolist(), p.std(0).tolist(), len(points))


def build(points, g):
    lo, inv, dims = np.float32(g["lo"]), np.float32(1.0 / g["cell"]), g["dims"]
    c = np.floor((points - lo) * inv).astype(np.int64)
    c = np.clip(c, 0, np.array(dims) - 1)
    cell = (c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0]
    order = np.argsort(cell, kind="stable")
    cs = cell[order]
    n_cells = dims[0] * dims[1] * dims[2]
    start, end = np.zeros(n_cells, np.int64), np.zeros(n_cells, np.int64)
    for i, cc in enumerate(cs):
        if i == 0 or cs[i - 1] != cc:
            start[cc] = i
        if i == len(cs) - 1 or cs[i + 1] != cc:
            end[cc] = i + 1
    return order, start, end


def query(points, g, order, start, end, q, K, skip):
    lo, inv, dims, cellf = np.float32(g["lo"]), np.float32(1.0 / g["cell"]), g["dims"], np.float32(g["cell"])
    c = np.clip(np.floor((q - lo) * inv).astype(np.int64), 0, np.array(dims) - 1)
    cx, cy, cz = int(c[0]), int(c[1]), int(c[2])
    r_max = max(cx, dims[0] - 1 - cx, cy, dims[1] - 1 - cy, cz, dims[2] - 1 - cz)
    delta = np.float32(max(dims)) * np.float32(2.0 ** -18)  # the fp32 binning slack, in cells
    d, ids = [], []

    def insert(d2, i):
        if len(d) == K and not d2 < d[-1]:
            return
        pos = len(d) if len(d) < K else K - 1
        if len(d) < K:
            d.append(None)
            ids.append(None)
        while pos > 0 and d[pos - 1] > d2:
            d[pos], ids[pos] = d[pos - 1], ids[pos - 1]
            pos -= 1
        d[pos], ids[pos] = d2, i

    def scan(cell):
        for j in range(start[cell], end[cell]):
            p = points[order[j]]
            dx, dy, dz = np.float32(p[0] - q[0]), np.float32(p[1] - q[1]), np.float32(p[2] - q[2])
            insert(np.float32(np.float32(dx * dx + dy * dy) + dz * dz), int(order[j]))

    visited = 0
    for r in range(r_max + 1):
        for z in range(max(cz - r, 0), min(cz + r, dims[2] - 1) + 1):
            zf = z == cz - r or z == cz + r
            for y in range(max(cy - r, 0), min(cy + r, dims[1] - 1) + 1):
                row = (z * dims[1] + y) * dims[0]
                if zf or y == cy - r or y == cy + r:
                    for x in range(max(cx - r, 0), min(cx + r, dims[0] - 1) + 1):
                        scan(row + x)
                        visited += 1
                else:
                    if cx - r >= 0:
                        scan(row + cx - r)
                        visited += 1
                    if cx + r < dims[0]:
                        scan(row + cx + r)
                        visited += 1
        reach = max(np.float32(r) - delta, np.float32(0)) * cellf
        if len(d) == K and d[K - 1] <= np.float32(reach * reach):
            break
    return ids[skip:], visited


def sk(points, queries, K):
    from sklearn.neighbors import NearestNeighbors

    dist, idx = NearestNeighbors(n_neighbors=K, algorithm="auto", metric="euclidean").fit(points).kneighbors(queries)
    return dist, idx


CASES = {
    "blob_with_outliers": lambda r: np.concatenate([r.normal(size=(1500, 3)), r.normal(size=(12, 3)) * 40.0]),
    "flat_sheet": lambda r: np.concatenate([r.uniform(-2, 2, size=(1200, 2)), r.normal(size=(1200, 1)) * 1e-3], axis=1),
    "anisotropic": lambda r: r.normal(size=(1000, 3)) * np.array([8.0, 1.0, 0.2]),
    "tiny": lambda r: r.normal(size=(20, 3)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_grid_search_equals_sklearn(name):
    r = np.random.default_rng(sum(map(ord, name)))
    pts = CASES[name](r).astype(np.float32)
    g = grid_for(pts)
    assert all(1 <= d <= 256 for d in g["dims"])
    order, start, end = build(pts, g)
    assert int((end - start).sum()) == len(pts)  # every point is in exactly one cell (outliers clamped)
    q_in = pts[r.choice(len(pts), 40, replace=len(pts) < 40)] + r.normal(size=(40, 3)).astype(np.float32) * 0.05
    q_out = (pts.mean(0) + r.normal(size=(10, 3)) * pts.std(0) * 6).astype(np.float32)  # well outside the grid box
    queries = np.concatenate([q_in, q_out]).astype(np.float32)
    K = min(17, len(pts))
    dist, idx = sk(pts, queries, K)
    total_cells = g["dims"][0] * g["dims"][1] * g["dims"][2]
    visited_in = []
    for qi, q in enumerate(queries):
        got, visited = query(pts, g, order, start, end, q, K, skip=1)
        want = idx[qi, 1:].tolist()
        if got != want:  # only acceptable when two neighbours are equidistant to fp32 precision
            dg = np.linalg.norm(pts[got].astype(np.float64) - q, axis=1)
            np.testing.assert_allclose(dg, dist[qi, 1:], rtol=1e-5)
        if qi < 40:
            visited_in.append(visited)
    if name != "tiny":  # the bound prunes: queries near the data touch a small part of the grid
        assert np.mean(visited_in) < 0.35 * total_cells, (np.mean(visited_in), total_cells)


# Binning in fp32 moves cell boundaries: the query lands at u = 158.99998 (cell 158), A at 160.0 (cell 160), B at
# 157.99998 (cell 157).  A is nearer than B by 5.4e-6 relative, far outside the fp32 tie band, but A sits two cells
# away and B only one, so a stop rule of "K-th distance <= r * cell" returns B after shell 1.
STOP_RULE_GRID = {"lo": [-2.3644726, 0.0, 0.0], "cell": 0.013844357633743604, "dims": [256, 1, 1]}
STOP_RULE_POINTS = [[-0.14937554, 0.0, 0.0], [-0.17706418, 0.0, 0.0]]  # A (nearest), B
STOP_RULE_QUERY = [-0.16321982, 0.0, 0.0]


def test_stop_rule_covers_the_fp32_binning_error():
    pts = np.array(STOP_RULE_POINTS, np.float32)
    q = np.array(STOP_RULE_QUERY, np.float32)
    g = STOP_RULE_GRID
    inv = np.float32(1.0 / g["cell"])
    u = [float(np.float32(np.float32(x - np.float32(g["lo"][0])) * inv)) for x in (q[0], pts[0, 0], pts[1, 0])]
    assert [math.floor(v) for v in u] == [158, 160, 157]  # the case still straddles the cells as described
    d = np.abs(pts[:, 0].astype(np.float64) - float(q[0]))
    assert d[0] < d[1] * (1 - 5e-6)
    order, start, end = build(pts, g)
    got, _ = query(pts, g, order, start, end, q, 1, skip=0)
    assert got == [0]


def test_fewer_points_than_k():
    pts = np.random.default_rng(0).normal(size=(5, 3)).astype(np.float32)
    g = grid_for(pts)
    order, start, end = build(pts, g)
    got, _ = query(pts, g, order, start, end, pts[0], 17, skip=1)
    assert len(got) == 4 and 0 not in got  # all the other points; the kernel pads the remaining columns with -1


def test_choose_grid_degenerate_inputs():
    g = choose_grid([0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], 1)
    assert g["dims"] == [1, 1, 1] and g["cell"] > 0 and math.isfinite(g["cell"])
    g = choose_grid([-1e6, -1, -1], [1e6, 1, 1], [0, 0, 0], [1, 1, 1], 10_000_000)
    assert max(g["dims"]) <= 256
