"""The binning reference (oracle/binning_ref.py) against independent statements of the same contract, on the CPU:
gsplat_ref.isect_tiles for the exact lists, integer supertile arithmetic for the list boxes, and brute force over pixel
centres plus a bounded least-squares solve for the reachability test."""
import numpy as np
import pytest
import torch
from scipy.optimize import lsq_linear

from oracle import binning_ref as BR
from oracle import gsplat_ref as G
from oracle import project_ref as P

KINDS = ["random", "edge_on", "rank1"]


def _project(kind, seed, n=3000, width=96, height=72):
    """gsplat_ref's fp32 projection of a project_ref case, and its depth keys (-1 where culled)."""
    case = (P.edge_on_case(n, seed, width=width, height=height) if kind == "edge_on"
            else P.random_case(n, seed, kind=kind, width=width, height=height))
    s = case.params["scales"] if case.activated else torch.exp(case.params["scales"])
    proj = G.project_gaussians(case.params["means"], case.params["quats"], s, case.viewmat, case.K, width, height,
                               eps2d=case.eps2d, near_plane=case.near_plane, far_plane=case.far_plane)
    keys = torch.where(proj["radii"] > 0, proj["depths"].view(torch.int32), torch.tensor(-1, dtype=torch.int32))
    return proj, keys


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", [(96, 72), (200, 130)])
def test_expected_lists_equal_gsplat_isect_tiles(kind, size):
    W, H = size
    proj, keys = _project(kind, seed=KINDS.index(kind) + W, width=W, height=H)
    _, _, flat, offsets, _ = G.isect_tiles(proj["means2d"], proj["radii"], proj["depths"], 16, W, H)
    ids, offs = BR.expected_lists(proj["means2d"].numpy(), proj["radii"].numpy(), keys.numpy(), 16, W, H)
    assert ids.size > 1000, "premise: a populated frame"
    assert np.array_equal(ids, flat.numpy()), kind
    assert np.array_equal(offs[:-1], offsets.numpy().astype(np.int64)) and offs[-1] == ids.size, kind


def _boxes(seed, n=20000, width=1000, height=600):
    """Means on and far off the frame, radii from 1 to beyond the frame, some exactly on tile edges."""
    rng = np.random.default_rng(seed)
    m = np.stack([rng.uniform(-3000, width + 3000, n), rng.uniform(-3000, height + 3000, n)], 1).astype(np.float32)
    m[: n // 4] = (rng.integers(-40, 80, (n // 4, 2)) * 16).astype(np.float32)  # on a 16 px edge
    r = np.exp(rng.uniform(0, np.log(5000), n)).astype(np.int32)
    r[: n // 8] = rng.integers(1, 8, n // 8) * 16  # and a whole number of tiles from it
    r[-50:] = 0
    return m, r


@pytest.mark.parametrize("shift", [1, 2, 3])
@pytest.mark.parametrize("size", [(1000, 600), (1920, 1080), (100, 70)])
def test_list_box_is_the_supertiles_of_the_tile_box(shift, size):
    """Scaling by a power of two is exact, so the box at 16 << s holds exactly the supertiles that cover the 16 px box:
    [x0 >> s, (x1 + 2^s - 1) >> s) wherever the 16 px box is not empty.  (A box clamped empty at 16 px past the right or
    bottom tile may still name the last supertile there; the raster's own tile-box test never composites such a pair.)"""
    W, H = size
    m, r = _boxes(shift + W)
    tx, ty = BR.lists_xy(W, H, 16)
    lx, ly = BR.lists_xy(W, H, 16 << shift)
    x0, y0, x1, y1 = BR.list_box(m, r, 16, tx, ty)
    X0, Y0, X1, Y1 = BR.list_box(m, r, 16 << shift, lx, ly)
    ne = (x1 > x0) & (y1 > y0)
    assert ne.sum() > 1000 and (~ne & (r > 0)).sum() > 1000, "premise: boxes on and off the frame"
    up = (1 << shift) - 1
    for got, want in ((X0, x0 >> shift), (Y0, y0 >> shift), (X1, (x1 + up) >> shift), (Y1, (y1 + up) >> shift)):
        assert np.array_equal(got[ne], want[ne])


def _splats(seed, n, W, H):
    """Conics and opacities: ordinary splats, needles (axis ratio up to 1:2000), splats larger than the frame, centres
    off-screen on every side."""
    rng = np.random.default_rng(seed)
    s1 = np.exp(rng.uniform(np.log(0.3), np.log(400.0), n))
    ratio = np.where(rng.random(n) < 0.3, np.exp(rng.uniform(0, np.log(2000.0), n)), rng.uniform(1, 4, n))
    s2 = s1 / ratio
    eps = np.where(rng.random(n) < 0.5, 0.3, 1e-3)
    th = rng.uniform(0, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    a = c * c * s1 * s1 + s * s * s2 * s2 + eps
    b = c * s * (s1 * s1 - s2 * s2)
    cc = s * s * s1 * s1 + c * c * s2 * s2 + eps
    det = a * cc - b * b
    con = np.stack([cc / det, -b / det, a / det], 1).astype(np.float32)
    lam = 0.5 * (a + cc) + np.sqrt(np.maximum(0.25 * (a - cc) ** 2 + b * b, 0.01))
    radius = np.ceil(3 * np.sqrt(lam)).astype(np.int32)
    m = np.stack([rng.uniform(-0.5 * W, 1.5 * W, n), rng.uniform(-0.5 * H, 1.5 * H, n)], 1).astype(np.float32)
    op = np.exp(rng.uniform(np.log(1.0 / 255), 0, n)).astype(np.float32)
    ok = (con[:, 0].astype(np.float64) * con[:, 2] - con[:, 1].astype(np.float64) ** 2 > 0)
    return m[ok], con[ok], op[ok], radius[ok]


def _lsq_min_sigma(m, con, rect):
    """min over the rectangle of 0.5 d^T Q d = 0.5 |L^T d|^2 (Q = L L^T) by bounded least squares (BVLS)."""
    Q = np.array([[con[0], con[1]], [con[1], con[2]]], dtype=np.float64)
    Lt = np.linalg.cholesky(Q).T
    px0, px1, py0, py1 = rect
    lo = np.array([px0 + 0.5 - m[0], py0 + 0.5 - m[1]])
    hi = np.array([px1 - 0.5 - m[0], py1 - 0.5 - m[1]])
    if np.array_equal(lo, hi):
        return 0.5 * float(np.sum((Lt @ lo) ** 2))
    res = lsq_linear(Lt, np.zeros(2), bounds=(lo, hi + 1e-300 * (hi == lo)), method="bvls", tol=1e-14)
    return 0.5 * float(np.sum((Lt @ res.x) ** 2))


@pytest.mark.parametrize("ts", [16, 32, 64, 128])
@pytest.mark.parametrize("seed", range(3))
def test_needed_matches_brute_force(ts, seed):
    """On a small frame, every pair of the list boxes: the closed form over the continuous rectangle equals a bounded
    least-squares solve, and it keeps every pair that some pixel centre passes (brute force)."""
    W, H = 150, 94  # not a multiple of any list tile
    m, con, op, r = _splats(seed * 10 + ts, 400, W, H)
    lx, ly = BR.lists_xy(W, H, ts)
    gid, lid = BR.box_pairs(m, r, ts, lx, ly)
    rects = BR.pair_rects(m, r, gid, lid, ts, W, H)
    sig = BR.min_sigma(m, con, gid, rects)
    closed = BR.reaches(op[gid], sig)
    brute = BR.needed_discrete(m, con, op, r, gid, lid, ts, W, H)
    assert brute.sum() > 200 and (~brute).sum() > 100, "premise: pairs on both sides"
    miss = brute & ~closed
    assert not miss.any(), f"closed form drops a pair brute force keeps: {np.nonzero(miss)[0][:5]}"
    fin = np.isfinite(sig)
    rng = np.random.default_rng(seed)
    pick = rng.choice(np.nonzero(fin)[0], size=min(600, int(fin.sum())), replace=False)
    for k in pick:
        want = _lsq_min_sigma(m[gid[k]].astype(np.float64), con[gid[k]].astype(np.float64), [int(v[k]) for v in rects])
        assert abs(sig[k] - want) <= 1e-7 * (1.0 + want), (k, sig[k], want)
    # and it is tight: few of the pairs it keeps fall between the pixel centres
    extra = closed & ~brute
    assert extra.sum() <= 0.1 * closed.sum(), (int(extra.sum()), int(closed.sum()))
    # the wrapper agrees
    g2, l2 = BR.needed(m, con, op, r, ts, W, H)
    assert np.array_equal(g2, gid[closed]) and np.array_equal(l2, lid[closed])


def test_truncated_keeps_emission_order():
    """Three Gaussians, depth order 2, 0, 1: emission is G2's lists, then G0's, then G1's, each row-major."""
    keys = np.array([0x3F000000, 0x40000000, 0x3E000000], dtype=np.uint32)
    # lists: G0 -> {0, 1, 4}, G1 -> {1, 5}, G2 -> {4, 5}
    gid = np.array([0, 0, 0, 1, 1, 2, 2])
    lid = np.array([0, 1, 4, 1, 5, 4, 5])
    ids, offs = BR._lists(gid, lid, keys, 6)
    assert ids.tolist() == [0, 0, 1, 2, 0, 2, 1] and offs.tolist() == [0, 1, 3, 3, 3, 5, 7]
    for cap, want_ids, want_offs in ((7, [0, 0, 1, 2, 0, 2, 1], [0, 1, 3, 3, 3, 5, 7]),
                                     (3, [0, 2, 2], [0, 1, 1, 1, 1, 2, 3]),
                                     (2, [2, 2], [0, 0, 0, 0, 0, 1, 2]),
                                     (0, [], [0] * 7)):
        t_ids, t_offs = BR.truncated(ids, offs, keys, cap)
        assert t_ids.tolist() == want_ids and t_offs.tolist() == want_offs, cap
