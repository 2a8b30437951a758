"""CPU checks of the neighbour-search oracles of oracle/normals_ref.py: knn_fast == knn (brute force) and search_mirror ==
knn on the clouds of tests/test_gpu_depth_normals.py, a 64 x 48 golden frame, exact-tie lattices and the constructed
clouds of tests/normals_search_cases.py; each constructed cloud reaches the branch it is named for; each of SEARCH_SLIPS
changes some query's neighbour multiset or examined count on those clouds."""
import numpy as np
import pytest

from oracle import normals_ref as R
from tests import normals_search_cases as S
from tests.test_depth_normals_cpu import golden_points
from tests.test_gpu_depth_normals import clouds as gpu_clouds


def _tie_lattices():
    i, j, k = np.meshgrid(np.arange(9), np.arange(9), np.arange(9), indexing="ij")
    cube = np.c_[i.ravel(), j.ravel(), k.ravel()] * 0.25
    ii, jj = np.meshgrid(np.arange(30), np.arange(30))
    plane = np.c_[ii.ravel() * 0.5, jj.ravel() * 0.5, np.zeros(900)]
    return {"cube_9": cube, "plane_30": plane, "plane_dups": np.r_[plane, plane[::7]]}


def _cases():
    out = {f"gpu_{n}": (p, k) for n, p in gpu_clouds().items() for k in (3, 30, 200)}
    out["golden_frame"] = (golden_points("omnidata")[1], 200)
    out.update({n: (p, k) for n, p in _tie_lattices().items() for k in (6, 30, 200)})
    out.update({n: (p, k) for n, (p, k, _) in S.clouds().items()})
    return out


def _rows(pts):
    return np.unique(R.unique_positions(pts)[3], return_index=True)[1]


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(np.sort(x), np.sort(y)) for x, y in zip(a, b))


@pytest.mark.parametrize("name", list(_cases()))
def test_fast_and_mirror_equal_brute_force(name):
    pts, k = _cases()[name]
    rows = _rows(pts)
    want = R.knn(pts, k, queries=rows)
    assert _same(R.knn_fast(pts, k, rows), want)
    mir = R.search_mirror(pts, k, rows)
    assert _same(mir["nbrs"], want)
    assert (mir["examined"][mir["shortcut"]] == 0).all() and (mir["examined"][~mir["shortcut"]] > 0).all()


def test_constructed_clouds_reach_their_branch():
    cl = S.clouds()
    for name, (pts, k, q) in cl.items():
        rows = _rows(pts) if q is None else q
        mir = R.search_mirror(pts, k, rows)
        assert not mir["everything"].any() and not mir["shortcut"].any(), name
        if name == "morton_discontinuity":  # the window's k-th distance at least twice the true one
            kd = np.array([R.sq_dist(pts[r], pts[w]).max() for r, w in zip(rows, R.knn_fast(pts, k, rows))])
            assert (mir["R"] >= 2 * np.sqrt(kd)).any()
        elif name == "level_clamped":
            assert mir["level_clamped"].any()
        elif name == "split":
            assert mir["split"].any()
        elif name == "subnormal":  # squared distances to other positions that are 0 and subnormal
            d2 = R.sq_dist(pts[0], pts[1:])
            assert (d2 == 0).any() and ((d2 > 0) & (d2 < 2.0 ** -1022)).any() and (mir["R"] == R.R_FLOOR).any()
        elif name == "signed_zero":
            z = np.signbit(pts) & (pts == 0)
            assert z.any() and (~z & (pts == 0)).any() and (R.unique_positions(pts)[2] == 2).any()
        elif name == "offset_1e4":
            assert pts.min() > 1e4 - 1 and np.ptp(pts, 0).max() < 0.02 and mir["box_clamped"].any()
        elif name == "margin":
            assert not np.array_equal(R.search_mirror(pts, k, rows, slip="no_margin")["examined"], mir["examined"])


def test_full_frame_branches():
    """The mirror on a 1920 x 1440 frame with five pixels 10^5 m away: fine grid levels and mid-scan compactions (a
    sample of the queries the GPU test checks)."""
    depth, (fx, fy, cx, cy), c2w = S.frames()["distant"]
    h, w = depth.shape
    pts = R.backproject(depth, fx, fy, cx, cy, w, h, c2w)[0]
    rows = S.frame_queries(depth, pts, n_random=2000)[::10]
    mir = R.search_mirror(pts, S.K, rows)
    assert mir["compactions"].max() > 0 and mir["level"].max() < 12
    assert _same(mir["nbrs"], R.knn_fast(pts, S.K, rows))


@pytest.mark.parametrize("slip", list(R.SEARCH_SLIPS))
def test_each_slip_is_caught(slip):
    caught = []
    for name, (pts, k, q) in S.clouds().items():
        rows = _rows(pts) if q is None else q
        a, b = R.search_mirror(pts, k, rows), R.search_mirror(pts, k, rows, slip=slip)
        if not _same(a["nbrs"], b["nbrs"]) or not np.array_equal(a["examined"], b["examined"]):
            caught.append(name)
    assert caught, slip
