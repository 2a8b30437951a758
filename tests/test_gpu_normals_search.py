"""dnr_dn_normals per query against oracle/normals_ref.py at capture resolution: neighbour multisets exactly equal to the
fp64 k-NN under the tie rule (knn_fast), the candidates each search examined exactly equal to the numpy restatement of
the search geometry (search_mirror), covariances within their fp64 bound, normals under the eigen-gap rule, orientation
outside its rounding band and the consistency pass on every pixel, on depth frames (256 x 192 with every position,
1920 x 1440 at 2 % / 40 % holes under a rotated and translated pose, a nearest-resized coarse depth map, an exact
lattice, k - 1 / k / k + 1 holes, five pixels 10^5 m away) and on constructed clouds (tests/normals_search_cases.py).
Prints the worst fraction of each bound, the ill-conditioned share and the examined-per-search distribution."""
import numpy as np
import pytest
import torch

from dn_splatter_b200 import depth_normals as DN
from oracle import normals_ref as R
from tests import normals_search_cases as S

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -52
WORST = {}


def _note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), float(v))


def _run(pts_dev, k, center):
    n = pts_dev.shape[0]
    ex = torch.zeros(n, dtype=torch.int32, device="cuda")
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    normals, cov, nbr = DN.estimate_normals(pts_dev, k, center=center, examined=ex, stats=stats, debug=True)
    return normals, cov, nbr, ex, stats


def _check(name, pts, k, rows, center, all_positions):
    """One case: the kernel at every point, compared at `rows` (point indices)."""
    pts_dev = torch.as_tensor(pts, device="cuda")
    normals, cov, nbr, ex, stats = _run(pts_dev, k, center)
    rows_dev = torch.as_tensor(rows, device="cuda")
    g_nbr = nbr[rows_dev].cpu().numpy()  # only the sampled rows leave the device
    g_cov = cov[rows_dev].cpu().numpy().reshape(-1, 3, 3)
    g_nrm = normals[rows_dev].cpu().numpy()
    g_ex = ex[rows_dev].cpu().numpy()
    n = len(pts)
    kk = min(k, n)
    want = R.knn_fast(pts, k, rows)
    mir = R.search_mirror(pts, k, rows)
    assert (g_nbr[:, kk:] == -1).all(), name
    for r, got, w, m in zip(rows, g_nbr, want, mir["nbrs"]):
        np.testing.assert_array_equal(np.sort(got[:kk]), np.sort(w), err_msg=f"{name} row {r}")
        np.testing.assert_array_equal(np.sort(m), np.sort(w), err_msg=f"{name} mirror row {r}")
    np.testing.assert_array_equal(g_ex, mir["examined"], err_msg=name)
    if all_positions:  # rows holds one point of every distinct position
        s = stats.cpu().numpy()
        assert s[1] == len(rows) and s[0] == mir["examined"].sum(), (name, s, len(rows), mir["examined"].sum())
    # covariance, normal, orientation
    ill = 0
    for i, (r, w) in enumerate(zip(rows, want)):
        c = R.covariance(pts, w)
        scale = (np.asarray(pts)[w] ** 2).sum(1).max() + 1e-300
        bound = 8 * kk * (EPS * scale + 2.0 ** -1074)  # plus a subnormal ulp per term for the subnormal cloud
        err = np.abs(g_cov[i] - c).max()
        assert err <= bound, (name, r, err, bound)
        _note("covariance", err / bound)
        v = R.fast_eigen3x3(c)
        if len(np.unique(w)) == 1 or np.linalg.norm(v) == 0:
            # one position (the camera centre of a frame's holes: its covariance is rounding noise) or a covariance that
            # rounded to 0 (the subnormal cloud): no normal to compare
            ill += 1
            continue
        ev = np.linalg.eigvalsh(c)
        gap = ev[1] - ev[0]
        nb = 1e3 * bound / gap + 1e-9 if gap > 0 else np.inf
        if not (gap > 1e-6 * max(ev[2], 1e-300) and kk >= 3):
            ill += 1
            continue
        e = min(np.abs(g_nrm[i] - v).max(), np.abs(g_nrm[i] + v).max())
        assert e <= nb, (name, r, e, gap)
        _note("normal", e / nb)
        if nb >= 0.1:  # the covariance's rounding (|p| large against the neighbourhood) leaves the normal undetermined
            ill += 1
            continue
        if center is not None:
            ray = pts[r] - center
            ref = -v if ray @ v > 0 else v
            if abs(ray @ ref) > 1e-9 * np.linalg.norm(ray):
                assert g_nrm[i] @ ref > 0, (name, r)
    return normals, ex, mir, ill


def _rerun_identical(pts_dev, k, center, normals, ex):
    n2, _, _, ex2, _ = _run(pts_dev, k, center)
    assert torch.equal(normals, n2) and torch.equal(ex, ex2)


def _consistency(normals, c2w, pts, seed):
    """dnr_dn_consistency on every pixel with the kernel's own normals against the oracle."""
    mono = np.random.default_rng(seed).integers(0, 256, (len(pts), 3), dtype=np.uint8)
    nrm = normals.cpu().numpy()
    for mode, thr in (("omnidata", 20.0), ("dsine", 15.0), ("depth_to_normal", 10.0)):
        enc, deg, mask = DN.depth_normal_consistency(normals, mono, c2w, mode, thr)
        d_ref, m_ref, e_ref = R.consistency(nrm, mono, c2w, mode, thr)
        deg = deg.cpu().numpy()
        err = np.abs(deg - d_ref)
        assert np.nanmax(err) <= 1e-9, mode
        _note("degrees", np.nanmax(err) / 1e-9)
        near = np.abs(d_ref - thr) <= 1e-9
        assert ((mask.cpu().numpy() == 255) == m_ref)[~near].all(), mode
        enc = enc.cpu().numpy()
        assert (np.abs(enc.astype(int) - e_ref.astype(int)) <= 1).all()
        clear = np.abs(nrm * 127.5 % 1 - 0.5).min(1) > 1e-6
        np.testing.assert_array_equal(enc[clear], e_ref[clear])


ILL = {}
EXAMINED = {}


@pytest.mark.parametrize("name", list(S.frames()))
def test_frame(name):
    depth, (fx, fy, cx, cy), c2w = S.frames()[name]
    pts_dev = DN.backproject_depth(depth, fx, fy, cx, cy, c2w)
    pts = pts_dev.cpu().numpy()
    every = depth.size <= 256 * 192
    if every:
        rows = np.unique(R.unique_positions(pts)[3], return_index=True)[1]
    else:
        rows = S.frame_queries(depth, pts, *((300, 300) if name.startswith("holes_") else ()))
        rows = rows[np.unique(R.unique_positions(pts)[3][rows], return_index=True)[1]]  # one query per position
        assert (depth == 0).sum() == 0 or (depth.reshape(-1)[rows] == 0).any()
    centre = c2w[:3, 3]
    normals, ex, mir, ill = _check(name, pts, S.K, rows, centre, every)
    _rerun_identical(pts_dev, S.K, centre, normals, ex)
    ILL[name] = (ill, len(rows))
    assert ill <= 0.05 * len(rows), (name, ill, len(rows))
    EXAMINED[name] = np.percentile(mir["examined"], [50, 90, 99, 100])
    if not every:
        _consistency(normals, c2w, pts, 7)
    holes = int((depth == 0).sum())
    if name == "holes_199":
        assert not mir["shortcut"].any()
    if name in ("holes_200", "holes_201"):
        assert mir["shortcut"].any() and bool((mir["split"] & mir["shortcut"]).any()) == (holes > S.K)
    if name == "distant":
        assert mir["compactions"].max() > 0
    if name != "room_256":
        assert mir["box_clamped"].any() and not mir["everything"].any()
    print(f"\n{name}: {len(rows)} queries, ill-conditioned {ill} ({ill / len(rows):.2%}), examined p50/p90/p99/max "
          f"{EXAMINED[name].tolist()}, levels {np.unique(mir['level']).tolist()}, compactions {int(mir['compactions'].sum())}, "
          f"worst bound fractions {WORST}")


def _branch(name, mir, pts, k):
    if name == "morton_discontinuity":
        kd = np.array([R.sq_dist(pts[r], pts[w]).max() for r, w in zip(_rows(name), R.knn_fast(pts, k, _rows(name)))])
        assert (mir["R"] >= 2 * np.sqrt(kd)).any()
    elif name == "level_clamped":
        assert mir["level_clamped"].any()
    elif name == "split":
        assert (mir["split"] & ~mir["shortcut"]).any()
    elif name == "subnormal":
        assert (mir["R"] == R.R_FLOOR).any()
    elif name == "margin":
        assert not R.search_mirror(pts, k, _rows(name), slip="no_margin")["examined"].tolist() == mir["examined"].tolist()


def _rows(name):
    pts, k, q = S.clouds()[name]
    return np.unique(R.unique_positions(pts)[3], return_index=True)[1] if q is None else q


@pytest.mark.parametrize("name", list(S.clouds()))
def test_cloud(name):
    pts, k, q = S.clouds()[name]
    rows = _rows(name)
    centre = np.asarray(pts).mean(0)
    normals, ex, mir, ill = _check(name, pts, k, rows, centre, q is None)
    _rerun_identical(torch.as_tensor(pts, device="cuda"), k, centre, normals, ex)
    _branch(name, mir, pts, k)
    print(f"\n{name}: ill-conditioned {ill} of {len(rows)}, worst bound fractions {WORST}")
