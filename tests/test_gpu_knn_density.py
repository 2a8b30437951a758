"""GPU tests of the grid k-NN (csrc/knn.cu) and the SuGaR density kernels (csrc/density.cu) per query, per sample and per
ray against fp64 references built here on the device from the same fp32 inputs.

k-NN.  The reference is brute force over fp64 differences (not the |x|^2 + |y|^2 - 2xy form).  Every returned row must
hold unique ids in [0, n), -1 / inf exactly in the trailing columns when fewer than K = k + skip points exist,
non-decreasing distances equal bit for bit to the fp32 expression of the kernel (knn.cu is built with -fmad=false), and at
every rank j the fp64 squared distance of the returned id within TIE of the j-th smallest fp64 squared distance.  The fp32
squared distance of fp32 points is within 5 eps of the exact one (eps = 2^-24: the three differences, three products and
two sums), so two neighbours can trade places only when their squared distances agree to 10 eps; TIE = 16 eps also
covers the rounding of the stop rule's reach.  A missed neighbour shows as a rank whose distance is too large.

Density.  Each Gaussian term's error is bounded from its own quantities: the fp32 squared Mahalanobis distance d2 is
off by at most dd2 = 2 sqrt(d2) h + h^2 + 13 eps d2, h = sum_c is_c (56 eps |x - mu| + e_x) (56 eps: the rotation entries
of a normalised fp32 quaternion are within 30 eps absolute, the dot products add 4 eps; 13 eps: 1 / max(exp(s), 1e-3),
the squares and sums; e_x: the error of the sample position, 0 for dnr_density); the weight's error is the spread of
op exp(-d2 / 2) over d2 +- dd2 plus 8 eps of the weight (sigmoid, exp, product); the sum adds (k - 1) eps of itself.
Where the fp64 sum lies within its bound of 1 either side of the d / (d + 1e-5) squash is accepted, and counted.

Set DNR_KNN_DENSITY_REPORT=<file> to append one JSON line per check with the worst ratio of error to bound.
"""
import ctypes as C
import json
import math
import os
import types

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from dn_splatter_b200 import sugar as SG
from oracle import gsplat_ref as G
from tests.test_knn_grid_cpu import STOP_RULE_GRID, STOP_RULE_POINTS, STOP_RULE_QUERY

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

EPS = 2.0 ** -24
TIE = 16 * EPS
KS = (1, 2, 3, 16, 31, 32)
ATOL_W = 1e-44  # a weight in fp32 denormals is off by a few 2^-149 in absolute terms
DEV = "cuda"
PARAMS = ("means", "quats", "scales", "opacities")
L_E = {"NULL": -1, "SIZE": -2, "OPTION": -3, "WORKSPACE": -5}  # DNR_E_* of include/dnr.h


def report(check, **kw):
    path = os.environ.get("DNR_KNN_DENSITY_REPORT")
    if path:
        with open(path, "a") as fh:
            fh.write(json.dumps(dict(check=check, **kw)) + "\n")


# ----------------------------------------------------------------------------------------------------------- k-NN


def ref_sorted_d2(points, queries, K):
    """fp64 squared distances of the min(K, n) nearest points of every query, ascending."""
    x = points.double()
    out = []
    for q in queries.double().split(512):
        d2 = ((q[:, None, :] - x[None]) ** 2).sum(-1)
        out.append(d2.topk(min(K, x.shape[0]), dim=1, largest=False, sorted=True).values)
    return torch.cat(out)


def f32_dist(points, queries, idx):
    """The kernel's own fp32 expression: sqrt((dx dx + dy dy) + dz dz), d = p - q, no contraction."""
    d = points[idx] - queries[:, None, :]
    return torch.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def check_rows(name, points, queries, k, skip, idx, dist, ref):
    """The per-row pass rule of the module docstring; returns the worst rank error as a share of TIE."""
    n, m = points.shape[0], queries.shape[0]
    K = k + int(skip)
    valid = max(min(n, K) - int(skip), 0)
    assert idx.shape == (m, k) and dist.shape == (m, k), name
    assert bool((idx[:, valid:] == -1).all()), f"{name}: padding columns hold ids"
    assert bool((dist[:, valid:] == math.inf).all()), f"{name}: padding columns hold finite distances"
    if valid == 0:
        return 0.0
    v = idx[:, :valid]
    assert bool(((v >= 0) & (v < n)).all()), f"{name}: ids outside [0, {n})"
    s = v.sort(dim=1).values
    assert bool((s[:, 1:] != s[:, :-1]).all()), f"{name}: an id repeats within a row"
    dv = dist[:, :valid]
    assert bool((dv[:, 1:] >= dv[:, :-1]).all()), f"{name}: distances decrease along a row"
    same = dv.view(torch.int32) == f32_dist(points, queries, v).view(torch.int32)
    assert bool(same.all()), f"{name}: {int((~same).sum())} distances differ from the fp32 recomputation"
    d64 = ((points.double()[v] - queries.double()[:, None, :]) ** 2).sum(-1)
    want = ref[:, int(skip):int(skip) + valid]
    ratio = (d64 - want).abs() / (TIE * want + 2.0 ** -126)
    worst = float(ratio.max())
    if worst > 1.0:
        r, c = divmod(int(ratio.argmax()), valid)
        raise AssertionError(f"{name}: query {r} rank {c + int(skip)}: id {int(v[r, c])} at d2 {float(d64[r, c])!r}, "
                             f"the fp64 rank holds {float(want[r, c])!r} ({worst:.3g} x the tie band)")
    return worst


def blob_outliers(g):
    far = torch.randn(12, 3, generator=g)
    far = far / far.norm(dim=1, keepdim=True)
    return torch.cat([torch.randn(3000, 3, generator=g), far[:8] * 40.0, far[8:] * 1e6])


def flat_sheet(g):
    return torch.cat([torch.rand(2500, 2, generator=g) * 4 - 2, torch.zeros(2500, 1)], dim=1)


def line(g):
    return torch.cat([torch.rand(1500, 1, generator=g) * 6 - 3, torch.zeros(1500, 2)], dim=1)


def hollow_box(g):
    """Surface samples of [-1, 1]^3: six faces, one coordinate pinned to +-1."""
    p = torch.rand(4000, 3, generator=g) * 2 - 1
    axis = torch.randint(0, 3, (4000,), generator=g)
    side = torch.randint(0, 2, (4000,), generator=g).float() * 2 - 1
    p[torch.arange(4000), axis] = side
    return p


def lattice(g):
    r = torch.arange(12, dtype=torch.float32)
    return torch.stack(torch.meshgrid(r, r, r, indexing="ij"), dim=-1).reshape(-1, 3)


def duplicates(g):
    base = torch.randn(600, 3, generator=g)
    x = torch.cat([base, base[:400], base[:100]])
    return x[torch.randperm(x.shape[0], generator=g)]


def offset_blob(g):
    return 1e4 + torch.randn(3000, 3, generator=g)


POINT_SETS = {"blob_outliers": blob_outliers, "flat_sheet": flat_sheet, "line": line, "hollow_box": hollow_box,
              "lattice": lattice, "duplicates": duplicates, "offset_blob": offset_blob}


def queries_for(x, grid, g):
    """(queries, number of leading queries that are data points): data points, jittered data points, points on cell
    boundaries of `grid`, points far outside the grid box."""
    n = x.shape[0]
    data = x[torch.randperm(n, generator=g)[:400]]
    jitter = x[torch.randint(0, n, (400,), generator=g)] + torch.randn(400, 3, generator=g) * 0.3 * grid["cell"]
    dims = torch.tensor(grid["dims"], dtype=torch.float64)
    c = torch.floor(torch.rand(300, 3, generator=g, dtype=torch.float64) * (dims + 1))
    bound = (torch.tensor(grid["lo"], dtype=torch.float64) + c * grid["cell"]).float()
    centre = torch.tensor(grid["lo"], dtype=torch.float64) + dims * grid["cell"] / 2
    span = float(dims.max()) * grid["cell"]
    u = torch.randn(120, 3, generator=g, dtype=torch.float64)
    u = u / u.norm(dim=1, keepdim=True)
    far = (centre + u * torch.cat([torch.full((100, 1), 20.0 * span + 10.0), torch.full((20, 1), 2e6)])).float()
    return torch.cat([data, jitter, bound, far]).contiguous(), data.shape[0]


@pytest.mark.parametrize("name", sorted(POINT_SETS))
def test_knn_per_query_against_fp64(name):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = POINT_SETS[name](g).float().contiguous()
    xc = x.to(DEV)
    index = SG.KnnIndex(xc)
    grid = index.grid
    if name in ("flat_sheet", "line"):
        assert max(grid["dims"]) == 256, grid
    q, n_data = queries_for(x, grid, g)
    qc = q.to(DEV)
    ref = ref_sorted_d2(xc, qc, 33)
    worst = 0.0
    for k in KS:
        for skip in (False, True):
            idx, dist = index.query(qc, k, skip_first=skip, return_distances=True)
            worst = max(worst, check_rows(f"{name} k={k} skip={skip}", xc, qc, k, skip, idx, dist, ref))
            if skip:  # the same search as k + 1 without the skip, first column dropped
                idx1, dist1 = index.query(qc, k + 1, skip_first=False, return_distances=True)
                assert torch.equal(idx, idx1[:, 1:]) and torch.equal(dist, dist1[:, 1:]), f"{name} k={k}"
                assert bool((dist1[:n_data, 0] == 0).all()), f"{name} k={k}: a data point's dropped column is not at 0"
            else:
                assert bool((dist[:n_data, 0] == 0).all()), f"{name} k={k}: a data point is not its own nearest"
    # two builds and two queries give the same bits
    a = index.query(qc, 16, skip_first=True, return_distances=True)
    b = SG.KnnIndex(xc).query(qc, 16, skip_first=True, return_distances=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)), name
    report(f"knn-{name}", worst=worst, queries=int(q.shape[0]), dims=grid["dims"])


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("skip", [False, True])
def test_knn_fewer_points_than_k(k, skip):
    K = k + int(skip)
    for n in sorted({1, K - 1, K} - {0}):
        g = torch.Generator().manual_seed(1000 * k + 10 * n + int(skip))
        x = torch.randn(n, 3, generator=g).to(DEV)
        q = torch.cat([x, torch.randn(20, 3, generator=g).to(DEV) * 3])
        idx, dist = SG.KnnIndex(x).query(q, k, skip_first=skip, return_distances=True)
        check_rows(f"n={n} k={k} skip={skip}", x, q, k, skip, idx, dist, ref_sorted_d2(x, q, K))


def abi_knn(points, grid, queries, k, skip):
    """dnr_knn_build / dnr_knn_query with a hand-set DnrKnnGrid."""
    lib = L.load()
    gs = SG._grid_struct(grid)
    n, m = points.shape[0], queries.shape[0]
    nbytes = lib.dnr_knn_workspace_bytes(n, C.byref(gs))
    assert nbytes > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    assert lib.dnr_knn_build(points.data_ptr(), n, C.byref(gs), ws.data_ptr(), nbytes, SG._stream()) == 0
    idx = torch.empty((m, k), dtype=torch.int64, device=DEV)
    dist = torch.empty((m, k), dtype=torch.float32, device=DEV)
    assert lib.dnr_knn_query(n, C.byref(gs), ws.data_ptr(), queries.data_ptr(), m, k, int(skip), idx.data_ptr(),
                             dist.data_ptr(), SG._stream()) == 0
    return idx, dist


def test_knn_stop_rule_covers_fp32_binning():
    """The constructed case of tests/test_knn_grid_cpu.py: A is nearer than B by 5.4e-6 relative but lies two cells from
    the query after fp32 binning, B one.  A stop rule that trusts r * cell returns B."""
    pts = torch.tensor(STOP_RULE_POINTS, dtype=torch.float32, device=DEV)
    q = torch.tensor([STOP_RULE_QUERY], dtype=torch.float32, device=DEV)
    idx, dist = abi_knn(pts, STOP_RULE_GRID, q, 1, False)
    assert idx.tolist() == [[0]], f"returned point {idx.tolist()} at {dist.tolist()}, point 0 is nearer"
    check_rows("stop-rule", pts, q, 1, False, idx, dist, ref_sorted_d2(pts, q, 1))


HAND_GRIDS = {
    "one_cell": {"lo": [0.0, 0.0, 0.0], "cell": 1.0, "dims": [1, 1, 1]},
    "coarse": {"lo": [-2.0, -1.5, -1.0], "cell": 1.3, "dims": [3, 2, 2]},
    "fine": {"lo": [-3.0, -3.0, -3.0], "cell": 0.05, "dims": [120, 120, 120]},
    "off_data": {"lo": [5.0, 5.0, 5.0], "cell": 0.25, "dims": [8, 8, 8]},  # every point clamps into the corner cell
    "long_axis": {"lo": [-3.0, -0.5, -0.5], "cell": 3e-4, "dims": [20000, 1, 1]},
}


@pytest.mark.parametrize("name", sorted(HAND_GRIDS))
def test_knn_hand_set_grid(name):
    grid = HAND_GRIDS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    far = torch.randn(3, 3, generator=g)
    x = torch.cat([torch.randn(1500, 3, generator=g), torch.randn(20, 3, generator=g) * 50,
                   far / far.norm(dim=1, keepdim=True) * 1e6]).to(DEV)
    q = torch.cat([x[:200], x[200:400] + 0.01 * torch.randn(200, 3, generator=g).to(DEV),
                   torch.randn(100, 3, generator=g).to(DEV) * 30])
    ref = ref_sorted_d2(x, q, 33)
    worst = 0.0
    for k, skip in ((1, False), (16, True), (32, True), (32, False)):
        idx, dist = abi_knn(x, grid, q, k, skip)
        worst = max(worst, check_rows(f"{name} k={k} skip={skip}", x, q, k, skip, idx, dist, ref))
    report(f"knn-grid-{name}", worst=worst)


def test_knn_abi_rejections():
    lib = L.load()
    x = torch.randn(50, 3, device=DEV)
    gs = SG._grid_struct(SG.KnnIndex(x).grid)
    nbytes = lib.dnr_knn_workspace_bytes(50, C.byref(gs))
    assert nbytes > 0 and lib.dnr_knn_workspace_bytes(0, C.byref(gs)) == -1
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    st = SG._stream()
    assert lib.dnr_knn_build(x.data_ptr(), 0, C.byref(gs), ws.data_ptr(), nbytes, st) == L_E["SIZE"]
    assert lib.dnr_knn_build(x.data_ptr(), 50, C.byref(gs), ws.data_ptr(), nbytes - 1, st) == L_E["WORKSPACE"]
    assert lib.dnr_knn_build(x.data_ptr(), 50, C.byref(gs), ws.data_ptr(), nbytes, st) == 0
    q = x[:5].contiguous()
    out = torch.empty((5, 40), dtype=torch.int64, device=DEV)
    for k, skip, want in ((33, 1, "OPTION"), (34, 0, "OPTION"), (33, 0, None), (32, 1, None), (0, 0, "SIZE"),
                          (-1, 1, "SIZE")):
        rc = lib.dnr_knn_query(50, C.byref(gs), ws.data_ptr(), q.data_ptr(), 5, k, skip, out.data_ptr(), None, st)
        assert rc == (0 if want is None else L_E[want]), (k, skip, rc)
    assert lib.dnr_knn_query(0, C.byref(gs), ws.data_ptr(), q.data_ptr(), 5, 4, 0, out.data_ptr(), None, st) == L_E["SIZE"]
    assert lib.dnr_knn_query(50, C.byref(gs), ws.data_ptr(), q.data_ptr(), 0, 4, 0, out.data_ptr(), None, st) == L_E["SIZE"]


# -------------------------------------------------------------------------------------------------------- density


def gaussians(n, g, cluster=0):
    """Scales over [-9, 1] (across the 1e-3 clamp at -6.9), quaternions of norm 0.1 to 10, opacity logits up to +-10;
    the first `cluster` Gaussians are wide and opaque around the origin, so samples there sum past 1."""
    means = torch.randn(n, 3, generator=g) * 2.0
    scales = torch.rand(n, 3, generator=g) * 10 - 9
    quats = torch.randn(n, 4, generator=g)
    quats = quats / quats.norm(dim=1, keepdim=True) * 10.0 ** (torch.rand(n, 1, generator=g) * 2 - 1)
    opac = torch.rand(n, 1, generator=g) * 20 - 10
    opac[n // 2: n // 2 + n // 10] = 10.0
    opac[n // 2 + n // 10: n // 2 + n // 5] = -10.0
    means[:cluster] = torch.randn(cluster, 3, generator=g) * 0.1
    scales[:cluster] = torch.rand(cluster, 3, generator=g) - 0.5
    opac[:cluster] = 10.0
    return {k: v.float().contiguous().to(DEV) for k, v in (("means", means), ("quats", quats), ("scales", scales),
                                                            ("opacities", opac))}


def density_ref(samples64, idx, p, ex=None):
    """fp64 sum of the valid terms of every sample and the bound on the fp32 kernel's pre-squash sum (module docstring).
    `idx` holds one row per sample; ids < 0 or >= n contribute nothing, as in the kernel.  `ex`: per-sample bound on the
    absolute error of the kernel's own sample position."""
    n = p["means"].shape[0]
    valid = (idx >= 0) & (idx < n)
    j = idx.clamp(0, n - 1)
    mu, s = p["means"].double()[j], p["scales"].double()[j]
    R = G.quat_to_rotmat(p["quats"].double()[j])
    inv = 1.0 / torch.exp(s).clamp(min=1e-3)
    d = samples64[:, None, :] - mu
    a = (R.transpose(-1, -2) @ d[..., None])[..., 0] * inv
    d2 = (a * a).sum(-1)
    e = 56 * EPS * d.norm(dim=-1)[..., None]
    if ex is not None:
        e = e + ex[:, None, None]
    h = (inv * e).sum(-1)
    dd2 = 2 * d2.sqrt() * h + h * h + 13 * EPS * d2
    op = torch.sigmoid(p["opacities"].double()[j][..., 0])

    def w_at(x):
        return op * torch.exp(-0.5 * x.clamp(0.0, 1e8))

    w = w_at(d2)
    dw = torch.maximum(w_at(d2 - dd2) - w, w - w_at(d2 + dd2)) + 8 * EPS * w + ATOL_W
    w, dw = torch.where(valid, w, 0.0), torch.where(valid, dw, 0.0)
    tot = w.sum(-1)
    bound = dw.sum(-1) + (idx.shape[1] - 1) * EPS * tot
    clamped_terms = int((valid & (d2 > 1e8)).sum())
    return tot, bound, clamped_terms


def judge_density(name, out, tot, bound, clamp_min=None):
    """out = max(squash(d32), clamp_min) with |d32 - tot| <= bound.  Returns (intervals of the two squash branches, the
    worst decided ratio, the number of samples whose squash decision is accepted either way)."""
    cm = -math.inf if clamp_min is None else float(np.float32(clamp_min))
    o = out.double()
    lo1, hi1 = (tot - bound).clamp(min=cm), torch.minimum(tot + bound, torch.ones_like(tot)).clamp(min=cm)
    f = tot / (tot + 1e-5)
    fb = 1e-5 * bound + 3 * EPS * f
    lo2, hi2 = f - fb, f + fb
    below, above = tot + bound < 1.0, tot - bound >= 1.0
    amb = ~below & ~above
    ok1 = (o >= lo1) & (o <= hi1)
    ok2 = (o >= lo2) & (o <= hi2)
    ok = torch.where(below, ok1, torch.where(above, ok2, ok1 | ok2))
    if not bool(ok.all()):
        i = int((~ok).nonzero()[0, 0])
        raise AssertionError(f"{name}: {int((~ok).sum())} samples outside their bound; sample {i}: got {float(o[i])!r}, "
                             f"fp64 sum {float(tot[i])!r} +- {float(bound[i]):.3g}")
    r1 = (o - tot.clamp(min=cm)).abs() / (bound + 1e-300)
    r2 = (o - f).abs() / fb
    worst = float(torch.where(below, r1, torch.where(above, r2, 0.0)).max())
    return (lo1, hi1, below | amb), (lo2, hi2, above | amb), worst, int(amb.sum())


def abi_density(samples, idx, per_row, p, clamp_min):
    out = torch.empty(samples.shape[0], dtype=torch.float32, device=DEV)
    rc = L.load().dnr_density(samples.data_ptr(), samples.shape[0], idx.data_ptr(), idx.shape[1], per_row,
                              p["means"].data_ptr(), p["scales"].data_ptr(), p["quats"].data_ptr(), p["opacities"].data_ptr(),
                              p["means"].shape[0], float(clamp_min), out.data_ptr(), SG._stream())
    assert rc == 0, rc
    return out


def density_case(g, p, rows, k, per_row):
    """Neighbour rows (cluster ids, random ids, -1 and >= n_gauss ids) and samples near the cluster, near each row's
    first Gaussian, far from it (d2 past the 1e8 clamp for the narrow ones) and anywhere."""
    n = p["means"].shape[0]
    idx = torch.randint(0, n, (rows, k), generator=g)
    kind = torch.arange(rows) % 4
    idx[kind == 0] = torch.randint(0, 40, (int((kind == 0).sum()), k), generator=g)
    bad = torch.rand(rows, k, generator=g)
    idx[bad < 0.08] = -1
    idx[(bad >= 0.08) & (bad < 0.12)] = n
    idx[(bad >= 0.12) & (bad < 0.14)] = n + 12345
    idx[rows - 1] = -1  # a row without any Gaussian
    first = idx[:, 0].clamp(0, n - 1)
    m = rows * per_row
    kind_s = kind.repeat_interleave(per_row)
    base = p["means"].cpu()[first].repeat_interleave(per_row, 0)
    ext = torch.exp(p["scales"].cpu()[first]).amax(1, keepdim=True).repeat_interleave(per_row, 0)
    u = torch.randn(m, 3, generator=g)
    u = u / u.norm(dim=1, keepdim=True)
    radius = torch.rand(m, 1, generator=g)
    samples = torch.where((kind_s == 0)[:, None], u * radius * 4.0, base + u * ext * radius * 3.0)
    samples = torch.where((kind_s == 2)[:, None], base + u * (10.0 + 990.0 * radius), samples)
    samples = torch.where((kind_s == 3)[:, None], torch.rand(m, 3, generator=g) * 8 - 4, samples)
    return samples.float().contiguous().to(DEV), idx.contiguous().to(DEV)


@pytest.mark.parametrize("per_row", [1, 3])
def test_density_per_sample_against_fp64(per_row):
    g = torch.Generator().manual_seed(70 + per_row)
    p = gaussians(3000, g, cluster=40)
    worst, amb, squashed, clamped, total = 0.0, 0, 0, 0, 0
    for k in (1, 2, 5, 16, 31, 32):
        samples, idx = density_case(g, p, 600, k, per_row)
        tot, bound, n_clamped = density_ref(samples.double(), idx.repeat_interleave(per_row, 0), p)
        for cm in (1e-4, 0.0):
            out = abi_density(samples, idx, per_row, p, cm)
            _, _, w, a = judge_density(f"density k={k} per_row={per_row} clamp={cm}", out, tot, bound, cm)
            worst, amb = max(worst, w), amb + a
        squashed += int((tot - bound >= 1.0).sum())
        clamped += n_clamped
        total += samples.shape[0]
    assert squashed > 0 and clamped > 0, (squashed, clamped)  # both the squash and the 1e8 clamp were reached
    assert amb <= 0.01 * 2 * total, amb
    report(f"density-per_row{per_row}", worst=worst, ambiguous=amb, squashed=squashed, clamped_terms=clamped, samples=total)


def test_density_inputs_reach_the_clamps():
    g = torch.Generator().manual_seed(71)
    p = gaussians(3000, g, cluster=40)
    s = p["scales"]
    assert bool((s < math.log(1e-3)).any()) and bool((s > math.log(1e-3)).any())
    qn = p["quats"].norm(dim=1)
    assert float(qn.min()) < 0.2 and float(qn.max()) > 5.0
    _, idx = density_case(g, p, 600, 16, 1)
    assert bool((idx == -1).any()) and bool((idx >= 3000).any()) and bool((idx[-1] == -1).all())


def test_get_density_and_get_sdf_against_fp64():
    """get_density (clamp 1e-4) and get_sdf = sqrt(-2 log density) through the same bound: the sdf must lie in the
    image of the accepted density interval(s), widened by the fp32 log and sqrt."""
    g = torch.Generator().manual_seed(72)
    p = gaussians(2000, g, cluster=40)
    model = types.SimpleNamespace(gauss_params=p)
    samples, idx = density_case(g, p, 800, 16, 1)
    tot, bound, _ = density_ref(samples.double(), idx, p)
    dens = SG.get_density(model, samples, idx)
    (lo1, hi1, use1), (lo2, hi2, use2), worst, amb = judge_density("get_density", dens, tot, bound, 1e-4)
    sdf = SG.get_sdf(model, samples, idx).double()

    def sdf_of(x):
        return torch.sqrt(-2.0 * torch.log(x.clamp(max=1.0)))

    tol = 8 * EPS * sdf  # fp32 log (1 ulp), sqrt and the doubling
    ok1 = use1 & (sdf >= sdf_of(hi1) - tol) & (sdf <= sdf_of(lo1) + tol)
    ok2 = use2 & (sdf >= sdf_of(hi2) - tol) & (sdf <= sdf_of(lo2) + tol)
    bad = ~(ok1 | ok2)
    assert not bool(bad.any()), f"get_sdf: {int(bad.sum())} samples outside the image of their density bound"
    report("get_density", worst=worst, ambiguous=amb)


def test_density_abi_rejections():
    lib = L.load()
    one = torch.zeros(64, device=DEV)
    oi = torch.zeros(64, dtype=torch.int64, device=DEV)
    st = SG._stream()
    args = lambda m, k, per, ng: (one.data_ptr(), m, oi.data_ptr(), k, per, one.data_ptr(), one.data_ptr(),  # noqa: E731
                                  one.data_ptr(), one.data_ptr(), ng, 0.0, one.data_ptr(), st)
    assert lib.dnr_density(*args(4, 0, 1, 4)) == L_E["SIZE"]
    assert lib.dnr_density(*args(4, 2, 0, 4)) == L_E["SIZE"]
    assert lib.dnr_density(*args(4, 2, 1, 0)) == L_E["SIZE"]
    cam = (C.c_float * 3)(0.0, 0.0, 0.0)
    for n_range in (1, 20, 22):
        rc = lib.dnr_ray_densities(one.data_ptr(), 2, oi.data_ptr(), 2, cam, one.data_ptr(), one.data_ptr(), one.data_ptr(),
                                   one.data_ptr(), 4, n_range, 3.0, one.data_ptr(), one.data_ptr(), one.data_ptr(), st)
        assert rc == L_E["OPTION"], (n_range, rc)


# ----------------------------------------------------------------------------------------------- ray densities


def ray_ref(points, idx, p, cam):
    """fp64 directions, first-neighbour std (0 when that id is not a Gaussian: the kernel's choice; the reference's
    std[idx] would read the last Gaussian for -1), and bounds on the kernel's dirs and std."""
    n = p["means"].shape[0]
    pts, c = points.double(), cam.double()
    dirs = torch.nn.functional.normalize(pts - c, dim=-1)
    g0 = idx[:, 0]
    ok = (g0 >= 0) & (g0 < n)
    j = g0.clamp(0, n - 1)
    v = torch.nn.functional.normalize(c - p["means"].double()[j], dim=-1)
    es = torch.exp(p["scales"].double()[j])
    a = es * (G.quat_to_rotmat(p["quats"].double()[j]).transpose(-1, -2) @ v[..., None])[..., 0]
    std = torch.where(ok, a.norm(dim=-1), 0.0)
    std_bound = torch.where(ok, 64 * EPS * es.sum(-1) + 4 * EPS * std, 0.0)
    return dirs, std, std_bound


def kernel_std(t):
    """The fp32 std the kernel multiplied torch's linspace by: the one value that reproduces the whole row of t."""
    lin = torch.linspace(-3.0, 3.0, 21).to(DEV)
    c = (t[:, 20].double() / 3.0).float()
    for cand in (c, torch.nextafter(c, torch.full_like(c, math.inf)), torch.nextafter(c, torch.full_like(c, -math.inf))):
        hit = (lin[None] * cand[:, None]).view(torch.int32) == t.view(torch.int32)
        c = torch.where(hit.all(1), cand, c)
    exact = ((lin[None] * c[:, None]).view(torch.int32) == t.view(torch.int32)).all(1)
    return c, exact


def abi_rays(points, idx, p, cam):
    P = points.shape[0]
    dens = torch.empty((P, 21), dtype=torch.float32, device=DEV)
    t = torch.empty((P, 21), dtype=torch.float32, device=DEV)
    dirs = torch.empty((P, 3), dtype=torch.float32, device=DEV)
    c = (C.c_float * 3)(*cam.tolist())
    rc = L.load().dnr_ray_densities(points.data_ptr(), P, idx.data_ptr(), idx.shape[1], c, p["means"].data_ptr(),
                                    p["scales"].data_ptr(), p["quats"].data_ptr(), p["opacities"].data_ptr(), p["means"].shape[0],
                                    21, 3.0, dens.data_ptr(), t.data_ptr(), dirs.data_ptr(), SG._stream())
    assert rc == 0, rc
    return dens, t, dirs


def check_rays(name, points, idx, p, cam):
    """Checks dirs, std, t and the 21 densities of every ray; returns what the level-crossing check needs."""
    dens, t, dirs = abi_rays(points, idx, p, cam)
    dirs64, std64, std_b = ray_ref(points, idx, p, cam)
    derr = float(((dirs.double() - dirs64).abs() / (8 * EPS)).max())
    assert derr <= 1.0, f"{name}: dirs off by {derr:.3g} x 8 eps"
    std32, exact = kernel_std(t)
    assert bool(exact.all()), f"{name}: {int((~exact).sum())} rays' t is not torch.linspace(-3, 3, 21) * std"
    serr = (std32.double() - std64).abs() / (std_b + 1e-300)
    assert bool(((std32.double() - std64).abs() <= std_b).all()), f"{name}: std off by {float(serr.max()):.3g} x its bound"
    no_first = (idx[:, 0] < 0) | (idx[:, 0] >= p["means"].shape[0])
    assert bool((t[no_first] == 0).all()), f"{name}: a ray without a first Gaussian has t != 0"
    lin64 = torch.linspace(-3.0, 3.0, 21, dtype=torch.float64, device=DEV)
    lin_err = (torch.linspace(-3.0, 3.0, 21).to(DEV).double() - lin64).abs()  # fp32 step: up to 8 eps at -0.3 and 0.3
    t64 = lin64[None] * std64[:, None]
    dt = lin64.abs()[None] * std_b[:, None] + lin_err[None] * std64[:, None] + 2 * EPS * t64.abs()
    pos64 = points.double()[:, None, :] + t64[..., None] * dirs64[:, None, :]
    ex = 16 * EPS * t64.abs() + dt + 2 * EPS * (points.double().abs().sum(-1, keepdim=True) + t64.abs())
    tot, bound, _ = density_ref(pos64.reshape(-1, 3), idx.repeat_interleave(21, 0), p, ex.reshape(-1))
    _, _, worst, amb = judge_density(name, dens.reshape(-1), tot, bound)
    # the squashed fp64 density and its bound; where the squash could go either way the two outcomes differ by ~1e-5
    f = tot / (tot + 1e-5)
    ref = torch.where(tot >= 1.0, f, tot)
    rb = torch.where(tot - bound >= 1.0, 1e-5 * bound + 3 * EPS * f, torch.where(tot + bound < 1.0, bound, bound + 2e-5))
    return dict(dens=dens, t=t, ref=ref.view(-1, 21), bound=rb.view(-1, 21), t64=t64, dt=dt, worst=worst, amb=amb,
                dirs=derr, std=float(serr.max()))


def check_level_crossings(name, r, level):
    """_level_crossings on the kernel's output against the fp64 pipeline.  A ray is ambiguous when a comparison it
    depends on (sample 0 under the level; every sample up to the first one above) could flip inside that sample's
    bound; every other ray must take the same keep decision and land t* within the bound carried through the
    interpolation.  Returns (ambiguous rays, worst t* ratio)."""
    L32 = float(np.float32(level))
    tot, B = r["ref"], r["bound"] + abs(L32 - level)
    keep, ts = SG._level_crossings(r["dens"], r["t"], level)
    above64 = tot > level
    first64 = torch.where(above64.any(1), above64.float().argmax(1), 20)
    upto = torch.arange(21, device=DEV)[None] <= first64[:, None]
    amb = ((tot - level).abs() <= B) & upto
    amb = amb.any(1)
    from oracle import sugar_ref as S

    keep64, ts64 = S.level_crossings(tot, r["t64"], level)
    dec = ~amb
    assert torch.equal(keep[dec], keep64[dec]), f"{name} level {level}: {int((keep != keep64)[dec].sum())} keep flips"
    both = keep & keep64 & dec
    pos = torch.cumsum(keep.long(), 0) - 1
    pos64 = torch.cumsum(keep64.long(), 0) - 1
    got, want = ts[pos[both]].double(), ts64[pos64[both]]
    f = first64[both]
    rows = both.nonzero()[:, 0]
    d0, d1 = tot[rows, f - 1], tot[rows, f]
    b0, b1 = B[rows, f - 1], B[rows, f]
    t0, t1 = r["t64"][rows, f - 1], r["t64"][rows, f]
    e0, e1 = r["dt"][rows, f - 1], r["dt"][rows, f]
    x, y = level - d0, d1 - level
    a = x / (x + y)
    da = (b0 * y + b1 * x) / ((x + y) * (x + y - b0 - b1))
    bound = da * (t1 - t0).abs() + a * (e0 + e1) + e0 + 6 * EPS * ((a * (t1 - t0)).abs() + want.abs() + t0.abs())
    ratio = (got - want).abs() / (bound + 1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    assert worst <= 1.0, f"{name} level {level}: t* off by {worst:.3g} x its bound"
    assert both.any(), f"{name} level {level}: no decided ray crosses the level"
    return int(amb.sum()), worst


def golden_rays():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "dn_sugar_a.npz"))
    p = {k: torch.from_numpy(z["in_" + k]).float().contiguous().to(DEV) for k in PARAMS}
    return (p, torch.from_numpy(z["knn_points"]).contiguous().to(DEV), torch.from_numpy(z["knn_idx"]).contiguous().to(DEV),
            torch.from_numpy(z["cam_c2w"])[:3, 3].float().to(DEV))


def synthetic_rays():
    """1000 rays (not a multiple of the 128-thread block) through the extreme Gaussians of `gaussians`, 16 neighbours
    from the k-NN, some first neighbours -1 and some later ones -1 or >= n_gauss."""
    g = torch.Generator().manual_seed(73)
    p = gaussians(2000, g, cluster=40)
    cam = torch.tensor([0.3, -7.0, 1.5], device=DEV)
    centres = p["means"][torch.randint(0, 2000, (1000,), generator=g).to(DEV)]
    points = (centres + 0.05 * torch.randn(1000, 3, generator=g).to(DEV)).contiguous()
    idx = SG.knn_gpu(p["means"], points, 16).clone()
    idx[::17, 0] = -1
    idx[5::13, 3] = -1
    idx[7::29, 8] = 2000
    return p, points, idx.contiguous(), cam


@pytest.mark.parametrize("case", ["golden", "synthetic"])
def test_ray_densities_and_level_crossings_against_fp64(case):
    p, points, idx, cam = golden_rays() if case == "golden" else synthetic_rays()
    r = check_rays(case, points, idx, p, cam)
    amb = {}
    worst_t = 0.0
    for level in (0.1, 0.3, 0.5):
        a, w = check_level_crossings(case, r, level)
        amb[str(level)], worst_t = a, max(worst_t, w)
        assert a <= max(3, 0.02 * points.shape[0]), (case, level, a)
    report(f"rays-{case}", rays=int(points.shape[0]), density_worst=r["worst"], density_ambiguous=r["amb"], dirs_worst=r["dirs"],
           std_worst=r["std"], tstar_worst=worst_t, level_ambiguous=amb)
