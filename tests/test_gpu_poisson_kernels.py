"""Screened Poisson (csrc/poisson.cu) per node, per cycle and per vertex against oracle/poisson_ref.py in fp64.

  * the splat (`dnr_poisson_splat`) at depths 4 to 10 on a sphere with a denser half, an axis-aligned plane and a box
    room on cell faces, a lattice of cell faces and centres with a cell size whose reciprocal is inexact, samples on the
    outer walls (scale 1), 10^5 duplicates in one cell, a single sample and, at depth 10, the 8 corner cells: density,
    a_p (input order), area_scale, S, the three face grids and the colour grid, each node within its fp32 bound, every
    node the samples cannot reach (and every wall face) exactly 0, two runs bit-identical;
  * the multigrid (`dnr_poisson_solve`), one V-cycle at a time from the kernel's own iterate, at depths 4 to 7, sigma = 0
    and the default screening; the reported residual against the fp64 residual of the kernel's own chi at depths 4 to
    10; the stop rule;
  * the steps after the solve (`poisson_solve_points`): iso-value, vertex densities and colours, and the mesh.

The case builders and acceptance rules need no GPU: tests/test_poisson_ref_cpu.py runs them on the oracle to show that
each restated kernel mistake (poisson_ref.SLIPS) fails them by at least 10x.

Bounds (EPS = 2^-24, each first order with the safety factor poisson_ref.BOUND_K = 2):
  * a splat node: the m_n sequential fp32 additions of the node's thread and the terms' own roundings,
    (m_n + 6) T_n + 2 W_n (`poisson_ref.splat_bound`); the density adds 7 EPS per 8-child sum; the colour grid sums in
    double, so only its terms' roundings count (`poisson_ref.color_bound`); rho_p, a_p and area_scale carry the
    density's bound through the interpolation and the fp32 rounding of the sample's level-2 coordinate
    (`poisson_ref.sample_weights`);
  * a V-cycle: CYCLE_ROUNDINGS roundings, each relative to the largest value the cycle touches at a finest node
    (`cycle_bound`);
  * the reported residual: the fp32 evaluation floor of ||b - A chi|| (`poisson_ref.residual_floor`);
  * a trilinear read (`grid_sample`): 12 roundings of the weighted corner sum and 4 of the fp32 weights (`read_bound`).
"""
import math

import numpy as np
import pytest
import torch

from oracle import poisson_ref as P

F32 = np.float32
EPS = P.EPS
K = P.BOUND_K
# a finest node in one cycle: PRE + POST sweeps, each a residual of 8 roundings (six neighbour differences, the
# screening, the subtraction) and 2 for the update; the prolongation's 8-term sum (12); the coarse correction carries
# its own levels' roundings relative to its size, which the prolongation (a convex combination) does not grow
CYCLE_ROUNDINGS = (P.PRE_SWEEPS + P.POST_SWEEPS) * 10 + 12
WORST = {}  # bound name -> largest fraction used, printed by the last test


def _used(name, frac):
    WORST[name] = max(WORST.get(name, 0.0), float(frac))


def _unit(g, n):
    v = g.normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)


def _grid_for(points, depth, scale=1.1):
    """poisson_grid's cube, as the fp32 struct holds it."""
    o, h = P.grid_for(points, depth, scale)
    return tuple(float(F32(x)) for x in o), float(F32(h))


# ------------------------------------------------------------------------------------------------------ clouds
def cloud(name, depth):
    """(points, normals, colours, origin, cell) of a named cloud at a depth; host arrays, seeded."""
    from tests.test_gpu_poisson import _sphere, _torus

    R = 1 << depth
    g = np.random.default_rng(depth * 31 + len(name))
    if name == "sphere":  # the z > 0 half 10x denser
        p, n = _sphere(2500, dense_half=10, seed=depth)
        o, h = _grid_for(p, depth)
    elif name == "torus":
        p, n = _torus(30000, seed=depth)
        o, h = _grid_for(p, depth)
    elif name == "sphere30k":
        p, n = _sphere(30000, seed=depth)
        o, h = _grid_for(p, depth)
    elif name == "plane":  # z = 0 is the box's centre: a cell face
        p = np.concatenate([g.uniform(-0.5, 0.5, (20000, 2)), np.zeros((20000, 1))], 1).astype(F32)
        n = np.tile(np.array([[0, 0, 1]], F32), (20000, 1))
        o, h = _grid_for(p, depth)
    elif name == "box":  # the walls of [-0.5, 0.5]^3 at u = R/4 and 3R/4, normals inward
        q = g.uniform(-0.5, 0.5, (6, 3000, 3))
        n = np.zeros_like(q)
        for f in range(6):
            q[f, :, f // 2] = 0.5 if f & 1 else -0.5
            n[f, :, f // 2] = -1.0 if f & 1 else 1.0
        p, n = q.reshape(-1, 3).astype(F32), n.reshape(-1, 3).astype(F32)
        o, h = (-1.0, -1.0, -1.0), 2.0 / R
    elif name == "lattice":  # every coordinate on a cell face or centre, 0 .. R; 1/h is inexact in fp64
        h = 3.0 * 2.0 ** -(depth + 2)
        o = (-R * h / 2,) * 3
        p = (np.array(o) + g.integers(0, 2 * R + 1, (20000, 3)) * (h / 2)).astype(F32)
        n = _unit(g, p.shape[0])
    elif name == "scale1":  # the extreme samples on the outer walls: the clamp and the dropped wall flux
        p, n = _sphere(15000, seed=depth)
        o, h = _grid_for(p, depth, 1.0)
    elif name == "dups":  # 10^5 copies of one sample in one cell, on a sphere of 2000
        s, sn = _sphere(2000, seed=depth)
        p = np.concatenate([s, np.repeat(s[:1], 100000, 0)])
        n = np.concatenate([sn, _unit(g, 100000)])
        o, h = _grid_for(p, depth)
    elif name == "single":
        p = np.array([[0.37, 0.61, 0.18]], F32)
        n = _unit(g, 1)
        o, h = (0.0, 0.0, 0.0), 1.0 / R
    elif name == "corners":  # 50 samples in each of the 8 corner cells
        c = np.array(list(np.ndindex(2, 2, 2))) * (R - 1)
        p = ((np.repeat(c, 50, 0) + g.uniform(0, 1, (400, 3))) / R).astype(F32)
        n = _unit(g, 400)
        o, h = (0.0, 0.0, 0.0), 1.0 / R
    else:
        raise KeyError(name)
    col = g.uniform(0, 1, p.shape).astype(F32)
    return np.ascontiguousarray(p, F32), np.ascontiguousarray(n, F32), col, tuple(float(F32(x)) for x in o), float(F32(h))


SPLAT_CASES = ([("sphere", d) for d in range(4, 11)] + [("plane", 5), ("plane", 9), ("box", 6), ("box", 8),
               ("lattice", 4), ("lattice", 7), ("lattice", 10), ("scale1", 5), ("scale1", 9), ("dups", 6),
               ("dups", 9), ("single", 4), ("single", 8), ("corners", 10)])
SPARSE_FROM = 8  # the dense oracle up to depth 7, the nodes the samples reach above it
GRIDS = ("screen", "face0", "face1", "face2")


# ------------------------------------------------------------------------------------------------- splat rule
def _frac(diff, bound):
    """Largest |diff| / bound; a nonzero diff against a zero bound counts as inf."""
    diff, bound = np.abs(diff), np.asarray(bound)
    if diff.size == 0:
        return 0.0
    bad = (bound <= 0) & (diff > 0)
    if bad.any():
        return math.inf
    return float((diff / np.where(bound > 0, bound, 1.0)).max())


def _at_nodes(g, size, x):
    """x (per entry of the oracle dict g) as a dense array of `size` nodes."""
    if "idx" not in g:
        return x
    out = np.zeros((size,) + x.shape[1:])
    out[g["idx"]] = x
    return out


def check_splat(got, case, want=None):
    """(failures, {bound: worst fraction}) of splat outputs `got` on a case:
    got = {"weights" [n], "area_scale", "density" [(R/4)^3], "color" [(R/4)^3, 4] and, per finest grid,
    (values at want[grid]["idx"] or at every node, the grid's nonzero count)}.  want: `splat_nodes` of the case with
    got's own weights (computed when None), so S, the faces and the colours are compared at the kernel's a_p."""
    p, n, col, o, h, depth = case
    R = 1 << depth
    if want is None:
        want = P.splat_nodes(p, n, col, o, h, depth, weights=got["weights"], sparse=depth >= SPARSE_FROM)
    dens, dbound = P.density(want["count"], R)
    sw = P.sample_weights(*want["cells"], dens, dbound, R)
    worst = {"density": _frac(got["density"] - dens.reshape(-1), dbound.reshape(-1)),
             "a_p": _frac(got["weights"] - sw["a"], sw["a_bound"]),
             "area_scale": _frac(got["area_scale"] - sw["area_scale"], sw["area_bound"])}
    fails = []
    for g in GRIDS:
        vals, nnz = got[g]
        w = want[g]
        key = "faces" if g.startswith("face") else g
        worst[key] = max(worst.get(key, 0.0), _frac(vals - w["val"], P.splat_bound(w)))
        if (vals[w["T"] == 0] != 0).any():
            fails.append(f"{g}: a node no sample reaches is not 0")
        if nnz != np.count_nonzero(vals):
            fails.append(f"{g}: {nnz - np.count_nonzero(vals)} nonzero nodes outside the samples' reach")
    wc, N4 = want["color"], (R >> 2) ** 3
    worst["color"] = _frac(got["color"] - _at_nodes(wc, N4, wc["val"]), _at_nodes(wc, N4, P.color_bound(wc)))
    fails += [f"{k}: {v:.3g} of its bound" for k, v in worst.items() if v > 1]
    return fails, worst


def _splat_gpu(case):
    from dn_splatter_b200.poisson import PoissonGrid, poisson_splat

    p, n, col, o, h, depth = case
    pt, nt, ct = (torch.from_numpy(x).cuda() for x in (p, n, col))
    return poisson_splat(pt, nt, ct, PoissonGrid(o, h, depth))


def gpu_splat_got(case):
    """(check_splat's `got` from the kernel, gathered on the device at the oracle's nodes from SPARSE_FROM on, whether a
    second run was bit-identical, the oracle's `want`)."""
    p, n, col, o, h, depth = case
    R = 1 << depth
    a, b = _splat_gpu(case), _splat_gpu(case)
    same = all(torch.equal(a[k], b[k]) for k in a)
    del b
    got = {"weights": a["weights"].double().cpu().numpy(), "area_scale": float(a["area_scale"]),
           "density": a["density"].double().cpu().numpy(), "color": a["colors"].double().cpu().numpy()}
    grids = {"screen": a["screen"], "face0": a["faces"][0], "face1": a["faces"][1], "face2": a["faces"][2]}
    want = P.splat_nodes(p, n, col, o, h, depth, weights=got["weights"], sparse=depth >= SPARSE_FROM)
    if depth >= SPARSE_FROM:
        for g, t in grids.items():
            idx = torch.from_numpy(want[g]["idx"]).cuda()
            got[g] = (t.index_select(0, idx).double().cpu().numpy(), int(torch.count_nonzero(t)))
    else:
        for g, t in grids.items():
            got[g] = (t.double().cpu().numpy(), int(torch.count_nonzero(t)))
    walls = [a["faces"][ax].view(R, R, R).select(ax, R - 1) for ax in range(3)]
    got["walls_zero"] = all(int(torch.count_nonzero(w)) == 0 for w in walls)
    return got, same, want


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("name,depth", SPLAT_CASES)
def test_splat_per_node(name, depth):
    case = cloud(name, depth) + (depth,)
    got, same, want = gpu_splat_got(case)
    assert same, "two runs of the splat differ"
    assert got["walls_zero"]
    fails, worst = check_splat(got, case, want)
    print(f"{name} depth {depth}: n {case[0].shape[0]}; " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert not fails, fails
    for k, v in worst.items():
        _used(f"splat {k}", v)



# --------------------------------------------------------------------------------------------------- V-cycles
MG_CASES = [(c, d) for d in (4, 5, 6) for c in ("torus", "sphere30k", "wall")] + [("sphere30k", 7)]
MG_ALPHAS = (0.0, 4.0)  # sigma = 0 and the default point weight
MG_CYCLES = 3


def mg_inputs(name, depth, splat):
    """(screen [R,R,R], faces [3,R,R,R], area_scale) in fp32 of a multigrid case.  splat(case) -> (screen, faces,
    area_scale) is the kernel's (or, without a GPU, the oracle's rounded to fp32).  "wall": the sphere's screening with
    one large isolated flux on the last interior x face and a smaller one on the wall face behind it, which the
    right-hand side reads as stored: a net source, so at sigma = 0 the coarsest level's mean removal matters."""
    S, V, area = splat(cloud("sphere30k" if name == "wall" else name, depth) + (depth,))
    if name == "wall":
        R = 1 << depth
        V = np.zeros_like(V)
        V[0, R - 2, R // 2, R // 3] = F32(1000.0)
        V[0, R - 1, R // 2, R // 3] = F32(500.0)
    return S, V, area


def cycle_bound(prev, u, m_prev, m_now):
    """K EPS CYCLE_ROUNDINGS times the magnitudes a finest node meets in the cycle: the iterate it starts from (the
    kernel's own at sigma = 0 carries the mean m_prev the returned chi had removed), the update, and the mean the final
    removal subtracts."""
    return K * EPS * CYCLE_ROUNDINGS * (np.abs(prev).max() + abs(m_prev) + np.abs(u).max() + abs(m_now))


def check_cycles(chis, S, V, sigma, slip=None):
    """(failures, worst fraction) of the iterates chis[c] (c = 0 .. MG_CYCLES, chis[0] = 0) against one oracle V-cycle
    (with `slip`) from chis[c - 1] each; at sigma = 0 both sides have their mean removed."""
    b = P.rhs(V.astype(np.float64))
    S = S.astype(np.float64)
    worst, m = 0.0, 0.0
    fails = []
    for c in range(1, len(chis)):
        prev = chis[c - 1].astype(np.float64)
        want = P.vcycle(prev, b, S, sigma, slip)
        u = want - prev
        m_now = m + (float(u.mean()) if float(F32(sigma)) == 0 else 0.0)
        if float(F32(sigma)) == 0:
            want = want - want.mean()
        frac = _frac(chis[c].astype(np.float64) - want, cycle_bound(prev, u, m, m_now))
        worst = max(worst, frac)
        if frac > 1:
            fails.append(f"cycle {c}: {frac:.3g} of its bound")
        m = m_now
    return fails, worst


def _gpu_mg_splat(case):
    s = _splat_gpu(case)
    R = 1 << case[-1]
    return (s["screen"].cpu().numpy().reshape(R, R, R), s["faces"].cpu().numpy().reshape(3, R, R, R),
            float(s["area_scale"]))


def _solve(depth, S, V, sigma, cycles, tol=0.0):
    from dn_splatter_b200.poisson import PoissonGrid, poisson_solve

    R = 1 << depth
    chi, hist = poisson_solve(PoissonGrid((0.0, 0.0, 0.0), 1.0, depth), torch.from_numpy(S.reshape(-1)).cuda(),
                              torch.from_numpy(V.reshape(3, -1)).cuda(), sigma, tol=tol, max_cycles=cycles)
    return chi.view(R, R, R), hist


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("alpha", MG_ALPHAS)
@pytest.mark.parametrize("name,depth", MG_CASES)
def test_vcycle_per_node(name, depth, alpha):
    S, V, area = mg_inputs(name, depth, _gpu_mg_splat)
    sigma = float(F32(alpha * area))
    chis = [np.zeros(S.shape, F32)]
    for c in range(1, MG_CYCLES + 1):
        chi, hist = _solve(depth, S, V, sigma, c)
        assert len(hist) == c + 1
        chis.append(chi.cpu().numpy())
    again, _ = _solve(depth, S, V, sigma, MG_CYCLES)
    assert np.array_equal(again.cpu().numpy(), chis[-1]), "two runs of the solve differ"
    fails, worst = check_cycles(chis, S, V, sigma)
    print(f"{name} depth {depth} alpha {alpha}: worst {worst:.3g} of the per-cycle bound")
    assert not fails, fails
    _used("v-cycle", worst)



# ----------------------------------------------------------------------------------------- reported residual
def _residual_torch(chi, faces, screen, sigma, mean_removed, slab=32):
    """(||b - A chi||, ||b||, ||floor||) in float64 on the device, slab by slab along x: the 7-point stencil of
    poisson_ref.residual and the per-node floor of poisson_ref.residual_floor, for grids too large for the host."""
    R = chi.shape[0]
    V, S = faces.view(3, R, R, R), screen.view(R, R, R)
    r2 = b2 = f2 = 0.0
    for i0 in range(0, R, slab):
        i1 = min(R, i0 + slab)
        lo, hi = max(0, i0 - 1), min(R, i1 + 1)
        x = chi[lo:hi].double()
        acc, dsum, asum = torch.zeros_like(x), torch.zeros_like(x), torch.zeros_like(x)
        for a in range(3):
            m = x.shape[a] - 1
            d = torch.diff(x, dim=a)
            acc.narrow(a, 0, m).sub_(d)
            acc.narrow(a, 1, m).add_(d)
            dsum.narrow(a, 0, m).add_(d.abs())
            dsum.narrow(a, 1, m).add_(d.abs())
            if mean_removed:
                e = x.narrow(a, 0, m).abs() + x.narrow(a, 1, m).abs()
                asum.narrow(a, 0, m).add_(e)
                asum.narrow(a, 1, m).add_(e)
        k = i0 - lo
        x, acc, dsum, asum = (t[k:k + i1 - i0] for t in (x, acc, dsum, asum))
        b, vsum = torch.zeros_like(x), torch.zeros_like(x)
        for a in range(3):
            cur = V[a, i0:i1].double()
            below = torch.zeros_like(cur)
            if a == 0:
                below[1:] = cur[:-1]
                if i0 > 0:
                    below[0] = V[0, i0 - 1].double()
            else:
                below.narrow(a, 1, R - 1).copy_(cur.narrow(a, 0, R - 1))
            b -= cur - below
            vsum += cur.abs() + below.abs()
        sx = sigma * S[i0:i1].double() * x
        r = b - acc - sx
        per = K * EPS * (6 * vsum + 8 * dsum + 3 * sx.abs() + 2 * asum)
        r2, b2, f2 = r2 + float((r * r).sum()), b2 + float((b * b).sum()), f2 + float((per * per).sum())
    return math.sqrt(r2), math.sqrt(b2), math.sqrt(f2)


def residual_check(chi, faces, screen, sigma, depth, host=None):
    """(fp64 relative residual of chi, its fp32 evaluation floor): the oracle up to depth 8, torch on the device above.
    host: (b, S, face sums) of the oracle, computed here when None."""
    R = 1 << depth
    chi = chi.view(R, R, R)
    mean_removed = float(F32(sigma)) == 0
    if depth <= 8:
        if host is None:
            V = faces.cpu().numpy().reshape(3, R, R, R).astype(np.float64)
            host = P.rhs(V), screen.cpu().numpy().reshape(R, R, R).astype(np.float64), P.face_sums(V)
        b, S, vsum = host
        x = chi.cpu().numpy().reshape(R, R, R).astype(np.float64)
        return P.relative_residual(x, b, S, sigma), P.residual_floor(x, b, S, sigma, vsum, mean_removed)
    r, b, f = _residual_torch(chi, faces, screen, float(F32(sigma)), mean_removed)
    return r / b, f / b


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("depth", range(4, 11))
def test_reported_residual(depth):
    from dn_splatter_b200.poisson import PoissonGrid, poisson_solve

    case = cloud("sphere30k", depth) + (depth,)
    s = _splat_gpu(case)
    grid = PoissonGrid((0.0, 0.0, 0.0), 1.0, depth)
    host = None
    if depth <= 8:
        R = 1 << depth
        V = s["faces"].cpu().numpy().reshape(3, R, R, R).astype(np.float64)
        host = P.rhs(V), s["screen"].cpu().numpy().reshape(R, R, R).astype(np.float64), P.face_sums(V)
        del V
    for alpha in MG_ALPHAS:
        sigma = float(F32(alpha * float(s["area_scale"])))
        full = None
        for c in range(MG_CYCLES, 0, -1):
            chi, hist = poisson_solve(grid, s["screen"], s["faces"], sigma, tol=0.0, max_cycles=c)
            assert len(hist) == c + 1 and hist[0] == 1.0
            full = full or hist
            assert hist == full[:c + 1], "the history is not reproduced by a shorter run"
            rel, floor = residual_check(chi, s["faces"], s["screen"], sigma, depth, host)
            frac = abs(hist[c] - rel) / (floor * (1 + rel) + 4 * EPS * rel)
            print(f"depth {depth} alpha {alpha} cycle {c}: reported {hist[c]:.6e} fp64 {rel:.6e} floor {floor:.2e} "
                  f"({frac:.3g} of it)")
            assert frac <= 1
            _used("reported residual", frac)
            del chi
    del s
    torch.cuda.empty_cache()



@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_stop_rule():
    depth = 6
    s = _splat_gpu(cloud("sphere30k", depth) + (depth,))
    S, V = s["screen"].cpu().numpy(), s["faces"].cpu().numpy()
    sigma = float(F32(4.0 * float(s["area_scale"])))
    R = 1 << depth
    _, full = _solve(depth, S, V, sigma, 8)
    assert len(full) == 9 and all(full[i + 1] < full[i] for i in range(8))
    for k in (2, 5):
        for tol in (full[k], float(np.nextafter(F32(full[k]), F32(0)))):
            chi, hist = _solve(depth, S, V, sigma, 30, tol)
            stop = next(c for c in range(1, 9) if full[c] <= tol)  # the first cycle at or below tol
            assert len(hist) == stop + 1 and hist == full[:stop + 1], (k, tol, hist)
            # the decision is the kernel's fp32 estimate; the fp64 residual agrees with it up to the floor
            rel, floor = residual_check(chi, s["faces"], s["screen"], sigma, depth)
            assert rel <= tol + floor * (1 + rel) + 4 * EPS * rel
    chi, hist = _solve(depth, S, V, sigma, 5, 0.0)
    assert len(hist) == 6  # max_cycles is honoured
    chi, hist = _solve(depth, S, np.zeros_like(V), sigma, 5, 1e-5)
    assert hist == [0.0] and int(torch.count_nonzero(chi)) == 0
    chi, hist = _solve(depth, S, np.zeros_like(V), 0.0, 5, 1e-5)
    assert hist == [0.0] and int(torch.count_nonzero(chi)) == 0 and chi.shape == (R, R, R)


# --------------------------------------------------------------------------------------------- after the solve
def read_bound(values, origin, cell, points):
    """K EPS (12 sum_c w_c |v_c| + 4 max_c |v_c|) per point of grid_sample's fp32 read of values (corner weights from
    an fp32 t: three products, 1 - t; eight products and sums)."""
    cs = P._corners(np.abs(np.asarray(values, np.float64)), (np.asarray(points, np.float64) - np.asarray(origin)) / cell)
    s = sum((w[:, None] if v.ndim == 2 else w) * v for w, v in cs)
    top = np.max([v for _, v in cs], axis=0)
    return K * EPS * (12 * s + 4 * top)


def check_after_solve(r, weights, points, slip=None):
    """(failures, worst) of a PoissonResult-like r (grid, chi [R,R,R], iso, vertices, densities, colours, the density
    and colour grids, as host arrays) against the fp64 reads of the kernel's own grids."""
    (o, h, depth), chi = r["grid"], r["chi"].astype(np.float64)
    R4 = (1 << depth) >> 2
    at = P.sample(chi, o, h, points)
    iso = float((at * weights).sum() / points.shape[0])
    iso_b = float((read_bound(chi, o, h, points) * weights).sum() / points.shape[0]) + 2 * EPS * abs(iso)
    dens, cgrid = r["density"].reshape(R4, R4, R4), r["color_grid"].reshape(R4, R4, R4, 4)
    v = r["vertices"].astype(np.float64)
    d, col = P.vertex_attributes(dens, cgrid, o, h, v, slip)
    db = read_bound(dens, o, 4 * h, v)
    cs = P.sample(cgrid, o, 4 * h, v)
    cb = read_bound(cgrid, o, 4 * h, v)
    den = np.maximum(cs[:, 3:], 1e-30)
    colb = (cb[:, :3] + np.abs(col) * cb[:, 3:]) / den + 2 * EPS * np.abs(col)
    worst = {"iso": _frac(r["iso"] - iso, iso_b), "vertex density": _frac(r["densities"] - d, db),
             "vertex colour": _frac(r["colors"] - col, colb)}
    return [f"{k}: {x:.3g} of its bound" for k, x in worst.items() if x > 1], worst


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
@pytest.mark.parametrize("depth", [5, 6, 7])
def test_after_the_solve_per_vertex(depth):
    from dn_splatter_b200.mesh import marching_cubes
    from dn_splatter_b200.poisson import poisson_solve_points

    p, n, col, _, _ = cloud("sphere", depth)
    pt, nt, ct = (torch.from_numpy(x).cuda() for x in (p, n, col))
    res = poisson_solve_points(pt, nt, ct, depth=depth)
    mc = marching_cubes(res.chi, res.iso, [x + 0.5 * res.grid.cell for x in res.grid.origin], res.grid.cell)
    o, h = tuple(float(F32(x)) for x in res.grid.origin), float(F32(res.grid.cell))  # as the kernels read them
    s = _splat_gpu((p, n, col, o, h, depth))
    assert torch.equal(mc.vertices, res.mesh.vertices) and torch.equal(mc.faces, res.mesh.faces)
    assert res.mesh.faces.shape[0] > 1000
    r = {"grid": (o, h, depth), "chi": res.chi.cpu().numpy(), "iso": res.iso,
         "vertices": res.mesh.vertices.cpu().numpy(), "densities": res.densities.cpu().numpy(),
         "colors": res.mesh.colors.cpu().numpy(), "density": s["density"].cpu().numpy(),
         "color_grid": s["colors"].cpu().numpy()}
    fails, worst = check_after_solve(r, s["weights"].double().cpu().numpy(), p)
    print(f"depth {depth}: V {r['vertices'].shape[0]}; " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert not fails, fails
    for k, v in worst.items():
        _used(k, v)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_zz_report_worst_fraction_of_each_bound():
    """Prints the largest fraction of each bound the tests before this one used (pytest -s shows it)."""
    print("\nworst fraction of each bound used:", {k: round(v, 4) for k, v in sorted(WORST.items())})
