"""oracle/poisson_ref.py's per-node splat and V-cycle, the rules tests/test_gpu_poisson_kernels.py holds the kernels to.

  * the per-node splat (values, T_n, W_n, m_n) equals a scalar loop over each node's 27 cells, and the sparse splat
    equals the dense one;
  * the V-cycle equals a scalar per-node restatement, and iterated from zero it converges to the direct solve;
  * each kernel mistake the oracle restates (poisson_ref.SLIPS) leaves the GPU test's bound on the GPU test's own cases
    by at least 10x; the multigrid ones still pass the converged-chi check of test_gpu_poisson.py, which is why the
    per-cycle test exists.
"""
import math

import numpy as np
import pytest

from oracle import poisson_ref as P
from tests import test_gpu_poisson_kernels as T

F32 = np.float32


def _case(name, depth):
    return T.cloud(name, depth) + (depth,)


# ---------------------------------------------------------------------------------------------- scalar loops
def scalar_splat(c, f, R, vals, off, wall_axis=None):
    """Per node: (value, T, W, m) by walking the samples of its (up to 27) cells, one Python float at a time."""
    cells = {}
    for q in range(c.shape[0]):
        cells.setdefault(tuple(int(x) for x in c[q]), []).append(q)
    out = np.zeros((R, R, R, 4))
    for i, j, k in np.ndindex(R, R, R):
        if wall_axis is not None and (i, j, k)[wall_axis] == R - 1:
            continue
        for ci in range(max(i - 1, 0), min(i + 2, R)):
            for cj in range(max(j - 1, 0), min(j + 2, R)):
                for ck in range(max(k - 1, 0), min(k + 2, R)):
                    for q in cells.get((ci, cj, ck), []):
                        t = [max(0.0, 1.0 - abs(float(cc) + float(f[q, a]) - nn - off[a]))
                             for a, (cc, nn) in enumerate(((ci, i), (cj, j), (ck, k)))]
                        v = float(vals[q])
                        out[i, j, k, 0] += v * t[0] * t[1] * t[2]
                        out[i, j, k, 1] += abs(v) * t[0] * t[1] * t[2]
                        out[i, j, k, 2] += abs(v) * (t[0] * t[1] + t[1] * t[2] + t[2] * t[0])
                        out[i, j, k, 3] += 1
    return out


def test_splat_nodes_equal_a_scalar_loop():
    depth, R = 4, 16
    g = np.random.default_rng(0)
    p = np.concatenate([g.uniform(0, 1, (40, 3)), g.integers(0, 33, (20, 3)) / 32.0]).astype(F32)  # faces, centres
    n = T._unit(g, p.shape[0])
    col = g.uniform(0, 1, p.shape).astype(F32)
    a = g.uniform(0.5, 2, p.shape[0])
    got = P.splat_nodes(p, n, col, (0.0, 0.0, 0.0), 1.0 / R, depth, weights=a)
    c, f = got["cells"]
    assert np.array_equal(f, f.astype(F32)) and (f == 0).any() and (f == 0.5).any()
    for name, vals, off, wall in (("count", np.ones(p.shape[0]), (0.5,) * 3, None), ("screen", a, (0.5,) * 3, None),
                                  ("face1", a * n[:, 1], (0.5, 1.0, 0.5), 1)):
        want = scalar_splat(c, f, R, vals, off, wall).reshape(-1, 4)
        gg = got[name]
        for col_i, key in enumerate(("val", "T", "W")):
            np.testing.assert_allclose(gg[key], want[:, col_i], rtol=1e-12, atol=1e-15)
        reached = want[:, 3] > 0
        assert (gg["m"][reached] >= want[reached, 3]).all()  # m_n counts every gathered sample, reaching or not
    # m_n against the 27 cells directly
    cnt = np.zeros((R + 2,) * 3)
    np.add.at(cnt, tuple((c + 1).T), 1)
    box = sum(cnt[1 + d[0]:R + 1 + d[0], 1 + d[1]:R + 1 + d[1], 1 + d[2]:R + 1 + d[2]] for d in P._OFFS)
    assert np.array_equal(got["screen"]["m"], box.reshape(-1))
    want = scalar_splat(c >> 2, ((c & 3) + f) / 4.0, R // 4, a * col[:, 0], (0.5,) * 3).reshape(-1, 4)
    np.testing.assert_allclose(got["color"]["val"][:, 0], want[:, 0], rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("name,depth", [("sphere", 4), ("lattice", 5), ("scale1", 5), ("single", 4)])
def test_sparse_splat_equals_dense(name, depth):
    p, n, col, o, h, _ = _case(name, depth)
    R = 1 << depth
    d = P.splat_nodes(p, n, col, o, h, depth)
    s = P.splat_nodes_sparse(p, n, col, o, h, depth)
    for g in ("count", "screen", "face0", "face1", "face2", "color"):
        Rg = R >> 2 if g == "color" else R
        idx = s[g]["idx"]
        for key in ("val", "T", "W", "m"):
            np.testing.assert_array_equal(s[g][key], d[g][key][idx])
        rest = np.setdiff1d(np.arange(Rg ** 3), idx)
        assert not d[g]["val"][rest].any() and not d[g]["T"][rest].any() and not d[g]["W"][rest].any()


def test_per_node_splat_equals_the_whole_grid_oracle():
    p, n, col, o, h, depth = _case("sphere", 5)
    R = 1 << depth
    new = P.splat_nodes(p, n, col, o, h, depth)
    old = P.splat(p, n, col, o, h, depth)
    dens, db = P.density(new["count"], R)
    sw = P.sample_weights(*new["cells"], dens, db, R)
    # the two differ only in the fp32 rounding of the fractions
    assert np.abs(dens - old["density"]).max() <= 1e-6 * dens.max()
    assert np.abs(sw["a"] - old["weights"]).max() <= 1e-6 * sw["a"].max()
    assert abs(sw["area_scale"] / old["area_scale"] - 1) <= 1e-6
    new2 = P.splat_nodes(p, n, col, o, h, depth, weights=old["weights"])
    assert np.abs(P._dense(new2["screen"], R) - old["screen"]).max() <= 1e-6 * old["screen"].max()
    faces = np.stack([P._dense(new2[f"face{a}"], R) for a in range(3)])
    assert np.abs(faces - old["faces"]).max() <= 1e-6 * np.abs(old["faces"]).max()
    assert np.abs(P._dense(new2["color"], R // 4) - old["colors"]).max() <= 1e-6 * old["colors"].max()


def scalar_vcycle(chi, b, S, sigma):
    """One V-cycle node by node in Python floats, every stage as poisson.cu's kernels state it."""
    sigma = float(F32(sigma))
    R0 = chi.shape[0]
    levels = []
    Sl = S.astype(np.float64)
    R = R0
    while True:
        levels.append(Sl)
        if R == P.COARSEST_R:
            break
        R //= 2
        Sn = np.zeros((R, R, R))
        for I, J, Kk in np.ndindex(R, R, R):
            Sn[I, J, Kk] = sum(Sl[2 * I + (c >> 2), 2 * J + ((c >> 1) & 1), 2 * Kk + (c & 1)] for c in range(8))
        Sl = Sn
    L = len(levels) - 1

    def res(x, bb, Sx, cl, i, j, k):
        R = x.shape[0]
        acc, nb = 0.0, 0
        for d in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)):
            q = (i + d[0], j + d[1], k + d[2])
            if all(0 <= v < R for v in q):
                acc += x[i, j, k] - x[q]
                nb += 1
        s = sigma * Sx[i, j, k]
        return bb[i, j, k] - cl * acc - s * x[i, j, k], cl * nb + s

    def sweep(x, bb, Sx, cl):
        for color in (0, 1):
            for i, j, k in np.ndindex(*x.shape):
                if (i + j + k) & 1 == color:
                    r, dg = res(x, bb, Sx, cl, i, j, k)
                    if dg > 0:
                        x[i, j, k] += r / dg

    def cycle(l, x, bb):
        cl = 2.0 ** l
        if l == L:
            bb = bb.copy()
            if sigma == 0:
                bb -= sum(bb.reshape(-1)) / bb.size
            x = np.zeros_like(bb)
            for _ in range(P.COARSE_SWEEPS):
                sweep(x, bb, levels[l], cl)
            if sigma == 0:
                x -= sum(x.reshape(-1)) / x.size
            return x
        x = x.copy()
        for _ in range(P.PRE_SWEEPS):
            sweep(x, bb, levels[l], cl)
        Rc = x.shape[0] // 2
        bc = np.zeros((Rc, Rc, Rc))
        for I, J, Kk in np.ndindex(Rc, Rc, Rc):
            bc[I, J, Kk] = sum(res(x, bb, levels[l], cl, 2 * I + (c >> 2), 2 * J + ((c >> 1) & 1), 2 * Kk + (c & 1))[0]
                               for c in range(8))
        xc = cycle(l + 1, np.zeros_like(bc), bc)
        for i, j, k in np.ndindex(*x.shape):
            lo, hi, t = [], [], []
            for pp in (i, j, k):
                q = pp >> 1
                if pp & 1:
                    lo.append(q), hi.append(min(q + 1, Rc - 1)), t.append(0.25)
                else:
                    lo.append(max(q - 1, 0)), hi.append(q), t.append(0.75)
            v = 0.0
            for c in range(8):
                w, idx = 1.0, []
                for a in range(3):
                    bit = (c >> (2 - a)) & 1
                    w *= t[a] if bit else 1.0 - t[a]
                    idx.append(hi[a] if bit else lo[a])
                v += w * xc[tuple(idx)]
            x[i, j, k] += v
        for _ in range(P.POST_SWEEPS):
            sweep(x, bb, levels[l], cl)
        return x

    return cycle(0, chi.astype(np.float64), b.astype(np.float64))


@pytest.mark.parametrize("alpha", [0.0, 4.0])
def test_vcycle_equals_a_scalar_loop(alpha):
    S, V, area = T.mg_inputs("torus", 4, oracle_mg_splat)
    b = P.rhs(V.astype(np.float64))
    sigma = alpha * area
    chi = np.random.default_rng(1).normal(size=b.shape)
    want = scalar_vcycle(chi, b, S, sigma)
    got = P.vcycle(chi, b, S, sigma)
    assert np.abs(got - want).max() <= 1e-11 * np.abs(want).max()
    np.testing.assert_allclose(P.rhs(V.astype(np.float64)), -P.divergence(V.astype(np.float64)), atol=1e-12)


@pytest.mark.parametrize("depth", [4, 5])
@pytest.mark.parametrize("alpha", [0.0, 4.0])
def test_vcycles_from_zero_converge_to_the_direct_solve(depth, alpha):
    S, V, area = T.mg_inputs("torus", depth, oracle_mg_splat)
    sigma = float(F32(alpha * area))
    chi, hist = P.multigrid(S, V, sigma, 40)
    want = P.solve(S.astype(np.float64), V.astype(np.float64), sigma)
    if alpha == 0:
        want = want - want.mean()
    assert hist[-1] <= 1e-10
    assert np.abs(chi - want).max() <= 1e-8 * (want.max() - want.min())
    b = P.rhs(V.astype(np.float64))
    assert abs(P.relative_residual(chi, b, S, sigma) - hist[-1]) <= 1e-12


@pytest.mark.parametrize("alpha", [0.0, 4.0])
def test_device_residual_equals_the_oracle(alpha):
    """The float64 torch stencil the GPU test uses above depth 8 (run here on host tensors, in slabs that do not divide
    R) equals poisson_ref.relative_residual and residual_floor."""
    import torch

    S, V, area = T.mg_inputs("wall", 5, oracle_mg_splat)
    sigma = float(F32(alpha * area))
    chi, _ = P.multigrid(S, V, sigma, 2)
    chi = chi.astype(F32)
    b = P.rhs(V.astype(np.float64))
    want = (P.relative_residual(chi, b, S, sigma), P.residual_floor(chi, b, S, sigma, P.face_sums(V), alpha == 0))
    r, bb, f = T._residual_torch(torch.from_numpy(chi), torch.from_numpy(V.reshape(3, -1)),
                                 torch.from_numpy(S.reshape(-1)), sigma, alpha == 0, slab=7)
    np.testing.assert_allclose((r / bb, f / bb), want, rtol=1e-12)


# ----------------------------------------------------------------------------------------------------- slips
def oracle_mg_splat(case):
    """The multigrid inputs of a case from the oracle's splat, rounded to fp32 like the kernel's."""
    p, n, _, o, h, depth = case
    s = P.splat(p, n, None, o, h, depth)
    return s["screen"].astype(F32), s["faces"].astype(F32), float(F32(s["area_scale"]))


def oracle_splat_got(case, slip=None):
    """check_splat's `got` from the oracle with a slip (dense: depths below SPARSE_FROM)."""
    p, n, col, o, h, depth = case
    R = 1 << depth
    base = P.splat_nodes(p, n, None, o, h, depth)
    dens, db = P.density(base["count"], R)
    sw = P.sample_weights(*base["cells"], dens, db, R, slip, base["count"])
    s = P.splat_nodes(p, n, col, o, h, depth, weights=sw["a"], slip=slip)
    got = {"weights": sw["a"], "area_scale": sw["area_scale"], "density": dens.reshape(-1), "color": s["color"]["val"]}
    for g in T.GRIDS:
        got[g] = (s[g]["val"], int(np.count_nonzero(s[g]["val"])))
    return got


SLIP_SPLAT_CASES = [("sphere", 5), ("box", 6), ("lattice", 4), ("scale1", 5)]  # GPU cases with samples on the walls
SLIP_MG_CASES = [c for c in T.MG_CASES if c[1] <= 5]


def _after_solve_r(slip=None):
    """check_after_solve's `r` on the GPU test's depth-5 sphere from the oracle (vertices: the samples, which the
    mesh's vertices lie within a cell of)."""
    p, n, col, o, h, depth = _case("sphere", 5)
    R = 1 << depth
    s = P.splat(p, n, col, o, h, depth)
    chi = P.solve(s["screen"], s["faces"], float(F32(4.0 * s["area_scale"])))
    d, c = P.vertex_attributes(s["density"], s["colors"], o, h, p, slip)
    iso = float((P.sample(chi, o, h, p) * s["weights"]).mean())
    return {"grid": (o, h, depth), "chi": chi, "iso": iso, "vertices": p, "densities": d, "colors": c,
            "density": s["density"].reshape(-1), "color_grid": s["colors"].reshape(-1, 4)}, s["weights"], p, R


def slip_factor(slip):
    """The largest fraction of the GPU test's bound the slip uses on the GPU test's own cases."""
    if slip in P.SPLAT_SLIPS:
        return max(max(T.check_splat(oracle_splat_got(_case(*c), slip), _case(*c))[1].values()) for c in SLIP_SPLAT_CASES)
    if slip == "color_offset":
        r, w, p, _ = _after_solve_r(slip)
        return max(T.check_after_solve(r, w, p)[1].values())
    worst = 0.0
    for name, depth in SLIP_MG_CASES:
        S, V, area = T.mg_inputs(name, depth, oracle_mg_splat)
        for alpha in T.MG_ALPHAS:
            sigma = float(F32(alpha * area))
            b = P.rhs(V.astype(np.float64))
            chis = [np.zeros(S.shape, F32)]
            for _ in range(T.MG_CYCLES):
                x = P.vcycle(chis[-1], b, S, sigma)
                chis.append((x - x.mean() if sigma == 0 else x).astype(F32))
            worst = max(worst, T.check_cycles(chis, S, V, sigma, slip)[1])
    return worst


def test_the_correct_oracle_passes_its_own_rules():
    for c in SLIP_SPLAT_CASES[:3]:
        fails, worst = T.check_splat(oracle_splat_got(_case(*c)), _case(*c))
        assert not fails and max(worst.values()) <= 1e-6, worst
    r, w, p, _ = _after_solve_r()
    fails, worst = T.check_after_solve(r, w, p)
    assert not fails and max(worst.values()) <= 1e-6, worst


@pytest.mark.parametrize("slip", P.SLIPS)
def test_slip_leaves_the_bound(slip):
    f = slip_factor(slip)
    print(f"slip {slip}: {f:.3g} x the GPU test's bound")
    assert f >= 10, (slip, f)


_SOLVED = {}


@pytest.mark.parametrize("slip", P.VCYCLE_SLIPS)
def test_multigrid_slip_still_converges(slip):
    """The converged chi of test_gpu_poisson.py's multigrid check (torus at 32^3, tol 1e-7, 40 cycles) passes its
    1e-4 bound with each multigrid slip but one: only a per-cycle comparison sees them.  The exception, S_l injected
    instead of summed, under-screens the coarse levels by 8x and diverges with screening, which that check sees."""
    S, V, area = T.mg_inputs("torus", 5, oracle_mg_splat)
    for alpha in (0.0, 4.0):
        sigma = float(F32(alpha * area))
        b = P.rhs(V.astype(np.float64))
        x = np.zeros(b.shape)
        for cycles in range(1, 41):
            x = P.vcycle(x, b, S, sigma, slip)
            if P.relative_residual(x, b, S, sigma) <= 1e-7:
                break
        if sigma not in _SOLVED:
            _SOLVED[sigma] = P.solve(S.astype(np.float64), V.astype(np.float64), sigma)
        want = _SOLVED[sigma]
        if alpha == 0:
            x, want = x - x.mean(), want - want.mean()
        err = np.abs(x - want).max() / (want.max() - want.min())
        print(f"slip {slip} alpha {alpha}: {cycles} cycles, chi err / range {err:.2e}")
        if slip == "screen_inject" and alpha > 0:
            assert not err <= 1e-4
        else:
            assert err <= 1e-4


def test_slips_are_named():
    assert set(P.SLIPS) == set(P.SPLAT_SLIPS) | set(P.VCYCLE_SLIPS) | {"color_offset"} and len(P.SLIPS) == 10
    assert not math.isnan(T.cycle_bound(np.zeros(1), np.ones(1), 0.0, 0.0))
