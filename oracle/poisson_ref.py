"""fp64 numpy / scipy restatement of the dense-grid screened Poisson system of csrc/poisson.cu (DESIGN.md §2 (6)):
splat and sample weights, MAC face grids, divergence / gradient, screening diagonal, the Neumann operator, a direct
sparse solve, and the trilinear interpolation used for the iso-value, the vertex densities and the vertex colours.

For the per-node tests (tests/test_gpu_poisson_kernels.py):
  * `splat_nodes` / `splat_nodes_sparse`: the splat per node with the error terms its fp32 bound is built from (T_n,
    the sum of |term|; W_n, the first-order weight of the fp32 tent arguments; m_n, the samples the node's thread
    gathers), dense or as the nodes the samples reach, at the kernel's fp32 cell fractions;
  * `sample_weights`: rho_p, a_p and area_scale with a first-order bound of their fp32 evaluation;
  * `vcycle` / `relative_residual`: one V-cycle of the solver restated stage by stage, and ||b - A chi|| / ||b||;
  * `SLIPS`: plausible kernel mistakes, each applied to the restatement through `slip=`, so that
    tests/test_poisson_ref_cpu.py can show the GPU test's bounds would see them.
Test infrastructure only."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

AREA_FACTOR = 16.0  # (R / (R/4))^2: cells^2 of a surface through one level-2 cell
EPS = 2.0 ** -24    # fp32 unit roundoff
COARSE_SWEEPS, PRE_SWEEPS, POST_SWEEPS = 400, 2, 2
COARSEST_R = 4
SLIPS = ("prolong_zero_outside",  # prolongation reads 0 past the wall instead of clamping to the outer coarse node
         "prolong_half",          # prolongation weights 0.5 / 0.5 instead of 0.75 / 0.25
         "coeff_4l",              # level-l Laplacian coefficient 4^l instead of 2^l
         "screen_inject",         # S_l injected (one child) instead of the 8-child sum
         "coarse_b_mean",         # the coarsest level keeps b's mean at sigma = 0
         "one_pre_sweep",         # one pre-smoothing sweep instead of two
         "face_tent_half",        # the face grids' tent offset 0.5 (a node's) instead of 1 along the face axis
         "wall_face_kept",        # the wall face (past the last cell) keeps its flux
         "density_one_level",     # rho from the count grid restricted one level (R/2) instead of two
         "color_offset")          # the R/4 colour grid read with the finest grid's half-cell node offset
SPLAT_SLIPS = ("face_tent_half", "wall_face_kept", "density_one_level")
VCYCLE_SLIPS = ("prolong_zero_outside", "prolong_half", "coeff_4l", "screen_inject", "coarse_b_mean", "one_pre_sweep")


def tent(d):
    return np.maximum(0.0, 1.0 - np.abs(d))


def grid_for(points, depth, scale=1.1):
    """(origin, cell) of the cube of side scale * largest extent, centred on the bounding box."""
    p = np.asarray(points, np.float64)
    lo, hi = p.min(0), p.max(0)
    side = max(float((hi - lo).max()), 1e-12) * scale
    return 0.5 * (lo + hi) - 0.5 * side, side / (1 << depth)


def _cells(points, origin, h, R):
    u = (np.asarray(points, np.float32).astype(np.float64) - np.asarray(origin, np.float32).astype(np.float64)) / np.float64(np.float32(h))
    c = np.clip(np.floor(u), 0, R - 1).astype(np.int64)
    return c, u - c


def _splat(c, f, R, vals, node_off):
    """sum_p vals_p * prod_a tent(c_a + f_a - node_a - node_off_a) over the nodes within reach; node_off 0.5 on a
    cell-centred axis, 1.0 on a face axis (face i at u = i + 1, i <= R - 2)."""
    out = np.zeros((R, R, R))
    for d in np.ndindex(3, 3, 3):
        idx = c + (np.array(d) - 1)
        w = np.ones(c.shape[0])
        ok = np.ones(c.shape[0], bool)
        for a in range(3):
            w *= tent(c[:, a] + f[:, a] - idx[:, a] - node_off[a])
            ok &= (idx[:, a] >= 0) & (idx[:, a] <= (R - 2 if node_off[a] == 1.0 else R - 1))
        ok &= w > 0
        np.add.at(out, (idx[ok, 0], idx[ok, 1], idx[ok, 2]), vals[ok] * w[ok])
    return out


def restrict_sum(x):
    R = x.shape[0] // 2
    return x.reshape(R, 2, R, 2, R, 2, *x.shape[3:]).sum(axis=(1, 3, 5))


def sample(values, origin, cell, points):
    """Trilinear interpolation of the cell-centred grid values [X,Y,Z(,C)] at points, clamped to the outer centres."""
    v = np.asarray(values, np.float64)
    x = (np.asarray(points, np.float64) - np.asarray(origin, np.float64)) / cell - 0.5
    i0 = np.floor(x)
    t = x - i0
    i0 = i0.astype(np.int64)
    dims = np.array(v.shape[:3])
    low, high = i0 < 0, i0 >= dims - 1
    t[low | high] = 0.0
    i0 = np.where(low, 0, np.where(high, dims - 1, i0))
    i1 = np.minimum(i0 + 1, dims - 1)
    out = 0.0
    for c in np.ndindex(2, 2, 2):
        w = np.ones(x.shape[0])
        idx = []
        for a in range(3):
            w *= t[:, a] if c[a] else 1.0 - t[:, a]
            idx.append(i1[:, a] if c[a] else i0[:, a])
        val = v[idx[0], idx[1], idx[2]]
        out = out + (w[:, None] * val if val.ndim == 2 else w * val)
    return out


def splat(points, normals, colors, origin, h, depth):
    """Everything dnr_poisson_splat produces: screen S, faces [3,R,R,R], density (R/4)^3, colour grid
    {sum a w c, sum a w} [(R/4)^3,4], weights a_p, area_scale."""
    R = 1 << depth
    c, f = _cells(points, origin, h, R)
    n = np.asarray(normals, np.float32).astype(np.float64)
    count = _splat(c, f, R, np.ones(c.shape[0]), (0.5, 0.5, 0.5))
    density = restrict_sum(restrict_sum(count))
    u = c + f
    rho = sample(density, (0.0, 0.0, 0.0), 4.0, u)
    inv = 1.0 / np.maximum(rho, 1e-20)
    a = inv / inv.mean()
    S = _splat(c, f, R, a, (0.5, 0.5, 0.5))
    faces = np.stack([_splat(c, f, R, a * n[:, ax], tuple(1.0 if b == ax else 0.5 for b in range(3))) for ax in range(3)])
    col = None
    if colors is not None:
        cc = np.asarray(colors, np.float32).astype(np.float64)
        R4 = R // 4
        c4 = np.floor(u / 4.0).astype(np.int64)
        f4 = u / 4.0 - c4
        wsum = _splat(c4, f4, R4, a, (0.5, 0.5, 0.5))
        num = np.stack([_splat(c4, f4, R4, a * cc[:, ch], (0.5, 0.5, 0.5)) for ch in range(3)], axis=-1)
        col = np.concatenate([num, wsum[..., None]], axis=-1)
    return {"screen": S, "faces": faces, "density": density, "colors": col, "weights": a,
            "area_scale": AREA_FACTOR * inv.mean()}


def _diff(R, axis):
    """Forward difference onto the R-1 interior faces of one axis, as a sparse [faces, R^3] matrix (faces indexed like
    the nodes, the last one per axis omitted)."""
    d1 = sp.diags([-np.ones(R - 1), np.ones(R - 1)], [0, 1], shape=(R - 1, R))
    I = sp.identity(R)
    ops = [I, I, I]
    ops[axis] = d1
    return sp.kron(sp.kron(ops[0], ops[1]), ops[2]).tocsr()


def _face_rows(R, axis):
    idx = np.arange(R ** 3).reshape(R, R, R)
    sl = [slice(None)] * 3
    sl[axis] = slice(0, R - 1)
    return idx[tuple(sl)].reshape(-1)


def gradient(R):
    """G: chi [R^3] -> the three face grids [3, R^3] (zero on the wall faces), as a list of per-axis operators."""
    return [_diff(R, a) for a in range(3)]


def divergence(faces):
    """div_h V at every node (the wall faces carry zero flux)."""
    R = faces.shape[1]
    out = np.zeros(R ** 3)
    for a, G in enumerate(gradient(R)):
        out -= G.T @ faces[a].reshape(-1)[_face_rows(R, a)]
    return out.reshape(R, R, R)


def laplacian(R):
    """-Lap_h = G^T G, the 7-point Neumann Laplacian (unit spacing), sparse [R^3, R^3]."""
    return sum((G.T @ G) for G in gradient(R)).tocsr()


def solve(screen, faces, sigma, direct_max=32 ** 3):
    """chi of (-Lap + sigma S) chi = -div V.  Up to direct_max unknowns a direct sparse solve (SuperLU; at sigma == 0
    with chi[0] pinned); beyond it SuperLU's fill-in makes a 64^3 solve take minutes, so conjugate gradients run to a
    relative residual of 1e-13, which is the same solution to fp64 rounding.  At sigma == 0 chi's mean is removed."""
    R = screen.shape[0]
    A = (laplacian(R) + sigma * sp.diags(screen.reshape(-1))).tocsc()
    b = -divergence(faces).reshape(-1)
    if sigma == 0:
        b = b - b.mean()  # compatible right-hand side of the singular Neumann problem
    if R ** 3 <= direct_max:
        if sigma == 0:
            x = np.zeros(R ** 3)
            x[1:] = spla.spsolve(A[1:, 1:], b[1:])
        else:
            x = spla.spsolve(A, b)
    else:
        x, info = spla.cg(A.tocsr(), b, rtol=1e-13, atol=0.0, maxiter=20000)
        assert info == 0, f"cg did not converge ({info})"
    if sigma == 0:
        x -= x.mean()
    return x.reshape(R, R, R)


def reconstruct_field(points, normals, depth, point_weight, colors=None, scale=1.1):
    """(chi, iso, origin, h, splat dict) of the whole pipeline in fp64."""
    origin, h = grid_for(points, depth, scale)
    s = splat(points, normals, colors, origin, h, depth)
    chi = solve(s["screen"], s["faces"], point_weight * s["area_scale"])
    iso = float((sample(chi, origin, h, points) * s["weights"]).mean())
    return chi, iso, origin, h, s


# ------------------------------------------------------------------------------------------- the splat per node
_OFFS = np.array(list(np.ndindex(3, 3, 3))) - 1  # a node's offsets from the cells within one cell of it
BOUND_K = 2.0  # every first-order fp32 bound below is used with this safety factor


def fractions(points, origin, h, R):
    """(cell [n,3], fraction [n,3]) as the kernel stores them: u = (p - origin) / h in fp64 of the fp32 inputs, the cell
    floor(u) clamped to the grid, the fraction u - cell rounded once to fp32 (the sorted copy holds it as a float).
    Everything after is fp64."""
    c, f = _cells(points, origin, h, R)
    return c, f.astype(np.float32).astype(np.float64)


def _reach(c, f, R, off):
    """Every (sample, node within one cell of the sample's cell and inside the grid) with two or more positive tents
    tent(c_a + f_a - node_a - off_a): (sample index, node linear index, product of the three tents,
    t_x t_y + t_y t_z + t_z t_x).  A term with a zero tent is exactly 0 in fp32 too (the tent arguments are monotone
    in f and the thresholds 1.5, 2 are representable), so the kernel's nonzero nodes are among those with T_n > 0."""
    d = np.arange(-1, 2)
    node = [c[:, a, None] + d for a in range(3)]                                   # [n, 3] per axis
    t = [tent(f[:, a, None] - d - off[a]) for a in range(3)]
    ok = [(node[a] >= 0) & (node[a] < R) for a in range(3)]
    x, y, z = t[0][:, :, None, None], t[1][:, None, :, None], t[2][:, None, None, :]
    pair = x * y + y * z + z * x
    sel = (pair > 0) & ok[0][:, :, None, None] & ok[1][:, None, :, None] & ok[2][:, None, None, :]
    p = np.nonzero(sel)
    lin = (node[0][p[0], p[1]] * R + node[1][p[0], p[2]]) * R + node[2][p[0], p[3]]
    return p[0], lin, (x * y * z)[sel], pair[sel]


def _gathered(idx, R, cell_lin):
    """m_n: the samples in the (up to 27) cells within one cell of each node idx, the run node n's thread walks."""
    if idx.shape[0] == R ** 3:  # dense: a 3x3x3 box sum of the cell counts
        cnt = np.pad(np.bincount(cell_lin, minlength=R ** 3).reshape(R, R, R), 1)
        return sum(cnt[1 + d[0]:R + 1 + d[0], 1 + d[1]:R + 1 + d[1], 1 + d[2]:R + 1 + d[2]] for d in _OFFS).reshape(-1)
    uc, cnt = np.unique(cell_lin, return_counts=True)
    ijk = np.stack(np.unravel_index(idx, (R, R, R)), -1)
    m = np.zeros(idx.shape[0], np.int64)
    for d in _OFFS:
        q = ijk + d
        ok = ((q >= 0) & (q < R)).all(-1)
        ql = (q[:, 0] * R + q[:, 1]) * R + q[:, 2]
        pos = np.minimum(np.searchsorted(uc, ql), uc.shape[0] - 1)
        m += np.where(ok & (uc[pos] == ql), cnt[pos], 0)
    return m


def _accumulate(c, f, R, vals, off, sparse, drop_axis=None):
    """{"idx" (sparse), "val", "T", "W", "m"} of sum_p vals_p * prod tent over the nodes: T_n = sum |term|, W_n = sum
    |vals_p| * pairwise tent products, m_n = samples gathered.  vals [n] or [n, C].  drop_axis: the nodes whose index
    along that axis is R - 1 (the wall face) are 0."""
    p, lin, w, pair = _reach(c, f, R, off)
    if drop_axis is not None:
        keep = np.unravel_index(lin, (R, R, R))[drop_axis] < R - 1
        p, lin, w, pair = p[keep], lin[keep], w[keep], pair[keep]
    v = vals[p]
    wb = w if v.ndim == 1 else w[:, None]
    pb = pair if v.ndim == 1 else pair[:, None]
    if sparse:
        idx, inv = np.unique(lin, return_inverse=True)
        size = idx.shape[0]
    else:
        idx, inv, size = np.arange(R ** 3), lin, R ** 3
    acc = lambda x: (np.bincount(inv, x, size) if x.ndim == 1  # noqa: E731
                     else np.stack([np.bincount(inv, x[:, ch], size) for ch in range(x.shape[1])], -1))
    out = {"val": acc(v * wb), "T": acc(np.abs(v) * wb), "W": acc(np.abs(v) * pb),
           "m": _gathered(idx, R, (c[:, 0] * R + c[:, 1]) * R + c[:, 2])}
    if sparse:
        out["idx"] = idx
    return out


def splat_bound(g):
    """First-order fp32 bound of a finest-grid splat node: the m_n sequential fp32 additions (m_n - 1 roundings of the
    partial sums, each at most T_n), four roundings inside a term (tent products, a_p, the normal), and an absolute
    1.5 EPS on each tent from rounding its argument (1 + f, f - 1, f - 0.5), which weighs the other two tents: W_n."""
    T, W = g["T"], g["W"]
    m = g["m"] if T.ndim == 1 else g["m"][:, None]
    return BOUND_K * EPS * ((m + 6) * T + 2 * W)


def color_bound(g):
    """fp32 bound of a colour-grid node: the sums are in double, so only the terms' own roundings count (the tent
    arguments ((fine bits) + f) / 4 + offset round to 5 EPS absolute, the weight products and the colour product to
    6 EPS relative), plus the final cast to float."""
    return BOUND_K * EPS * (9 * g["T"] + 6 * g["W"])


def splat_nodes(points, normals, colors, origin, h, depth, weights=None, sparse=False, slip=None):
    """The splat per node at the kernel's fp32 fractions: {"count", "screen", "face0", "face1", "face2", "color"} each
    `_accumulate`'s dict (finest grid; the colour grid at R/4 with channels {a c_r, a c_g, a c_b, a}), and "cells"
    (cell, fraction).  weights: the a_p to splat with (the kernel's own, so that each stage is compared at its own
    inputs); None uses `sample_weights` of this count grid.  sparse: the nodes the samples reach only, with "idx"."""
    R = 1 << depth
    c, f = fractions(points, origin, h, R)
    n = c.shape[0]
    out = {"cells": (c, f), "count": _accumulate(c, f, R, np.ones(n), (0.5, 0.5, 0.5), sparse)}
    if weights is None:
        d, db = density(out["count"], R)
        weights = sample_weights(c, f, d, db, R)["a"]
    a = np.asarray(weights, np.float64)
    nrm = np.asarray(normals, np.float32).astype(np.float64)
    out["screen"] = _accumulate(c, f, R, a, (0.5, 0.5, 0.5), sparse)
    for ax in range(3):
        off = tuple((0.5 if slip == "face_tent_half" else 1.0) if b == ax else 0.5 for b in range(3))
        out[f"face{ax}"] = _accumulate(c, f, R, a * nrm[:, ax], off, sparse,
                                       None if slip == "wall_face_kept" else ax)
    if colors is not None:
        col = np.asarray(colors, np.float32).astype(np.float64)
        vals = np.concatenate([a[:, None] * col, a[:, None]], 1)
        out["color"] = _accumulate(c >> 2, ((c & 3) + f) / 4.0, R >> 2, vals, (0.5, 0.5, 0.5), sparse)
    return out


def splat_nodes_sparse(points, normals, colors, origin, h, depth, weights=None, slip=None):
    """splat_nodes over the nodes the samples reach only (each grid with "idx"): depths 8 to 10 with 10^5 samples."""
    return splat_nodes(points, normals, colors, origin, h, depth, weights, True, slip)


def _dense(g, R, key="val"):
    """An `_accumulate` entry as an [R,R,R(,C)] grid."""
    if "idx" not in g:
        return g[key].reshape((R, R, R) + g[key].shape[1:])
    out = np.zeros((R ** 3,) + g[key].shape[1:])
    out[g["idx"]] = g[key]
    return out.reshape((R, R, R) + g[key].shape[1:])


def density(count, R, levels=2):
    """(density, its fp32 bound) at R >> levels: the count grid sum-restricted `levels` times; the bound adds the
    children's splat bounds and, per fp32 8-child sum (7 roundings of nonnegative partial sums), 7 EPS."""
    lin = count.get("idx", np.arange(R ** 3))
    ijk = np.stack(np.unravel_index(lin, (R, R, R)), -1) >> levels
    Rl = R >> levels
    cl = (ijk[:, 0] * Rl + ijk[:, 1]) * Rl + ijk[:, 2]
    d = np.bincount(cl, count["val"], Rl ** 3)
    b = np.bincount(cl, splat_bound(count), Rl ** 3) + BOUND_K * 7 * levels * EPS * d
    return d.reshape(Rl, Rl, Rl), b.reshape(Rl, Rl, Rl)


def _corners(values, x):
    """The 8 trilinear corners of the cell-centred grid values at x (in grid units, node I at I + 0.5), clamped as
    `sample` and the kernels do: [(weight [n], value [n, ...]) x 8]."""
    v = np.asarray(values, np.float64)
    x = np.asarray(x, np.float64) - 0.5
    i0 = np.floor(x)
    t = x - i0
    i0 = i0.astype(np.int64)
    dims = np.array(v.shape[:3])
    low, high = i0 < 0, i0 >= dims - 1
    t[low | high] = 0.0
    i0 = np.where(low, 0, np.where(high, dims - 1, i0))
    i1 = np.minimum(i0 + 1, dims - 1)
    out = []
    for cc in np.ndindex(2, 2, 2):
        w = np.ones(x.shape[0])
        idx = []
        for a in range(3):
            w *= t[:, a] if cc[a] else 1.0 - t[:, a]
            idx.append(i1[:, a] if cc[a] else i0[:, a])
        out.append((w, v[idx[0], idx[1], idx[2]]))
    return out


def sample_weights(c, f, dens, dens_bound, R, slip=None, count=None):
    """{"rho", "rho_bound", "a", "a_bound", "area_scale", "area_bound"}: rho_p = the density grid interpolated at the
    sample (level-2 units x = (c >> 2) + ((c & 3) + f) / 4), a_p = (1 / rho_p) / mean(1 / rho), area_scale = 16 mean.
    rho's bound: the corners' bounds interpolated, x's fp32 rounding (2 EPS (|x| + 1) per axis) times the largest
    corner (a bound of the slope), and 12 EPS for the weights and the sum.  a_p and area_scale inherit rho's relative
    error (area_scale the 1/rho-weighted mean of it), plus a few roundings.  slip "density_one_level" interpolates
    the count grid restricted once (count: the splat_nodes count dict)."""
    if slip == "density_one_level":
        dens, dens_bound = density(count, R, 1)
        x = (c + f) / 2.0
    else:
        x = (c >> 2) + ((c & 3) + f) / 4.0
    cs = _corners(dens, x)
    rho = sum(w * v for w, v in cs)
    top = np.max([v for _, v in cs], axis=0)
    dx = 2 * EPS * (np.abs(x) + 1)
    rb = BOUND_K * (sum(w * v for w, v in _corners(dens_bound, x)) + dx.sum(1) * top + 12 * EPS * rho)
    inv = 1.0 / np.maximum(rho, 1e-20)
    mean = inv.mean()
    eps_p = rb / np.maximum(rho, 1e-300)
    eps_mean = float((inv * eps_p).sum() / inv.sum())
    return {"rho": rho, "rho_bound": rb, "a": inv / mean, "a_bound": inv / mean * (eps_p + eps_mean + 6 * EPS),
            "area_scale": AREA_FACTOR * mean, "area_bound": AREA_FACTOR * mean * (eps_mean + 4 * EPS)}


# ----------------------------------------------------------------------------------------------------- V-cycle
def rhs(faces):
    """b = -div V as rhs_kernel forms it: the face below the first cell is the wall (0); the last face per axis is read
    as stored (the splat writes 0 there)."""
    V = np.asarray(faces)
    out = np.zeros(V.shape[1:], V.dtype)
    for a in range(3):
        lo = [slice(None)] * 3
        lo[a] = slice(1, None)
        hi = [slice(None)] * 3
        hi[a] = slice(0, -1)
        d = V[a].copy()
        d[tuple(lo)] -= V[a][tuple(hi)]
        out -= d
    return out


def _neigh(x):
    """(sum over the face neighbours nb of x_n - x_nb, the number of face neighbours) on the Neumann grid."""
    acc = np.zeros_like(x)
    nb = np.zeros(x.shape, np.int64)
    for a in range(3):
        d = np.diff(x, axis=a)
        lo = [slice(None)] * 3
        lo[a] = slice(0, -1)
        hi = [slice(None)] * 3
        hi[a] = slice(1, None)
        acc[tuple(lo)] -= d
        acc[tuple(hi)] += d
        nb[tuple(lo)] += 1
        nb[tuple(hi)] += 1
    return acc, nb


def residual(x, b, S, sigma, c=1.0):
    """b - c sum_nb (x_n - x_nb) - sigma S_n x_n (the kernel's difference form)."""
    acc, _ = _neigh(x)
    return b - c * acc - sigma * S * x


def _parity(R):
    i, j, k = np.meshgrid(*(np.arange(R),) * 3, indexing="ij")
    return (i + j + k) & 1


def _smooth(x, b, S, sigma, c, sweeps):
    """Red-black Gauss-Seidel in place: colour (i + j + k) & 1, colour 0 first, x_n += r_n / (c nb + sigma S_n)."""
    par = _parity(x.shape[0])
    _, nb = _neigh(x)
    diag = c * nb + sigma * S
    for _ in range(sweeps):
        for color in (0, 1):
            m = (par == color) & (diag > 0)
            r = residual(x, b, S, sigma, c)
            x[m] += r[m] / diag[m]


def prolong(xc, slip=None):
    """Cell-centred trilinear interpolation of the coarse grid onto the fine one: fine p takes 0.75 of coarse p >> 1
    and 0.25 of its neighbour on p's side, clamped at the walls."""
    out = xc
    for a in range(3):
        Rc = out.shape[a]
        p = np.arange(2 * Rc)
        q, odd = p >> 1, (p & 1).astype(bool)
        a0, a1 = np.where(odd, q, q - 1), np.where(odd, q + 1, q)
        t = np.full(2 * Rc, 0.5) if slip == "prolong_half" else np.where(odd, 0.25, 0.75)
        shape = [1, 1, 1]
        shape[a] = 2 * Rc
        v0 = np.take(out, np.clip(a0, 0, Rc - 1), axis=a)
        v1 = np.take(out, np.clip(a1, 0, Rc - 1), axis=a)
        if slip == "prolong_zero_outside":
            v0 = v0 * (a0 >= 0).reshape(shape)
            v1 = v1 * (a1 <= Rc - 1).reshape(shape)
        out = (1 - t).reshape(shape) * v0 + t.reshape(shape) * v1
    return out


def _coarse_solve(b, S, sigma, c, slip=None):
    """coarse_solve_kernel: b's mean removed at sigma = 0, COARSE_SWEEPS red-black sweeps from zero, x's mean removed
    at sigma = 0.  The 4^3 operator as a dense matrix, colour by colour (a colour couples only to the other)."""
    R = b.shape[0]
    A = (c * laplacian(R) + sigma * sp.diags(S.reshape(-1))).toarray()
    bb = b.reshape(-1).copy()
    if sigma == 0 and slip != "coarse_b_mean":
        bb -= bb.mean()
    par = _parity(R).reshape(-1)
    x = np.zeros(R ** 3)
    d = np.diag(A)
    for _ in range(COARSE_SWEEPS):
        for color in (0, 1):
            m = par == color
            x[m] += (bb[m] - A[m] @ x) / d[m]
    if sigma == 0:
        x -= x.mean()
    return x.reshape(R, R, R)


def vcycle(chi, b, S, sigma, slip=None):
    """One V-cycle of dnr_poisson_solve applied to the finest iterate chi [R,R,R] (fp64): levels l = 0 .. L with R >> l
    cells per axis down to 4^3, operator c_l (-Lap_unit) + sigma S_l with c_l = 2^l and S_l the 8-child sum of S_(l-1);
    PRE_SWEEPS red-black sweeps, the residual's 8-child sum as the next level's b with x zeroed, the recursion, the
    clamped prolongation added, POST_SWEEPS sweeps; the coarsest level solved by `_coarse_solve`.  sigma is used at
    fp32 precision as the kernel receives it.  Returns the new iterate without the final mean removal (`multigrid`)."""
    sigma = float(np.float32(sigma))
    S_l = [np.asarray(S, np.float64)]
    while S_l[-1].shape[0] > COARSEST_R:
        S_l.append(S_l[-1][::2, ::2, ::2].copy() if slip == "screen_inject" else restrict_sum(S_l[-1]))
    L = len(S_l) - 1
    base = 4.0 if slip == "coeff_4l" else 2.0

    def cycle(l, x, bl):
        c = base ** l
        if l == L:
            return _coarse_solve(bl, S_l[l], sigma, c, slip)
        x = x.copy()
        _smooth(x, bl, S_l[l], sigma, c, 1 if slip == "one_pre_sweep" else PRE_SWEEPS)
        bc = restrict_sum(residual(x, bl, S_l[l], sigma, c))
        x += prolong(cycle(l + 1, np.zeros_like(bc), bc), slip)
        _smooth(x, bl, S_l[l], sigma, c, POST_SWEEPS)
        return x

    return cycle(0, np.asarray(chi, np.float64), np.asarray(b, np.float64))


def relative_residual(chi, b, S, sigma):
    """||b - A chi|| / ||b|| in fp64 (A = -Lap + sigma S at the finest level; sigma at fp32 precision)."""
    b = np.asarray(b, np.float64)
    r = residual(np.asarray(chi, np.float64), b, np.asarray(S, np.float64), float(np.float32(sigma)))
    return float(np.sqrt((r * r).sum() / (b * b).sum()))


def face_sums(faces):
    """Per node, the sum of |V| over its six faces (the wall below the first cell is 0): what b's fp32 rounding scales
    with."""
    V = np.abs(np.asarray(faces, np.float64))
    out = V.sum(0)
    for a in range(3):
        hi = [slice(None)] * 3
        hi[a] = slice(1, None)
        lo = [slice(None)] * 3
        lo[a] = slice(0, -1)
        out[tuple(hi)] += V[a][tuple(lo)]
    return out


def residual_floor(chi, b, S, sigma, vsum, mean_removed=False):
    """The fp32 evaluation floor of the kernel's reported residual, per node K EPS (6 vsum (`face_sums`: b's own
    rounding), 8 sum_nb |x_n - x_nb| (the differences and their sum), 3 |sigma S_n x_n|), in the 2-norm, over ||b||.
    mean_removed: chi is the kernel's iterate less its mean (sigma = 0), rounded once more, which adds
    2 sum_nb (|x_n| + |x_nb|) per node."""
    x = np.asarray(chi, np.float64)
    sigma = float(np.float32(sigma))
    dsum = np.zeros_like(x)
    asum = np.zeros_like(x)
    for a in range(3):
        hi = [slice(None)] * 3
        hi[a] = slice(1, None)
        lo = [slice(None)] * 3
        lo[a] = slice(0, -1)
        d = np.abs(np.diff(x, axis=a))
        dsum[tuple(lo)] += d
        dsum[tuple(hi)] += d
        if mean_removed:
            e = np.abs(x[tuple(lo)]) + np.abs(x[tuple(hi)])
            asum[tuple(lo)] += e
            asum[tuple(hi)] += e
    per = BOUND_K * EPS * (6 * vsum + 8 * dsum + 3 * np.abs(sigma * np.asarray(S, np.float64) * x) + 2 * asum)
    b = np.asarray(b, np.float64)
    return float(np.sqrt((per * per).sum() / (b * b).sum()))


def multigrid(screen, faces, sigma, cycles, slip=None):
    """(chi, [relative residual before the first and after each cycle]) of `cycles` fp64 V-cycles from zero, chi's
    mean removed at sigma = 0 when a cycle ran."""
    b = rhs(np.asarray(faces, np.float64))
    S = np.asarray(screen, np.float64)
    x = np.zeros_like(b)
    hist = [1.0 if (b * b).sum() > 0 else 0.0]
    for _ in range(cycles):
        x = vcycle(x, b, S, sigma, slip)
        hist.append(relative_residual(x, b, S, sigma))
    if float(np.float32(sigma)) == 0 and cycles > 0:
        x = x - x.mean()
    return x, hist


def vertex_attributes(dens, color_grid, origin, h, verts, slip=None):
    """(density, colour) at the mesh vertices as poisson_solve_points reads them: the R/4 grids (node I at
    origin + (I + 0.5) 4h) interpolated, the colour the ratio of the interpolated sums.  slip "color_offset" reads the
    colour grid with its nodes at origin + (4 I + 0.5) h, the finest grid's half-cell offset."""
    o = np.asarray(origin, np.float64)
    d = sample(dens, o, 4 * h, verts)
    cw = sample(color_grid, o - (1.5 * h if slip == "color_offset" else 0.0), 4 * h, verts)
    return d, cw[:, :3] / np.maximum(cw[:, 3:], 1e-30)
