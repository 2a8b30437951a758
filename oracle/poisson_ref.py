"""fp64 numpy / scipy restatement of the dense-grid screened Poisson system of csrc/poisson.cu (DESIGN.md §2 (6)):
splat and sample weights, MAC face grids, divergence / gradient, screening diagonal, the Neumann operator, a direct
sparse solve, and the trilinear interpolation used for the iso-value, the vertex densities and the vertex colours.
Test infrastructure only."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

AREA_FACTOR = 16.0  # (R / (R/4))^2: cells^2 of a surface through one level-2 cell


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
