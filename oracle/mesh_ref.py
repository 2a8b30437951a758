"""numpy restatement of the mesh-export kernels (csrc/mesh.cu): TSDF integration of one view and marching cubes over the
generated tables (dn_splatter_b200/mc_tables.py).  Test infrastructure only.

`integrate(..., dtype=np.float32)` repeats the kernel's fp32 operations in its order (the kernel is compiled with
-fmad=false) and keeps the colour as the voxel does, a fixed-point mean in units of 2^-13 of a level rounded half up on
each update; `dtype=np.float64` is the same rule in fp64 with an exact colour mean.  The colour array's dtype says how the
mean is kept: float32 (the voxel's fixed point, as levels: every value a multiple of 2^-13 below 256, which fp32 holds
exactly), float64 (exact) or float16 (the voxel layout before the fixed point).
`integrate(..., slip=...)` restates one kernel mistake (SLIPS), so the tests can show that their rules would see it.
`marching_cubes` produces the kernel's welded, ordered output: vertices by (sample index, edge axis), faces by cube index
then table order."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from dn_splatter_b200 import mc_tables

_NTRI = np.array(mc_tables.tables()[0], dtype=np.int64)
_TRI = mc_tables.table_array().astype(np.int64)
_EDGE_C0 = np.array(mc_tables.EDGE_C0, dtype=np.int64)
_EDGE_AXIS = np.array(mc_tables.EDGE_AXIS, dtype=np.int64)

COLOR_FRAC_BITS = 13  # voxel colour unit: 2^-13 of a level; three 21-bit fields r | g << 21 | b << 42
_FIELD = (1 << 21) - 1

# integrate's branch codes: which test stopped the voxel (UPDATED: none did)
UPDATED, BEHIND, OUTSIDE, NO_DEPTH, TOO_FAR = 0, 1, 2, 3, 4

# kernel mistakes integrate can restate: rounding u_f / v_f to the nearest pixel instead of truncating, `>=` in the sdf
# test (sdf >= -sdf_trunc updates), `>=` for depth_trunc (d >= depth_trunc is no depth), the ray multiplier from u_f, v_f
# instead of the integer pixel, and the colour rounded instead of truncated.  fp16 colour storage is the float16 colour array.
SLIPS = ("round_uf", "sdf_ge", "depth_trunc_ge", "ray_from_uf", "round_color")


def empty_volume(dims, dtype=np.float32, color_dtype=None):
    """tsdf [X,Y,Z], weight [X,Y,Z], colour [X,Y,Z,3] in levels: the voxel's fixed point held in float32 for the fp32
    restatement, exact float64 for fp64; color_dtype overrides (np.float16: the fp16 layout)."""
    cdt = color_dtype if color_dtype is not None else dtype
    return np.zeros(dims, dtype), np.zeros(dims, dtype), np.zeros(tuple(dims) + (3,), cdt)


def color_levels(color) -> np.ndarray:
    """A colour array of any of the three kinds as float64 levels (0..255)."""
    return color.astype(np.float64)


def _units(levels) -> np.ndarray:
    """float32 fixed-point levels -> int64 units of 2^-13 level (exact: asserts the levels lie on the grid)."""
    u = np.asarray(levels, np.float64) * (1 << COLOR_FRAC_BITS)
    assert (u == np.round(u)).all() and ((u >= 0) & (u <= _FIELD)).all()
    return u.astype(np.int64)


def unpack_voxels(q):
    """[N,4] float32 voxels of the kernel -> tsdf [N], weight [N], colour [N,3] in levels (float32, exact)."""
    q = np.ascontiguousarray(q, dtype=np.float32)
    bits = q[:, 2:4].copy().view(np.uint64)[:, 0].astype(np.int64)
    col = np.stack([(bits >> (21 * ch)) & _FIELD for ch in range(3)], axis=1)
    return q[:, 0].copy(), q[:, 1].copy(), (col * 2.0 ** -COLOR_FRAC_BITS).astype(np.float32)


def pack_voxels(tsdf, weight, color) -> np.ndarray:
    """Inverse of unpack_voxels: [N,4] float32 voxels from tsdf, weight and the fixed-point colour in levels."""
    color = _units(np.asarray(color).reshape(-1, 3))
    bits = (color[:, 0] | (color[:, 1] << 21) | (color[:, 2] << 42)).astype(np.uint64)
    q = np.zeros((color.shape[0], 4), np.float32)
    q[:, 0], q[:, 1] = np.asarray(tsdf, np.float32).reshape(-1), np.asarray(weight, np.float32).reshape(-1)
    q[:, 2:4] = bits.view(np.float32).reshape(-1, 2)
    return q


def project(shape, origin, voxel, sdf_trunc, depth, rgb, mask, cam, depth_trunc, dtype=np.float32, slip=None):
    """The per-voxel decisions and values of one view over a [X,Y,Z] grid, without the update: a dict of z, uf, vf (the
    pixel coordinates before truncation), u, v (the pixel read), d (the depth used), sdf, t, c (the integer colour
    [X,Y,Z,3]) and branch (UPDATED / BEHIND / OUTSIDE / NO_DEPTH / TOO_FAR)."""
    f = dtype
    X, Y, Z = shape
    H, W = depth.shape
    cam = np.asarray(cam, dtype=f)
    fx, fy, cx, cy, E = cam[0], cam[1], cam[2], cam[3], cam[4:].reshape(3, 4)
    o, vx, tr = np.asarray(origin, dtype=f), f(voxel), f(sdf_trunc)
    i, j, k = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
    p = [o[a] + (idx.astype(f) + f(0.5)) * vx for a, idx in enumerate((i, j, k))]
    cx_, cy_, cz_ = [E[r, 0] * p[0] + E[r, 1] * p[1] + E[r, 2] * p[2] + E[r, 3] for r in range(3)]
    branch = np.full(shape, UPDATED, np.int64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        front = cz_ > 0
        branch[~front] = BEHIND
        uf = fx * cx_ / cz_ + cx + f(0.5)
        vf = fy * cy_ / cz_ + cy + f(0.5)
        eps = f(1e-4)
        ok = front & (uf >= eps) & (uf < f(W) - eps) & (vf >= eps) & (vf < f(H) - eps)
        branch[front & ~ok] = OUTSIDE
        if slip == "round_uf":
            u = np.where(ok, np.minimum(np.floor(uf + f(0.5)), W - 1), 0).astype(np.int64)
            v = np.where(ok, np.minimum(np.floor(vf + f(0.5)), H - 1), 0).astype(np.int64)
        else:
            u = np.where(ok, uf, 0).astype(np.int64)
            v = np.where(ok, vf, 0).astype(np.int64)
        d = depth.astype(f)[v, u]
        far = (d >= f(depth_trunc)) if slip == "depth_trunc_ge" else (d > f(depth_trunc))
        drop = far | (d < 0)
        if mask is not None:
            drop |= mask[v, u] == 0
        d = np.where(drop, f(0), d)
        branch[ok & ~(d > 0)] = NO_DEPTH
        ok &= d > 0
        if slip == "ray_from_uf":
            a = (uf - f(0.5) - cx) / fx
            b = (vf - f(0.5) - cy) / fy
        else:
            a = (u.astype(f) - cx) / fx
            b = (v.astype(f) - cy) / fy
        sdf = (d - cz_) * np.sqrt(f(1) + a * a + b * b)
        near = (sdf >= -tr) if slip == "sdf_ge" else (sdf > -tr)
        branch[ok & ~near] = TOO_FAR
        ok &= near
        t = np.minimum(f(1), sdf / tr)
        # the reference's uint8 colour, truncated (clamped, NaN -> 0 as fmaxf / fminf do)
        c = np.nan_to_num(rgb.astype(f)[v, u] * f(255), nan=0.0)
        c = np.clip(c, 0, 255)
        c = (np.floor(c + f(0.5)) if slip == "round_color" else c).astype(np.int64)
    return dict(z=cz_, uf=uf, vf=vf, u=np.where(ok, u, -1), v=np.where(ok, v, -1), d=d, sdf=sdf, t=t,
                c=np.minimum(c, 255), branch=branch)


def integrate(tsdf, weight, color, origin, voxel, sdf_trunc, depth, rgb, mask, cam, depth_trunc, dtype=np.float32, slip=None):
    """Fuses one view in place.  cam: 16 floats {fx, fy, cx, cy, world->camera [3,4]}.  Returns the pixel (u, v) each
    voxel read, -1 where the voxel was not updated."""
    f = dtype
    r = project(tsdf.shape, origin, voxel, sdf_trunc, depth, rgb, mask, cam, depth_trunc, dtype, slip)
    ok = r["branch"] == UPDATED
    w = weight[ok]
    w1 = w + f(1)
    tsdf[ok] = (tsdf[ok] * w + r["t"][ok]) / w1
    c = r["c"][ok]
    if color.dtype == np.float32:  # the voxel's fixed point: round half up of (m w + c 2^13) / (w + 1), in integers
        wi = w.astype(np.int64)[:, None]
        num = _units(color[ok]) * wi + (c << COLOR_FRAC_BITS)
        color[ok] = (((2 * num + (wi + 1)) // (2 * (wi + 1))) * 2.0 ** -COLOR_FRAC_BITS).astype(np.float32)
    else:
        col = color[ok].astype(f)
        color[ok] = ((col * w[:, None] + c.astype(f)) / w1[:, None]).astype(color.dtype)
    weight[ok] = w1
    return r["u"], r["v"]


def marching_cubes(values, iso, origin, spacing, valid: Optional[np.ndarray] = None,
                   colors: Optional[np.ndarray] = None, dtype=np.float32) -> Tuple[np.ndarray, np.ndarray, Optional[np.ndarray]]:
    """values [X,Y,Z] fp32 (valid [X,Y,Z] bool or None, colors [X,Y,Z,3] in 0..255 or None) -> vertices [V,3], faces
    [F,3] int64, vertex colours [V,3] in [0,1] or None.  The topology comes from the fp32 values; dtype=np.float64
    interpolates the vertices and colours in fp64."""
    f = dtype
    values = np.asarray(values, dtype=np.float32)
    X, Y, Z = values.shape
    iso = np.float32(iso)
    inside = values < iso
    ok = np.ones(values.shape, bool) if valid is None else np.asarray(valid, bool)
    case = np.zeros((max(X - 1, 0), max(Y - 1, 0), max(Z - 1, 0)), np.int64)
    cvalid = np.ones(case.shape, bool)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        sl = (slice(dx, X - 1 + dx), slice(dy, Y - 1 + dy), slice(dz, Z - 1 + dz))
        case |= inside[sl].astype(np.int64) << c
        cvalid &= ok[sl]
    ntri = np.where(cvalid, _NTRI[case], 0)
    ci, cj, ck = np.nonzero(ntri)  # ascending cube index
    cases = case[ci, cj, ck]
    edges = _TRI[cases]  # [n, 3 * max_tri]
    used = np.arange(edges.shape[1])[None, :] < 3 * ntri[ci, cj, ck][:, None]
    rows = np.nonzero(used)
    e = edges[rows]
    c0 = _EDGE_C0[e]
    vi = ci[rows[0]] + (c0 & 1)
    vj = cj[rows[0]] + ((c0 >> 1) & 1)
    vk = ck[rows[0]] + ((c0 >> 2) & 1)
    keys = ((vi * Y + vj) * Z + vk) * 3 + _EDGE_AXIS[e]
    uniq = np.unique(keys)
    faces = np.searchsorted(uniq, keys).reshape(-1, 3)
    lin, axis = uniq // 3, uniq % 3
    idx = np.stack([lin // (Y * Z), (lin // Z) % Y, lin % Z], axis=1)
    nb = idx + np.eye(3, dtype=np.int64)[axis]
    f0 = values[idx[:, 0], idx[:, 1], idx[:, 2]].astype(f)
    f1 = values[nb[:, 0], nb[:, 1], nb[:, 2]].astype(f)
    t = (f(iso) - f0) / (f1 - f0)
    o = np.asarray(origin, dtype=f)
    s = f(spacing)
    pos = idx.astype(f)
    pos[np.arange(len(uniq)), axis] += t
    verts = (o[None, :] + s * pos).astype(f)
    vcol = None
    if colors is not None:
        c0 = colors[idx[:, 0], idx[:, 1], idx[:, 2]].astype(f)
        c1 = colors[nb[:, 0], nb[:, 1], nb[:, 2]].astype(f)
        vcol = ((c0 + t[:, None] * (c1 - c0)) / f(255)).astype(f)
    return verts, faces, vcol
