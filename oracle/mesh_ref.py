"""numpy restatement of the mesh-export kernels (csrc/mesh.cu): TSDF integration of one view and marching cubes over the
generated tables (dn_splatter_b200/mc_tables.py).  Test infrastructure only.

`integrate(..., dtype=np.float32)` repeats the kernel's fp32 operations in its order (the kernel is compiled with
-fmad=false) and rounds the colour to fp16 as the voxel stores it; `dtype=np.float64` is the same rule in fp64.
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


def empty_volume(dims, dtype=np.float32):
    """tsdf [X,Y,Z], weight [X,Y,Z], colour [X,Y,Z,3] (fp16 for the fp32 restatement, as the voxel stores it)."""
    cdt = np.float16 if dtype == np.float32 else dtype
    return np.zeros(dims, dtype), np.zeros(dims, dtype), np.zeros(tuple(dims) + (3,), cdt)


def integrate(tsdf, weight, color, origin, voxel, sdf_trunc, depth, rgb, mask, cam, depth_trunc, dtype=np.float32):
    """Fuses one view in place.  cam: 16 floats {fx, fy, cx, cy, world->camera [3,4]}.  Returns the pixel (u, v) each
    voxel read, -1 where the voxel was not updated."""
    f = dtype
    X, Y, Z = tsdf.shape
    H, W = depth.shape
    cam = np.asarray(cam, dtype=f)
    fx, fy, cx, cy, E = cam[0], cam[1], cam[2], cam[3], cam[4:].reshape(3, 4)
    o, vx, tr = np.asarray(origin, dtype=f), f(voxel), f(sdf_trunc)
    i, j, k = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
    p = [o[a] + (idx.astype(f) + f(0.5)) * vx for a, idx in enumerate((i, j, k))]
    cx_, cy_, cz_ = [E[r, 0] * p[0] + E[r, 1] * p[1] + E[r, 2] * p[2] + E[r, 3] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        uf = fx * cx_ / cz_ + cx + f(0.5)
        vf = fy * cy_ / cz_ + cy + f(0.5)
        eps = f(1e-4)
        ok = (cz_ > 0) & (uf >= eps) & (uf < f(W) - eps) & (vf >= eps) & (vf < f(H) - eps)
        u = np.where(ok, uf, 0).astype(np.int64)
        v = np.where(ok, vf, 0).astype(np.int64)
        d = depth.astype(f)[v, u]
        drop = (d > f(depth_trunc)) | (d < 0)
        if mask is not None:
            drop |= mask[v, u] == 0
        d = np.where(drop, f(0), d)
        ok &= d > 0
        a = (u.astype(f) - cx) / fx
        b = (v.astype(f) - cy) / fy
        sdf = (d - cz_) * np.sqrt(f(1) + a * a + b * b)
        ok &= sdf > -tr
        t = np.minimum(f(1), sdf / tr)
    c = np.clip(rgb.astype(f)[v, u] * f(255), 0, 255).astype(np.int64).astype(f)
    w = weight[ok]
    w1 = w + f(1)
    tsdf[ok] = (tsdf[ok] * w + t[ok]) / w1
    col = color[ok].astype(f)
    color[ok] = ((col * w[:, None] + c[ok]) / w1[:, None]).astype(color.dtype)
    weight[ok] = w1
    return np.where(ok, u, -1), np.where(ok, v, -1)


def marching_cubes(values, iso, origin, spacing, valid: Optional[np.ndarray] = None,
                   colors: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, Optional[np.ndarray]]:
    """values [X,Y,Z] fp32 (valid [X,Y,Z] bool or None, colors [X,Y,Z,3] in 0..255 or None) -> vertices [V,3] fp32,
    faces [F,3] int64, vertex colours [V,3] fp32 in [0,1] or None."""
    f = np.float32
    values = np.asarray(values, dtype=f)
    X, Y, Z = values.shape
    iso = f(iso)
    inside = values < iso
    ok = np.ones(values.shape, bool) if valid is None else np.asarray(valid, bool)
    case = np.zeros((X - 1, Y - 1, Z - 1), np.int64)
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
    f0 = values[idx[:, 0], idx[:, 1], idx[:, 2]]
    f1 = values[nb[:, 0], nb[:, 1], nb[:, 2]]
    t = (iso - f0) / (f1 - f0)
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
