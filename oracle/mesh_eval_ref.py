"""fp64 numpy restatement of the mesh evaluation of /root/reference/dn_splatter/eval/eval_mesh_vis_cull.py and
metrics.PDMetrics (the rules dn_splatter_b200.mesh_eval implements on the device):

- `ray_cast_depth`: z-depth of a triangle mesh by a per-pixel Moller-Trumbore ray cast (small sizes only), both faces,
  nearest hit with near <= z <= far, 0 elsewhere; `near_edge_pixels` marks pixel centres within tol px of a triangle's
  boundary, where a fp32 / fp64 pair may legitimately disagree about a hit.
- `depth_kernel_rule`: dnr_mesh_depth's own rule in fp64 from its fp32 inputs, in the kernel's operation order, so
  the depth bits are equal; `depth_kernel_mirror` also restates its box pass and item search; `DEPTH_SLIPS` /
  `VIS_SLIPS` name plausible kernel mistakes the two rules can restate.
- `visibility_counts`: obs / invalid of cull_from_one_pose + get_grid_culling_pattern (:68-149), in the operation order
  the CUDA kernel uses, so the counts are equal.
- `keep_faces`: the face rule of cull_mesh (:251-260); `subdivide_to_size`: trimesh.remesh.subdivide_to_size's rule
  [EXT] with welded midpoints; `cull_mesh`: the whole of :176-266 on in-memory inputs.
- `mesh_metrics` / `pd_accuracy` / `pd_completeness`: compute_metrics (:333-397) on given samples with
  scipy.spatial.cKDTree, and metrics.calculate_accuracy / calculate_completeness.
"""
from __future__ import annotations

import numpy as np

FLIP = np.diag([1.0, -1.0, -1.0, 1.0])


def camera_block(c2w, fx, fy, cx, cy) -> np.ndarray:
    """{fx, fy, cx, cy, world->camera [3,4]} (16 fp64) of an OpenGL / nerfstudio c2w ([3,4] or [4,4])."""
    m = np.eye(4)
    m[:3, :4] = np.asarray(c2w, np.float64).reshape(-1, 4)[:3]
    E = np.linalg.inv(m @ FLIP)[:3]
    return np.concatenate([np.array([fx, fy, cx, cy], np.float64), E.reshape(-1)])


def _split(cam):
    cam = np.asarray(cam, np.float64)
    return cam[0], cam[1], cam[2], cam[3], cam[4:].reshape(3, 4)


def _camera_space(verts, E):
    v = np.asarray(verts, np.float64)
    return v @ E[:, :3].T + E[:, 3]


def _pixel_rays(cam, W, H):
    fx, fy, cx, cy, _ = _split(cam)
    i, j = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    return np.stack([(i + 0.5 - cx) / fx, (j + 0.5 - cy) / fy, np.ones((H, W))], axis=-1).reshape(-1, 3)


def ray_cast_depth(verts, faces, cam, W, H, near=0.01, far=10.0, chunk=64) -> np.ndarray:
    """[H,W] fp64 depth: Moller-Trumbore from the camera centre along (x, y, 1) per pixel centre, so t is the z-depth."""
    fx, fy, cx, cy, E = _split(cam)
    P = _camera_space(verts, E)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    d = _pixel_rays(cam, W, H)
    best = np.full(d.shape[0], np.inf)
    for f0 in range(0, f.shape[0], chunk):
        A, B, Cc = P[f[f0:f0 + chunk, 0]], P[f[f0:f0 + chunk, 1]], P[f[f0:f0 + chunk, 2]]
        e1, e2 = B - A, Cc - A
        pvec = np.cross(d[:, None, :], e2[None])
        det = (e1[None] * pvec).sum(-1)
        ok = det != 0
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        tvec = -A
        u = (tvec[None] * pvec).sum(-1) * inv
        q = np.cross(tvec, e1)
        v = (d[:, None, :] * q[None]).sum(-1) * inv
        t = (e2 * q).sum(-1)[None] * inv
        hit = ok & (u >= 0) & (v >= 0) & (u + v <= 1) & (t >= near) & (t <= far)
        best = np.minimum(best, np.where(hit, t, np.inf).min(axis=1))
    return np.where(np.isfinite(best), best, 0.0).reshape(H, W)


def near_edge_pixels(verts, faces, cam, W, H, tol=1e-4, chunk=64) -> np.ndarray:
    """[H,W] bool: pixel centres within tol px (measured on the image plane, focal max(fx, fy)) of the boundary of some
    triangle's projection, i.e. on an edge line while on the inner side of (or within tol of) the other two."""
    fx, fy, cx, cy, E = _split(cam)
    P = _camera_space(verts, E)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    d = _pixel_rays(cam, W, H)
    out = np.zeros(d.shape[0], bool)
    scale = max(fx, fy)
    for f0 in range(0, f.shape[0], chunk):
        tri = [P[f[f0:f0 + chunk, k]] for k in range(3)]
        s = []
        for k in range(3):
            c = np.cross(tri[k], tri[(k + 1) % 3])
            norm = np.sqrt(c[:, 0] ** 2 + c[:, 1] ** 2)
            s.append((d @ c.T) / np.where(norm > 0, norm, np.inf)[None] * scale)
        s = np.stack(s, -1)  # [N, Fc, 3] signed distances in px to the three edge lines
        near = (np.abs(s).min(-1) < tol) & (((s > -tol).all(-1)) | ((s < tol).all(-1)))
        out |= near.any(axis=1)
    return out.reshape(H, W)


def visibility_counts(points, cams, W, H, rendered=None, gt=None, eps=0.02, slip=None):
    """obs, invalid (int64 [n]) summed over the views; cams: fp64 camera blocks, rendered / gt: float32 [H,W] maps.
    rendered None: no occlusion test (obs = in frustum); gt None: invalid stays 0.  `slip` (one of VIS_SLIPS) restates
    a kernel mistake: rendered + eps summed in fp64, px rounded instead of truncated, or px < W - 1."""
    p = np.asarray(points, np.float64)
    obs = np.zeros(p.shape[0], np.int64)
    inv = np.zeros(p.shape[0], np.int64)
    for v, cam in enumerate(cams):
        px, py, pz = project_points(p, cam)
        in_x = (0 <= px) & ((px < W - 1) if slip == "px_strict_max" else (px <= W - 1))
        inside = in_x & (0 <= py) & (py <= H - 1) & (pz > 0)
        with np.errstate(invalid="ignore"):
            u = np.clip(np.nan_to_num(np.rint(px) if slip == "px_rounded" else px), 0, W - 1).astype(np.int32)
            vv = np.clip(np.nan_to_num(py), 0, H - 1).astype(np.int32)
        if rendered is None:
            obs += inside
        else:
            r = np.asarray(rendered[v], np.float32)
            limit = r[vv, u].astype(np.float64) + float(np.float32(eps)) if slip == "eps_fp64" else r[vv, u] + np.float32(eps)
            obs += inside & (pz < limit)
        if gt is not None:
            inv += inside & (np.asarray(gt[v], np.float32)[vv, u] <= 0.0)
    return obs, inv


def keep_faces(obs, invalid, faces) -> np.ndarray:
    """cull_mesh's rule: some vertex with obs > 3, and not all three with invalid > 0.7 * obs."""
    f = np.asarray(faces, np.int64)
    o, i = np.asarray(obs)[f], np.asarray(invalid)[f]
    return (o > 3).any(axis=1) & ~(i > 0.7 * o).all(axis=1)


def remove_unreferenced(verts, faces):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    used = np.zeros(len(verts), bool)
    used[f.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return np.asarray(verts)[used], remap[f]


def edge_lengths(verts, faces):
    t = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return (np.diff(t[:, [0, 1, 2, 0]], axis=1) ** 2).sum(axis=2) ** 0.5


def subdivide_to_size(verts, faces, max_edge=0.015, max_iter=10):
    """(vertices fp64, faces, dropped): each round, faces with any edge > max_edge split 1 -> 4 at their (welded) edge
    midpoints (a + b) / 2; the others are final.  Faces still too long after max_iter rounds are dropped (`dropped`)."""
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    cur = np.asarray(faces, np.int64).reshape(-1, 3)
    done = []
    dropped = 0
    for it in range(max_iter + 1):
        long_ = (edge_lengths(v, cur) > max_edge).any(axis=1)
        done.append(cur[~long_])
        cur = cur[long_]
        if cur.shape[0] == 0:
            break
        if it == max_iter:
            dropped = cur.shape[0]
            break
        e = np.concatenate([cur[:, [0, 1]], cur[:, [1, 2]], cur[:, [2, 0]]])
        e = np.sort(e, axis=1)
        key, inv = np.unique(e[:, 0] * v.shape[0] + e[:, 1], return_inverse=True)
        a, b = key // v.shape[0], key % v.shape[0]
        mid = (v[a] + v[b]) / 2
        m = (v.shape[0] + inv.reshape(3, -1)).T  # midpoints of edges (0,1), (1,2), (2,0)
        v = np.concatenate([v, mid])
        f0, f1, f2 = cur[:, 0], cur[:, 1], cur[:, 2]
        cur = np.concatenate([np.stack([f0, m[:, 0], m[:, 2]], 1), np.stack([m[:, 0], f1, m[:, 1]], 1),
                              np.stack([m[:, 2], m[:, 1], f2], 1), np.stack([m[:, 0], m[:, 1], m[:, 2]], 1)])
    return v, np.concatenate(done), dropped


def triangle_multiset(verts, faces) -> np.ndarray:
    """Sorted [F,9] rows of each triangle's vertex coordinates (corners sorted), for order-free comparisons."""
    t = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    order = np.lexsort((t[..., 2], t[..., 1], t[..., 0]), axis=1)
    t = np.take_along_axis(t, order[..., None], axis=1).reshape(-1, 9)
    return t[np.lexsort(t.T[::-1])]


def cull_mesh(verts, faces, cams, W, H, gt_depths=None, remove_missing_depth=True, remove_occlusion=True, subdivide=True,
              max_edge=0.015, eps=0.02, near=0.01, far=10.0, depths=None):
    """cull_mesh (:176-266): depth of the unsubdivided mesh (ray cast, or `depths` when given), counts on the subdivided
    vertices, the face rule, unreferenced vertices dropped.  Returns (vertices, faces, obs, invalid)."""
    v, f = remove_unreferenced(verts, faces)
    if depths is None and remove_occlusion:
        depths = [ray_cast_depth(v, f, c, W, H, near, far).astype(np.float32) for c in cams]
    sv, sf = (subdivide_to_size(v, f, max_edge)[:2]) if subdivide else (np.asarray(v, np.float64), f)
    obs, inv = visibility_counts(sv, cams, W, H, depths if remove_occlusion else None,
                                 gt_depths if remove_missing_depth else None, eps)
    keep = keep_faces(obs, inv, sf)
    out_v, out_f = remove_unreferenced(sv, sf[keep])
    return out_v, out_f, obs, inv


def triangle_areas(verts, faces):
    t = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return 0.5 * np.linalg.norm(np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]), axis=1)


def face_normals(verts, faces):
    t = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def distance_p2p(points_src, normals_src, points_tgt, normals_tgt):
    from scipy.spatial import cKDTree

    dist, idx = cKDTree(points_tgt).query(points_src)
    ns = normals_src / np.linalg.norm(normals_src, axis=-1, keepdims=True)
    nt = normals_tgt / np.linalg.norm(normals_tgt, axis=-1, keepdims=True)
    return dist, np.abs((nt[idx] * ns).sum(axis=-1))


def mesh_metrics(pred_points, pred_normals, gt_points, gt_normals, threshold=0.05):
    """compute_metrics (:333-397) on given samples: points as float32 (as the reference casts them), normals fp64.
    Precision / recall are the reference's float32 means, and F = 2PR/(P+R) its float32 value (NaN when P+R = 0)."""
    pp, gp = np.asarray(pred_points, np.float32), np.asarray(gt_points, np.float32)
    comp, comp_n = distance_p2p(gp, np.asarray(gt_normals, np.float64), pp, np.asarray(pred_normals, np.float64))
    acc, acc_n = distance_p2p(pp, np.asarray(pred_normals, np.float64), gp, np.asarray(gt_normals, np.float64))
    recall = (comp <= threshold).astype(np.float32).mean()
    precision = (acc <= threshold).astype(np.float32).mean()
    with np.errstate(invalid="ignore", divide="ignore"):
        f = float(2 * precision * recall / (precision + recall))  # float32, as the reference evaluates it
    return {"Acc": float(acc.mean()), "Comp": float(comp.mean()), "C-L1": float(0.5 * (comp.mean() + acc.mean())),
            "NC": float(0.5 * comp_n.mean() + 0.5 * acc_n.mean()), "F-score": f}


def pd_accuracy(pred_points, gt_points, percentile=90):
    from scipy.spatial import cKDTree

    d, _ = cKDTree(gt_points).query(pred_points)
    return float(np.percentile(d, percentile))


def pd_completeness(pred_points, gt_points, threshold=0.05):
    from scipy.spatial import cKDTree

    d, _ = cKDTree(pred_points).query(gt_points)
    return float(np.sum(d < threshold) / len(d) * 100)


# ---- dnr_mesh_depth's rule, bit for bit ----------------------------------------------------------------------------
# csrc/mesh_eval.cu works in fp64 from fp32 vertices and an fp32 camera block, without FMA (-fmad=false), so numpy in
# the same operation order reproduces its hit mask and its depth bits.  The rule per (face, pixel):
#   camera-space vertices   E[r,0] x + E[r,1] y + E[r,2] z + E[r,3], left to right
#   edge planes             e_k = P_a x P_b from the endpoints in ascending vertex-index order, negated otherwise
#   normal, numerator       n = (P1 - P0) x (P2 - P0), num = n . P0; faces with n = 0 or an index outside [0, n_verts)
#                           are skipped
#   ray                     dx = (i + 0.5 - cx) / fx, dy = (j + 0.5 - cy) / fy
#   inside                  e = dx ex + dy ey + ez for all three edges; all >= 0 or all <= 0 (a zero counts for both)
#   depth                   den = dx nx + dy ny + nz, skipped when 0; z = num / den, kept when near <= z <= far
#   pixel                   the min over faces, rounded once to fp32 (the kernel's atomicMin on positive fp32 bits)
# `depth_kernel_rule` evaluates it on pixel boxes of its own, wider than the kernel's; `depth_kernel_mirror` restates the
# kernel's box pass, scan and item -> face search, so a slip there shows up as a pixel the rule has and the mirror lacks.

PIX_PER_ITEM = 256
DEPTH_SLIPS = ("no_near_clip", "no_box_margin", "strict_inside", "strict_near", "strict_far", "fp32_z", "no_half_pixel",
               "item_search_ge")
VIS_SLIPS = ("eps_fp64", "px_rounded", "px_strict_max")
DECISIONS = ("hit", "near", "near_equal", "far", "far_equal", "edge_zero", "den_zero", "tie")


def kernel_camera(cam32):
    """(fx, fy, cx, cy, E [3,4]) in fp64 from the fp32 camera block the kernel reads."""
    c = np.asarray(cam32)
    if c.dtype != np.float32:
        raise TypeError("kernel_camera: the depth kernel reads a float32 camera block")
    c = c.astype(np.float64)
    return c[0], c[1], c[2], c[3], c[4:].reshape(3, 4)


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def kernel_to_camera(verts32, E):
    v = np.asarray(verts32, np.float32).reshape(-1, 3).astype(np.float64)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    return np.stack([E[r, 0] * x + E[r, 1] * y + E[r, 2] * z + E[r, 3] for r in range(3)], 1)


def triangle_setup(verts32, faces, E):
    """tri_setup per face: camera-space corners P [F,3,3], edge planes e [F,3,3], normal n, num and ok."""
    v = np.asarray(verts32, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    valid = ((f >= 0) & (f < v.shape[0])).all(1)
    fi = np.where(valid[:, None], f, 0)
    Pv = kernel_to_camera(v, E)
    Q = [Pv[fi[:, k]] for k in range(3)]
    e = []
    for k in range(3):
        a, b = k, (k + 1) % 3
        e.append(np.where((fi[:, a] <= fi[:, b])[:, None], _cross(Q[a], Q[b]), -_cross(Q[b], Q[a])))
    n = _cross(Q[1] - Q[0], Q[2] - Q[0])
    num = n[:, 0] * Q[0][:, 0] + n[:, 1] * Q[0][:, 1] + n[:, 2] * Q[0][:, 2]
    ok = valid & (n != 0).any(1)
    return {"P": np.stack(Q, 1), "e": np.stack(e, 1), "n": n, "num": num, "ok": ok, "valid": valid}


def _project(fx, fy, cx, cy, X, Y, Z):
    return fx * X / Z + cx, fy * Y / Z + cy


def kernel_boxes(T, cam32, W, H, near, far, slip=None):
    """depth_box_kernel: (boxes [F,4] int64 (x0, x1, y0, y1), (0, -1, 0, -1) when empty; item counts [F])."""
    fx, fy, cx, cy, _ = kernel_camera(cam32)
    near, far = float(np.float32(near)), float(np.float32(far))
    P = T["P"]
    z = P[..., 2]
    live = T["ok"] & ~(z < near).all(1) & ~(z > far).all(1)
    F = P.shape[0]
    x0, x1, y0, y1 = (np.full(F, s * np.inf) for s in (1, -1, 1, -1))

    def add(m, X, Y, Z):
        nonlocal x0, x1, y0, y1
        with np.errstate(divide="ignore", invalid="ignore"):
            u, v = _project(fx, fy, cx, cy, X, Y, Z)
        x0, x1 = np.where(m, np.fmin(x0, u), x0), np.where(m, np.fmax(x1, u), x1)
        y0, y1 = np.where(m, np.fmin(y0, v), y0), np.where(m, np.fmax(y1, v), y1)

    for k in range(3):
        a, b = P[:, k], P[:, (k + 1) % 3]
        if slip == "no_near_clip":
            add(live, a[:, 0], a[:, 1], a[:, 2])
            continue
        add(live & (a[:, 2] >= near), a[:, 0], a[:, 1], a[:, 2])
        cross = live & ((a[:, 2] < near) != (b[:, 2] < near))
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (near - a[:, 2]) / (b[:, 2] - a[:, 2])
            add(cross, a[:, 0] + s * (b[:, 0] - a[:, 0]), a[:, 1] + s * (b[:, 1] - a[:, 1]), np.full(F, near))
    m = 0.0 if slip == "no_box_margin" else 1.0
    with np.errstate(invalid="ignore"):
        lo_x, hi_x = np.fmax(np.ceil(x0 - 0.5) - m, 0.0), np.fmin(np.floor(x1 - 0.5) + m, float(W - 1))
        lo_y, hi_y = np.fmax(np.ceil(y0 - 0.5) - m, 0.0), np.fmin(np.floor(y1 - 0.5) + m, float(H - 1))
        keep = live & (lo_x <= hi_x) & (lo_y <= hi_y)
    boxes = np.tile(np.array([0, -1, 0, -1], np.int64), (F, 1))
    boxes[keep] = np.stack([lo_x, hi_x, lo_y, hi_y], 1)[keep].astype(np.int64)
    area = (boxes[:, 1] - boxes[:, 0] + 1) * (boxes[:, 3] - boxes[:, 2] + 1)
    counts = np.where(keep, (area + PIX_PER_ITEM - 1) // PIX_PER_ITEM, 0)
    return boxes, counts


def item_faces(counts, slip=None):
    """The raster kernel's binary search: per work item the first face whose inclusive scan exceeds it (with the slip
    item_search_ge: reaches it), and that face's exclusive scan."""
    scan = np.cumsum(counts)
    items = np.arange(int(scan[-1]) if scan.size else 0, dtype=np.int64)
    f = np.searchsorted(scan, items, side="left" if slip == "item_search_ge" else "right")
    f = np.minimum(f, len(counts) - 1)
    first = np.where(f == 0, 0, scan[np.maximum(f - 1, 0)])
    return items, f, first


def _expand(starts, lengths):
    """(row, offset) pairs of row r covering starts[r] .. starts[r] + lengths[r] - 1."""
    lengths = np.maximum(lengths, 0)
    row = np.repeat(np.arange(len(lengths)), lengths)
    off = np.arange(row.size) - np.repeat(np.cumsum(lengths) - lengths, lengths)
    return row, starts[row] + off


def kernel_pairs(boxes, counts, slip=None):
    """(face, i, j) of every pixel test the raster kernel makes, item by item."""
    items, f, first = item_faces(counts, slip)
    b = boxes[f]
    bw = b[:, 1] - b[:, 0] + 1
    area = bw * (b[:, 3] - b[:, 2] + 1)
    p0 = (items - first) * PIX_PER_ITEM
    p1 = np.minimum(p0 + PIX_PER_ITEM, area)
    row, p = _expand(p0, p1 - p0)
    bw_r = np.maximum(bw[row], 1)
    return f[row], b[row, 0] + p % bw_r, b[row, 2] + p // bw_r


def eval_pairs(T, cam32, f, i, j, near, far, slip=None):
    """Per (face, pixel) pair: (z fp64 where the kernel would atomicMin it, else inf; decision flags)."""
    fx, fy, cx, cy, _ = kernel_camera(cam32)
    near, far = float(np.float32(near)), float(np.float32(far))
    half = 0.0 if slip == "no_half_pixel" else 0.5
    dx = (i.astype(np.float64) + half - cx) / fx
    dy = (j.astype(np.float64) + half - cy) / fy
    e, n = T["e"][f], T["n"][f]
    ek = [dx * e[:, k, 0] + dy * e[:, k, 1] + e[:, k, 2] for k in range(3)]
    if slip == "strict_inside":
        inside = ((ek[0] > 0) & (ek[1] > 0) & (ek[2] > 0)) | ((ek[0] < 0) & (ek[1] < 0) & (ek[2] < 0))
    else:
        inside = ((ek[0] >= 0) & (ek[1] >= 0) & (ek[2] >= 0)) | ((ek[0] <= 0) & (ek[1] <= 0) & (ek[2] <= 0))
    inside &= T["ok"][f]
    den = dx * n[:, 0] + dy * n[:, 1] + n[:, 2]
    num = T["num"][f]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        z = num / den
        if slip == "fp32_z":
            z = (num.astype(np.float32) / den.astype(np.float32)).astype(np.float64)
    live = inside & (den != 0)
    lo = z > near if slip == "strict_near" else z >= near
    hi = z < far if slip == "strict_far" else z <= far
    hit = live & lo & hi
    flags = {"near": live & (z < near), "near_equal": live & (z == near), "far": live & (z > far),
             "far_equal": live & (z == far), "edge_zero": inside & ((ek[0] == 0) | (ek[1] == 0) | (ek[2] == 0)),
             "den_zero": inside & (den == 0)}
    return np.where(hit, z, np.inf), flags


def _resolve(pix, z, flags, n_pix):
    """min z per pixel rounded once to fp32 (0 without a hit), and the count of pixels reaching each decision."""
    best = np.full(n_pix, np.inf)
    np.minimum.at(best, pix, z)
    hit = np.isfinite(best)
    out = np.where(hit, best, 0.0).astype(np.float32)
    at_min = np.isfinite(z) & (z.astype(np.float32) == out[pix])
    stats = {"hit": int(hit.sum()), "tie": int((np.bincount(pix[at_min], minlength=n_pix) > 1).sum())}
    for k, v in flags.items():
        stats[k] = int(np.unique(pix[v]).size)
    return out, stats


def oracle_boxes(T, cam32, W, H, near, far, margin=2, whole_frame_straddlers=True):
    """The rule's own pixel boxes [F,4] (x0, x1, y0, y1; x1 < x0 when the face cannot hit).  Faces with every corner in
    front of near (to 1e-6 relative) or beyond far are dropped; the others with a corner in front of near take the whole
    frame, or with whole_frame_straddlers=False the box of the face clipped at near / 2; the rest the box of their
    three projected corners.  Every box is widened by `margin` px (the kernel's is 1)."""
    fx, fy, cx, cy, _ = kernel_camera(cam32)
    near, far = float(np.float32(near)), float(np.float32(far))
    P = T["P"]
    z = P[..., 2]
    zmin, zmax = z.min(1), z.max(1)
    drop = ~T["ok"] | (zmax < near * (1 - 1e-6)) | (zmin > far * (1 + 1e-6))
    strad = ~drop & (zmin < near)
    clip = near / 2 if not whole_frame_straddlers else near
    F = P.shape[0]
    x0, x1, y0, y1 = (np.full(F, s * np.inf) for s in (1, -1, 1, -1))
    for k in range(3):
        a, b = P[:, k], P[:, (k + 1) % 3]
        pts = [(a[:, 2] >= clip, a[:, 0], a[:, 1], a[:, 2])]
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (clip - a[:, 2]) / (b[:, 2] - a[:, 2])
            pts.append(((a[:, 2] < clip) != (b[:, 2] < clip), a[:, 0] + s * (b[:, 0] - a[:, 0]),
                        a[:, 1] + s * (b[:, 1] - a[:, 1]), np.full(F, clip)))
        for m, X, Y, Z in pts:
            m = m & ~drop
            with np.errstate(divide="ignore", invalid="ignore"):
                u, v = _project(fx, fy, cx, cy, X, Y, Z)
            x0, x1 = np.where(m, np.minimum(x0, u), x0), np.where(m, np.maximum(x1, u), x1)
            y0, y1 = np.where(m, np.minimum(y0, v), y0), np.where(m, np.maximum(y1, v), y1)
    with np.errstate(invalid="ignore"):
        box = np.stack([np.clip(np.floor(x0) - margin, 0, W - 1), np.clip(np.ceil(x1) + margin, -1, W - 1),
                        np.clip(np.floor(y0) - margin, 0, H - 1), np.clip(np.ceil(y1) + margin, -1, H - 1)], 1)
    box = np.nan_to_num(box, nan=-1.0)
    if whole_frame_straddlers:
        box[strad] = [0, W - 1, 0, H - 1]
    box[drop] = [0, -1, 0, -1]
    return box.astype(np.int64)


def depth_kernel_rule(verts32, faces, cam32, W, H, near=0.01, far=10.0, pixels=None, slip=None, margin=2,
                      whole_frame_straddlers=True, max_pairs=1 << 22):
    """The kernel's rule on the rule's own boxes: ([H,W] float32 depth, or [len(pixels)] at the flat pixel indices
    `pixels`; decision counts).  With `pixels`, candidate faces are found through a 16-px grid of the boxes."""
    _, _, _, _, E = kernel_camera(cam32)
    T = triangle_setup(verts32, faces, E)
    boxes = oracle_boxes(T, cam32, W, H, near, far, margin, whole_frame_straddlers)
    bw = np.maximum(boxes[:, 1] - boxes[:, 0] + 1, 0)
    bh = np.maximum(boxes[:, 3] - boxes[:, 2] + 1, 0)
    fs = np.nonzero(bw * bh > 0)[0]
    chunks = []
    if pixels is None:
        n_out, slot = W * H, None
        area = (bw * bh)[fs]
        cut = np.searchsorted(np.cumsum(area), np.arange(1, area.sum() // max_pairs + 2) * max_pairs)
        for part in np.split(fs, np.unique(np.minimum(cut, len(fs)))):
            if part.size == 0:
                continue
            r, p = _expand(np.zeros(len(part), np.int64), (bw * bh)[part])
            f = part[r]
            chunks.append((f, boxes[f, 0] + p % bw[f], boxes[f, 2] + p // bw[f]))
    else:
        pixels = np.asarray(pixels, np.int64)
        n_out = pixels.size
        G = 16
        ncx, ncy = (W + G - 1) // G, (H + G - 1) // G
        cw = boxes[fs, 1] // G - boxes[fs, 0] // G + 1
        ch = boxes[fs, 3] // G - boxes[fs, 2] // G + 1
        r, q = _expand(np.zeros(len(fs), np.int64), cw * ch)
        cell = (boxes[fs[r], 2] // G + q // cw[r]) * ncx + boxes[fs[r], 0] // G + q % cw[r]
        order = np.argsort(cell, kind="stable")
        cell_faces = fs[r][order]
        start = np.searchsorted(cell[order], np.arange(ncx * ncy + 1))
        pi, pj = pixels % W, pixels // W
        pc = (pj // G) * ncx + pi // G
        cnt = start[pc + 1] - start[pc]
        cut = np.searchsorted(np.cumsum(cnt), np.arange(1, cnt.sum() // max_pairs + 2) * max_pairs)
        for part in np.split(np.arange(n_out), np.unique(np.minimum(cut, n_out))):
            if part.size == 0:
                continue
            r, k = _expand(start[pc[part]], cnt[part])
            f, s = cell_faces[k], part[r]
            b = boxes[f]
            m = (pi[s] >= b[:, 0]) & (pi[s] <= b[:, 1]) & (pj[s] >= b[:, 2]) & (pj[s] <= b[:, 3])
            chunks.append((f[m], pi[s[m]], pj[s[m]], s[m]))
    pix_all, z_all, fl_all = [], [], {k: [] for k in DECISIONS[1:-1]}
    for c in chunks:
        f, i, j = c[:3]
        z, fl = eval_pairs(T, cam32, f, i, j, near, far, slip)
        pix_all.append(j * W + i if pixels is None else c[3])
        z_all.append(z)
        for k in fl_all:
            fl_all[k].append(fl[k])
    if not z_all:
        return (np.zeros(n_out, np.float32) if pixels is not None else np.zeros((H, W), np.float32)), \
            {k: 0 for k in DECISIONS}
    pix = np.concatenate(pix_all)
    out, stats = _resolve(pix, np.concatenate(z_all), {k: np.concatenate(v) for k, v in fl_all.items()}, n_out)
    return (out if pixels is not None else out.reshape(H, W)), stats


def depth_kernel_mirror(verts32, faces, cam32, W, H, near=0.01, far=10.0, slip=None):
    """dnr_mesh_depth's three passes restated (box, scan, item -> face search, pixel tests): ([H,W] float32, counts,
    boxes, item counts).  Equal to depth_kernel_rule whenever the kernel's boxes hold every pixel the rule hits."""
    _, _, _, _, E = kernel_camera(cam32)
    T = triangle_setup(verts32, faces, E)
    boxes, counts = kernel_boxes(T, cam32, W, H, near, far, slip)
    f, i, j = kernel_pairs(boxes, counts, slip)
    z, fl = eval_pairs(T, cam32, f, i, j, near, far, slip)
    out, stats = _resolve(j * W + i, z, fl, W * H)
    return out.reshape(H, W), stats, boxes, counts


def depth_scalar(verts32, faces, cam32, W, H, near=0.01, far=10.0):
    """The rule as a plain per-pixel, per-face loop in Python floats (fp64), every face over the whole frame."""
    fx, fy, cx, cy, E = (float(x) if np.ndim(x) == 0 else x.tolist() for x in kernel_camera(cam32))
    near, far = float(np.float32(near)), float(np.float32(far))
    V = np.asarray(verts32, np.float32).astype(np.float64).tolist()
    F = np.asarray(faces, np.int64).reshape(-1, 3).tolist()

    def cam(p):
        return [E[r][0] * p[0] + E[r][1] * p[1] + E[r][2] * p[2] + E[r][3] for r in range(3)]

    def cross(a, b):
        return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]

    tris = []
    for ids in F:
        if any(k < 0 or k >= len(V) for k in ids):
            continue
        P = [cam(V[k]) for k in ids]
        e = []
        for k in range(3):
            a, b = k, (k + 1) % 3
            e.append(cross(P[a], P[b]) if ids[a] <= ids[b] else [-c for c in cross(P[b], P[a])])
        n = cross([P[1][k] - P[0][k] for k in range(3)], [P[2][k] - P[0][k] for k in range(3)])
        if n == [0.0, 0.0, 0.0]:
            continue
        tris.append((e, n, n[0] * P[0][0] + n[1] * P[0][1] + n[2] * P[0][2]))
    out = np.zeros((H, W), np.float32)
    for j in range(H):
        dy = (j + 0.5 - cy) / fy
        for i in range(W):
            dx = (i + 0.5 - cx) / fx
            best = np.inf
            for e, n, num in tris:
                s = [dx * ek[0] + dy * ek[1] + ek[2] for ek in e]
                if not (all(v >= 0.0 for v in s) or all(v <= 0.0 for v in s)):
                    continue
                den = dx * n[0] + dy * n[1] + n[2]
                if den == 0.0:
                    continue
                z = num / den
                if near <= z <= far:
                    best = min(best, z)
            if best < np.inf:
                out[j, i] = np.float32(best)
    return out


def project_points(points, cam):
    """dnr_mesh_visibility's projection of fp64 points by an fp64 block: (px, py, pz)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    fx, fy, cx, cy, E = _split(cam)
    X = E[0, 0] * x + E[0, 1] * y + E[0, 2] * z + E[0, 3]
    Y = E[1, 0] * x + E[1, 1] * y + E[1, 2] * z + E[1, 3]
    Z = E[2, 0] * x + E[2, 1] * y + E[2, 2] * z + E[2, 3]
    pz = Z + 1e-8
    with np.errstate(divide="ignore", invalid="ignore"):
        return (fx * X + cx * Z) / pz, (fy * Y + cy * Z) / pz, pz
