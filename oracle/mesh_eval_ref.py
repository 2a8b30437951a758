"""fp64 numpy restatement of the mesh evaluation of /root/reference/dn_splatter/eval/eval_mesh_vis_cull.py and
metrics.PDMetrics (the rules dn_splatter_b200.mesh_eval implements on the device):

- `ray_cast_depth`: z-depth of a triangle mesh by a per-pixel Moller-Trumbore ray cast (small sizes only), both faces,
  nearest hit with near <= z <= far, 0 elsewhere; `near_edge_pixels` marks pixel centres within tol px of a triangle's
  boundary, where a fp32 / fp64 pair may legitimately disagree about a hit.
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


def visibility_counts(points, cams, W, H, rendered=None, gt=None, eps=0.02):
    """obs, invalid (int64 [n]) summed over the views; cams: fp64 camera blocks, rendered / gt: float32 [H,W] maps.
    rendered None: no occlusion test (obs = in frustum); gt None: invalid stays 0."""
    p = np.asarray(points, np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    obs = np.zeros(p.shape[0], np.int64)
    inv = np.zeros(p.shape[0], np.int64)
    for v, cam in enumerate(cams):
        fx, fy, cx, cy, E = _split(cam)
        X = E[0, 0] * x + E[0, 1] * y + E[0, 2] * z + E[0, 3]
        Y = E[1, 0] * x + E[1, 1] * y + E[1, 2] * z + E[1, 3]
        Z = E[2, 0] * x + E[2, 1] * y + E[2, 2] * z + E[2, 3]
        pz = Z + 1e-8
        px = (fx * X + cx * Z) / pz
        py = (fy * Y + cy * Z) / pz
        inside = (0 <= px) & (px <= W - 1) & (0 <= py) & (py <= H - 1) & (pz > 0)
        with np.errstate(invalid="ignore"):
            u = np.clip(np.nan_to_num(px), 0, W - 1).astype(np.int32)
            vv = np.clip(np.nan_to_num(py), 0, H - 1).astype(np.int32)
        if rendered is None:
            obs += inside
        else:
            r = np.asarray(rendered[v], np.float32)
            obs += inside & (pz < (r[vv, u] + np.float32(eps)))
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
