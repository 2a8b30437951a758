"""Mesh evaluation on the device: the reference's `eval/eval_mesh_vis_cull.py` (visibility culling, then Acc / Comp /
C-L1 / NC / F-score at 0.05) and `metrics.PDMetrics` (/root/reference/dn_splatter/eval/eval_mesh_vis_cull.py,
dn_splatter/metrics.py:39-56) without pyrender, trimesh or open3d.

- `render_mesh_depth` ray-casts z-depth maps of a triangle mesh (`dnr_mesh_depth`: no back-face culling, nearest hit,
  watertight on shared edges) instead of two pyrender passes with flipped winding.
- `cull_mesh` counts, per vertex of the subdivided mesh, the views that see it unoccluded and the views whose sensor depth
  is missing there (`dnr_mesh_visibility`, fp64 projection, chunks of views), and keeps the reference's faces.
- `subdivide_to_size`, `sample_surface` and the metric reductions are torch ops on the device; nearest neighbours are
  `sugar.KnnIndex`.
- `evaluate_mesh` / `evaluate_mesh_files` are the script's `main`; `read_triangle_mesh` reads general PLY meshes.

Deviations are listed in DESIGN.md §2 (exact fp32 ray-cast depth, the canonical-edge coverage rule, torch sample draws,
Python floats in mesh_metrics.json).  No CPU path: the kernels need CUDA tensors.
"""
from __future__ import annotations

import json
import logging
import os
from typing import Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib as L
from .mesh import TriangleMesh, _quantile_sorted, _views, write_ply
from .sugar import KnnIndex

log = logging.getLogger(__name__)

CULL_NAME = "mesh_cull.ply"
METRICS_NAME = "mesh_metrics.json"
METRIC_KEYS = ("Acc", "Comp", "C-L1", "NC", "F-score")
# eval_mesh_vis_cull.py:400-407: the ScanNet++ gt mesh is brought to the poses' frame
SCANNETPP_TRANSFORM = np.array([[1, 0, 0, 0], [0, 0, 1, 0], [0, -1, 0, 0], [0, 0, 0, 1]], np.float64)


def _device(device=None) -> torch.device:
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda" or not torch.cuda.is_available():
        raise L.DnrError("dn_splatter_b200.mesh_eval needs a CUDA device (no CPU path)")
    return dev


def _mesh_on(mesh: TriangleMesh, dev, dtype=torch.float32) -> Tuple[Tensor, Tensor]:
    v = torch.as_tensor(mesh.vertices).to(device=dev, dtype=dtype).reshape(-1, 3).contiguous()
    f = torch.as_tensor(mesh.faces).to(device=dev, dtype=torch.int64).reshape(-1, 3).contiguous()
    return v, f


def _image_size(views) -> Tuple[int, int]:
    sizes = {(int(v.width.flatten()[0]), int(v.height.flatten()[0])) for v in views}
    if len(sizes) != 1:
        raise ValueError(f"mesh_eval: all views must share one image size, got {sorted(sizes)}")
    return sizes.pop()


def camera_blocks(cameras, dtype=torch.float32, device=None) -> Tensor:
    """[n,16] {fx, fy, cx, cy, world->camera [3,4]} per view (TSDFVolume.camera_block's layout); the world->camera
    matrix is inverse(c2w @ diag(1, -1, -1, 1)) in fp64, rounded to `dtype`."""
    rows = []
    for cam in _views(cameras):
        c2w = np.eye(4)
        c2w[:3, :4] = cam.camera_to_worlds.detach().reshape(-1, 3, 4)[0].cpu().double().numpy()
        E = np.linalg.inv(c2w @ np.diag([1.0, -1.0, -1.0, 1.0]))[:3]
        intr = [float(getattr(cam, k).flatten()[0]) for k in ("fx", "fy", "cx", "cy")]
        rows.append(np.concatenate([np.asarray(intr, np.float64), E.reshape(-1)]))
    return torch.from_numpy(np.stack(rows)).to(device=_device(device), dtype=dtype)


def _depth_call(v: Tensor, f32: Tensor, cams: Tensor, W: int, H: int, near: float, far: float) -> Tensor:
    n = cams.shape[0]
    out = torch.empty((n, H, W), dtype=torch.float32, device=v.device)
    if f32.shape[0] == 0:
        return out.zero_()
    lib = L.load()
    ws, nbytes = L.workspace(lib.dnr_mesh_depth_workspace_bytes, f32.shape[0], device=v.device)
    L.check(lib.dnr_mesh_depth(v.data_ptr(), v.shape[0], f32.data_ptr(), f32.shape[0], cams.data_ptr(), n, W, H, float(near),
                               float(far), ws.data_ptr(), nbytes, out.data_ptr(), L.stream()), "dnr_mesh_depth")
    return out


@torch.no_grad()
def render_mesh_depth(mesh: TriangleMesh, cameras, near: float = 0.01, far: float = 10.0, device=None) -> Tensor:
    """[n,H,W] float32 z-depth of `mesh` from every view (nerfstudio / OpenGL c2w): the nearest surface on the ray through
    each pixel centre, both faces of each triangle, 0 where no hit lies in [near, far].  The reference's pyrender
    defaults are near = 0.01 and far = 10."""
    dev = _device(device)
    views = _views(cameras)
    W, H = _image_size(views)
    v, f = _mesh_on(mesh, dev)
    return _depth_call(v, f.to(torch.int32).contiguous(), camera_blocks(views, torch.float32, dev), W, H, near, far)


def remove_unreferenced(vertices: Tensor, faces: Tensor) -> Tuple[Tensor, Tensor]:
    used = torch.zeros(vertices.shape[0], dtype=torch.bool, device=vertices.device)
    used[faces.reshape(-1)] = True
    remap = torch.cumsum(used.to(torch.int64), 0) - 1
    return vertices[used], remap[faces]


def _edge_lengths(v: Tensor, f: Tensor) -> Tensor:
    t = v[f]
    d = t[:, [1, 2, 0]] - t
    return (d * d).sum(dim=2).sqrt()


@torch.no_grad()
def subdivide_to_size(mesh: TriangleMesh, max_edge: float = 0.015, max_iter: int = 10) -> TriangleMesh:
    """trimesh.remesh.subdivide_to_size's rule [EXT]: each round, every face with an edge longer than max_edge splits
    1 -> 4 at its edge midpoints (a + b) / 2 (welded across faces); the other faces are final.  Faces still too long
    after max_iter rounds are dropped with a warning, as trimesh does.  fp64 vertices, int64 faces, on the device."""
    dev = _device()
    v, cur = _mesh_on(mesh, dev, torch.float64)
    done = []
    for it in range(max_iter + 1):
        long_ = (_edge_lengths(v, cur) > max_edge).any(dim=1)
        done.append(cur[~long_])
        cur = cur[long_]
        if cur.shape[0] == 0:
            break
        if it == max_iter:
            log.warning("subdivide_to_size: %d faces still have edges over %g after %d rounds; dropped", cur.shape[0],
                        max_edge, max_iter)
            break
        nv = v.shape[0]
        e = torch.cat([cur[:, [0, 1]], cur[:, [1, 2]], cur[:, [2, 0]]]).sort(dim=1).values
        key, inv = torch.unique(e[:, 0] * nv + e[:, 1], return_inverse=True)
        a, b = key // nv, key % nv
        v = torch.cat([v, (v[a] + v[b]) / 2])
        m = (nv + inv).reshape(3, -1)
        f0, f1, f2 = cur[:, 0], cur[:, 1], cur[:, 2]
        cur = torch.cat([torch.stack([f0, m[0], m[2]], 1), torch.stack([m[0], f1, m[1]], 1),
                         torch.stack([m[2], m[1], f2], 1), torch.stack([m[0], m[1], m[2]], 1)])
    return TriangleMesh(v, torch.cat(done), None)


def _as_depth_maps(gt_depths):
    if gt_depths is None:
        return None
    if isinstance(gt_depths, (list, tuple)):
        return [torch.as_tensor(np.asarray(d) if not isinstance(d, Tensor) else d) for d in gt_depths]
    return gt_depths


@torch.no_grad()
def visibility_counts(points: Tensor, cameras, rendered: Optional[Tensor] = None, gt_depths=None, eps: float = 0.02,
                      chunk: int = 16) -> Tuple[Tensor, Tensor]:
    """obs / invalid int32 counts of get_grid_culling_pattern (eval_mesh_vis_cull.py:68-149) at points [n,3] (fp64 on the
    device): rendered [n_views,H,W] (None: no occlusion test), gt_depths [n_views,H,W] or a list of [H,W] maps (None: no
    missing-depth test).  Views go to the kernel in chunks of `chunk`."""
    views = _views(cameras)
    W, H = _image_size(views)
    dev = points.device
    p = points.to(torch.float64).contiguous()
    cams = camera_blocks(views, torch.float64, dev)
    obs = torch.zeros(p.shape[0], dtype=torch.int32, device=dev)
    inv = torch.zeros(p.shape[0], dtype=torch.int32, device=dev)
    if p.shape[0] == 0:
        return obs, inv
    gts = _as_depth_maps(gt_depths)
    for c0 in range(0, len(views), chunk):
        c1 = min(c0 + chunk, len(views))
        r = None if rendered is None else rendered[c0:c1].to(device=dev, dtype=torch.float32).contiguous()
        g = None
        if gts is not None:
            g = torch.stack([torch.as_tensor(gts[k]).to(device=dev, dtype=torch.float32).reshape(H, W) for k in range(c0, c1)])
        L.check(L.load().dnr_mesh_visibility(p.data_ptr(), p.shape[0], cams[c0:c1].contiguous().data_ptr(),
                                             None if r is None else r.data_ptr(), None if g is None else g.data_ptr(), c1 - c0,
                                             W, H, float(eps), obs.data_ptr(), inv.data_ptr(), L.stream()), "dnr_mesh_visibility")
    return obs, inv


def keep_faces(obs: Tensor, invalid: Tensor, faces: Tensor) -> Tensor:
    """eval_mesh_vis_cull.py:251-260: some vertex with obs > 3, and not all three with invalid > 0.7 * obs."""
    o, i = obs[faces].to(torch.float64), invalid[faces].to(torch.float64)
    return (o > 3).any(dim=1) & ~(i > 0.7 * o).all(dim=1)


@torch.no_grad()
def cull_mesh(mesh: TriangleMesh, cameras, gt_depths=None, *, remove_missing_depth: bool = True, remove_occlusion: bool = True,
              subdivide: bool = True, max_edge: float = 0.015, eps: float = 0.02, far: float = 10.0, chunk: int = 16,
              device=None) -> TriangleMesh:
    """eval_mesh_vis_cull.py:176-266: the unsubdivided mesh (unreferenced vertices removed) is rendered from every view;
    the obs / invalid counts are taken on the vertices of the subdivided mesh; a face survives when some vertex has
    obs > 3 and not all three have invalid > 0.7 * obs; unreferenced vertices are dropped.  gt_depths: the views'
    sensor depth maps ([n,H,W] or a list of [H,W]; 0 = missing), required by remove_missing_depth.  Depth maps are rendered
    and counted `chunk` views at a time.  Returns fp64 vertices and int64 faces on the device."""
    if remove_missing_depth and gt_depths is None:
        raise ValueError("cull_mesh: remove_missing_depth needs gt_depths (pass remove_missing_depth=False without them)")
    dev = _device(device)
    views = _views(cameras)
    W, H = _image_size(views)
    v64, f = _mesh_on(mesh, dev, torch.float64)
    v64, f = remove_unreferenced(v64, f)
    v32, f32 = v64.float().contiguous(), f.to(torch.int32).contiguous()
    sub = subdivide_to_size(TriangleMesh(v64, f, None), max_edge) if subdivide else TriangleMesh(v64, f, None)
    points = sub.vertices.contiguous()
    obs = torch.zeros(points.shape[0], dtype=torch.int32, device=dev)
    inv = torch.zeros_like(obs)
    cams32 = camera_blocks(views, torch.float32, dev)
    gts = _as_depth_maps(gt_depths) if remove_missing_depth else None
    for c0 in range(0, len(views), chunk):
        c1 = min(c0 + chunk, len(views))
        rendered = _depth_call(v32, f32, cams32[c0:c1].contiguous(), W, H, 0.01, far) if remove_occlusion else None
        o, i = visibility_counts(points, views[c0:c1], rendered, None if gts is None else gts[c0:c1], eps, chunk=c1 - c0)
        obs += o
        inv += i
    keep = keep_faces(obs, inv, sub.faces)
    cv, cf = remove_unreferenced(points, sub.faces[keep])
    return TriangleMesh(cv, cf, None)


def mesh_area(mesh: TriangleMesh) -> float:
    v, f = _mesh_on(mesh, _device(), torch.float64)
    t = v[f]
    return float(0.5 * torch.linalg.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]).norm(dim=1).sum())


@torch.no_grad()
def sample_surface(mesh: TriangleMesh, count: int, generator: Optional[torch.Generator] = None, return_index: bool = False):
    """trimesh.sample.sample_surface's rule [EXT]: faces drawn with probability proportional to their area (uniform draws
    scaled by the fp64 cumulative area, searchsorted), uniform barycentrics by parallelogram folding.  Returns float32
    points [count,3] and the unit normals of their faces (and the face indices with return_index).  Draws come from
    `generator` (a CUDA torch.Generator)."""
    dev = _device(generator.device if generator is not None else None)
    v, f = _mesh_on(mesh, dev, torch.float64)
    t = v[f]
    e1, e2 = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    cr = torch.linalg.cross(e1, e2)
    cum = torch.cumsum(0.5 * cr.norm(dim=1), 0)
    r = torch.rand(count, dtype=torch.float64, device=dev, generator=generator) * cum[-1]
    idx = torch.searchsorted(cum, r).clamp_(max=f.shape[0] - 1)
    lengths = torch.rand((count, 2), dtype=torch.float64, device=dev, generator=generator)
    fold = lengths.sum(dim=1) > 1.0
    lengths[fold] -= 1.0
    lengths = lengths.abs()
    pts = t[idx, 0] + e1[idx] * lengths[:, :1] + e2[idx] * lengths[:, 1:]
    n = cr[idx]
    n = n / n.norm(dim=1, keepdim=True)
    out = (pts.float(), n.float())
    return out + (idx,) if return_index else out


def _nearest(data: Tensor, queries: Tensor) -> Tuple[Tensor, Tensor]:
    if data.shape[0] == 0 or queries.shape[0] == 0:
        raise ValueError("mesh_eval: nearest neighbours of an empty point set")
    idx, dist = KnnIndex(data).query(queries, 1, skip_first=False, return_distances=True)
    return dist[:, 0], idx[:, 0]


@torch.no_grad()
def metrics_from_samples(pred_points: Tensor, pred_normals: Tensor, gt_points: Tensor, gt_normals: Tensor,
                         threshold: float = 0.05) -> Dict[str, float]:
    """compute_metrics (eval_mesh_vis_cull.py:333-397) on given samples: Acc / Comp are the mean nearest-neighbour
    distances pred -> gt / gt -> pred, C-L1 their mean, NC the mean of the two directions' mean |n . n'|, F-score
    2PR / (P + R) of the fractions within `threshold` (<=), NaN when P + R = 0.  Reductions in fp64."""
    pp, gp = pred_points.float().contiguous(), gt_points.float().contiguous()
    pn = torch.nn.functional.normalize(pred_normals.double(), dim=-1)
    gn = torch.nn.functional.normalize(gt_normals.double(), dim=-1)
    comp, ci = _nearest(pp, gp)
    acc, ai = _nearest(gp, pp)
    comp_n = (pn[ci] * gn).sum(-1).abs().mean()
    acc_n = (gn[ai] * pn).sum(-1).abs().mean()
    hits = torch.stack([(acc <= threshold).sum(), (comp <= threshold).sum()]).double()
    vals = torch.cat([torch.stack([acc.double().mean(), comp.double().mean(), comp_n, acc_n]), hits]).cpu().tolist()
    a, c, cn, an = vals[:4]
    p, r = vals[4] / acc.shape[0], vals[5] / comp.shape[0]  # exact fractions: P = R = 1 gives F = 1
    f = 2 * p * r / (p + r) if p + r > 0 else float("nan")
    return {"Acc": a, "Comp": c, "C-L1": 0.5 * (a + c), "NC": 0.5 * cn + 0.5 * an, "F-score": f}


@torch.no_grad()
def compute_metrics(pred: TriangleMesh, gt: TriangleMesh, threshold: float = 0.05,
                    generator: Optional[torch.Generator] = None) -> Dict[str, float]:
    """eval_mesh_vis_cull.py:333-397: int(area * 1e4) area-weighted samples per mesh, then `metrics_from_samples`.
    Without a generator the draws are seeded with 0."""
    if generator is None:
        generator = torch.Generator(device=_device()).manual_seed(0)
    n_p, n_g = int(mesh_area(pred) * 1e4), int(mesh_area(gt) * 1e4)
    pp, pn = sample_surface(pred, n_p, generator)
    gp, gn = sample_surface(gt, n_g, generator)
    return metrics_from_samples(pp, pn, gp, gn, threshold)


@torch.no_grad()
def point_cloud_metrics(pred_points: Tensor, gt_points: Tensor, percentile: float = 90,
                        threshold: float = 0.05) -> Tuple[float, float]:
    """metrics.PDMetrics (metrics.py:39-56): (accuracy, completeness) = (numpy's linear-interpolation `percentile` of the
    pred -> gt distances, 100 * the fraction of gt -> pred distances < threshold (strict, unlike the F-score's <=))."""
    dev = _device()
    pp = torch.as_tensor(pred_points).to(dev, torch.float32)
    gp = torch.as_tensor(gt_points).to(dev, torch.float32)
    d_acc, _ = _nearest(gp, pp)
    d_comp, _ = _nearest(pp, gp)
    acc = _quantile_sorted(d_acc.double().sort().values, percentile / 100.0)
    comp = 100.0 * (d_comp < threshold).double().mean()
    return float(acc), float(comp)


@torch.no_grad()
def evaluate_mesh(pred: TriangleMesh, gt: TriangleMesh, cameras, output_dir: str, gt_depths=None, *, threshold: float = 0.05,
                  max_edge: float = 0.015, generator: Optional[torch.Generator] = None,
                  rename_output_file: Optional[str] = None) -> Dict[str, float]:
    """The script's main (eval_mesh_vis_cull.py:439-470) on in-memory inputs: cull gt and pred to the views (the
    missing-depth test only with gt_depths), write the culled pred mesh as `output_dir/mesh_cull.ply`, compute the
    metrics and write them as `output_dir/mesh_metrics.json` (or rename_output_file).  Returns the metrics."""
    kw = dict(remove_missing_depth=gt_depths is not None, remove_occlusion=True, subdivide=True, max_edge=max_edge)
    gt_c = cull_mesh(gt, cameras, gt_depths, **kw)
    pred_c = cull_mesh(pred, cameras, gt_depths, **kw)
    os.makedirs(output_dir, exist_ok=True)
    write_ply(os.path.join(output_dir, CULL_NAME), TriangleMesh(pred_c.vertices.float(), pred_c.faces.to(torch.int32), None))
    rst = compute_metrics(pred_c, gt_c, threshold, generator)
    with open(os.path.join(output_dir, rename_output_file or METRICS_NAME), "w") as fh:
        json.dump(rst, fh)
    return rst


def _read_png(path: str) -> np.ndarray:
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im)


def resize_nearest(img: np.ndarray, W: int, H: int) -> np.ndarray:
    """cv2.resize(img, (W, H), interpolation=cv2.INTER_NEAREST)'s index rule [EXT]: destination pixel x reads source
    column min(floor(x * src_w / W), src_w - 1), likewise for rows."""
    h, w = img.shape[:2]
    xs = np.minimum(np.floor(np.arange(W) * (w / W)).astype(np.int64), w - 1)
    ys = np.minimum(np.floor(np.arange(H) * (h / H)).astype(np.int64), h - 1)
    return img[ys[:, None], xs[None, :]]


def load_dataset_views(transformation_file: str, dataset_path: str, dataset: str = "scannetpp"):
    """(cameras, gt depth maps [n,H,W] float32) of a transforms json (eval_mesh_vis_cull.py:198-227).  Replica: depth
    PNG / 6553.5 and c2w[:3, 1:3] *= -1; ScanNet++: depth/<frame name>.png / 1000, resized to (W, H) nearest."""
    from .cameras import Cameras

    if dataset not in ("scannetpp", "replica"):
        raise ValueError(f"evaluate_mesh_files: dataset must be 'scannetpp' or 'replica', got {dataset!r}")
    with open(transformation_file) as fh:
        tf = json.load(fh)
    H, W = int(tf["h"]), int(tf["w"])
    views, depths = [], []
    for frame in tf["frames"]:
        c2w = np.array(frame["transform_matrix"], np.float32)[:3, :4]
        if dataset == "scannetpp":
            name = frame["file_path"].split("/")[-1].split(".")[0]
            d = _read_png(os.path.join(dataset_path, "depth", name + ".png")) / 1000.0
            d = resize_nearest(d, W, H)
        else:
            d = (_read_png(os.path.join(dataset_path, frame["depth_file_path"])) / 6553.5).astype(np.float32)
            c2w[0:3, 1:3] *= -1
        views.append(Cameras(torch.from_numpy(c2w)[None], tf["fl_x"], tf["fl_y"], tf["cx"], tf["cy"], W, H))
        depths.append(np.asarray(d, np.float32))
    return views, np.stack(depths)


def evaluate_mesh_files(gt_mesh_path: str, pred_mesh_path: str, transformation_file: str, dataset_path: str,
                        dataset: str = "scannetpp", output: Optional[str] = None, rename_output_file: Optional[str] = None,
                        align: bool = False, generator: Optional[torch.Generator] = None) -> Dict[str, float]:
    """eval_mesh_vis_cull.py:410-478: reads both meshes (PLY), brings a ScanNet++ gt mesh to the poses' frame, culls both
    with the dataset's views and depth maps, writes `mesh_cull.ply` and `mesh_metrics.json` to `output` (default: the
    pred mesh's directory) and returns the metrics."""
    if align:
        raise NotImplementedError("evaluate_mesh_files: ICP alignment (align=True) is not implemented")
    gt = read_triangle_mesh(str(gt_mesh_path))
    pred = read_triangle_mesh(str(pred_mesh_path))
    if dataset == "scannetpp":
        v = gt.vertices.double().numpy()
        v = v @ SCANNETPP_TRANSFORM[:3, :3].T + SCANNETPP_TRANSFORM[:3, 3]
        gt = TriangleMesh(torch.from_numpy(v), gt.faces, gt.colors)
    views, depths = load_dataset_views(str(transformation_file), str(dataset_path), dataset)
    out = str(output) if output is not None else os.path.dirname(os.path.abspath(str(pred_mesh_path)))
    return evaluate_mesh(pred, gt, views, out, depths, generator=generator, rename_output_file=rename_output_file)


# ---- PLY -----------------------------------------------------------------------------------------------------------
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def _ply_type(name: str, path: str) -> str:
    if name not in _PLY_TYPES:
        raise ValueError(f"{path}: unsupported PLY property type {name!r}")
    return _PLY_TYPES[name]


def _parse_header(data: bytes, path: str):
    if not data.startswith(b"ply"):
        raise ValueError(f"{path}: not a PLY file")
    end = data.find(b"end_header")
    if end < 0:
        raise ValueError(f"{path}: PLY header has no end_header")
    nl = data.find(b"\n", end)
    body = nl + 1 if nl >= 0 else len(data)
    fmt, elements = None, []
    for line in data[:end].decode("ascii", errors="replace").splitlines()[1:]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append({"name": tok[1], "count": int(tok[2]), "props": []})
        elif tok[0] == "property":
            if not elements:
                raise ValueError(f"{path}: PLY property before any element")
            if tok[1] == "list":
                elements[-1]["props"].append((tok[4], _ply_type(tok[2], path), _ply_type(tok[3], path)))
            else:
                elements[-1]["props"].append((tok[2], _ply_type(tok[1], path), None))
        else:
            raise ValueError(f"{path}: unexpected PLY header line {line!r}")
    if fmt not in ("ascii", "binary_little_endian", "binary_big_endian"):
        raise ValueError(f"{path}: unsupported PLY format {fmt!r}")
    return fmt, elements, body


def _read_binary_element(data: bytes, off: int, el, order: str, path: str):
    """(dict name -> array (lists: a list of per-row arrays, or an [n,k] array when every row has k items), new offset)."""
    props, n = el["props"], el["count"]
    if all(p[2] is None for p in props):
        dt = np.dtype([(p[0], order + p[1]) for p in props])
        if off + dt.itemsize * n > len(data):
            raise ValueError(f"{path}: PLY data ends inside element {el['name']!r}")
        arr = np.frombuffer(data, dt, n, off)
        return {p[0]: arr[p[0]] for p in props}, off + dt.itemsize * n
    if n > 0 and sum(p[2] is not None for p in props) == 1:  # fast path: one list with the same length on every row
        fields, k_off = [], off
        for name, t, it in props:
            if it is None:
                k_off += np.dtype(t).itemsize
            else:
                if k_off + np.dtype(t).itemsize > len(data):
                    raise ValueError(f"{path}: PLY data ends inside element {el['name']!r}")
                k = int(np.frombuffer(data, order + t, 1, k_off)[0])
                break
        for name, t, it in props:
            if it is None:
                fields.append((name, order + t))
            else:
                fields.append(("__n_" + name, order + t))
                fields.append((name, order + it, (k,)) if k > 0 else (name, order + it, (0,)))
        dt = np.dtype(fields)
        if off + dt.itemsize * n <= len(data):
            arr = np.frombuffer(data, dt, n, off)
            lname = next(p[0] for p in props if p[2] is not None)
            if (arr["__n_" + lname] == k).all():
                return {p[0]: arr[p[0]] for p in props}, off + dt.itemsize * n
    out = {p[0]: [] for p in props}  # general rows, one at a time
    for _ in range(n):
        for name, t, it in props:
            ts = np.dtype(order + t)
            if off + ts.itemsize > len(data):
                raise ValueError(f"{path}: PLY data ends inside element {el['name']!r}")
            val = np.frombuffer(data, ts, 1, off)[0]
            off += ts.itemsize
            if it is None:
                out[name].append(val)
            else:
                its = np.dtype(order + it)
                cnt = int(val)
                if off + its.itemsize * cnt > len(data):
                    raise ValueError(f"{path}: PLY data ends inside element {el['name']!r}")
                out[name].append(np.frombuffer(data, its, cnt, off).copy())
                off += its.itemsize * cnt
    return {p[0]: (np.asarray(out[p[0]]) if p[2] is None else out[p[0]]) for p in props}, off


def _read_ascii(data: bytes, body: int, elements, path: str):
    tokens = data[body:].split()
    pos, result = 0, {}
    for el in elements:
        cols = {p[0]: [] for p in el["props"]}
        for _ in range(el["count"]):
            for name, t, it in el["props"]:
                if pos >= len(tokens):
                    raise ValueError(f"{path}: PLY data ends inside element {el['name']!r}")
                if it is None:
                    cols[name].append(float(tokens[pos]))
                    pos += 1
                else:
                    cnt = int(tokens[pos])
                    if pos + 1 + cnt > len(tokens):
                        raise ValueError(f"{path}: PLY data ends inside element {el['name']!r}")
                    cols[name].append(np.array([float(x) for x in tokens[pos + 1:pos + 1 + cnt]], np.float64).astype(np.int64))
                    pos += 1 + cnt
        result[el["name"]] = {p[0]: (np.asarray(cols[p[0]], np.dtype(p[1])) if p[2] is None else cols[p[0]]) for p in el["props"]}
    return result


def _fan(lists) -> np.ndarray:
    if isinstance(lists, np.ndarray) and lists.ndim == 2:
        k = lists.shape[1]
        if k < 3:
            return np.zeros((0, 3), np.int64)
        return np.stack([np.stack([lists[:, 0], lists[:, j], lists[:, j + 1]], 1) for j in range(1, k - 1)], 1).reshape(
            -1, 3).astype(np.int64)
    tris = [np.stack([np.full(len(p) - 2, p[0]), p[1:-1], p[2:]], 1) for p in lists if len(p) >= 3]
    return np.concatenate(tris).astype(np.int64) if tris else np.zeros((0, 3), np.int64)


def read_triangle_mesh(path: str) -> TriangleMesh:
    """General PLY mesh reader: ascii, binary little- and big-endian; float or double x, y, z and any other vertex
    properties (red / green / blue, when present, become colours in [0, 1]: integer types / 255); faces from a
    `vertex_indices` or `vertex_index` list of any count / index type, polygons fan-triangulated.  Vertices are float32,
    or float64 when stored as double; faces int32 on the host."""
    with open(path, "rb") as fh:
        data = fh.read()
    fmt, elements, body = _parse_header(data, path)
    if fmt == "ascii":
        parsed = _read_ascii(data, body, elements, path)
    else:
        order = "<" if fmt == "binary_little_endian" else ">"
        parsed, off = {}, body
        for el in elements:
            parsed[el["name"]], off = _read_binary_element(data, off, el, order, path)
    if "vertex" not in parsed:
        raise ValueError(f"{path}: PLY file has no vertex element")
    vert = parsed["vertex"]
    if not all(k in vert for k in ("x", "y", "z")):
        raise ValueError(f"{path}: PLY vertices need x, y and z properties")
    double = any(p[1] == "f8" for el in elements if el["name"] == "vertex" for p in el["props"] if p[0] in "xyz")
    xyz = np.stack([np.asarray(vert[k], np.float64) for k in "xyz"], 1).astype(np.float64 if double else np.float32)
    colors = None
    if all(k in vert for k in ("red", "green", "blue")):
        c = np.stack([np.asarray(vert[k]) for k in ("red", "green", "blue")], 1)
        colors = torch.from_numpy((c.astype(np.float32) / 255.0) if np.issubdtype(c.dtype, np.integer) else c.astype(np.float32))
    faces = np.zeros((0, 3), np.int64)
    if "face" in parsed:
        face = parsed["face"]
        key = "vertex_indices" if "vertex_indices" in face else ("vertex_index" if "vertex_index" in face else None)
        if key is None:
            raise ValueError(f"{path}: PLY faces need a vertex_indices or vertex_index list")
        faces = _fan(face[key])
        if faces.size and (faces.min() < 0 or faces.max() >= xyz.shape[0]):
            raise ValueError(f"{path}: PLY face index out of range")
    return TriangleMesh(torch.from_numpy(np.ascontiguousarray(xyz)), torch.from_numpy(faces.astype(np.int32)), colors)
