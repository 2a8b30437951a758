"""SuGaR-style density / level-set queries on the device (SURVEY.md §8f-4) — the host-side mirror of the reference's
`DNSplatterModel.get_closest_gaussians / get_density / get_sdf / get_sdf_weight / get_density_grad /
compute_level_surface_points` (/root/reference/dn_splatter/dn_model.py:1061-1494) and of `utils/knn.py: knn_sk`.

The two heavy pieces are CUDA kernels behind the C ABI: a grid-hash k-NN (`dnr_knn_build / dnr_knn_query`, instead of
sklearn on the CPU) and the per-ray density evaluation (`dnr_ray_densities`: 21 samples x 16 neighbours per pixel, instead
of 2M-sample torch passes that materialise [2M,16,3,3] tensors); the level-crossing search and the normal modes are
small gather ops on the device.  No CPU path.

The algorithms are pinned on the CPU (oracle/sugar_ref.py against goldens from the reference's own functions; a numpy
mirror of the grid search against sklearn) and the kernels against those on the GPU (tests/test_gpu_sugar.py).
"""
from __future__ import annotations

import ctypes as C
import math
import random
from typing import Dict, Optional, Sequence, Tuple

import torch
from torch import Tensor

from . import _lib as L
# module-level names that this module's functions look up at call time: the CPU proxy tests substitute _need_cuda here
# to run the host logic on CPU tensors, and the GPU kernel tests take the stream from here
from ._lib import need_cuda as _need_cuda
from ._lib import stream as _stream

KNN = 16
MAX_DIM = 256
TARGET_PER_CELL = 4.0


def choose_grid(lo: Sequence[float], hi: Sequence[float], mean: Sequence[float], std: Sequence[float], n: int) -> Dict:
    """Uniform grid over mean +- 3 sigma (clipped to the bounding box): outliers are clamped into the border cells by the
    kernels, so a few far-away Gaussians do not coarsen the grid where the points are.  ~4 points per cell."""
    glo = [max(l, m - 3.0 * s) for l, m, s in zip(lo, mean, std)]
    ghi = [min(h, m + 3.0 * s) for h, m, s in zip(hi, mean, std)]
    ext = [max(h - l, 1e-6) for l, h in zip(glo, ghi)]
    cell = (ext[0] * ext[1] * ext[2] * TARGET_PER_CELL / max(n, 1)) ** (1.0 / 3.0)
    cell = max(cell, max(ext) / MAX_DIM, 1e-9)
    dims = [max(1, min(MAX_DIM, int(math.ceil(e / cell)))) for e in ext]
    return {"lo": glo, "cell": cell, "dims": dims}


def _grid_struct(g: Dict) -> "L.DnrKnnGrid":
    s = L.DnrKnnGrid()
    s.lo[0], s.lo[1], s.lo[2] = g["lo"]
    s.cell, s.inv_cell = g["cell"], 1.0 / g["cell"]
    s.dims[0], s.dims[1], s.dims[2] = g["dims"]
    return s


class KnnIndex:
    """Grid-hash index over a point set; `query(y, k, skip_first)` mirrors knn_sk(x, y, k) when skip_first=True."""

    def __init__(self, points: Tensor):
        _need_cuda(points)
        self.points = points.detach().float().contiguous()
        n = self.points.shape[0]
        stats = torch.stack([self.points.amin(0), self.points.amax(0), self.points.mean(0),
                             self.points.std(0, unbiased=False) if n > 1 else torch.zeros(3, device=points.device)]).cpu()
        self.grid = choose_grid(stats[0].tolist(), stats[1].tolist(), stats[2].tolist(), stats[3].tolist(), n)
        self._g = _grid_struct(self.grid)
        lib = L.load()
        self.ws, nbytes = L.workspace(lib.dnr_knn_workspace_bytes, n, C.byref(self._g), device=points.device)
        L.check(lib.dnr_knn_build(self.points.data_ptr(), n, C.byref(self._g), self.ws.data_ptr(), nbytes, _stream()), "dnr_knn_build")

    def query(self, queries: Tensor, k: int, skip_first: bool = True, return_distances: bool = False):
        _need_cuda(queries)
        q = queries.detach().float().contiguous()
        m = q.shape[0]
        idx = torch.empty((m, k), dtype=torch.int64, device=q.device)
        dist = torch.empty((m, k), dtype=torch.float32, device=q.device) if return_distances else None
        if m > 0:
            L.check(L.load().dnr_knn_query(self.points.shape[0], C.byref(self._g), self.ws.data_ptr(), q.data_ptr(), m, k,
                                           int(skip_first), idx.data_ptr(), None if dist is None else dist.data_ptr(), _stream()),
                    "dnr_knn_query")
        return (idx, dist) if return_distances else idx


def knn_gpu(x: Tensor, y: Tensor, k: int) -> Tensor:
    """Drop-in for the reference's knn_sk(x, y, k): the k+1 nearest x of every y, nearest one dropped."""
    return KnnIndex(x).query(y, k, skip_first=True)


def k_nearest(x: Tensor, k: int) -> Tuple[Tensor, Tensor]:
    """nerfstudio's k_nearest_sklearn [EXT] on the device: distances / indices of the k nearest OTHER points."""
    idx, dist = KnnIndex(x).query(x, k, skip_first=True, return_distances=True)
    return dist, idx


def _params(model) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    gp = model.gauss_params
    out = tuple(gp[k].detach().float().contiguous() for k in ("means", "scales", "quats", "opacities"))
    _need_cuda(*out)
    return out


def _density_call(samples: Tensor, idx: Tensor, model, samples_per_row: int, clamp_min: float) -> Tensor:
    means, scales, quats, opac = _params(model)
    s = samples.detach().float().contiguous()
    idx = idx.long().contiguous()
    out = torch.empty(s.shape[0], dtype=torch.float32, device=s.device)
    if s.shape[0] > 0:
        L.check(L.load().dnr_density(s.data_ptr(), s.shape[0], idx.data_ptr(), idx.shape[1], samples_per_row, means.data_ptr(),
                                     scales.data_ptr(), quats.data_ptr(), opac.data_ptr(), means.shape[0], float(clamp_min),
                                     out.data_ptr(), _stream()), "dnr_density")
    return out


def get_closest_gaussians(model, samples: Tensor) -> Tensor:
    """dn_model.py:1061-1075."""
    return knn_gpu(model.gauss_params["means"].data, samples, KNN)


@torch.no_grad()
def get_density(model, sdf_samples: Tensor, closest_gaussians: Optional[Tensor] = None) -> Tensor:
    """dn_model.py:1077-1135 (forward value; the mesh exporters call it without gradients)."""
    if closest_gaussians is None:
        closest_gaussians = get_closest_gaussians(model, sdf_samples)
    return _density_call(sdf_samples, closest_gaussians, model, 1, 1e-4)


@torch.no_grad()
def get_sdf(model, sdf_samples: Tensor, closest_gaussians: Optional[Tensor] = None) -> Tensor:
    """dn_model.py:1137-1158."""
    return torch.sqrt(-2.0 * torch.log(get_density(model, sdf_samples, closest_gaussians)))


@torch.no_grad()
def get_sdf_weight(model, closest_gaussians_idx: Tensor) -> Tensor:
    """dn_model.py:1160-1165."""
    return torch.exp(model.gauss_params["scales"]).min(dim=-1)[0][closest_gaussians_idx].mean(dim=1)


def sample_points_in_gaussians(model, num_samples: int, vis_indices: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """dn_model.py:954-1004: pick Gaussians with probability given by the CUMULATIVE volume fractions (the reference
    hands the cumulative sums, not the volumes, to torch.multinomial — kept), then draw one point from each."""
    gp = model.gauss_params
    ext = torch.exp(gp["scales"] if vis_indices is None else gp["scales"][vis_indices])
    vol = (ext[..., 0] * ext[..., 1] * ext[..., 2]).abs()
    weights = vol.cumsum(dim=-1) / vol.sum(dim=-1, keepdim=True)
    picked = torch.multinomial(weights, num_samples=num_samples, replacement=True)
    if vis_indices is not None:
        picked = vis_indices[picked]
    noise = torch.randn(size=(len(picked), 3), device=gp["means"].device, dtype=torch.float)
    local = torch.exp(gp["scales"][picked]) * noise
    offsets = torch.bmm(_quat_to_rotmat(gp["quats"][picked]), local[..., None]).squeeze()
    return gp["means"][picked] + offsets, picked


def get_ideal_sdf(model, sdf_samples: Tensor, depth: Tensor, camera, mask: Optional[Tensor] = None,
                  min_depth: float = 0.01) -> Tuple[Tensor, Tensor]:
    """dn_model.py:1006-1058: rendered depth at the pixel a sample projects to, minus the sample's own z-depth.
    Reference quirks kept: fx is used for BOTH focal lengths, and pixel row / column 0 count as invalid (strict > 0)."""
    from .utils.camera_utils import project_pix

    c2w = camera.camera_to_worlds.squeeze(0)
    c2w = c2w @ torch.diag(torch.tensor([1, -1, -1, 1], device=c2w.device, dtype=c2w.dtype))
    fx = float(camera.fx.flatten()[0])
    proj = project_pix(sdf_samples, fx=fx, fy=fx, cx=float(camera.cx.flatten()[0]), cy=float(camera.cy.flatten()[0]),
                       c2w=c2w, device=sdf_samples.device, return_z_depths=True)
    uv = torch.floor(proj[:, :2]).long()
    W, H = int(camera.width.flatten()[0]), int(camera.height.flatten()[0])
    in_image = (uv[:, 0] > 0) & (uv[:, 0] < W) & (uv[:, 1] > 0) & (uv[:, 1] < H)
    valid = in_image
    if mask is not None:
        valid = in_image.detach().clone()
        valid[in_image] = mask[uv[in_image, 1], uv[in_image, 0]][..., 0]
    return depth[uv[valid, 1], uv[valid, 0], 0] - proj[valid][..., -1], valid


@torch.no_grad()
def get_sdf_loss_weight(model, valid_indices: Tensor, mode: str = "std") -> Optional[Tensor]:
    """dn_model.py:1167-1204: per-Gaussian weight of the sdf loss — product of the two largest extents ("area") or the
    standard deviation along the direction to the camera of the last rendered view ("std")."""
    gp = model.gauss_params
    if mode == "area":
        ext = torch.exp(gp["scales"][valid_indices]).clone().detach()
        return torch.prod(torch.gather(ext, dim=-1, index=torch.topk(ext, k=2, dim=-1)[1]), dim=-1)
    if mode == "std":
        cam_pos = model.camera.camera_to_worlds.detach()[..., :3, 3]
        view = cam_pos - gp["means"][valid_indices].detach()
        view = view / view.norm(dim=-1, keepdim=True)
        Rt = _quat_to_rotmat(gp["quats"][valid_indices]).transpose(-1, -2)  # R(q^-1)
        return (torch.exp(gp["scales"][valid_indices]) * torch.bmm(Rt, view[..., None])[..., 0]).norm(dim=-1)
    return None


def _quat_to_rotmat(q: Tensor) -> Tensor:
    w, x, y, z = torch.unbind(torch.nn.functional.normalize(q, dim=-1), dim=-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1),
    ], dim=-2)


def _mahalanobis(model, samples: Tensor, idx: Tensor):
    gp = model.gauss_params
    inv = 1.0 / torch.exp(gp["scales"].detach()[idx]).clamp(min=1e-3)
    Minv = _quat_to_rotmat(gp["quats"].detach()[idx]) * inv[..., None, :]
    man = Minv.transpose(-1, -2) @ (samples[:, None, :] - gp["means"].detach()[idx])[..., None]
    d2 = (man[..., 0] * man[..., 0]).sum(dim=-1).clamp(min=0.0, max=1e8)
    return d2, man, Minv


@torch.no_grad()
def get_density_grad(model, samples: Tensor, num_closest_gaussians: Optional[int] = None,
                     closest_gaussians: Optional[Tensor] = None) -> Tensor:
    """dn_model.py:1449-1494 (the weights are the clamped squared distances, as in the reference)."""
    if closest_gaussians is None:
        closest_gaussians = get_closest_gaussians(model, samples)
    if num_closest_gaussians is not None:
        assert num_closest_gaussians >= 1
        closest_gaussians = closest_gaussians[..., :num_closest_gaussians]
    d2, man, Minv = _mahalanobis(model, samples, closest_gaussians)
    return -torch.nn.functional.normalize((d2[..., None] * (Minv @ man)[..., 0]).sum(dim=-2), dim=-1)


@torch.no_grad()
def ray_densities(model, points: Tensor, idx: Tensor, cam_pos: Tensor, n_range: int = 21, range_size: float = 3.0):
    """Densities at the n_range samples of every pixel ray: (densities [P,n], offsets t [P,n], unit directions [P,3])."""
    means, scales, quats, opac = _params(model)
    p = points.detach().float().contiguous()
    idx = idx.long().contiguous()
    P = p.shape[0]
    dens = torch.empty((P, n_range), dtype=torch.float32, device=p.device)
    t = torch.empty((P, n_range), dtype=torch.float32, device=p.device)
    dirs = torch.empty((P, 3), dtype=torch.float32, device=p.device)
    if P > 0:
        cam = (C.c_float * 3)(*[float(v) for v in cam_pos.detach().cpu().reshape(3).tolist()])
        L.check(L.load().dnr_ray_densities(p.data_ptr(), P, idx.data_ptr(), idx.shape[1], cam, means.data_ptr(),
                                           scales.data_ptr(), quats.data_ptr(), opac.data_ptr(), means.shape[0], n_range,
                                           float(range_size), dens.data_ptr(), t.data_ptr(), dirs.data_ptr(), _stream()),
                "dnr_ray_densities")
    return dens, t, dirs


def _level_crossings(dens: Tensor, t: Tensor, level: float):
    under, above = dens - level < 0, dens - level > 0
    first = above.float().argmax(dim=-1, keepdim=True)
    keep = ~(~under[:, 0] | (first[:, 0] == 0))
    f = first[keep]
    d1, d0 = dens[keep].gather(1, f).view(-1), dens[keep].gather(1, f - 1).view(-1)
    t1, t0 = t[keep].gather(1, f).view(-1), t[keep].gather(1, f - 1).view(-1)
    return keep, (level - d0) / (d1 - d0) * (t1 - t0) + t0


@torch.no_grad()
def compute_level_surface_points(model, camera, num_samples: int, mask: Optional[Tensor] = None,
                                 surface_levels: Tuple[float, ...] = (0.1, 0.3, 0.5),
                                 return_normal: str = "closest_gaussian") -> Dict[float, Dict[str, Tensor]]:
    """dn_model.py:1207-1447: level-surface intersections along every pixel ray of `camera`, their normals and colours."""
    from .utils.camera_utils import get_colored_points_from_depth

    c2w = camera.camera_to_worlds.squeeze(0)
    dev = model.device
    flip = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0])).to(device=c2w.device, dtype=c2w.dtype)
    outputs = model.get_outputs(camera)
    depth, rgb = outputs["depth"], outputs["rgb"]
    W, H = int(camera.width.flatten()[0]), int(camera.height.flatten()[0])
    points, colors = get_colored_points_from_depth(depths=depth, rgbs=rgb, fx=float(camera.fx.flatten()[0]),
                                                   fy=float(camera.fy.flatten()[0]), cx=float(camera.cx.flatten()[0]),
                                                   cy=float(camera.cy.flatten()[0]), img_size=(W, H), c2w=(c2w @ flip).to(dev))
    points, colors = points.view(H, W, -1), colors.view(H, W, 3)
    if mask is not None:
        mask = mask.to(points.device)
        points, depth = points * mask, depth * mask
    has_depth = ~(depth <= 0.0)[..., 0]
    points, colors = points[has_depth], colors[has_depth]
    idx = knn_gpu(model.gauss_params["means"].data, points, KNN)
    cam_pos = camera.camera_to_worlds.detach().reshape(3, 4)[:3, 3]
    dens, t, dirs = ray_densities(model, points, idx, cam_pos)
    all_outputs = {}
    for level in surface_levels:
        keep, ts = _level_crossings(dens, t, level)
        xp = points[keep] + ts[:, None] * dirs[keep]
        if return_normal == "analytical":
            d2, man, Minv = _mahalanobis(model, xp, idx[keep])
            w = torch.sigmoid(model.gauss_params["opacities"].detach()[idx[keep]])[..., 0] * torch.exp(-0.5 * d2)
            normals = -torch.nn.functional.normalize((w[..., None] * (Minv @ man)[..., 0]).sum(dim=-2), dim=-1)
        elif return_normal == "closest_gaussian":
            normals = model.normals[idx[keep][:, 0]]
        else:
            raise NotImplementedError
        n = xp.shape[0]
        pick = torch.tensor(random.sample(range(n), num_samples if num_samples < n else n), dtype=torch.long, device=xp.device)
        all_outputs[level] = {"points": xp[pick], "normals": normals[pick], "colors": colors[keep][pick]}
    return all_outputs
