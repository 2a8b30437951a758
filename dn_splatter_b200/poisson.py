"""Screened Poisson surface reconstruction on the device, and the three exporters of the reference that end in
Open3D's `TriangleMesh.create_from_point_cloud_poisson` (/root/reference/dn_splatter/export_mesh.py:128-696):

- `poisson_reconstruct` is that call: a dense-grid screened Poisson solve (csrc/poisson.cu: deterministic splat of the
  oriented samples onto MAC face grids, multigrid V-cycles) followed by marching cubes (mesh.marching_cubes) at the
  iso-value of the samples.  Untrimmed; `trim_low_density` is the reference's 1 % density-quantile clean-up.
- Point-cloud helpers with Open3D's rules [EXT]: `remove_statistical_outlier`, `voxel_down_sample`,
  `filter_smooth_laplacian`, `write_point_cloud_ply` / `read_point_cloud_ply`.
- `export_dn_poisson_mesh` (`gs-mesh dn`), `export_gaussians_poisson_mesh` (`gs-mesh gaussians`),
  `export_level_set_poisson_mesh` (`gs-mesh sugar-coarse`).

Deviations from the reference are listed in DESIGN.md §2 (6).  No CPU path: the kernels need CUDA tensors.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings
from typing import Dict, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from . import _lib as L
from .mesh import TriangleMesh, _quantile_sorted, _views, marching_cubes, write_ply
from .sugar import knn_gpu, sample_points_in_gaussians

DEFAULT_POINT_WEIGHT = 4.0
"""Screening weight alpha: a node on a uniformly sampled surface is screened with about alpha (in units where the
finest-cell Laplacian's diagonal is 6) at every depth, because S is scaled by the surface area per unit sample weight
(`area_scale`).  0 is plain Poisson."""
DEFAULT_MAX_BYTES = 40 << 30
"""Device bytes a reconstruction may allocate (depth 10 with 2 M samples needs about 26 GiB)."""
TOL = 1e-5
MAX_CYCLES = 30
DN_PCD_NAME = "DepthAndNormalMapsPoisson_pcd.ply"
DN_MESH_NAME = "DepthAndNormalMapsPoisson_poisson_mesh.ply"
GAUSSIANS_MESH_NAME = "GaussiansToPoisson_poisson_mesh.ply"
GAUSSIANS_PCD_NAME = "GaussiansToPoisson_pcd.ply"


class PoissonGrid(NamedTuple):
    origin: Tuple[float, float, float]  # corner of cell (0, 0, 0)
    cell: float                         # finest cell edge h
    depth: int                          # R = 2^depth cells per axis

    @property
    def R(self) -> int:
        return 1 << self.depth

    def struct(self) -> "L.DnrPoissonGrid":
        g = L.DnrPoissonGrid()
        g.origin[0], g.origin[1], g.origin[2] = self.origin
        g.cell, g.depth = self.cell, self.depth
        return g


def poisson_grid(points: Tensor, depth: int, scale: float = 1.1) -> PoissonGrid:
    """The cube of side scale * (largest extent of the points' bounding box) centred on the box, 2^depth cells per axis
    (Open3D's default scale is 1.1 [EXT])."""
    if not (L.POISSON_MIN_DEPTH <= depth <= L.POISSON_MAX_DEPTH):
        raise ValueError(f"poisson: depth must be in [{L.POISSON_MIN_DEPTH}, {L.POISSON_MAX_DEPTH}], got {depth}")
    if not scale >= 1.0:
        raise ValueError(f"poisson: scale must be >= 1, got {scale}")
    lo, hi = (t.double().cpu().numpy() for t in torch.aminmax(points.detach(), dim=0))
    side = max(float((hi - lo).max()), 1e-12) * scale
    centre = 0.5 * (lo + hi)
    return PoissonGrid(tuple(float(c - 0.5 * side) for c in centre), side / (1 << depth), int(depth))


def required_bytes(depth: int, n_points: int, max_cycles: int = MAX_CYCLES) -> int:
    """Peak device bytes of poisson_reconstruct: the splat workspace with its outputs, then the solver's."""
    lib = L.load()
    g = PoissonGrid((0.0, 0.0, 0.0), 1.0, depth).struct()
    N = (1 << depth) ** 3
    outputs = 4 * N * 4 + 4 * (N // 64) * 4 + 4 * n_points  # S, faces, density, colour grid, weights
    splat = L.workspace_bytes(lib.dnr_poisson_splat_workspace_bytes, C.byref(g), max(n_points, 1))
    solve = L.workspace_bytes(lib.dnr_poisson_solve_workspace_bytes, C.byref(g), max_cycles) + 4 * N  # + chi
    return outputs + max(splat, solve)


def _check_budget(depth: int, n: int, max_bytes: int) -> None:
    need = required_bytes(depth, n)
    if need > max_bytes:
        R = 1 << depth
        raise ValueError(f"poisson: depth {depth} ({R}^3 = {R ** 3} nodes) with {n} samples needs {need / 2**30:.2f} GiB, "
                         f"over max_bytes = {max_bytes / 2**30:.2f} GiB; use a smaller depth")


def _prep(t: Optional[Tensor], n: int, what: str) -> Optional[Tensor]:
    if t is None:
        return None
    L.need_cuda(t)
    t = t.detach().float().reshape(-1, 3).contiguous()
    if t.shape[0] != n:
        raise ValueError(f"poisson: {what} has {t.shape[0]} rows, points has {n}")
    return t


def poisson_splat(points: Tensor, normals: Tensor, colors: Optional[Tensor], grid: PoissonGrid) -> Dict[str, Tensor]:
    """dnr_poisson_splat: {"screen" [R^3], "faces" [3,R^3], "density" [(R/4)^3], "colors" [(R/4)^3,4] ({sum a w c, sum a w}) or None,
    "weights" [n] (a_p, mean 1), "area_scale" [1]} on the device."""
    L.need_cuda(points)
    p = points.detach().float().reshape(-1, 3).contiguous()
    n = p.shape[0]
    if n == 0:
        raise ValueError("poisson: no samples")
    nrm, col = _prep(normals, n, "normals"), _prep(colors, n, "colors")
    lib, dev, R = L.load(), p.device, grid.R
    g = grid.struct()
    ws, nbytes = L.workspace(lib.dnr_poisson_splat_workspace_bytes, C.byref(g), n, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    out = {"screen": torch.empty(R ** 3, **f32), "faces": torch.empty(3, R ** 3, **f32),
           "density": torch.empty((R // 4) ** 3, **f32), "colors": None if col is None else torch.empty((R // 4) ** 3, 4, **f32),
           "weights": torch.empty(n, **f32), "area_scale": torch.empty(1, **f32)}
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    L.check(lib.dnr_poisson_splat(C.byref(g), p.data_ptr(), nrm.data_ptr(), ptr(col), n, ws.data_ptr(), nbytes,
                                  out["screen"].data_ptr(), out["faces"].data_ptr(), out["density"].data_ptr(), ptr(out["colors"]),
                                  out["weights"].data_ptr(), out["area_scale"].data_ptr(), L.stream()), "dnr_poisson_splat")
    return out


def poisson_solve(grid: PoissonGrid, screen: Tensor, faces: Tensor, screen_weight: float, tol: float = TOL,
                  max_cycles: int = MAX_CYCLES) -> Tuple[Tensor, list]:
    """dnr_poisson_solve: chi [R^3] and the relative residual before the first and after each V-cycle."""
    lib, dev = L.load(), screen.device
    g = grid.struct()
    ws, nbytes = L.workspace(lib.dnr_poisson_solve_workspace_bytes, C.byref(g), int(max_cycles), device=dev)
    chi = torch.empty(grid.R ** 3, dtype=torch.float32, device=dev)
    hist = (C.c_float * (max_cycles + 1))()
    cycles = C.c_int32(0)
    L.check(lib.dnr_poisson_solve(C.byref(g), screen.data_ptr(), faces.data_ptr(), float(screen_weight), float(tol), int(max_cycles),
                                  ws.data_ptr(), nbytes, chi.data_ptr(), hist, C.byref(cycles), L.stream()), "dnr_poisson_solve")
    return chi, [float(hist[i]) for i in range(cycles.value + 1)]


def grid_sample(values: Tensor, origin: Sequence[float], cell: float, points: Tensor) -> Tensor:
    """dnr_grid_sample: trilinear interpolation of a cell-centred grid values [X,Y,Z] or [X,Y,Z,C] (node (i,j,k) at
    origin + (index + 0.5) * cell) at points [n,3], clamped to the outer node centres.  Returns [n] or [n,C]."""
    L.need_cuda(values, points)
    v = values.detach().float().contiguous()
    ch = 1 if v.dim() == 3 else v.shape[3]
    d = L.DnrGridDesc()
    d.origin[0], d.origin[1], d.origin[2] = [float(o) for o in origin]
    d.cell, d.channels = float(cell), ch
    d.dims[0], d.dims[1], d.dims[2] = v.shape[:3]
    p = points.detach().float().reshape(-1, 3).contiguous()
    out = torch.empty((p.shape[0], ch), dtype=torch.float32, device=p.device)
    L.check(L.load().dnr_grid_sample(C.byref(d), v.data_ptr(), p.data_ptr(), p.shape[0], out.data_ptr(), L.stream()), "dnr_grid_sample")
    return out[:, 0] if v.dim() == 3 else out


class PoissonResult(NamedTuple):
    mesh: TriangleMesh
    densities: Tensor
    grid: PoissonGrid
    chi: Tensor            # [R,R,R]
    iso: float
    residuals: list        # relative residual before the first and after each cycle
    screen_weight: float   # point_weight * area_scale


@torch.no_grad()
def poisson_solve_points(points: Tensor, normals: Tensor, colors: Optional[Tensor] = None, *, depth: int = 9,
                         scale: float = 1.1, point_weight: float = DEFAULT_POINT_WEIGHT, max_bytes: int = DEFAULT_MAX_BYTES,
                         tol: float = TOL, max_cycles: int = MAX_CYCLES) -> PoissonResult:
    """poisson_reconstruct with the solver's state (grid, chi, iso-value, residual history) kept."""
    if not point_weight >= 0:
        raise ValueError(f"poisson: point_weight must be >= 0, got {point_weight}")
    n = int(points.reshape(-1, 3).shape[0])
    grid = poisson_grid(points.reshape(-1, 3), depth, scale)
    _check_budget(depth, n, max_bytes)
    sp = poisson_splat(points, normals, colors, grid)
    sigma = float(point_weight) * float(sp["area_scale"])
    chi, hist = poisson_solve(grid, sp["screen"], sp["faces"], sigma, tol, max_cycles)
    if hist[-1] > tol:
        warnings.warn(f"poisson: the solve stopped after {max_cycles} V-cycles at a relative residual of {hist[-1]:.2e}, "
                      f"above tol = {tol:.0e}; the mesh comes from an unconverged chi", RuntimeWarning, stacklevel=2)
    del sp["screen"], sp["faces"]
    R, h = grid.R, grid.cell
    chi = chi.view(R, R, R)
    p = points.detach().float().reshape(-1, 3)
    iso = float((grid_sample(chi, grid.origin, h, p).double() * sp["weights"].double()).sum() / n)
    mesh = marching_cubes(chi, iso, [o + 0.5 * h for o in grid.origin], h)
    R4 = R // 4
    dens = grid_sample(sp["density"].view(R4, R4, R4), grid.origin, 4 * h, mesh.vertices)
    cols = None
    if sp["colors"] is not None:
        cw = grid_sample(sp["colors"].view(R4, R4, R4, 4), grid.origin, 4 * h, mesh.vertices)
        cols = cw[:, :3] / cw[:, 3:].clamp_min(1e-30)
    return PoissonResult(TriangleMesh(mesh.vertices, mesh.faces, cols), dens, grid, chi, iso, hist, sigma)


def poisson_reconstruct(points: Tensor, normals: Tensor, colors: Optional[Tensor] = None, *, depth: int = 9,
                        scale: float = 1.1, point_weight: float = DEFAULT_POINT_WEIGHT,
                        max_bytes: int = DEFAULT_MAX_BYTES) -> Tuple[TriangleMesh, Tensor]:
    """The `create_from_point_cloud_poisson(pcd, depth)` equivalent on the device: oriented samples points / normals
    [n,3] (colors [n,3] in [0,1] or None) -> (mesh, per-vertex density), untrimmed.  Faces wind counter-clockwise seen
    from the side the normals point to; vertex colours are the sample-weighted mean colour at R/4: the interpolated
    weighted sums divided by the interpolated weight.  Raises ValueError when the grids would need more than max_bytes of device memory."""
    r = poisson_solve_points(points, normals, colors, depth=depth, scale=scale, point_weight=point_weight, max_bytes=max_bytes)
    return r.mesh, r.densities


def trim_low_density(mesh: TriangleMesh, densities: Tensor, quantile: float = 0.01) -> TriangleMesh:
    """The reference's `mesh.remove_vertices_by_mask(densities < np.quantile(densities, 0.01))`: drops those vertices
    and every face that uses one of them."""
    if densities.numel() == 0:
        return mesh
    thr = _quantile_sorted(densities.detach().double().sort().values, quantile)
    keep = densities.double() >= thr
    remap = torch.cumsum(keep.long(), 0) - 1
    f = mesh.faces.long()
    fk = keep[f].all(dim=1)
    return TriangleMesh(mesh.vertices[keep], remap[f[fk]].to(torch.int32), None if mesh.colors is None else mesh.colors[keep])


# ---------------------------------------------------------------------------------------------- point-cloud helpers
def remove_statistical_outlier(points: Tensor, nb_neighbors: int = 20, std_ratio: float = 2.0) -> Tensor:
    """Open3D's PointCloud.remove_statistical_outlier [EXT]: the mean distance of each point to its nb_neighbors nearest
    points, the point itself included (distance 0), kept where <= mean + std_ratio * std (sample std) over the cloud.
    Returns the kept indices (ascending)."""
    L.need_cuda(points)
    p = points.detach().float().reshape(-1, 3).contiguous()
    n = p.shape[0]
    if n <= nb_neighbors:
        return torch.arange(n, device=p.device)
    # knn_gpu searches k + 1 and drops the nearest (the point itself): k = nb_neighbors - 1 gives the other neighbours
    idx = knn_gpu(p, p, nb_neighbors - 1)
    dist = (p[idx.clamp_min(0)] - p[:, None]).norm(dim=-1).double()
    avg = dist.sum(dim=1) / nb_neighbors
    mean, std = avg.mean(), avg.std(unbiased=True)
    return torch.nonzero(avg <= mean + std_ratio * std).reshape(-1)


def voxel_down_sample(points: Tensor, normals: Optional[Tensor], colors: Optional[Tensor], voxel: float):
    """Open3D's PointCloud.voxel_down_sample [EXT]: one point per occupied voxel with the mean position, normal and colour
    of its points.  Voxel index floor((p - (min - voxel / 2)) / voxel): Open3D's grid starts half a voxel below the
    bounding box.  Voxels come out in lexicographic (x, y, z) index order (Open3D's order is its hash map's)."""
    p = points.detach().float().reshape(-1, 3)
    if not voxel > 0:
        raise ValueError("voxel_down_sample: voxel must be positive")
    key = torch.floor((p.double() - (p.double().min(dim=0).values - 0.5 * voxel)) / voxel).long()
    _, inv = torch.unique(key, dim=0, return_inverse=True)
    m = int(inv.max()) + 1 if inv.numel() else 0
    cnt = torch.zeros(m, dtype=torch.float64, device=p.device).index_add_(0, inv, torch.ones_like(inv, dtype=torch.float64))

    def mean(x):
        if x is None:
            return None
        s = torch.zeros((m, 3), dtype=torch.float64, device=p.device).index_add_(0, inv, x.detach().double().reshape(-1, 3))
        return (s / cnt[:, None]).float()

    return mean(p), mean(normals), mean(colors)


def filter_smooth_laplacian(mesh: TriangleMesh, iterations: int = 1, lam: float = 0.5) -> TriangleMesh:
    """Open3D's TriangleMesh.filter_smooth_laplacian with its default scope (all attributes) [EXT]:
    x <- x + lam * (sum_j w_ij x_j / sum_j w_ij - x) over the edge neighbours j, for the positions and, with the same
    weights, the colours; w_ij = 1 / |v_i - v_j| (Open3D's inverse-distance weights), all vertices updated at once."""
    v = mesh.vertices.detach().double()
    col = None if mesh.colors is None else mesh.colors.detach().double()
    f = mesh.faces.long()
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    e = torch.unique(torch.sort(torch.cat([e, e.flip(1)]), dim=1).values, dim=0)
    src, dst = torch.cat([e[:, 0], e[:, 1]]), torch.cat([e[:, 1], e[:, 0]])
    for _ in range(iterations):
        w = 1.0 / (v[src] - v[dst]).norm(dim=1).clamp_min(1e-12)
        den = torch.zeros(v.shape[0], dtype=v.dtype, device=v.device).index_add_(0, src, w)
        has = (den > 0)[:, None]

        def step(x):
            avg = torch.zeros_like(x).index_add_(0, src, w[:, None] * x[dst]) / den.clamp_min(1e-300)[:, None]
            return x + lam * (torch.where(has, avg, x) - x)

        v, col = step(v), None if col is None else step(col)
    return TriangleMesh(v.float(), mesh.faces, None if col is None else col.float())


_PCD_VERTEX = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                        ("red", "u1"), ("green", "u1"), ("blue", "u1")])


def write_point_cloud_ply(path: str, points: Tensor, normals: Tensor, colors: Optional[Tensor]) -> None:
    """Binary PLY of x, y, z, nx, ny, nz (float) and red, green, blue (uchar, round(clamp(c, 0, 1) * 255); grey 128
    without colours)."""
    p = points.detach().cpu().float().numpy().reshape(-1, 3)
    v = np.empty(p.shape[0], _PCD_VERTEX)
    nrm = normals.detach().cpu().float().numpy().reshape(-1, 3)
    for a, name in enumerate("xyz"):
        v[name], v["n" + name] = p[:, a], nrm[:, a]
    rgb = (np.full(p.shape, 128, np.uint8) if colors is None
           else np.round(np.clip(colors.detach().cpu().float().numpy().reshape(-1, 3), 0.0, 1.0) * 255.0).astype(np.uint8))
    v["red"], v["green"], v["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    head = ("ply\nformat binary_little_endian 1.0\n"
            f"element vertex {p.shape[0]}\n"
            "property float x\nproperty float y\nproperty float z\n"
            "property float nx\nproperty float ny\nproperty float nz\n"
            "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(head.encode("ascii"))
        fh.write(v.tobytes())


def read_point_cloud_ply(path: str) -> Tuple[Tensor, Tensor, Tensor]:
    """Reads what write_point_cloud_ply writes: (points, normals, colours as uint8 / 255), host tensors."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    n = int(next(h for h in head if h.startswith("element vertex")).split()[-1])
    v = np.frombuffer(data, _PCD_VERTEX, n, end)
    pts = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
    nrm = np.stack([v["nx"], v["ny"], v["nz"]], axis=1).astype(np.float32)
    col = np.stack([v["red"], v["green"], v["blue"]], axis=1).astype(np.float32) / 255.0
    return torch.from_numpy(pts), torch.from_numpy(nrm), torch.from_numpy(col)


# ---------------------------------------------------------------------------------------------- host logic of the exporters
def samples_per_frame(total_points: int, num_frames: int) -> int:
    """export_mesh.py:355 (and :549)."""
    return (total_points + num_frames) // num_frames


def find_depth_edges(depth_im: Tensor, threshold: float = 0.01, dilation_itr: int = 3) -> Tensor:
    """export_mesh.py:58-90: pixels near a jump of inverse depth (Laplacian > threshold), dilated dilation_itr times
    with a 3x3 box; depth_im [H,W,1] -> [H,W,1] of 0.0 / 1.0."""
    lap_k = torch.tensor([[0, 1, 0], [1, -4, 1], [0, 1, 0]], dtype=depth_im.dtype, device=depth_im.device)[None, None]
    lap = F.conv2d((1.0 / (depth_im + 1e-6)).unsqueeze(0).unsqueeze(0).squeeze(-1), lap_k, padding=1)
    edges = (lap.squeeze(0).squeeze(0).unsqueeze(-1) > threshold) * 1.0
    box = lap_k * 0.0 + 1.0
    for _ in range(dilation_itr):
        edges = F.conv2d(edges.unsqueeze(0).unsqueeze(0).squeeze(-1), box, padding=1).squeeze(0).squeeze(0).unsqueeze(-1)
    return (edges > 0.0) * 1.0


def flipped_c2w(camera) -> Tensor:
    """[3,4] camera-to-world with the y and z axes flipped (OpenGL -> OpenCV), export_mesh.py:370-375."""
    c2w = torch.eye(4, dtype=torch.float32, device=camera.camera_to_worlds.device)
    c2w[:3, :4] = camera.camera_to_worlds.reshape(3, 4)
    return (c2w @ torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0], device=c2w.device)))[:3, :4]


def surface_normals_to_world(surface_normal: Tensor, c2w: Tensor) -> Tensor:
    """export_mesh.py:408-428 up to the index: the [H,W,3] surface-normal map in [0,1] -> world normals [H*W,3] with
    the flipped c2w [3,4]."""
    h, w, _ = surface_normal.shape
    nm = 2 * surface_normal.reshape(-1, 3) - 1
    nm = nm @ torch.diag(torch.tensor([1.0, -1.0, -1.0], device=nm.device, dtype=torch.float))
    nm = nm.view(h, w, 3).permute(2, 0, 1).reshape(3, -1)
    nm = c2w[:3, :3] @ F.normalize(nm, p=2, dim=0)
    return nm.permute(1, 0).reshape(h, w, 3).view(-1, 3)


def _pick(valid: Tensor, k: int, gen: torch.Generator) -> Tensor:
    """pick_indices_at_random (export_mesh.py:50-55) with a seeded generator."""
    idx = torch.nonzero(valid.reshape(-1)).reshape(-1)
    if k < idx.shape[0]:
        idx = idx[torch.randperm(idx.shape[0], generator=gen, device=gen.device)[:k]]
    return idx


def _finish(path: str, name: str, points: Tensor, normals: Tensor, colors: Optional[Tensor], depth: int) -> TriangleMesh:
    mesh, dens = poisson_reconstruct(points, normals, colors, depth=depth)
    mesh = trim_low_density(mesh, dens)
    write_ply(os.path.join(path, name), mesh)
    return mesh


def _clean(points, normals, colors, down_sample_voxel, outlier_removal, std_ratio):
    if down_sample_voxel is not None:
        points, normals, colors = voxel_down_sample(points, normals, colors, down_sample_voxel)
    if outlier_removal:
        keep = remove_statistical_outlier(points, 20, std_ratio)
        points, normals, colors = points[keep], normals[keep], None if colors is None else colors[keep]
    return points, normals, colors


@torch.no_grad()
def export_dn_poisson_mesh(model, cameras, path: str, *, total_points: int = 2_000_000,
                           masks: Optional[Sequence[Tensor]] = None, filter_edges_from_depth_maps: bool = False,
                           edge_threshold: float = 0.004, edge_dilation_iterations: int = 10,
                           down_sample_voxel: Optional[float] = None, outlier_removal: bool = False, std_ratio: float = 2.0,
                           poisson_depth: int = 9, normal_method: str = "normal_maps", seed: int = 0):
    """The `dn` exporter (DepthAndNormalMapsPoisson, export_mesh.py:313-510): render rgb, depth and surface normals of
    every view, draw samples_per_frame pixels with depth != 0 (and, with filter_edges_from_depth_maps, away from depth
    edges; upstream the edge filter alone decides, so it can draw depth-0 pixels) per view, back-project them with their world normals and colours, optionally down-sample and remove
    outliers, write `path/DepthAndNormalMapsPoisson_pcd.ply`, reconstruct, drop the vertices below the 1 % density
    quantile and write `path/DepthAndNormalMapsPoisson_poisson_mesh.ply`.  masks[i] ([H,W] bool, device) limits view i's
    samples to the mask (the reference zeroes masked depth after sampling, which back-projects onto the camera centre).
    Samples on the 1-pixel image border carry a zero normal, as upstream: the depth-derived normal map is undefined
    there; they add no flux.
    normal_method="density_grad" is broken upstream and raises NotImplementedError.  Returns (mesh, (points, normals,
    colors))."""
    if normal_method != "normal_maps":
        raise NotImplementedError("normal_method='density_grad' is broken in the reference (export_mesh.py:442 rebinds "
                                  "the normals list, :472 then fails); only 'normal_maps' is supported")
    points, normals, colors = dn_point_cloud(model, cameras, total_points=total_points, masks=masks,
                                             filter_edges_from_depth_maps=filter_edges_from_depth_maps,
                                             edge_threshold=edge_threshold, edge_dilation_iterations=edge_dilation_iterations,
                                             seed=seed)
    points, normals, colors = _clean(points, normals, colors, down_sample_voxel, outlier_removal, std_ratio)
    os.makedirs(path, exist_ok=True)
    write_point_cloud_ply(os.path.join(path, DN_PCD_NAME), points, normals, colors)
    return _finish(path, DN_MESH_NAME, points, normals, colors, poisson_depth), (points, normals, colors)


@torch.no_grad()
def dn_point_cloud(model, cameras, *, total_points: int = 2_000_000, masks: Optional[Sequence[Tensor]] = None,
                   filter_edges_from_depth_maps: bool = False, edge_threshold: float = 0.004,
                   edge_dilation_iterations: int = 10, seed: int = 0) -> Tuple[Tensor, Tensor, Tensor]:
    """The oriented, coloured point cloud of export_dn_poisson_mesh (its arguments) before down-sampling and outlier
    removal: (points, world normals, colours) on the device."""
    from .render_service import ViewRenderer
    from .utils.camera_utils import get_colored_points_from_depth

    views = _views(cameras)
    spf = samples_per_frame(total_points, len(views))
    gen = torch.Generator(device=model.device).manual_seed(seed)
    pts, nrms, cols = [], [], []
    for idx, maps in ViewRenderer(model, keys=("rgb", "depth", "surface_normal"), to_host=False).render(views):
        cam = views[idx]
        depth = maps["depth"]
        valid = depth != 0
        if filter_edges_from_depth_maps:
            valid = valid & (find_depth_edges(depth, edge_threshold, edge_dilation_iterations) < 0.2)
        if masks is not None:
            valid = valid & masks[idx].reshape(valid.shape).to(valid.device, torch.bool)
        pick = _pick(valid, spf, gen)
        if pick.numel() == 0:
            continue
        c2w = flipped_c2w(cam).to(depth.device)
        H, W = depth.shape[0], depth.shape[1]
        xyz, rgb = get_colored_points_from_depth(depths=depth, rgbs=maps["rgb"], c2w=c2w, fx=float(cam.fx.flatten()[0]),
                                                 fy=float(cam.fy.flatten()[0]), cx=float(cam.cx.flatten()[0]),
                                                 cy=float(cam.cy.flatten()[0]), img_size=(W, H), mask=pick)
        pts.append(xyz)
        cols.append(rgb)
        nrms.append(surface_normals_to_world(maps["surface_normal"], c2w)[pick])
    if not pts:
        raise ValueError("export_dn_poisson_mesh: no view has a pixel with depth")
    return torch.cat(pts), torch.cat(nrms), torch.cat(cols)


def _mask_filter(positions: Tensor, cameras, masks) -> Tensor:
    """export_mesh.py:172-225: a Gaussian whose mean projects strictly inside a view (pixel floor(uv - 0.5), both > 0)
    onto a pixel outside that view's mask is removed.  Returns the keep mask."""
    from .utils.camera_utils import project_pix

    keep = torch.ones(positions.shape[0], dtype=torch.bool, device=positions.device)
    for cam, mask in zip(_views(cameras), masks):
        c2w = flipped_c2w(cam).to(positions.device)
        H, W = int(cam.height.flatten()[0]), int(cam.width.flatten()[0])
        uvz = project_pix(positions, float(cam.fx.flatten()[0]), float(cam.fy.flatten()[0]), float(cam.cx.flatten()[0]),
                          float(cam.cy.flatten()[0]), c2w, positions.device, return_z_depths=True)
        uv = torch.floor(uvz[:, :2] - 0.5).long()
        inside = (uv[:, 0] > 0) & (uv[:, 0] < W) & (uv[:, 1] > 0) & (uv[:, 1] < H)
        m = mask.reshape(H, W).to(positions.device, torch.bool)
        hit = torch.zeros_like(keep)
        hit[inside] = ~m[uv[inside, 1], uv[inside, 0]]
        keep &= ~hit
    return keep


@torch.no_grad()
def export_gaussians_poisson_mesh(model, path: str, *, cameras=None, masks: Optional[Sequence[Tensor]] = None,
                                  min_opacity: Optional[float] = None, mask_color: Optional[Sequence[float]] = None,
                                  densify_gaussians: Optional[int] = None, down_sample_voxel: Optional[float] = None,
                                  outlier_removal: bool = False, std_ratio: float = 2.0, poisson_depth: int = 9):
    """The `gaussians` exporter (GaussiansToPoisson, export_mesh.py:128-310): Gaussian means with `model.normals` as the
    last render left them and clamped colours; masks (with cameras) remove Gaussians that project outside a mask
    (:172-225); min_opacity compares the raw opacity parameter as the reference does; mask_color keeps the Gaussians
    whose colour differs from it in every channel (:239-252); densify_gaussians adds points drawn inside the Gaussians.  Writes `GaussiansToPoisson_poisson_mesh.ply` and `GaussiansToPoisson_pcd.ply`.
    Returns (mesh, (points, normals, colors))."""
    positions = model.means.detach().float()
    normals = model.normals.detach().float()
    opacities = model.opacities.detach()
    colors = torch.clamp(model.colors.detach().clone(), 0.0, 1.0).float()
    if masks is not None:
        keep = _mask_filter(positions, cameras, masks)
        positions, normals, opacities, colors = positions[keep], normals[keep], opacities[keep], colors[keep]
    if min_opacity is not None:
        keep = (opacities > min_opacity)[..., 0]
        positions, normals, colors = positions[keep], normals[keep], colors[keep]
    if mask_color is not None:
        keep = torch.all(colors != torch.tensor([mask_color], dtype=colors.dtype, device=colors.device), dim=-1)
        positions, normals, colors = positions[keep], normals[keep], colors[keep]
    if densify_gaussians is not None:
        extra, gs = sample_points_in_gaussians(model, num_samples=densify_gaussians)
        positions = torch.cat([positions, extra.float()])
        normals = torch.cat([normals, model.normals.detach().float()[gs]])
        colors = torch.cat([colors, torch.clamp(model.colors.detach()[gs], 0.0, 1.0).float()])
    points, normals, colors = _clean(positions, normals, colors, down_sample_voxel, outlier_removal, std_ratio)
    os.makedirs(path, exist_ok=True)
    mesh = _finish(path, GAUSSIANS_MESH_NAME, points, normals, colors, poisson_depth)
    write_point_cloud_ply(os.path.join(path, GAUSSIANS_PCD_NAME), points, normals, colors)
    return mesh, (points, normals, colors)


@torch.no_grad()
def export_level_set_poisson_mesh(model, cameras, path: str, *, total_points: int = 2_000_000,
                                  masks: Optional[Sequence[Tensor]] = None, surface_levels: Sequence[float] = (0.1, 0.3, 0.5),
                                  return_normal: str = "closest_gaussian", poisson_depth: int = 9) -> Dict[float, TriangleMesh]:
    """The `sugar-coarse` exporter (LevelSetExtractor, export_mesh.py:513-696): level-surface points of every view
    (sugar.compute_level_surface_points), per level: `before_clean_points_…`, outlier removal with std_ratio = 20,
    `after_clean_points_…`, Poisson + density trim `poisson_mesh_surface_level_…`, and two Laplacian smoothings
    `smoothed_1_…` / `smoothed_2_…`.  Returns the trimmed mesh per level."""
    from .sugar import compute_level_surface_points

    views = _views(cameras)
    spf = samples_per_frame(total_points, len(views))
    acc = {lv: {"points": [], "colors": [], "normals": []} for lv in surface_levels}
    for i, cam in enumerate(views):
        out = compute_level_surface_points(model, cam, spf, mask=None if masks is None else masks[i],
                                           surface_levels=tuple(surface_levels), return_normal=return_normal)
        for lv in surface_levels:
            for k in acc[lv]:
                acc[lv][k].append(out[lv][k])
    os.makedirs(path, exist_ok=True)
    meshes = {}
    for lv in surface_levels:
        p, c, n = (torch.cat(acc[lv][k]).float() for k in ("points", "colors", "normals"))
        tag = f"surface_level_{lv}_{return_normal}.ply"
        write_point_cloud_ply(os.path.join(path, f"before_clean_points_{tag}"), p, n, c)
        keep = remove_statistical_outlier(p, 20, 20.0)
        p, n, c = p[keep], n[keep], c[keep]
        write_point_cloud_ply(os.path.join(path, f"after_clean_points_{tag}"), p, n, c)
        mesh = meshes[lv] = _finish(path, f"poisson_mesh_{tag}", p, n, c, poisson_depth)
        mesh = filter_smooth_laplacian(mesh)
        write_ply(os.path.join(path, f"smoothed_1_poisson_mesh_{tag}"), mesh)
        write_ply(os.path.join(path, f"smoothed_2_poisson_mesh_{tag}"), filter_smooth_laplacian(mesh))
    return meshes
