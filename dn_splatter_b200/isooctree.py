"""AGS-Mesh's mesh extractor, the reference's dn_splatter/scripts/isooctree_dn.py, on the device.

The script fuses the rendered depth and normal maps of every frame into a normal-aware projective TSDF (`isoFunc`),
evaluated on the corners of an octree that the frames' back-projected pixels (the hint cloud) refine, and meshes it
with the third-party IsoOctree module.  Here:

- `FrameSet` keeps the F frames' depth and normal files resident on the device;
- `hint_samples` is Frame.get_samples of every frame (`dnr_iso_samples`);
- `build_octree` is this project's octree rule (DESIGN.md §2): the root cube is centred on the hint cloud's bounding box
  with side 1.05 x its longest extent, and a node splits iff it holds >= subdivision_threshold hint samples and its
  level is below max_depth (`dnr_iso_octree`, `dnr_iso_corners`);
- `iso_eval` is isoFunc in all its modes, in fp64 (`dnr_iso_eval`); every shared leaf corner is evaluated once;
- `fill_grid` spreads the corner values over the dense (2^max_depth + 1)^3 grid, each sample taking the trilinear value
  of the smallest leaf holding it (`dnr_iso_fill`), and `mesh.marching_cubes` meshes it at 0: one value per sample, so
  the mesh has no cracks, and coarse leaves give smooth, coarse patches.

Entry points with the script's names and defaults: `load_frame_metadata`, `build_mesh_projection`,
`isooctree_mesh_files` (and `python -m dn_splatter_b200.isooctree`), plus `export_isooctree_mesh`, which renders a model
straight into the frame buffers.  The fp64 restatement is oracle/isooctree_ref.py.  No CPU path: the kernels need CUDA.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch
from torch import Tensor

from . import _lib as L
from .mesh import TriangleMesh, marching_cubes, write_obj, write_ply

CAM_CONVENTION_CHANGE = np.diag([1.0, -1.0, -1.0, 1.0])
DEPTH_SCALE = 1 / 1000.0  # the depth files hold millimetres
MAX_VALID_DEPTH_REL_DELTA = 0.005
ROOT_SCALE = 1.05
DEFAULT_MAX_BYTES = 40 << 30


class CameraModel:
    """The one pinhole camera of a transforms file: resolution (w, h) and K (fl_x, fl_y, cx, cy)."""

    def __init__(self, data):
        self.resolution = int(data["w"]), int(data["h"])
        self.camera_matrix = np.array([[data["fl_x"], 0, data["cx"]], [0, data["fl_y"], data["cy"]], [0, 0, 1]], np.float64)
        self.inverse_camera_matrix = np.linalg.inv(self.camera_matrix)


class Frame:
    """One frame of a render folder: its pose and where its depth and normal files are.  With color_normal_data (set by
    camera_coordinate_normals) they are depth/raw/frame_<id>.npy and normal/frame_<id>.png, as render_model.py writes
    them; otherwise depth/frame_<id>.npy and normal/frame_<id>.npy (world-frame normals)."""

    def __init__(self, camera: CameraModel, data, root_folder: str):
        self.camera = camera
        c2w = np.array(data["transform_matrix"], np.float64)
        if c2w.shape[0] == 3:
            c2w = np.vstack([c2w, [0, 0, 0, 1]])
        self.pose_c2w = c2w @ CAM_CONVENTION_CHANGE
        self.pose_w2c = np.linalg.inv(self.pose_c2w)
        self.root_folder = root_folder
        self.image_id = data["file_path"].split("/")[-1].split("_")[1].split(".")[0]
        self.cam_coordinate_normals = False
        self.color_normal_data = False

    def image_path(self, kind: str) -> str:
        if self.color_normal_data:
            if kind == "normal":
                return os.path.join(self.root_folder, kind, f"frame_{self.image_id}.png")
            return os.path.join(self.root_folder, kind, "raw", f"frame_{self.image_id}.npy")
        return os.path.join(self.root_folder, kind, f"frame_{self.image_id}.npy")

    def image_data_exists(self) -> bool:
        return os.path.exists(self.image_path("depth")) and os.path.exists(self.image_path("normal"))


def pose_row(pose_c2w: np.ndarray, pose_w2c: np.ndarray) -> np.ndarray:
    """The DNR_ISO_POSE doubles of one frame: world->camera [3,4], c2w rotation, position, normal rotation, 3 of padding."""
    nrot = pose_c2w[:3, :3] @ CAM_CONVENTION_CHANGE[:3, :3]
    return np.concatenate([pose_w2c[:3].reshape(-1), pose_c2w[:3, :3].reshape(-1), pose_c2w[:3, 3], nrot.reshape(-1), np.zeros(3)])


def load_frame_metadata(root_dir: str, json_file_path: str, max_frames: Optional[int] = None, frame_stride: int = 1,
                        camera_coordinate_normals: bool = False) -> List[Frame]:
    """The frames of json_file_path (every frame_stride-th, at most max_frames) whose depth and normal files exist."""
    with open(json_file_path) as fh:
        data = json.load(fh)
    camera = CameraModel(data)
    frames = []
    for i, jf in enumerate(data["frames"]):
        if i % frame_stride != 0:
            continue
        f = Frame(camera, jf, root_dir)
        f.cam_coordinate_normals = camera_coordinate_normals
        f.color_normal_data = camera_coordinate_normals
        if not f.image_data_exists():
            continue
        frames.append(f)
        if max_frames is not None and len(frames) >= max_frames:
            break
    return frames


class FrameSet:
    """The depth [F,h,w] and normal [F,h,w,3] file values of F frames of one camera, resident on the device (f32: the
    PNG values 0..255 when cam_normals, world-frame normals otherwise), and their poses."""

    def __init__(self, camera: CameraModel, n_frames: int, cam_normals: bool, device="cuda"):
        w, h = camera.resolution
        if n_frames <= 0:
            raise ValueError("isooctree: no frames")
        self.camera, self.cam_normals = camera, bool(cam_normals)
        self.depth = torch.zeros((n_frames, h, w), dtype=torch.float32, device=device)
        self.normals = torch.zeros((n_frames, h, w, 3), dtype=torch.float32, device=device)
        self._poses = np.zeros((n_frames, L.ISO_POSE), np.float64)
        self.poses = None
        L.need_cuda(self.depth)

    @property
    def n_frames(self) -> int:
        return self.depth.shape[0]

    def set_pose(self, i: int, pose_c2w: np.ndarray, pose_w2c: np.ndarray) -> None:
        self._poses[i] = pose_row(pose_c2w, pose_w2c)
        self.poses = None

    @classmethod
    def from_files(cls, frames: Sequence[Frame], device="cuda") -> "FrameSet":
        from PIL import Image

        if not frames:
            raise ValueError("isooctree: no frames with depth and normal files")
        cam = frames[0].camera
        fs = cls(cam, len(frames), frames[0].color_normal_data, device)
        w, h = cam.resolution
        for i, f in enumerate(frames):
            d = np.load(f.image_path("depth"))
            p = f.image_path("normal")
            n = np.array(Image.open(p)) if p.endswith(".png") else np.load(p)
            if d.shape[:2] != (h, w) or n.shape[:2] != (h, w):
                raise ValueError(f"isooctree: frame {f.image_id} is {d.shape[:2]} / {n.shape[:2]}, the camera is {(h, w)}")
            fs.depth[i] = torch.from_numpy(np.ascontiguousarray(d[..., 0], np.float32))
            fs.normals[i] = torch.from_numpy(np.ascontiguousarray(n[..., :3], np.float32))
            fs.set_pose(i, f.pose_c2w, f.pose_w2c)
        return fs

    def struct(self) -> L.DnrIsoFrames:
        if self.poses is None:
            self.poses = torch.from_numpy(self._poses).to(self.depth.device)
        s = L.DnrIsoFrames()
        s.depth, s.normals, s.poses = self.depth.data_ptr(), self.normals.data_ptr(), self.poses.data_ptr()
        s.n_frames = self.n_frames
        s.width, s.height = self.camera.resolution
        s.cam_normals = int(self.cam_normals)
        s.K[:] = self.camera.camera_matrix.reshape(-1).tolist()
        s.inv_K[:] = self.camera.inverse_camera_matrix.reshape(-1).tolist()
        s.depth_scale, s.rel_delta = DEPTH_SCALE, MAX_VALID_DEPTH_REL_DELTA
        return s


def hint_samples(fs: FrameSet, pixel_stride: int, with_normals: bool = False):
    """(points [n,3] f64, normals [n,3] f64 or None): Frame.get_samples(stride=pixel_stride) of every frame, stacked in
    frame order.  One host read."""
    lib = L.load()
    s = fs.struct()
    w, h = fs.camera.resolution
    cap = fs.n_frames * (-(-h // pixel_stride)) * (-(-w // pixel_stride))
    dev = fs.depth.device
    ws, nbytes = L.workspace(lib.dnr_iso_samples_workspace_bytes, C.byref(s), int(pixel_stride), device=dev)
    pts = torch.empty((cap, 3), dtype=torch.float64, device=dev)
    nrm = torch.empty((cap, 3), dtype=torch.float64, device=dev) if with_normals else None
    count = C.c_int64()
    L.check(lib.dnr_iso_samples(C.byref(s), int(pixel_stride), ws.data_ptr(), nbytes, pts.data_ptr(),
                                None if nrm is None else nrm.data_ptr(), C.byref(count), L.stream()), "dnr_iso_samples")
    n = count.value
    return pts[:n], (None if nrm is None else nrm[:n])


class Octree(NamedTuple):
    grid: L.DnrIsoGrid
    leaves: Tensor          # [L] int64, level << 58 | Morton code, by level then code
    level_counts: tuple     # leaves per level 0..max_depth
    corner_keys: Tensor     # [N] int64 sorted lattice keys (i * (R+1) + j) * (R+1) + k
    corner_points: Tensor   # [N,3] f64
    leaf_corners: Tensor    # [L,8] int32 indices into the corners

    @property
    def origin(self):
        return list(self.grid.origin)

    @property
    def cell(self) -> float:
        return float(self.grid.cell)


def root_cube(hint: Tensor):
    """(origin [3], side) of the cube centred on the hint cloud's bounding box, side ROOT_SCALE x its longest extent."""
    lo, hi = (t.cpu().numpy() for t in torch.aminmax(hint, dim=0))
    side = max(float((hi - lo).max()), 1e-9) * ROOT_SCALE
    return 0.5 * (lo + hi) - 0.5 * side, side


def iso_grid(origin, side: float, max_depth: int, subdivision_threshold: int) -> L.DnrIsoGrid:
    if not 0 <= max_depth <= L.ISO_MAX_DEPTH:
        raise ValueError(f"isooctree: max_depth must be in [0, {L.ISO_MAX_DEPTH}] (the dense grid of depth 10 is "
                         f"1025^3 f32 = 4.3 GB), got {max_depth}")
    if subdivision_threshold < 1:
        raise ValueError(f"isooctree: subdivision_threshold must be >= 1, got {subdivision_threshold}")
    g = L.DnrIsoGrid()
    g.origin[:] = [float(o) for o in origin]
    g.cell = float(side) / (1 << max_depth)
    g.max_depth, g.threshold = int(max_depth), int(subdivision_threshold)
    return g


def build_octree(hint: Tensor, max_depth: int, subdivision_threshold: int) -> Octree:
    """The octree of the hint cloud [n,3] f64 (device), its leaves and their unique corners.  One host read per level."""
    L.need_cuda(hint)
    if hint.shape[0] == 0:
        raise ValueError("isooctree: the hint cloud is empty (no depth sample survived the validity tests)")
    lib = L.load()
    h = hint.detach().to(torch.float64).contiguous()
    origin, side = root_cube(h)
    g = iso_grid(origin, side, max_depth, subdivision_threshold)
    dev = h.device
    ws, nbytes = L.workspace(lib.dnr_iso_octree_workspace_bytes, C.byref(g), h.shape[0], device=dev)
    counts = (C.c_int64 * (max_depth + 1))()
    L.check(lib.dnr_iso_octree(C.byref(g), h.data_ptr(), h.shape[0], ws.data_ptr(), nbytes, counts, L.stream()), "dnr_iso_octree")
    n_leaves = sum(counts)
    ws2, cbytes = L.workspace(lib.dnr_iso_corners_workspace_bytes, C.byref(g), n_leaves, device=dev)
    leaves = torch.empty(n_leaves, dtype=torch.int64, device=dev)
    keys = torch.empty(8 * n_leaves, dtype=torch.int64, device=dev)
    pts = torch.empty((8 * n_leaves, 3), dtype=torch.float64, device=dev)
    lc = torch.empty((n_leaves, 8), dtype=torch.int32, device=dev)
    n_corners = C.c_int64()
    L.check(lib.dnr_iso_corners(C.byref(g), ws.data_ptr(), counts, ws2.data_ptr(), cbytes, leaves.data_ptr(), keys.data_ptr(),
                                pts.data_ptr(), lc.data_ptr(), C.byref(n_corners), L.stream()), "dnr_iso_corners")
    n = n_corners.value
    return Octree(g, leaves, tuple(int(c) for c in counts), keys[:n], pts[:n], lc)


def iso_eval(fs: FrameSet, points: Tensor, max_tsdf_rel: float = 0.05, max_angle_to_max_weight_normal_deg: float = 60,
             max_tsdf_abs: Optional[float] = None, choose_best_frame: bool = False, two_pass: bool = True,
             use_normals: bool = True) -> Tensor:
    """isoFunc of build_mesh_projection at points [n,3] (device): values [n] f32.  No host read."""
    L.need_cuda(points)
    if not use_normals:
        choose_best_frame, two_pass = False, False
    p = L.DnrIsoParams()
    p.max_tsdf_rel = float(max_tsdf_rel)
    p.max_tsdf_abs = math.inf if max_tsdf_abs is None else float(max_tsdf_abs)
    p.min_dot = float(np.cos(max_angle_to_max_weight_normal_deg / 180 * np.pi))
    p.use_normals = int(use_normals)
    p.passes = 1 if choose_best_frame else (3 if two_pass else 2)
    pts = points.detach().to(torch.float64).contiguous()
    out = torch.empty(pts.shape[0], dtype=torch.float32, device=pts.device)
    L.check(L.load().dnr_iso_eval(C.byref(fs.struct()), C.byref(p), pts.data_ptr(), pts.shape[0], out.data_ptr(), L.stream()),
            "dnr_iso_eval")
    return out


def fill_grid(tree: Octree, corner_values: Tensor) -> Tensor:
    """The dense grid [R+1, R+1, R+1] f32 over the root cube (sample (i, j, k) at origin + (i, j, k) * cell)."""
    R1 = (1 << tree.grid.max_depth) + 1
    v = corner_values.detach().float().contiguous()
    field = torch.empty((R1, R1, R1), dtype=torch.float32, device=v.device)
    counts = (C.c_int64 * len(tree.level_counts))(*tree.level_counts)
    L.check(L.load().dnr_iso_fill(C.byref(tree.grid), tree.leaves.data_ptr(), counts, tree.leaf_corners.data_ptr(), v.data_ptr(),
                                  field.data_ptr(), L.stream()), "dnr_iso_fill")
    return field


def required_bytes(n_frames: int, width: int, height: int, pixel_stride: int, max_depth: int,
                   subdivision_threshold: int) -> int:
    """An upper bound on the device bytes of build_mesh_projection: frames, hint cloud, octree and corner workspaces at
    their worst-case leaf count, corner values and the dense grid with marching cubes' count workspace."""
    lib = L.load()
    cand = n_frames * (-(-height // pixel_stride)) * (-(-width // pixel_stride))
    frames = n_frames * width * height * 16 + n_frames * L.ISO_POSE * 8
    hint = cand * (24 + 9) + 4096
    g = iso_grid((0.0, 0.0, 0.0), 1.0, max_depth, subdivision_threshold)
    octree = L.workspace_bytes(lib.dnr_iso_octree_workspace_bytes, C.byref(g), cand)
    by_count, bound, pw = cand // subdivision_threshold, 1, 1
    for _ in range(1, max_depth):
        pw *= 8
        bound = max(bound, min(pw, by_count))
    n_leaves = max_depth * 8 * bound + 1
    corners = L.workspace_bytes(lib.dnr_iso_corners_workspace_bytes, C.byref(g), n_leaves) + n_leaves * (8 + 8 * (8 + 24 + 4))
    R1 = (1 << max_depth) + 1
    mc = L.DnrMcField()
    mc.values, mc.dims[0], mc.dims[1], mc.dims[2], mc.spacing = 1, R1, R1, R1, 1.0
    field = 4 * R1 ** 3 + L.workspace_bytes(lib.dnr_mc_count_workspace_bytes, C.byref(mc))
    return frames + hint + octree + corners + field


def check_budget(n_frames: int, w: int, h: int, pixel_stride: int, max_depth: int, subdivision_threshold: int,
                 max_bytes: int) -> None:
    """Raises ValueError when required_bytes exceeds max_bytes."""
    need = required_bytes(n_frames, w, h, pixel_stride, max_depth, subdivision_threshold)
    if need > max_bytes:
        raise ValueError(f"isooctree: {n_frames} frames of {w}x{h}, pixel_stride {pixel_stride}, max_depth {max_depth} may "
                         f"need {need / 2**30:.2f} GiB, over max_bytes = {max_bytes / 2**30:.2f} GiB; use a smaller max_depth, "
                         "a larger pixel_stride or fewer frames")


@torch.no_grad()
def build_mesh_projection(frames, subdivision_threshold: int, pixel_stride: int, max_depth: int, max_tsdf_rel: float = 0.05,
                          max_angle_to_max_weight_normal_deg: float = 60, cache: bool = False,
                          max_tsdf_abs: Optional[float] = None, choose_best_frame: bool = False, two_pass: bool = True,
                          debug_ply_file: Optional[str] = None, use_normals: bool = True,
                          max_bytes: int = DEFAULT_MAX_BYTES) -> TriangleMesh:
    """The script's build_mesh_projection: frames (a list of Frame, or a FrameSet) -> the mesh of the isoFunc field at
    0 over this project's octree.  `cache` is accepted for the script's signature: the frames always stay on the
    device.  debug_ply_file receives the hint cloud and its normals."""
    fs = frames if isinstance(frames, FrameSet) else FrameSet.from_files(frames)
    if pixel_stride < 1:
        raise ValueError(f"isooctree: pixel_stride must be >= 1, got {pixel_stride}")
    iso_grid((0.0, 0.0, 0.0), 1.0, max_depth, subdivision_threshold)  # argument checks
    check_budget(fs.n_frames, *fs.camera.resolution, pixel_stride, max_depth, subdivision_threshold, max_bytes)
    hint, hint_normals = hint_samples(fs, pixel_stride, with_normals=debug_ply_file is not None)
    if debug_ply_file is not None:
        from .poisson import write_point_cloud_ply

        write_point_cloud_ply(debug_ply_file, hint.float(), hint_normals.float(), None)
    tree = build_octree(hint, max_depth, subdivision_threshold)
    values = iso_eval(fs, tree.corner_points, max_tsdf_rel, max_angle_to_max_weight_normal_deg, max_tsdf_abs, choose_best_frame,
                      two_pass, use_normals)
    field = fill_grid(tree, values)
    del values
    return marching_cubes(field, 0.0, tree.origin, tree.cell)


def write_mesh(mesh: TriangleMesh, path: str) -> None:
    """A PLY when path ends in .ply, else an OBJ as the script's writeMeshAsObj writes it."""
    if path.lower().endswith(".ply"):
        write_ply(path, mesh)
    else:
        write_obj(path, mesh)


def isooctree_mesh_files(root_folder: str, transformation_path: Optional[str] = None, camera_coordinate_normals: bool = False,
                         max_frames: Optional[int] = None, frame_stride: int = 1, pixel_stride: int = 6, max_depth: int = 10,
                         subdivision_threshold: int = 50, tsdf_rel: float = 0.05, tsdf_abs: Optional[float] = None,
                         disable_normals: bool = False, output_mesh_file: str = "", debug_ply_file: Optional[str] = None,
                         max_bytes: int = DEFAULT_MAX_BYTES) -> TriangleMesh:
    """The script's main(): mesh the render folder root_folder (poses from transformation_path, by default
    root_folder/transformations_colmap.json) and write it to output_mesh_file (default root_folder/mesh.obj)."""
    if transformation_path is None:
        transformation_path = os.path.join(root_folder, "transformations_colmap.json")
    frames = load_frame_metadata(root_folder, transformation_path, max_frames=max_frames, frame_stride=frame_stride,
                                 camera_coordinate_normals=camera_coordinate_normals)
    mesh = build_mesh_projection(frames, subdivision_threshold=subdivision_threshold, pixel_stride=pixel_stride,
                                 max_depth=max_depth, max_tsdf_rel=tsdf_rel, max_tsdf_abs=tsdf_abs,
                                 use_normals=not disable_normals, debug_ply_file=debug_ply_file, max_bytes=max_bytes)
    write_mesh(mesh, output_mesh_file or os.path.join(root_folder, "mesh.obj"))
    return mesh


def _views(cameras) -> list:
    if isinstance(cameras, (list, tuple)):
        return list(cameras)
    return [cameras[i] for i in range(cameras.shape[0])]


def camera_model_of(view) -> CameraModel:
    return CameraModel({"w": int(view.width.flatten()[0]), "h": int(view.height.flatten()[0]),
                        "fl_x": float(view.fx.flatten()[0]), "fl_y": float(view.fy.flatten()[0]),
                        "cx": float(view.cx.flatten()[0]), "cy": float(view.cy.flatten()[0])})


@torch.no_grad()
def render_frames(model, cameras) -> FrameSet:
    """Renders every view into a FrameSet as render_model.py's files would hold it: depth / 0.001 (millimetres, f32) and
    uint8(normal * 255) camera-frame normals (so the set reads as camera_coordinate_normals)."""
    from .render_service import ViewRenderer

    views = _views(cameras)
    if not views:
        raise ValueError("export_isooctree_mesh: no cameras")
    cam = camera_model_of(views[0])
    for v in views[1:]:
        c = camera_model_of(v)
        if c.resolution != cam.resolution or not np.array_equal(c.camera_matrix, cam.camera_matrix):
            raise ValueError("export_isooctree_mesh: all views must share one camera model (resolution and intrinsics)")
    fs = FrameSet(cam, len(views), cam_normals=True, device=model.device)
    w, h = cam.resolution
    for idx, maps in ViewRenderer(model, keys=("depth", "normal"), to_host=False).render(views):
        fs.depth[idx] = maps["depth"].reshape(h, w).float() / 0.001
        fs.normals[idx] = (maps["normal"].reshape(h, w, 3).float() * 255).to(torch.uint8).float()
        c2w = np.eye(4)
        c2w[:3, :4] = views[idx].camera_to_worlds.detach().reshape(3, 4).cpu().double().numpy()
        pose = c2w @ CAM_CONVENTION_CHANGE
        fs.set_pose(idx, pose, np.linalg.inv(pose))
    return fs


@torch.no_grad()
def export_isooctree_mesh(model, cameras, path: str, *, pixel_stride: int = 6, max_depth: int = 10,
                          subdivision_threshold: int = 50, tsdf_rel: float = 0.05, tsdf_abs: Optional[float] = None,
                          disable_normals: bool = False, mesh_file: str = "mesh.obj",
                          max_bytes: int = DEFAULT_MAX_BYTES) -> TriangleMesh:
    """Renders depth and normals of every view with the captured forward service straight into the device frame
    buffers, meshes them as isooctree_mesh_files(camera_coordinate_normals=True) would mesh render_model.py's files of
    the same renders, and writes path/mesh_file (.obj, or .ply)."""
    fs = render_frames(model, cameras)
    mesh = build_mesh_projection(fs, subdivision_threshold=subdivision_threshold, pixel_stride=pixel_stride, max_depth=max_depth,
                                 max_tsdf_rel=tsdf_rel, max_tsdf_abs=tsdf_abs, use_normals=not disable_normals,
                                 max_bytes=max_bytes)
    os.makedirs(path, exist_ok=True)
    write_mesh(mesh, os.path.join(path, mesh_file))
    return mesh


def main(argv=None) -> None:
    parser = argparse.ArgumentParser(description="Parse transformations.json file")
    parser.add_argument("root_folder", type=str, help="path to the render folder containing depth and normal images")
    parser.add_argument("--transformation_path", type=str, help="Root folder path containing transformations.json")
    parser.add_argument("-cam", "--camera_coordinate_normals", action="store_true",
                        help="Whether normals are in camera coordinates")
    parser.add_argument("--max_frames", type=int, default=None, help="Maximum number of frames to parse")
    parser.add_argument("--frame_stride", type=int, default=1, help="Use every Nth frame")
    parser.add_argument("--pixel_stride", type=int, default=6, help="Use every Nth pixel row & col")
    parser.add_argument("--max_depth", type=int, default=10, help="Max meshing octree depth")
    parser.add_argument("--subdivision_threshold", type=int, default=50,
                        help="Subdivision threshold (surface samples per node)")
    parser.add_argument("--tsdf_rel", default=0.05, type=float, help="TSDF fusion tuning param")
    parser.add_argument("--tsdf_abs", type=float, default=None, help="Max TSDF distance (absolute)")
    parser.add_argument("--disable_normals", action="store_true", help="do not use normals in TSDF fusion")
    parser.add_argument("--cache", action="store_true", help="accepted for compatibility: frames stay on the device")
    parser.add_argument("-o", "--output_mesh_file", default="", type=str, help="defaults to input_folder/mesh.obj")
    parser.add_argument("--debug_ply_file", type=str, default=None,
                        help="Path to an output PLY file with intermediary sample data for debug/visualization")
    args = parser.parse_args(argv)
    isooctree_mesh_files(args.root_folder, transformation_path=args.transformation_path,
                         camera_coordinate_normals=args.camera_coordinate_normals, max_frames=args.max_frames,
                         frame_stride=args.frame_stride, pixel_stride=args.pixel_stride, max_depth=args.max_depth,
                         subdivision_threshold=args.subdivision_threshold, tsdf_rel=args.tsdf_rel, tsdf_abs=args.tsdf_abs,
                         disable_normals=args.disable_normals, output_mesh_file=args.output_mesh_file,
                         debug_ply_file=args.debug_ply_file)


if __name__ == "__main__":
    main()
