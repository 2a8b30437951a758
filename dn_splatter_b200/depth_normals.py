"""AGS-Mesh depth confidence masks on the device: the reference's scripts/depth_normal_consistency.py
(`DepthNormalConsistency`) and scripts/depth_to_normal.py (`DepthToNormal`, the class the MuSHRoom and ScanNet++
dataparsers call when --load-depth-confidence-masks finds no masks).

Per frame (natural order of file_path): the depth file (PNG millimetres or .npy, both x 0.001, then f32), resized to the
camera's (w, h) by nearest neighbour, is back-projected (`dnr_dn_backproject`); every pixel, holes included, gets the
normal of its k = 200 nearest points, as Open3D's estimate_normals computes it, oriented towards the camera
(`dnr_dn_normals`); the mono normal PNG of normals_from_pretrain/ is compared with it and the normals image and the mask
(255 where the angle exceeds the threshold) are written as the scripts write them (`dnr_dn_consistency`).  AGS-Mesh reads
the mask back as confidence = 1 - mask / 255, so the JPEG bytes matter: they are written by PIL at quality 95, which gives
cv2.imwrite's bytes.  The next frame's files are read on a host thread while the device works on the current one.

    python -m dn_splatter_b200.depth_normals consistency --data-dir D --transforms-name T [--normal-format dsine]
    python -m dn_splatter_b200.depth_normals depth-to-normal --data-dir D --transforms-name T

The fp64 restatement is oracle/normals_ref.py.  No CPU path: the kernels need CUDA.  Deviation from the scripts
(DESIGN.md §2 (9)): non-finite depth, depth PNGs with more than one channel and mono-normal PNGs of another size than
the camera raise ValueError.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from . import _lib as L

SCALE_FACTOR = 0.001
OPENGL_TO_OPENCV = np.diag([1.0, -1.0, -1.0, 1.0])
KNN = 200
MORTON_CELLS = 1 << 21
DEFAULT_MAX_BYTES = 16 << 30
MODES = {"omnidata": L.DN_OMNIDATA, "dsine": L.DN_DSINE, "depth_to_normal": L.DN_DEPTH_TO_NORMAL}


# ---- host I/O, shared with the oracle's pipeline ----
def natural_key(s: str):
    """natsort's default key: digit runs compare as unsigned integers, the rest as strings."""
    parts = re.split(r"(\d+)", s)
    return tuple(int(p) if i % 2 else p for i, p in enumerate(parts))


def load_transforms(data_dir, transforms_name: str):
    """(frames in natural file_path order, (fx, fy, cx, cy, w, h)): the intrinsics at the top level when fl_x is there,
    else those of frame 0."""
    path = os.path.join(data_dir, transforms_name)
    if not os.path.exists(path):
        raise FileNotFoundError(f"Could not find {transforms_name}")
    with open(path, encoding="UTF-8") as fh:
        tf = json.load(fh)
    frames = sorted(tf["frames"], key=lambda f: natural_key(f["file_path"]))
    src = tf if "fl_x" in tf else tf["frames"][0]
    return frames, (src["fl_x"], src["fl_y"], src["cx"], src["cy"], int(src["w"]), int(src["h"]))


def c2w_of(frame) -> np.ndarray:
    c2w = np.array(frame["transform_matrix"])
    if c2w.shape[0] != 4:
        c2w = np.concatenate([c2w, np.array([[0, 0, 0, 1]])], axis=0)
    return c2w @ OPENGL_TO_OPENCV


def load_depth(path) -> np.ndarray:
    """The depth file in metres, f32, as the scripts' depth_path_to_array reads it; ValueError on non-finite values."""
    from PIL import Image

    path = Path(path)
    if path.suffix == ".png":
        depth = np.array(Image.open(path))
        if depth.ndim != 2:  # cv2.IMREAD_ANYDEPTH would convert a colour PNG to grey: not a depth map, refused here
            raise ValueError(f"{path}: a depth PNG must have one channel, got shape {depth.shape}")
    elif path.suffix == ".npy":
        depth = np.load(path, allow_pickle=True)
        if len(depth.shape) == 3:
            depth = depth[..., 0]
    else:
        raise ValueError(f"Format is not supported {path.suffix}")
    depth = (depth * SCALE_FACTOR).astype(np.float32)
    if not np.isfinite(depth).all():
        raise ValueError(f"{path}: the depth map holds non-finite values")
    return depth


def resize_nearest(img: np.ndarray, w: int, h: int) -> np.ndarray:
    """cv2.resize(img, (w, h), interpolation=cv2.INTER_NEAREST): source index min(floor(x * (1 / (w / sw))), sw - 1)."""
    sh, sw = img.shape[:2]
    if (sh, sw) == (h, w):
        return img
    xs = np.minimum(np.floor(np.arange(w) * (1.0 / (w / sw))).astype(np.int64), sw - 1)
    ys = np.minimum(np.floor(np.arange(h) * (1.0 / (h / sh))).astype(np.int64), sh - 1)
    return img[ys[:, None], xs[None, :]]


def read_mono(path, w: int, h: int) -> np.ndarray:
    from PIL import Image

    m = np.array(Image.open(path))
    if m.shape != (h, w, 3):
        raise ValueError(f"{path}: the mono normal image is {m.shape}, the camera is {(h, w, 3)}")
    return m


def write_image(path: str, img: np.ndarray) -> None:
    """cv2.imwrite(path, img) for a uint8 BGR [h,w,3] or grey [h,w] image: JPEG (quality 95) or PNG by extension."""
    from PIL import Image

    im = Image.fromarray(np.ascontiguousarray(img[..., ::-1]) if img.ndim == 3 else img)
    if path.lower().endswith((".jpg", ".jpeg")):
        im.save(path, format="JPEG", quality=95)
    else:
        im.save(path)


# ---- device ----
def _pose(rot: np.ndarray, t=None) -> L.DnrDnPose:
    p = L.DnrDnPose()
    p.rinv[:] = np.asarray(rot, np.float64).reshape(-1).tolist()
    p.t[:] = [0.0, 0.0, 0.0] if t is None else np.asarray(t, np.float64).reshape(-1).tolist()
    return p


@torch.no_grad()
def backproject_depth(depth, fx, fy, cx, cy, c2w: np.ndarray, with_camera: bool = False):
    """World points [h*w,3] f64 (device) of a depth frame [h,w] in metres, as the scripts' backproject forms them; with
    with_camera also the f32 camera coordinates [h*w,3]."""
    d = torch.as_tensor(depth, dtype=torch.float32, device="cuda").contiguous()
    L.need_cuda(d)
    h, w = d.shape
    if not bool(torch.isfinite(d).all()):
        raise ValueError("backproject_depth: the depth map holds non-finite values")
    pts = torch.empty((h * w, 3), dtype=torch.float64, device=d.device)
    cam = torch.empty((h * w, 3), dtype=torch.float32, device=d.device) if with_camera else None
    intr = (C.c_float * 4)(*[float(np.float32(v)) for v in (fx, fy, cx, cy)])
    c2w = np.asarray(c2w, np.float64)
    pose = _pose(np.linalg.inv(c2w[:3, :3]), c2w[:3, 3])
    L.check(L.load().dnr_dn_backproject(d.data_ptr(), w, h, intr, C.byref(pose), None if cam is None else cam.data_ptr(),
                                        pts.data_ptr(), L.stream()), "dnr_dn_backproject")
    return (pts, cam) if with_camera else pts


def required_bytes(n_points: int) -> int:
    """Device bytes of one estimate_normals call on n points: the search workspace, the points and the normals, plus the
    frame, mono image, angle and encoded outputs of a consistency pass."""
    ws = L.workspace_bytes(L.load().dnr_dn_normals_workspace_bytes, int(n_points))
    return ws + n_points * (24 + 24 + 4 + 3 + 8 + 1 + 3)


def check_budget(n_points: int, max_bytes: int) -> None:
    need = required_bytes(n_points)
    if need > max_bytes:
        raise ValueError(f"depth_normals: {n_points} points need {need / 2**30:.2f} GiB, over max_bytes = "
                         f"{max_bytes / 2**30:.2f} GiB")


@torch.no_grad()
def estimate_normals(points, knn: int = KNN, center=None, *, intrinsics=None, c2w=None, max_bytes: int = DEFAULT_MAX_BYTES,
                     stats: Optional[torch.Tensor] = None, examined: Optional[torch.Tensor] = None, debug: bool = False):
    """Normals [N,3] f64 (device) of a point cloud [N,3], or of a depth frame [h,w] when intrinsics (fx, fy, cx, cy) and
    c2w are given (then oriented towards the camera centre c2w[:3, 3]), as Open3D's
    estimate_normals(KDTreeSearchParamKNN(knn)) computes them [EXT].  center: orient a cloud's normals away from it
    ((p - center) . n <= 0).  stats: a device int64 [2] accumulating (candidates examined, searches, one per distinct
    position); examined: a device int32 [N] receiving the candidates the search of each point's position examined.  With debug, returns
    (normals, covariances [N,9], neighbours [N,knn] int32) for tests."""
    if intrinsics is not None:
        points = backproject_depth(points, *intrinsics, c2w)
        center = np.asarray(c2w, np.float64)[:3, 3]
    pts = torch.as_tensor(points, device="cuda").to(torch.float64).contiguous()
    L.need_cuda(pts)
    if pts.ndim != 2 or pts.shape[1] != 3 or pts.shape[0] == 0:
        raise ValueError(f"estimate_normals: points must be [N,3] with N > 0, got {tuple(pts.shape)}")
    if not 1 <= knn <= L.DN_MAX_K:
        raise ValueError(f"estimate_normals: knn must be in [1, {L.DN_MAX_K}], got {knn}")
    n = pts.shape[0]
    check_budget(n, max_bytes)
    lo, hi = torch.aminmax(pts, dim=0)
    lo, hi = lo.cpu().numpy(), hi.cpu().numpy()
    if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
        raise ValueError("estimate_normals: the points hold non-finite values")
    s = L.DnrDnSearch()
    s.lo[:] = lo.tolist()
    extent = float((hi - lo).max())
    s.cell = extent / MORTON_CELLS if extent > 0 else 1.0
    s.center[:] = [0.0, 0.0, 0.0] if center is None else np.asarray(center, np.float64).tolist()
    s.k, s.orient = int(knn), int(center is not None)
    lib = L.load()
    ws, nbytes = L.workspace(lib.dnr_dn_normals_workspace_bytes, n, device=pts.device)
    normals = torch.empty((n, 3), dtype=torch.float64, device=pts.device)
    cov = torch.empty((n, 9), dtype=torch.float64, device=pts.device) if debug else None
    nbr = torch.empty((n, knn), dtype=torch.int32, device=pts.device) if debug else None
    if examined is not None and (examined.dtype != torch.int32 or examined.numel() != n or not examined.is_contiguous()):
        raise ValueError("estimate_normals: examined must be a contiguous int32 tensor of N elements")
    L.check(lib.dnr_dn_normals(pts.data_ptr(), n, C.byref(s), ws.data_ptr(), nbytes, normals.data_ptr(),
                               None if examined is None else examined.data_ptr(), None if cov is None else cov.data_ptr(), None if nbr is None else nbr.data_ptr(),
                               None if stats is None else stats.data_ptr(), L.stream()), "dnr_dn_normals")
    return (normals, cov, nbr) if debug else normals


@torch.no_grad()
def depth_normal_consistency(normals, mono_u8, c2w: np.ndarray, mode: str = "omnidata", threshold: float = 20.0):
    """(normals image [N,3] u8 (channel 0 first, as the array cv2 writes), degrees [N] f64, mask [N] u8 0/255) on the
    device for oriented normals [N,3] and the mono PNG values [N,3] u8.  mode: "omnidata" / "dsine"
    (DepthNormalConsistency) or "depth_to_normal" (DepthToNormal: threshold 10)."""
    if mode not in MODES:
        raise ValueError(f"depth_normal_consistency: mode must be one of {sorted(MODES)}, got {mode!r}")
    nrm = torch.as_tensor(normals, device="cuda").to(torch.float64).contiguous()
    mono = torch.as_tensor(np.ascontiguousarray(mono_u8), device=nrm.device).reshape(-1, 3).to(torch.uint8).contiguous()
    n = nrm.shape[0]
    if mono.shape[0] != n:
        raise ValueError(f"depth_normal_consistency: {n} normals but {mono.shape[0]} mono normals")
    deg = torch.empty(n, dtype=torch.float64, device=nrm.device)
    mask = torch.empty(n, dtype=torch.uint8, device=nrm.device)
    enc = torch.empty((n, 3), dtype=torch.uint8, device=nrm.device)
    rot = _pose(np.transpose(np.linalg.inv(np.asarray(c2w, np.float64))[:3, :3]))
    L.check(L.load().dnr_dn_consistency(nrm.data_ptr(), mono.data_ptr(), n, C.byref(rot), MODES[mode], float(threshold),
                                        deg.data_ptr(), mask.data_ptr(), enc.data_ptr(), L.stream()), "dnr_dn_consistency")
    return enc, deg, mask


# ---- the scripts ----
def _frame_job(data_dir, frame, mono_dir, w, h):
    name = frame["file_path"].split("/")[-1]
    depth = resize_nearest(load_depth(Path(data_dir) / Path(frame["depth_file_path"])), w, h)
    mono = read_mono(os.path.join(mono_dir, name.replace("jpg", "png")), w, h)
    return name, depth, mono


def run_folder(data_dir, transforms_name: str, mode: str, threshold: float, rename_png: bool, knn: int = KNN,
               max_bytes: int = DEFAULT_MAX_BYTES) -> list:
    """Both scripts' main loop: returns the written (normals, mask) paths in frame order."""
    frames, (fx, fy, cx, cy, w, h) = load_transforms(data_dir, transforms_name)
    out_n, out_m = os.path.join(data_dir, "depth_normals"), os.path.join(data_dir, "depth_normals_mask")
    os.makedirs(out_n, exist_ok=True)
    os.makedirs(out_m, exist_ok=True)
    mono_dir = os.path.join(data_dir, "normals_from_pretrain")
    check_budget(w * h, max_bytes)
    written = []
    with ThreadPoolExecutor(max_workers=1) as pool:
        nxt = pool.submit(_frame_job, data_dir, frames[0], mono_dir, w, h) if frames else None
        for i, frame in enumerate(frames):
            name, depth, mono = nxt.result()
            if i + 1 < len(frames):
                nxt = pool.submit(_frame_job, data_dir, frames[i + 1], mono_dir, w, h)
            c2w = c2w_of(frame)
            normals = estimate_normals(depth, knn, intrinsics=(fx, fy, cx, cy), c2w=c2w, max_bytes=max_bytes)
            enc, _, mask = depth_normal_consistency(normals, mono, c2w, mode, threshold)
            save = name.replace("png", "jpg") if rename_png else name
            pn, pm = os.path.join(out_n, save), os.path.join(out_m, save)
            write_image(pn, enc.reshape(h, w, 3).cpu().numpy())
            write_image(pm, mask.reshape(h, w).cpu().numpy())
            written.append((pn, pm))
    return written


@dataclass
class DepthNormalConsistency:
    """Depth confidence masks from the consistency of depth normals with the pre-trained (mono) normals: writes
    depth_normals/ and depth_normals_mask/ (255 where the angle exceeds angle_treshold) under data_dir."""

    data_dir: Path = Path("dataset/room_datasets/vr_room/iphone/long_capture")
    transforms_name: str = "transformations_colmap.json"
    normal_format: str = "omnidata"  # "omnidata" or "dsine"
    angle_treshold: float = 20.0

    def main(self):
        if self.normal_format not in ("omnidata", "dsine"):
            raise ValueError(f"normal_format must be 'omnidata' or 'dsine', got {self.normal_format!r}")
        return run_folder(self.data_dir, self.transforms_name, self.normal_format, self.angle_treshold, rename_png=True)


@dataclass
class DepthToNormal:
    """Normals of raw sensor depth and the 10-degree consistency mask, written under the frames' own file names."""

    data_dir: Path = None
    transforms_name: str = "transformations_colmap.json"

    def main(self):
        return run_folder(self.data_dir, self.transforms_name, "depth_to_normal", 10.0, rename_png=False)


def main(argv=None) -> None:
    parser = argparse.ArgumentParser(description="Depth normals and depth confidence masks of a capture")
    parser.add_argument("script", choices=("consistency", "depth-to-normal"))
    parser.add_argument("--data-dir", type=Path, required=True, help="Path to data root")
    parser.add_argument("--transforms-name", type=str, default="transformations_colmap.json", help="transforms file name")
    parser.add_argument("--normal-format", choices=("omnidata", "dsine"), default="omnidata",
                        help="coordinate frame of the pre-trained normals (consistency only)")
    parser.add_argument("--angle-treshold", type=float, default=20.0,
                        help="angles above this many degrees are masked (consistency only)")
    args = parser.parse_args(argv)
    if args.script == "consistency":
        DepthNormalConsistency(args.data_dir, args.transforms_name, args.normal_format, args.angle_treshold).main()
    else:
        DepthToNormal(args.data_dir, args.transforms_name).main()


if __name__ == "__main__":
    main()
