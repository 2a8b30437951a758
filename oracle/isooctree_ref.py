"""fp64 numpy restatement of AGS-Mesh's mesh extractor, dn_splatter/scripts/isooctree_dn.py:19-458 of the reference
(`compute_depth_validity_mask`, `CameraModel`, `Frame.get_samples` / `get_depth_values`, `isoFunc` in its three modes),
plus the octree and the dense fill this project defines in place of the absent IsoOctree module (DESIGN.md §2).
Test infrastructure only.

Every product of a matrix with a vector is written out as ((a0 b0 + a1 b1) + a2 b2) (+ a3), the order
csrc/isooctree.cu uses with -fmad=false, so the kernels equal this file bit for bit; the reference's BLAS matmuls may
round the same sums differently in the last place (~1e-16 relative).

The reference's quirks, kept on purpose (each is named again where it happens):
  Q1  `astype(int)` truncates toward zero: a point projecting to x in (-1, 0) passes the in-image test with ix = 0 and
      tx < 0, so the bilinear weights extrapolate.
  Q2  the depth-validity mask is read at (iy, ix) only.
  Q3  ix1 / iy1 are clamped to the last column / row.
  Q4  get_depth_values reads the full-resolution depth with no 4 m cut; get_samples reads the stride-subsampled depth,
      cuts it at 4 and uses max_valid_depth_rel_delta * stride.
  Q5  rays are not normalised (depth_is_z).
  Q6  frames whose normal faces away from the point (normals . ray >= 0) are dropped.
  Q7  the normal pass takes a frame only when w > weight strictly: on a tie the earlier frame wins.
  Q8  back_mask turns unobserved points up to 25 % of the depth behind a surface into -1.
  Q9  values[~valid] = 1.
  Q10 with camera_coordinate_normals the PNG normals go from [0, 255] to [-1, 1]; get_samples rotates them by
      pose_c2w . CAM_CONVENTION_CHANGE and renormalises them, get_depth_values uses them as loaded.
  Q11 image_id is the part of file_path's base name between the first "_" and the first ".".
  Q12 choose_best_frame returns the best frame's TSDF value divided by its weight (values / weights after one normal
      pass).
"""
from __future__ import annotations

import json
import os
from typing import List, Optional, Sequence

import numpy as np

EPS = 1e-6
MIN_DEPTH = 1e-3
BACK_MASK_COEFF = 0.25
CAM_CONVENTION_CHANGE = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])
ROOT_SCALE = 1.05  # root cube side over the hint cloud's longest extent


def _mv(M, p):
    """Rows of M (r x 3 or r x 4) applied to points p [n,3] as ((m0 p0 + m1 p1) + m2 p2) (+ m3)."""
    cols = []
    for r in range(M.shape[0]):
        c = (p[:, 0] * M[r, 0] + p[:, 1] * M[r, 1]) + p[:, 2] * M[r, 2]
        if M.shape[1] == 4:
            c = c + M[r, 3]
        cols.append(c)
    return np.stack(cols, axis=1)


def _dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def compute_depth_validity_mask(depth_img, max_valid_depth_rel_delta):
    depth_dx = np.diff(depth_img, axis=1)
    depth_dy = np.diff(depth_img, axis=0)
    dx_ok = np.abs(depth_dx) < np.minimum(depth_img[:, 1:], depth_img[:, :-1]) * max_valid_depth_rel_delta
    dy_ok = np.abs(depth_dy) < np.minimum(depth_img[1:, :], depth_img[:-1, :]) * max_valid_depth_rel_delta
    valid = np.ones_like(depth_img, dtype=bool)
    valid[:, 1:] &= dx_ok
    valid[:, :-1] &= dx_ok
    valid[1:, :] &= dy_ok
    valid[:-1, :] &= dy_ok
    return valid


class CameraModel:
    def __init__(self, data):
        self.resolution = int(data["w"]), int(data["h"])
        self.camera_matrix = np.array([[data["fl_x"], 0, data["cx"]], [0, data["fl_y"], data["cy"]], [0, 0, 1]], dtype=np.float64)
        self.inverse_camera_matrix = np.linalg.inv(self.camera_matrix)

    def unproject(self, pixel_coordinates):
        return _mv(self.inverse_camera_matrix, np.hstack([pixel_coordinates, np.ones((pixel_coordinates.shape[0], 1))]))

    def project(self, points):
        projections = np.zeros((points.shape[0], 2))
        valid = points[:, 2] > EPS
        h = _mv(self.camera_matrix, points[valid])
        projections[valid] = h[:, :2] / h[:, 2:3]
        for i in range(2):
            proj_i = projections[:, i].astype(int)  # Q1: truncation toward zero
            valid = valid & (proj_i >= 0) & (proj_i < self.resolution[i])
        return projections, valid

    def all_pixels(self, stride=1):
        x = np.arange(0, self.resolution[0])[::stride].astype(float) + 0.5
        y = np.arange(0, self.resolution[1])[::stride].astype(float) + 0.5
        xv, yv = np.meshgrid(x, y)
        return np.stack([xv.ravel(), yv.ravel()], axis=1)


class Frame:
    """One view: the raw file contents (depth in millimetres [H,W] as stored, normals [H,W,3] as stored: uint8 PNG
    values when cam_coordinate_normals, world-frame floats otherwise) and its transforms.json pose."""

    depth_scale = 1 / 1000.0
    max_valid_depth_rel_delta = 0.005

    def __init__(self, camera: CameraModel, transform_matrix, depth_raw, normal_raw, cam_coordinate_normals=False):
        self.camera = camera
        c2w = np.array(transform_matrix, dtype=np.float64)
        if c2w.shape[0] == 3:
            c2w = np.vstack([c2w, [0, 0, 0, 1]])
        self.pose_c2w = c2w @ CAM_CONVENTION_CHANGE
        self.pose_w2c = np.linalg.inv(self.pose_c2w)
        self.cam_coordinate_normals = bool(cam_coordinate_normals)
        W, H = camera.resolution
        assert depth_raw.shape[:2] == (H, W) and normal_raw.shape[:2] == (H, W)
        self.depth_raw = depth_raw.reshape(H, W)
        self.normal_raw = normal_raw

    @property
    def position(self):
        return self.pose_c2w[:3, 3]

    def normal_rotation(self):
        return self.pose_c2w[:3, :3] @ CAM_CONVENTION_CHANGE[:3, :3]

    def depth(self, stride=1):
        return self.depth_raw[::stride, ::stride].astype(np.float64) * self.depth_scale

    def normals(self, stride=1):
        n = self.normal_raw[::stride, ::stride]
        if self.cam_coordinate_normals:
            return n.astype(float) / 255.0 * 2 - 1  # Q10
        return n.astype(np.float64)

    def world_to_camera(self, points):
        return _mv(self.pose_w2c[:3], points)

    def get_depth_values(self, points, return_normals=False, *, slip=None):
        pixel_coords, valid_mask = self.camera.project(self.world_to_camera(points))
        if slip == "floor":  # test slip: truncation done as floor
            for i in range(2):
                valid_mask &= np.floor(pixel_coords[:, i]) >= 0
        vp = pixel_coords[valid_mask]
        depths = np.zeros(points.shape[0])
        di = self.depth()  # Q4: full resolution, no 4 m cut
        if slip == "cut4":
            di = np.where(di <= 4, di, 0)
        depth_mask = compute_depth_validity_mask(di, self.max_valid_depth_rel_delta)
        normals = np.zeros((points.shape[0], 3))
        if valid_mask.any():
            rnd = np.floor if slip == "floor" else np.trunc
            ix, iy = rnd(vp[:, 0]).astype(int), rnd(vp[:, 1]).astype(int)
            tx, ty = vp[:, 0] - ix, vp[:, 1] - iy
            ix1 = np.minimum(ix + 1, di.shape[1] - 1)  # Q3
            iy1 = np.minimum(iy + 1, di.shape[0] - 1)
            dd = (di[iy, ix] * (1 - tx) * (1 - ty) + di[iy, ix1] * tx * (1 - ty) + di[iy1, ix] * (1 - tx) * ty
                  + di[iy1, ix1] * tx * ty)
            new_valid = depth_mask[iy, ix] & (dd > MIN_DEPTH)  # Q2
            if return_normals:
                normals[valid_mask] = self.normals()[iy, ix]  # Q10: unrotated in -cam mode
            depths[valid_mask] = dd
            valid_mask[valid_mask] = new_valid
        computed = self.world_to_camera(points)[:, 2]
        if return_normals:
            rays = points - self.position[None, :]
            valid_mask &= _dot(normals, rays) < 0  # Q6
            return depths, computed, normals, valid_mask
        return depths, computed, valid_mask

    def get_samples(self, stride=1):
        """(positions, normals, depths, rays) of the surviving stride-subsampled pixels, in row-major order."""
        pix = self.camera.all_pixels(stride=stride)
        rays = _mv(self.pose_c2w[:3, :3], self.camera.unproject(pix))  # Q5: not normalised
        d = self.depth(stride)
        d = np.where(d <= 4, d, 0)  # Q4
        mask = compute_depth_validity_mask(d, self.max_valid_depth_rel_delta * stride).ravel()
        depths = d.ravel()
        normals = self.normals(stride).reshape(-1, 3).astype(float)
        if self.cam_coordinate_normals:  # Q10
            normals = _mv(self.normal_rotation().astype(np.float64), normals)
            normals = normals / np.sqrt(_dot(normals, normals))[:, None]
        keep = (_dot(normals, rays) < 0) & mask
        pos = self.position[None, :] + rays * depths[:, None]
        return pos[keep], normals[keep], depths[keep], rays[keep]


def image_id(file_path: str) -> str:
    return file_path.split("/")[-1].split("_")[1].split(".")[0]  # Q11


def load_frames(root_dir, json_file_path, max_frames=None, frame_stride=1, camera_coordinate_normals=False) -> List[Frame]:
    """load_frame_metadata + load_image: the frames whose depth and normal files exist, read into memory."""
    from PIL import Image

    with open(json_file_path) as fh:
        data = json.load(fh)
    camera = CameraModel(data)
    frames = []
    for i, jf in enumerate(data["frames"]):
        if i % frame_stride != 0:
            continue
        iid = image_id(jf["file_path"])
        if camera_coordinate_normals:
            dpath = os.path.join(root_dir, "depth", "raw", f"frame_{iid}.npy")
            npath = os.path.join(root_dir, "normal", f"frame_{iid}.png")
        else:
            dpath = os.path.join(root_dir, "depth", f"frame_{iid}.npy")
            npath = os.path.join(root_dir, "normal", f"frame_{iid}.npy")
        if not (os.path.exists(dpath) and os.path.exists(npath)):
            continue
        depth = np.load(dpath)[..., 0]
        normal = np.array(Image.open(npath)) if npath.endswith(".png") else np.load(npath)
        frames.append(Frame(camera, jf["transform_matrix"], depth, normal, camera_coordinate_normals))
        if max_frames is not None and len(frames) >= max_frames:
            break
    return frames


def hint_cloud(frames: Sequence[Frame], pixel_stride: int):
    """(points, normals) of every frame's get_samples, stacked in frame order."""
    s = [f.get_samples(stride=pixel_stride) for f in frames]
    return np.vstack([x[0] for x in s]).reshape(-1, 3), np.vstack([x[1] for x in s]).reshape(-1, 3)


def iso_func(frames: Sequence[Frame], points, max_tsdf_rel=0.05, max_angle_to_max_weight_normal_deg=60,
             max_tsdf_abs=None, choose_best_frame=False, two_pass=True, use_normals=True, slip=None):
    """isoFunc of build_mesh_projection at points [n,3].  slip names a deliberate deviation, used by the tests to show
    that the GPU test's acceptance rule detects it: "floor", "tie" (w >= weights), "cut4", "no_back", "norm_ray"."""
    points = np.asarray(points, dtype=np.float64)
    md = np.cos(max_angle_to_max_weight_normal_deg / 180 * np.pi)
    if not use_normals:
        choose_best_frame, two_pass = False, False
    passes = [True] if choose_best_frame else ([True, False] if two_pass else [False])
    n = points.shape[0]
    mwn = np.zeros((n, 3))
    for normal_pass in passes:
        valid_mask = np.zeros(n, bool)
        back_mask = np.zeros(n, bool)
        values = np.zeros(n)
        weights = np.zeros(n)
        for frame in frames:
            r = frame.get_depth_values(points, return_normals=use_normals, slip=slip)
            if use_normals:
                pd, zc, normals, valid = r
            else:
                pd, zc, valid = r
            if slip == "norm_ray":  # test slip: the point's depth measured along a normalised ray
                cam = frame.world_to_camera(points)
                zc = np.sqrt(_dot(cam, cam))
            max_tsdf = max_tsdf_rel * pd[valid]
            if max_tsdf_abs is not None:
                max_tsdf = np.minimum(max_tsdf, max_tsdf_abs)
            tv = (pd[valid] - zc[valid]) / max_tsdf
            if slip != "no_back":
                back_mask[valid] |= (tv * max_tsdf_rel > -BACK_MASK_COEFF) & (tv < 0)  # Q8
            v1 = tv > -1
            tv = tv[v1]
            valid[valid] = v1
            tv = np.minimum(tv, 1)
            rays = points[valid] - frame.position[None, :]
            rays = rays / np.maximum(EPS, np.sqrt(_dot(rays, rays)))[:, None]
            if normal_pass or not use_normals:
                dir_weight = 1
            else:
                dir_weight = -_dot(normals[valid], rays)
            tv = tv * dir_weight
            w = dir_weight / np.maximum(EPS, pd[valid])
            if normal_pass:
                w = w * np.maximum(0, np.minimum(tv + 0.5, 1))
                v2 = (w >= weights[valid]) if slip == "tie" else (w > weights[valid])  # Q7
                valid[valid] = v2
                weights[valid] = w[v2]
                mwn[valid] = normals[valid]
                values[valid] = tv[v2]
            else:
                if use_normals:
                    has = _dot(mwn[valid], mwn[valid]) > 0
                    mnw = np.maximum(_dot(mwn[valid], normals[valid]) - md, 0) / (1 - md)
                    neg = 1 - np.maximum(0, np.minimum(tv[has] + 0.5, 1))
                    w[has] *= mnw[has] * neg + (1 - neg)
                values[valid] += tv * w
                weights[valid] += w
            valid_mask |= valid
        if normal_pass:
            valid_mask &= _dot(mwn, mwn) > 0
            mwn[valid_mask] /= np.sqrt(_dot(mwn[valid_mask], mwn[valid_mask]))[:, None]
    valid_mask &= weights > 0
    values[valid_mask] /= weights[valid_mask]  # Q12 in choose_best_frame mode
    values[~valid_mask] = 1  # Q9
    values[~valid_mask & back_mask] = -1  # Q8
    return values


# ---------------------------------------------------------------------------------------------- octree and fill
def root_cube(hint):
    """(origin [3], side): the cube centred on the hint cloud's bounding box, side ROOT_SCALE x its longest extent."""
    lo, hi = hint.min(axis=0), hint.max(axis=0)
    side = max(float((hi - lo).max()), 1e-9) * ROOT_SCALE
    return 0.5 * (lo + hi) - 0.5 * side, side


def finest_cells(hint, origin, cell, max_depth):
    R = 1 << max_depth
    return np.clip(np.floor((hint - origin[None, :]) / cell), 0, R - 1).astype(np.int64)


def morton(c, bits):
    code = np.zeros(c.shape[0], np.int64)
    for b in range(bits):
        for a in range(3):
            code |= ((c[:, a] >> b) & 1) << (3 * b + 2 - a)
    return code


def demorton(code, bits):
    c = np.zeros((code.shape[0], 3), np.int64)
    for b in range(bits):
        for a in range(3):
            c[:, a] |= ((code >> (3 * b + 2 - a)) & 1) << b
    return c


def octree(hint, max_depth, subdivision_threshold, origin=None, side=None):
    """Leaves as int64 level << 58 | Morton code of the node at its level, sorted (by level, then code).  A node splits
    iff it holds >= subdivision_threshold hint samples and its level is below max_depth; every child of a split node
    exists.  Returns (leaves, origin, finest cell)."""
    if origin is None:
        origin, side = root_cube(hint)
    cell = side / (1 << max_depth)
    keys = np.sort(morton(finest_cells(hint, origin, cell, max_depth), max_depth))
    leaves = []
    split = np.zeros(1, np.int64)
    if not (keys.shape[0] >= subdivision_threshold and max_depth > 0):
        return np.array([0], np.int64), origin, cell
    for level in range(1, max_depth + 1):
        children = (split[:, None] * 8 + np.arange(8)[None, :]).reshape(-1)
        shift = 3 * (max_depth - level)
        count = np.searchsorted(keys, (children + 1) << shift) - np.searchsorted(keys, children << shift)
        s = (count >= subdivision_threshold) & (level < max_depth)
        leaves.append((np.int64(level) << 58) | children[~s])
        split = children[s]
    return np.concatenate(leaves), origin, cell


def leaf_boxes(leaves, max_depth):
    """(level [n], lattice corner [n,3], size [n]) of each leaf on the (2^max_depth + 1)^3 sample lattice."""
    level = leaves >> 58
    code = leaves & ((1 << 58) - 1)
    c = demorton(code, max_depth)
    size = np.int64(1) << (max_depth - level)
    return level, c * size[:, None], size


def leaf_corners(leaves, max_depth):
    """Sorted unique lattice keys (i * (R+1) + j) * (R+1) + k of all leaf corners."""
    R1 = (1 << max_depth) + 1
    _, lo, size = leaf_boxes(leaves, max_depth)
    keys = []
    for q in range(8):
        p = lo + size[:, None] * np.array([(q >> 2) & 1, (q >> 1) & 1, q & 1])
        keys.append((p[:, 0] * R1 + p[:, 1]) * R1 + p[:, 2])
    return np.unique(np.concatenate(keys))


def corner_points(keys, origin, cell, max_depth):
    R1 = (1 << max_depth) + 1
    ijk = np.stack([keys // (R1 * R1), (keys // R1) % R1, keys % R1], axis=1)
    return origin[None, :] + ijk.astype(np.float64) * cell


def _lerp(a, b, t):
    return (np.float32(1) - t) * a + t * b


def fill(leaves, corner_keys, corner_values, max_depth):
    """The dense f32 grid [(R+1)^3]: leaves written coarse to fine, each over its closed cube, with the lerp-of-lerps
    (x, then y, then z) of its 8 corner values, so the smallest leaf containing a sample decides it and a corner
    sample keeps its evaluated value."""
    R1 = (1 << max_depth) + 1
    field = np.full((R1, R1, R1), np.nan, np.float32)
    vals = np.asarray(corner_values, np.float32)
    level, lo, size = leaf_boxes(leaves, max_depth)
    for n in np.argsort(level, kind="stable"):
        s = int(size[n])
        x0, y0, z0 = (int(v) for v in lo[n])
        cv = {}
        for q in range(8):
            dx, dy, dz = (q >> 2) & 1, (q >> 1) & 1, q & 1
            key = ((x0 + dx * s) * R1 + (y0 + dy * s)) * R1 + (z0 + dz * s)
            cv[(dx, dy, dz)] = vals[np.searchsorted(corner_keys, key)]
        t = (np.arange(s + 1, dtype=np.float32) / np.float32(s))
        tx, ty, tz = t[:, None, None], t[None, :, None], t[None, None, :]
        c00 = _lerp(cv[0, 0, 0], cv[1, 0, 0], tx)
        c01 = _lerp(cv[0, 0, 1], cv[1, 0, 1], tx)
        c10 = _lerp(cv[0, 1, 0], cv[1, 1, 0], tx)
        c11 = _lerp(cv[0, 1, 1], cv[1, 1, 1], tx)
        c0, c1 = _lerp(c00, c10, ty), _lerp(c01, c11, ty)
        field[x0:x0 + s + 1, y0:y0 + s + 1, z0:z0 + s + 1] = _lerp(c0, c1, tz)
    return field


def mesh_pipeline(frames, subdivision_threshold, pixel_stride, max_depth, **iso_kwargs):
    """build_mesh_projection with this project's octree and fill: (vertices, faces, hint) via oracle/mesh_ref.py's
    marching cubes at 0."""
    from oracle import mesh_ref

    hint, _ = hint_cloud(frames, pixel_stride)
    leaves, origin, cell = octree(hint, max_depth, subdivision_threshold)
    keys = leaf_corners(leaves, max_depth)
    vals = iso_func(frames, corner_points(keys, origin, cell, max_depth), **iso_kwargs).astype(np.float32)
    field = fill(leaves, keys, vals, max_depth)
    v, f, _ = mesh_ref.marching_cubes(field, 0.0, origin.astype(np.float32), np.float32(cell))
    return v, f, hint
