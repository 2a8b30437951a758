"""A box room with a block in it, rendered analytically (z-depth and world normals) from inside, and written as the render
folders isooctree_dn.py reads.  Shared by tests/golden/make_golden_isooctree.py and the isooctree tests."""
from __future__ import annotations

import json
import os

import numpy as np

W, H, F = 64, 48, 40.0  # fl_x = fl_y = 40, cx = 32, cy = 24: the dyadic poses below project exactly
ROOM = (np.array([-2.0, -1.5, 0.0]), np.array([3.0, 1.5, 2.5]))  # 5 m long: depths past the 4 m cut
BLOCK = (np.array([0.5, -0.5, 0.0]), np.array([1.25, 0.25, 0.75]))
CCC = np.diag([1.0, -1.0, -1.0, 1.0])


def camera_json():
    return {"w": W, "h": H, "fl_x": F, "fl_y": F, "cx": W / 2, "cy": H / 2}


def look_at_opencv(pos, target, up=(0.0, 0.0, 1.0)):
    pos, target, up = (np.asarray(v, np.float64) for v in (pos, target, up))
    fwd = target - pos
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([right, down, fwd], axis=1)
    c2w[:3, 3] = pos
    return c2w


def transform_matrix(c2w_opencv):
    """The transforms.json (OpenGL) matrix whose pose_c2w, as isooctree_dn.py forms it, is c2w_opencv."""
    return c2w_opencv @ CCC


# The first two look along +x / -y with dyadic positions: every product in their projections is exact, so query points
# can be placed exactly on pixel edges.
POSES = [
    np.array([[0.0, 0.0, 1.0, -1.5], [-1.0, 0.0, 0.0, 0.25], [0.0, -1.0, 0.0, 1.25], [0, 0, 0, 1]]),
    np.array([[1.0, 0.0, 0.0, 0.5], [0.0, 0.0, -1.0, 1.0], [0.0, -1.0, 0.0, 1.0], [0, 0, 0, 1]]),
    look_at_opencv((-1.0, 0.8, 1.6), (1.0, -0.2, 0.4)),
    look_at_opencv((2.2, 1.0, 1.8), (0.0, -0.5, 0.5)),
    look_at_opencv((0.0, -1.0, 2.0), (1.5, 0.5, 0.0)),
    look_at_opencv((2.5, -1.2, 0.9), (-1.5, 1.0, 1.2)),
]


def _box_hits(o, d, lo, hi, inside):
    """Ray parameter t and the hit face's outward axis sign of rays o + t d against an axis-aligned box."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (lo[None] - o[None]) / d
        t1 = (hi[None] - o[None]) / d
    tmin, tmax = np.minimum(t0, t1), np.maximum(t0, t1)
    if inside:
        t = tmax.min(axis=1)
        ax = tmax.argmin(axis=1)
        n = np.zeros_like(d)
        n[np.arange(d.shape[0]), ax] = -np.sign(d[np.arange(d.shape[0]), ax])  # room walls face inward
        return t, n
    tn, tf = tmin.max(axis=1), tmax.min(axis=1)
    ax = tmin.argmax(axis=1)
    hit = (tn <= tf) & (tn > 0)
    n = np.zeros_like(d)
    n[np.arange(d.shape[0]), ax] = -np.sign(d[np.arange(d.shape[0]), ax])
    return np.where(hit, tn, np.inf), n


def render(c2w_opencv, w=W, h=H, f=F):
    """(z-depth [h,w] in metres, world normals [h,w,3]) of the room seen from c2w_opencv (cx = w/2, cy = h/2)."""
    u, v = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    rc = np.stack([(u - w / 2) / f, (v - h / 2) / f, np.ones_like(u)], axis=-1).reshape(-1, 3)
    d = rc @ c2w_opencv[:3, :3].T  # camera z = 1: t is the z-depth
    o = c2w_opencv[:3, 3]
    t_room, n_room = _box_hits(o, d, *ROOM, inside=True)
    t_blk, n_blk = _box_hits(o, d, *BLOCK, inside=False)
    use_blk = t_blk < t_room
    t = np.where(use_blk, t_blk, t_room)
    n = np.where(use_blk[:, None], n_blk, n_room)
    return t.reshape(h, w), n.reshape(h, w, 3)


def frame_files(c2w_opencv, w=W, h=H, f=F):
    """The files of one frame: depth in millimetres [h,w,1] f32 (as render_model.py saves it), world normals f32
    [h,w,3] (.npy layout), and uint8 camera-frame normals (OpenGL axes, (n + 1) / 2 * 255 truncated: the PNG layout)."""
    z, n = render(c2w_opencv, w, h, f)
    depth_mm = (z.astype(np.float32) / np.float32(0.001))[..., None]
    R_gl = (c2w_opencv @ CCC)[:3, :3]
    n_cam = n @ R_gl  # world -> OpenGL camera
    png = (((n_cam + 1) / 2).astype(np.float32) * 255).astype(np.uint8)
    return depth_mm.astype(np.float32), n.astype(np.float32), png


def write_folder(root, cam, transforms, depths_mm, normals_npy, normals_png):
    """Writes both layouts of isooctree_dn.py: depth/frame_X.npy + normal/frame_X.npy, and depth/raw/frame_X.npy +
    normal/frame_X.png, plus transforms.json.  Returns the json path."""
    from PIL import Image

    for sub in ("depth/raw", "normal"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    frames = []
    for i, T in enumerate(transforms):
        iid = f"{i:05d}"
        np.save(os.path.join(root, "depth", f"frame_{iid}.npy"), depths_mm[i])
        np.save(os.path.join(root, "depth", "raw", f"frame_{iid}.npy"), depths_mm[i])
        np.save(os.path.join(root, "normal", f"frame_{iid}.npy"), normals_npy[i])
        Image.fromarray(normals_png[i]).save(os.path.join(root, "normal", f"frame_{iid}.png"))
        frames.append({"file_path": f"images/frame_{iid}.png", "transform_matrix": np.asarray(T).tolist()})
    path = os.path.join(root, "transforms.json")
    with open(path, "w") as fh:
        json.dump({**cam, "frames": frames}, fh)
    return path


def query_points(seed=0):
    """Points for isoFunc: near the surfaces, throughout the room, behind the walls (the back-mask band), behind the
    cameras, and exactly on pixel edges / projecting into (-1, 0) for the two dyadic poses."""
    g = np.random.default_rng(seed)
    pts = [g.uniform(ROOM[0] - 0.3, ROOM[1] + 0.3, (1500, 3))]
    for c2w in POSES:
        z, _ = render(c2w)
        ys, xs = g.integers(0, H, 300), g.integers(0, W, 300)
        rc = np.stack([(xs + g.uniform(0, 1, 300) - W / 2) / F, (ys + g.uniform(0, 1, 300) - H / 2) / F, np.ones(300)], 1)
        scale = z[ys, xs] * g.uniform(0.9, 1.2, 300)  # around the surface, some 10-20 % behind it
        pts.append(c2w[:3, 3][None] + (rc * scale[:, None]) @ c2w[:3, :3].T)
    # exact pixel edges for pose 0 (camera z = world x + 1.5): z = 2.5 -> px = 16 X + 32, py = 16 Y + 24
    for c2w in POSES[:2]:
        cam = []
        for px in (-0.5, -0.25, 0.0, 1.0, 31.0, 32.0, 63.0, 63.5, 64.0):
            for py in (-0.5, 0.0, 10.0, 24.0, 47.0, 47.75, 48.0):
                cam.append([(px - 32) / 16, (py - 24) / 16, 2.5])
        cam = np.array(cam)
        pts.append(c2w[:3, 3][None] + cam @ c2w[:3, :3].T)
        pts.append(c2w[:3, 3][None] + (cam * np.array([1, 1, -1])) @ c2w[:3, :3].T)  # behind the camera
    return np.concatenate(pts)


def eval_tolerance(oracle_values):
    """The GPU isoFunc test's acceptance bound per point: the kernel evaluates in fp64 and rounds to f32 once, so 4 f32
    ulps of the oracle's value (at least those of 1)."""
    return 4 * 2.0 ** -24 * np.maximum(np.abs(oracle_values), 1.0)


def tie_frames(frames):
    """Each frame followed by a copy with the same pose and depth but other normals: every weight of the normal pass
    ties between the two, and the earlier frame must win (isoFunc's strict w > weights)."""
    import copy

    out = []
    for f in frames:
        g = copy.copy(f)
        if f.cam_coordinate_normals:
            g.normal_raw = np.clip(f.normal_raw.astype(np.int64) + np.array([24, -16, 8]), 0, 255).astype(np.uint8)
        else:
            n = f.normal_raw + np.float32(0.35) * np.roll(f.normal_raw, 1, axis=-1)
            g.normal_raw = (n / np.linalg.norm(n, axis=-1, keepdims=True)).astype(np.float32)
        out += [f, g]
    return out
