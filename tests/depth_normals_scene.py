"""The capture folder of the depth-normal tests: the box room of tests/isooctree_scene.py seen by its six poses, written
as the reference's depth_normal_consistency.py / depth_to_normal.py read it.  Frame names sort differently naturally and
lexically (frame_2 < frame_10); depth comes as 16-bit PNG millimetres and as .npy millimetres (2-D and 3-D); one frame has
150 holes and one 400; the mono normals are the true camera-frame normals, rotated by 35 degrees over the x = -2 wall so
both mask values occur, in the omnidata or the dsine convention.  Shared by tests/golden/make_golden_normals.py and the
tests."""
from __future__ import annotations

import json
import os

import numpy as np

from tests import isooctree_scene as S

W, H = S.W, S.H
NAMES = ["frame_1.jpg", "frame_2.png", "frame_10.jpg", "frame_11.jpg", "frame_3.png", "frame_20.jpg"]
DEPTH_KIND = ["png", "npy", "npy3", "png", "npy", "png"]
HOLES = {1: 150, 4: 400}


def scene_arrays(seed=0):
    """(depth_mm [6,h,w] f32 with holes as 0, world normals [6,h,w,3], transforms [6,4,4] OpenGL)."""
    g = np.random.default_rng(seed)
    depths, normals = [], []
    for i, c2w in enumerate(S.POSES):
        z, n = S.render(c2w)
        d = np.round(z * 1000.0).astype(np.float32)
        if i in HOLES:
            flat = d.reshape(-1)
            flat[g.choice(flat.size, HOLES[i], replace=False)] = 0
        depths.append(d)
        normals.append(n)
    return np.stack(depths), np.stack(normals), np.stack([S.transform_matrix(p) for p in S.POSES])


def mono_png(world_normals, c2w_opencv, dsine=False):
    """uint8 [h,w,3] mono normal image of world normals seen from c2w_opencv (the camera frame the scripts decode)."""
    n = world_normals.copy()
    wall = n[..., 0] > 0.5  # the x = -2 wall faces +x
    a = np.deg2rad(35.0)
    rot = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    n[wall] = n[wall] @ rot.T
    cam = n @ c2w_opencv[:3, :3]
    if dsine:
        cam = cam * np.array([1.0, -1.0, -1.0])
    return np.clip(np.round((cam + 1) / 2 * 255), 0, 255).astype(np.uint8)


def write_folder(root, depth_mm, transforms, monos, transforms_name="transforms.json", intrinsics_in_frames=False):
    """Writes the capture folder; returns the transforms file name."""
    from PIL import Image

    for sub in ("depth", "normals_from_pretrain", "images"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    cam = S.camera_json()
    frames = []
    for i, name in enumerate(NAMES):
        stem = name.rsplit(".", 1)[0]
        kind = DEPTH_KIND[i]
        if kind == "png":
            dpath = f"depth/{stem}.png"
            Image.fromarray(depth_mm[i].astype(np.uint16)).save(os.path.join(root, dpath))
        else:
            dpath = f"depth/{stem}.npy"
            np.save(os.path.join(root, dpath), depth_mm[i][..., None] if kind == "npy3" else depth_mm[i])
        Image.fromarray(monos[i]).save(os.path.join(root, "normals_from_pretrain", name.replace("jpg", "png")))
        fr = {"file_path": f"images/{name}", "depth_file_path": dpath, "transform_matrix": np.asarray(transforms[i]).tolist()}
        if intrinsics_in_frames:
            fr.update(cam)
        frames.append(fr)
    body = {"frames": frames} if intrinsics_in_frames else {**cam, "frames": frames}
    with open(os.path.join(root, transforms_name), "w") as fh:
        json.dump(body, fh)
    return transforms_name


def build(root, dsine=False, intrinsics_in_frames=False, seed=0):
    depth, normals, transforms = scene_arrays(seed)
    monos = [mono_png(normals[i], S.POSES[i], dsine) for i in range(len(NAMES))]
    return write_folder(root, depth, transforms, monos, intrinsics_in_frames=intrinsics_in_frames)


def list_outputs(root):
    """{relative path: bytes} of every file the scripts wrote."""
    out = {}
    for sub in ("depth_normals", "depth_normals_mask"):
        d = os.path.join(root, sub)
        for f in sorted(os.listdir(d)):
            with open(os.path.join(d, f), "rb") as fh:
                out[f"{sub}/{f}"] = fh.read()
    return out
