"""normal_from_depth_image / pcd_to_normal with the reference's signatures
(/root/reference/dn_splatter/utils/normal_utils.py:9-48).  The depth->normal stencil runs in one CUDA kernel
(dnr_normal_from_depth) when c2w is the identity (every call site of the reference); a non-identity c2w is
applied afterwards as a rotation of the normals (equivalent, since the back-projection is linear in c2w)."""
from __future__ import annotations

import ctypes as C

import torch
from torch import Tensor

from .. import _lib as L


def normal_from_depth_image(depths: Tensor, fx: float, fy: float, cx: float, cy: float, img_size: tuple, c2w: Tensor,
                            device: torch.device, smooth: bool = False) -> Tensor:
    """estimate normals from a depth map [H,W,1] (or [H*W,1]) -> [H,W,3], zero 1-px border."""
    if smooth:
        raise NotImplementedError("smooth=True (cv2.GaussianBlur on the host) is outside the accelerated path")
    W, H = int(img_size[0]), int(img_size[1])
    if depths.device.type != "cuda":
        raise L.DnrError("normal_from_depth_image: CUDA tensor required (no CPU path)")
    d = depths.detach().float().contiguous().view(H, W)
    out = torch.empty(H, W, 3, dtype=torch.float32, device=d.device)
    a = L.DnrArgs()
    a.width, a.height = W, H
    a.flags = L.FLAG_HOST_CAMERA  # intrinsics by value: no upload
    a.host_cam[16], a.host_cam[17], a.host_cam[18], a.host_cam[19] = float(fx), float(fy), float(cx), float(cy)
    a.out_depth, a.out_surface_normal = d.data_ptr(), out.data_ptr()
    L.check(L.load().dnr_normal_from_depth(C.byref(a), L.stream()), "dnr_normal_from_depth")
    if c2w is not None and c2w.device.type == "cpu":  # identity test on the host only (a device tensor would sync)
        R = c2w[..., :3, :3].to(out)
        if not bool(torch.equal(c2w[..., :3, :3].float(), torch.eye(3))):
            # means3d @ inv(R) + t  =>  differences (and hence normals) are rotated by inv(R)
            out = torch.nn.functional.normalize(out @ torch.linalg.inv(R), dim=-1) * (out.norm(dim=-1, keepdim=True) > 0)
    return out


def pcd_to_normal(xyz: Tensor) -> Tensor:
    """[H,W,3] point map -> normals from the 4-neighbourhood (reference :9-22); torch ops (not on the hot path)."""
    H, W, _ = xyz.shape
    l2r = xyz[1:H - 1, 2:W] - xyz[1:H - 1, 0:W - 2]
    b2t = xyz[0:H - 2, 1:W - 1] - xyz[2:H, 1:W - 1]
    n = torch.nn.functional.normalize(torch.cross(l2r, b2t, dim=-1), p=2, dim=-1)
    return torch.nn.functional.pad(n.permute(2, 0, 1), (1, 1, 1, 1), mode="constant").permute(1, 2, 0)
