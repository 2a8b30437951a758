"""ORACLE (test infrastructure, NOT product code) — fp64 restatement of AGSMeshRegularization's depth and normal terms
(reference regularization_strategy.py:202-321, as dn_model.py:645-646, 715-725 calls them), quirks included.

Inputs are read as the kernels read them (csrc/ags_loss.cu): a uint8 map is `u8 * fp32(1/255)`, the signed normals are
`2x - 1` formed in fp32, a raw confidence map is gated on `1 - get_gt_img(c) * fp32(1/255) > 0` in fp32, and the
thresholds are fp32 (0.01, 0.1, the depth tolerance).  Everything after that is float64.  The two mask decisions are
reported with their fp64 margins, so a test can tell a kernel error from a decision that fp32 rounding may flip:
  * the Laplacian of r = 1 / (g + 1e-6) against 0.01, relative to the sum of |terms| (r itself is the fp32 reciprocal);
  * the angle acos(clip(sum_c s g, -1, 1)) against 0.1, in radians.
Only tests may import this.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
from torch import Tensor

F32, F64 = torch.float32, torch.float64
INV255 = torch.tensor(1 / 255, dtype=F32)
LO = torch.tensor(10 / 255, dtype=F32)
EDGE_T = float(torch.tensor(0.01, dtype=F32))
ANGLE_T = float(torch.tensor(0.1, dtype=F32))


def u8(t: Tensor) -> Tensor:
    """uint8 -> fp32 as the kernels read it (value * fp32(1/255))."""
    return t.to(F32) * INV255


def signed(t: Tensor) -> Tensor:
    """[H,W,3] [0,1] map (fp32 or uint8) -> signed fp32 [3,H,W]: 2x - 1 formed in fp32, as torch forms it."""
    x = u8(t) if t.dtype == torch.uint8 else t.to(F32)
    return (2 * x - 1).permute(2, 0, 1).contiguous()


def gate_map(conf: Tensor, raw: bool) -> Tensor:
    """The confidence the gate compares with 0: the batch map through 1 - get_gt_img(c) / 255 (fp32), or as given."""
    if not raw:
        return conf.to(F32)
    c = u8(conf) if conf.dtype == torch.uint8 else conf.to(F32)
    return 1 - c * INV255


def edge_image(img: Tensor) -> Tensor:
    """EdgeAwareLogL1's image: uint8 scaled and clamped below at 10/255 (dn_model.py:633), fp32 as given."""
    return torch.maximum(u8(img), LO) if img.dtype == torch.uint8 else img.to(F32)


def laplacian_r(g: Tensor):
    """Per channel: the Laplacian of r = fp32(1 / (g + fp32(1e-6))) with zero padding of r, in fp64, and the sum of the
    |terms| (the scale of its rounding error).  g: signed fp32 [3,H,W]."""
    r = (1.0 / (g + torch.tensor(1e-6, dtype=F32))).to(F64)
    rp = torch.nn.functional.pad(r, (1, 1, 1, 1))
    c = rp[:, 1:-1, 1:-1]
    nb = (rp[:, :-2, 1:-1], rp[:, 2:, 1:-1], rp[:, 1:-1, :-2], rp[:, 1:-1, 2:])
    lap = nb[0] + nb[1] + nb[2] + nb[3] - 4 * c
    scale = sum(t.abs() for t in nb) + 4 * c.abs()
    return lap, scale


def dilate(e: Tensor) -> Tensor:
    """3x3 box dilation per channel, clipped to the image.  e: bool [C,H,W]."""
    p = torch.nn.functional.pad(e.to(F64)[None], (1, 1, 1, 1))[0]
    H, W = e.shape[1:]
    out = torch.zeros_like(e)
    for dy in range(3):
        for dx in range(3):
            out |= p[:, dy:dy + H, dx:dx + W] > 0
    return out


def keep_mask(s: Tensor, g: Tensor, angle: bool) -> Dict[str, Tensor]:
    """The surface term's selection [3,H,W] (True: kept) and the margins of its decisions.
    Edge mode: `margin` [3,H,W] = (lap - 0.01) / sum|terms| per element (before the dilation).
    Angle mode: `margin` [H,W] = angle - 0.1 in radians."""
    if angle:
        dot = (s.to(F64) * g.to(F64)).sum(0)
        ang = torch.arccos(dot.clamp(-1.0, 1.0))
        keep = ~(ang > ANGLE_T)
        return {"keep": keep[None].expand(3, -1, -1).clone(), "margin": ang - ANGLE_T}
    lap, scale = laplacian_r(g)
    edges = lap > EDGE_T
    return {"keep": ~dilate(edges), "margin": (lap - EDGE_T) / scale.clamp(min=1e-300)}


def depth_sums(pd: Tensor, gd: Tensor, depth_type: int, tol: float, img: Optional[Tensor]):
    """(value, d value / d pred) of the depth term D, fp64, on [H,W] maps; `gd` already gated."""
    pd, gd = pd.to(F64).reshape(gd.shape), gd
    mask = gd.to(F32) > torch.tensor(tol, dtype=F32)
    gd = gd.to(F64)
    pd = pd.detach().clone().requires_grad_(True)
    e = pd - gd
    if depth_type in (1, 2):
        val = torch.log(1 + e.abs())
    elif depth_type == 3:
        val = e.abs()
    else:
        val = e * e
    if depth_type == 1:
        im = img.to(F64)
        wx = torch.exp(-(im[:, :-1] - im[:, 1:]).abs().mean(-1))
        wy = torch.exp(-(im[:-1] - im[1:]).abs().mean(-1))
        mx, my = mask[:, :-1], mask[:-1]
        D = (wx * val[:, :-1])[mx].mean() + (wy * val[:-1])[my].mean()
    else:
        D = val[mask].mean()
    if pd.requires_grad and torch.isfinite(D):
        (gr,) = torch.autograd.grad(D, pd, allow_unused=True)
    else:
        gr = torch.zeros_like(pd)
    return D.detach(), gr.detach()


def ags_loss(pred_depth, gt_depth, confidence, image, surf_normal, gt_normal, pred_normal, *, depth_type: int,
             depth_lambda: float, tol: float, normal_lambda: float, step: int, normal_mask_steps: int = 15000,
             confidence_raw: bool = True, keep: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """The regulariser's depth + normal value and gradients at `step`.  Normals are [H,W,3] [0,1] maps (fp32 or uint8);
    depth maps [H,W] or [H,W,1]; `keep` ([3,H,W] bool) replaces the selection with a given one (the kernel's).
    Returns value, depth / surface / pred terms, keep, margin, v_depth [H,W] and v_normal [H,W,3] (d value / d map)."""
    H, W = pred_normal.shape[:2]
    s, g, n = signed(surf_normal), signed(gt_normal), signed(pred_normal)
    lam = normal_lambda if step > 7000 else 0.0
    km = keep_mask(s, g, angle=not step < normal_mask_steps)
    sel = km["keep"] if keep is None else keep
    d_surf = (s.to(F64) - g.to(F64)).abs()
    surf = d_surf[sel].mean() * lam  # empty: nan, and 0 * nan stays nan
    dn = n.to(F64) - g.to(F64)
    pred = dn.abs().mean() * lam
    d_sign = torch.sign((n - g).to(F64))  # the sign of d as formed in fp32
    v_normal = (d_sign * (2.0 * lam / (3 * H * W))).permute(1, 2, 0).contiguous()
    if depth_type:
        gd = gt_depth.to(F32).reshape(H, W)
        if step >= 7000:
            gd = torch.where(gate_map(confidence, confidence_raw).reshape(H, W) > 0, gd, torch.zeros_like(gd))
        D, vD = depth_sums(pred_depth, gd, depth_type, tol, edge_image(image) if depth_type == 1 else None)
        depth, v_depth = D * depth_lambda, vD * depth_lambda
    else:
        depth, v_depth = torch.zeros((), dtype=F64), torch.zeros(H, W, dtype=F64)
    return {"value": depth + (surf + pred), "depth": depth, "surface": surf, "pred": pred, "keep": km["keep"],
            "margin": km["margin"], "v_depth": v_depth, "v_normal": v_normal, "lam": torch.tensor(lam, dtype=F64)}


def find_edges(g: Tensor) -> Tensor:
    """find_edges of a signed [3,H,W] map (reference :40-96, 3-channel branch), in fp64 after the fp32 reciprocal."""
    lap, _ = laplacian_r(g.to(F32))
    return dilate(lap > EDGE_T)


def mean_angular_error(s: Tensor, g: Tensor) -> Tensor:
    """acos of the fp32 dot ((s0 g0 + s1 g1) + s2 g2), clipped, in fp64: near parallel normals the angle is set by the
    dot's fp32 rounding, which is what the reference's map holds."""
    s, g = s.to(F32), g.to(F32)
    dot = (s[0] * g[0] + s[1] * g[1]) + s[2] * g[2]
    return torch.arccos(dot.to(F64).clamp(-1.0, 1.0))


def normal_loss_signed(step: int, s: Tensor, g: Tensor, n: Tensor, normal_lambda: float = 0.1,
                       normal_mask_steps: int = 15000) -> Tensor:
    """get_normal_loss on signed [3,H,W] maps (the strategy's own inputs), fp64."""
    lam = normal_lambda if step > 7000 else 0.0
    km = keep_mask(s.to(F32), g.to(F32), angle=not step < normal_mask_steps)
    surf = (s.to(F64) - g.to(F64)).abs()[km["keep"]].mean() * lam
    return surf + (n.to(F64) - g.to(F64)).abs().mean() * lam


def depth_loss_signed(step: int, pd: Tensor, gd: Tensor, conf: Tensor, img: Tensor, depth_type: int = 1,
                      depth_lambda: float = 0.2, tol: float = 0.1) -> Tensor:
    """get_depth_loss on the strategy's own inputs ([H,W,1] maps, a gate map, fp32 edge image), fp64."""
    H, W = pd.shape[:2]
    g = gd.to(F32).reshape(H, W)
    if step >= 7000:
        g = torch.where(conf.to(F32).reshape(H, W) > 0, g, torch.zeros_like(g))
    D, _ = depth_sums(pd.reshape(H, W), g, depth_type, tol, img.to(F32) if depth_type == 1 else None)
    return D * depth_lambda
