"""fp64 restatement of the render metrics (dn_splatter/metrics.py RGBMetrics / DepthMetrics / NormalMetrics, with
torchmetrics' PeakSignalNoiseRatio(data_range=1.0) and StructuralSimilarityIndexMeasure(data_range=1.0, kernel_size=11)).

Inputs are channels-last [B,H,W,C] tensors as the kernels read them.  A uint8 target is u8 * fp32(1/255), rounded once
in fp32.  The per-element values that a decision or a selection rests on are formed in fp32 exactly as csrc/metrics.cu
forms them (no contraction): the depth ratio max(gt/pred, pred/gt), the clamped normal dot (g0 p0 + g1 p1) + g2 p2 and
the |g - p| the median selects.  Everything else is fp64.  tests/golden/make_golden_metrics.py pins these functions to
the reference's own code; only tests may import this module.
"""
from __future__ import annotations

from typing import Dict

import torch
from torch import Tensor

INV255 = torch.tensor(1 / 255, dtype=torch.float32)
F64 = torch.float64


def target_as_read(t: Tensor) -> Tensor:
    t = t.detach().cpu()
    return t.float() * INV255 if t.dtype == torch.uint8 else t.float()


def rgb(pred: Tensor, gt: Tensor) -> Dict[str, Tensor]:
    """PSNR (pooled MSE), MSE and SSIM (mean over images of the interior mean) of [B,H,W,C] images, plus the per-image
    SSIM sums and squared-error sums."""
    from dn_splatter_b200.losses import ssim

    x, y = pred.detach().cpu().float().to(F64), target_as_read(gt).to(F64)
    B, H, W, C = x.shape
    sse = ((x - y) ** 2).sum(dim=(1, 2, 3))
    mse = sse.sum() / x.numel()
    per = torch.stack([ssim(y[b].permute(2, 0, 1)[None], x[b].permute(2, 0, 1)[None]) for b in range(B)])
    return {"mse": mse, "psnr": 10.0 * torch.log10(1.0 / mse), "ssim": per.mean(),
            "ssim_sum": per * ((H - 10) * (W - 10) * C), "sse": sse}


def depth_thresh(pred: Tensor, gt: Tensor) -> Tensor:
    """max(gt/pred, pred/gt) in fp32 (IEEE division), NaN when either ratio is."""
    r0, r1 = gt / pred, pred / gt
    return torch.where(torch.isnan(r0) | torch.isnan(r1), torch.full_like(r0, float("nan")), torch.maximum(r0, r1))


def depth(pred: Tensor, gt: Tensor, tolerance: float = 0.1) -> Dict[str, Tensor]:
    """DepthMetrics pooled over all elements with gt > tolerance (fp32 comparison)."""
    p, g = pred.detach().cpu().float().reshape(-1), gt.detach().cpu().float().reshape(-1)
    m = g > torch.tensor(tolerance, dtype=torch.float32)
    p, g = p[m], g[m]
    t = depth_thresh(p, g)
    n = torch.tensor(float(p.numel()), dtype=F64)
    pd, gd = p.to(F64), g.to(F64)
    d = gd - pd
    lg = (torch.log(gd) - torch.log(pd)).abs()
    ok = ~torch.isnan(lg)
    sums = torch.stack([n, (t < 1.25).sum().to(F64), (t < 1.5625).sum().to(F64), (t < 1.953125).sum().to(F64),
                        (d * d).sum(), (d.abs() / gd).sum(), (d * d / gd).sum(), lg[ok].sum(), ok.sum().to(F64)])
    return {"sums": sums, "abs_rel": sums[5] / n, "sq_rel": sums[6] / n, "rmse": torch.sqrt(sums[4] / n),
            "rmse_log": sums[7] / sums[8], "a1": sums[1] / n, "a2": sums[2] / n, "a3": sums[3] / n}


def normal_abs_err(pred: Tensor, gt: Tensor) -> Tensor:
    """|g - p| in fp32, [B,H,W,3]."""
    return (target_as_read(gt) - pred.detach().cpu().float()).abs()


def normal(pred: Tensor, gt: Tensor) -> Dict[str, Tensor]:
    """NormalMetrics of [B,H,W,3] maps: mae over all pixels, rmse / mean per image then averaged, lower median."""
    p, g = pred.detach().cpu().float(), target_as_read(gt)
    B, H, W, _ = p.shape
    dot = (g[..., 0] * p[..., 0] + g[..., 1] * p[..., 1]) + g[..., 2] * p[..., 2]
    ang = torch.acos(dot.clamp(-1.0, 1.0).to(F64))
    d = g.to(F64) - p.to(F64)
    acos_sum, sq_sum, abs_sum = ang.sum(dim=(1, 2)), (d * d).sum(dim=(1, 2, 3)), d.abs().sum(dim=(1, 2, 3))
    a = normal_abs_err(pred, gt).reshape(-1)
    med = a.sort().values[(a.numel() - 1) // 2]
    return {"acos_sum": acos_sum, "sq_sum": sq_sum, "abs_sum": abs_sum, "mae": acos_sum.sum() / (B * H * W),
            "rmse": torch.sqrt(sq_sum / (3 * H * W)).mean(), "mean_err": (abs_sum / (3 * H * W)).mean(), "med_err": med}
