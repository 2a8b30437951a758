"""Render metrics: a drop-in for dn_splatter/metrics.py's `mean_angular_error`, `RGBMetrics`, `DepthMetrics` and
`NormalMetrics`, used by DNSplatterModel.get_metrics_dict / get_image_metrics_and_images and the pipeline's eval average.

Every class takes the reference's [B,C,H,W] arguments and returns the reference's tuple of 0-d tensors.  CUDA tensors go
to the kernels (csrc/ssim.cu `dnr_rgb_metrics`, csrc/metrics.cu `dnr_depth_metrics` / `dnr_normal_metrics`): the sums
are fp64, and the result comes back to the host in one read per call, so the returned tensors live on the CPU.  A
[B,C,H,W] view of channels-last images (`img.permute(2, 0, 1)[None]`) reaches the kernels without a copy.  CPU tensors
take a plain-torch restatement of the reference code.

Semantics (the reference's, torchmetrics' where it delegates):
  * PSNR is 10 log10(1 / MSE) with the MSE pooled over the whole batch (torchmetrics' PeakSignalNoiseRatio(data_range=
    1.0)); identical images give inf.  SSIM is the mean over images of the mean SSIM over the (H-10)x(W-10) interior
    (StructuralSimilarityIndexMeasure(data_range=1.0, kernel_size=11)).
  * DepthMetrics pools every element with gt > tolerance; an empty mask gives NaN everywhere.  `rmse_log` is the
    reference's `sqrt((log gt - log pred)^2).nanmean()`, i.e. the mean |log gt - log pred|, not a root mean square;
    pred = 0 makes it inf.
  * NormalMetrics averages RMSE and the mean error per image and takes one lower median (torch.median) over all values.
    The vectors are compared as given, without renormalisation.
  * A uint8 target is read as value / 255 (the product u8 * fp32(1/255), as the loss kernels read it).  The reference
    would compare the raw 0..255 values with a [0,1] prediction.
  * LPIPS needs network weights, which this package never fetches: RGBMetrics returns None in its third slot unless a
    callable is passed as `lpips`, which is then called as lpips(pred, gt).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from .losses import ssim as _ssim

INV255 = torch.tensor(1 / 255, dtype=torch.float32)
SSIM_RADIUS = 5


def u8_as_float(t: Tensor) -> Tensor:
    """A uint8 image as the kernels read it: u8 * fp32(1/255), rounded once in fp32; other dtypes as fp32."""
    return t.float() * INV255.to(t.device) if t.dtype == torch.uint8 else t.float()


def tf_resize(img: Tensor, size: Sequence[int]) -> Tensor:
    """torchvision.transforms.functional.resize(img, size, antialias=None) of a [..., H, W] tensor: bilinear,
    align_corners=False, no antialiasing, computed in float32 (float64 kept) and rounded back for integer dtypes."""
    size = [int(s) for s in size]
    if list(img.shape[-2:]) == size:
        return img
    squeeze = img.dim() < 4
    x = img[None] if squeeze else img
    out_dtype = x.dtype
    if out_dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float32)
    x = F.interpolate(x, size=size, mode="bilinear", align_corners=False, antialias=False)
    if squeeze:
        x = x[0]
    if out_dtype != x.dtype:
        if not out_dtype.is_floating_point:
            x = torch.round(x)
        x = x.to(out_dtype)
    return x


# ---------------------------------------------------------------------------------------------------------- kernels
def _channels_last(t: Tensor) -> Tensor:
    """[B,C,H,W] -> contiguous [B,H,W,C]; free for a view of channels-last images."""
    return t.permute(0, 2, 3, 1).contiguous()


def _pred_target(pred: Tensor, gt: Tensor):
    if pred.shape != gt.shape or pred.dim() != 4:
        raise ValueError(f"expected two [B,C,H,W] tensors of one shape, got {tuple(pred.shape)} and {tuple(gt.shape)}")
    if gt.device != pred.device:
        raise ValueError(f"pred is on {pred.device}, gt on {gt.device}")
    p = _channels_last(pred.float())
    g = _channels_last(gt if gt.dtype == torch.uint8 else gt.float())
    return p, g, int(gt.dtype == torch.uint8)


def rgb_sums(pred: Tensor, gt: Tensor) -> Tensor:
    """[B,2] float64 on the host: per image the SSIM sum over the interior and the sum of squared errors."""
    from . import _lib as L

    p, g, u8 = _pred_target(pred, gt)
    B, H, W, Cn = p.shape
    out = torch.empty((B, 2), dtype=torch.float64, device=p.device)
    L.check(L.load().dnr_rgb_metrics(p.data_ptr(), g.data_ptr(), u8, B, H, W, Cn, out.data_ptr(), L.stream()),
            "dnr_rgb_metrics")
    return out.cpu()


def depth_sums(pred: Tensor, gt: Tensor, tolerance: float) -> Tensor:
    """[9] float64 on the host: the sums documented at dnr_depth_metrics (include/dnr.h)."""
    from . import _lib as L

    if pred.shape != gt.shape:
        raise ValueError(f"pred {tuple(pred.shape)} and gt {tuple(gt.shape)} differ in shape")
    if gt.device != pred.device:
        raise ValueError(f"pred is on {pred.device}, gt on {gt.device}")
    p, g = pred.float().contiguous(), gt.float().contiguous()
    out = torch.empty(9, dtype=torch.float64, device=p.device)
    L.check(L.load().dnr_depth_metrics(p.data_ptr(), g.data_ptr(), p.numel(), float(tolerance), out.data_ptr(), L.stream()),
            "dnr_depth_metrics")
    return out.cpu()


def normal_sums(pred: Tensor, gt: Tensor) -> Tensor:
    """[3B+1] float64 on the host: per image sum acos, sum (g-p)^2, sum |g-p|, then the median (dnr_normal_metrics)."""
    from . import _lib as L

    p, g, u8 = _pred_target(pred, gt)
    B, H, W, Cn = p.shape
    if Cn != 3:
        raise ValueError(f"normal maps have 3 channels, got {Cn}")
    lib = L.load()
    ws, ws_bytes = L.workspace(lib.dnr_normal_metrics_workspace_bytes, B, H, W, device=p.device)
    out = torch.empty(3 * B + 1, dtype=torch.float64, device=p.device)
    L.check(lib.dnr_normal_metrics(p.data_ptr(), g.data_ptr(), u8, B, H, W, ws.data_ptr(), ws_bytes, out.data_ptr(),
                                   L.stream()), "dnr_normal_metrics")
    return out.cpu()


def rgb_from_sums(s: Tensor, shape) -> Tuple[Tensor, Tensor, Tensor]:
    """(MSE, PSNR, SSIM) in float64 from rgb_sums of [B,C,H,W] images."""
    B, Cn, H, W = shape
    mse = s[:, 1].sum() / (B * Cn * H * W)
    psnr = 10.0 * torch.log10(1.0 / mse)
    ssim = (s[:, 0] / ((H - 2 * SSIM_RADIUS) * (W - 2 * SSIM_RADIUS) * Cn)).mean()
    return mse, psnr, ssim


def depth_from_sums(s: Tensor) -> Tuple[Tensor, ...]:
    """(abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3) in float64 from depth_sums."""
    n = s[0]
    return s[5] / n, s[6] / n, torch.sqrt(s[4] / n), s[7] / s[8], s[1] / n, s[2] / n, s[3] / n


def normal_from_sums(s: Tensor, shape) -> Tuple[Tensor, ...]:
    """(mae, rmse, mean_err, med_err) in float64 from normal_sums of [B,3,H,W] maps."""
    B, Cn, H, W = shape
    per = s[:3 * B].view(B, 3)
    mae = per[:, 0].sum() / (B * H * W)
    rmse = torch.sqrt(per[:, 1] / (Cn * H * W)).mean()
    mean_err = (per[:, 2] / (Cn * H * W)).mean()
    return mae, rmse, mean_err, s[3 * B]


def _f32(values) -> Tuple[Tensor, ...]:
    return tuple(v.to(torch.float32) for v in values)


# ---------------------------------------------------------------------------------------------------------- public
def mean_angular_error(pred: Tensor, gt: Tensor) -> Tensor:
    """[B,H,W] angle (radians) between [B,C,H,W] predicted and reference normals: acos of the clamped dot product."""
    dot_products = torch.sum(gt * pred, dim=1)
    dot_products = torch.clamp(dot_products, -1.0, 1.0)
    return torch.acos(dot_products)


def rgb_metrics(pred: Tensor, gt: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """(MSE, PSNR, SSIM) of [B,C,H,W] images as 0-d float32 tensors, from one kernel pass on CUDA tensors."""
    if pred.is_cuda:
        return _f32(rgb_from_sums(rgb_sums(pred, gt), pred.shape))
    return rgb_torch(pred, gt)


def rgb_torch(pred: Tensor, gt: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """The plain-torch (MSE, PSNR, SSIM) on any device: the CPU route."""
    pred, gt = pred.float(), u8_as_float(gt)
    if min(pred.shape[-2:]) <= 2 * SSIM_RADIUS:
        raise ValueError(f"SSIM with an 11x11 window needs H, W >= 11, got {tuple(pred.shape[-2:])}")
    mse = torch.mean((pred - gt) ** 2)
    psnr = 10.0 * torch.log10(1.0 / mse)
    return mse, psnr, _ssim(pred, gt)


class RGBMetrics(nn.Module):
    """(PSNR, SSIM, LPIPS) of predicted and ground truth [B,C,H,W] images; LPIPS is `lpips(pred, gt)` when a callable
    was given, else None (the weights are never fetched here)."""

    def __init__(self, lpips: Optional[Callable[[Tensor, Tensor], Tensor]] = None, **kwargs):
        super().__init__()
        self.lpips = lpips

    @torch.no_grad()
    def forward(self, pred: Tensor, gt: Tensor):
        _, psnr, ssim = rgb_metrics(pred, gt)
        lpips = self.lpips(pred, gt) if callable(self.lpips) else None
        return psnr, ssim, lpips


class DepthMetrics(nn.Module):
    """(abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3) of predicted and ground truth depths (https://arxiv.org/abs/1806.01260)
    over the elements with gt > tolerance, pooled over the batch.  rmse_log is the mean |log gt - log pred| over the
    terms that are not NaN (the reference's sqrt-then-nanmean), not a root mean square."""

    def __init__(self, tolerance: float = 0.1, **kwargs):
        super().__init__()
        self.tolerance = tolerance

    @torch.no_grad()
    def forward(self, pred: Tensor, gt: Tensor):
        if pred.is_cuda:
            return _f32(depth_from_sums(depth_sums(pred, gt, self.tolerance)))
        return depth_torch(pred, gt, self.tolerance)


def depth_torch(pred: Tensor, gt: Tensor, tolerance: float = 0.1) -> Tuple[Tensor, ...]:
    """DepthMetrics in plain torch on any device (the reference's code): the CPU route."""
    mask = gt > tolerance
    thresh = torch.max((gt[mask] / pred[mask]), (pred[mask] / gt[mask]))
    a1 = (thresh < 1.25).float().mean()
    a2 = (thresh < 1.25**2).float().mean()
    a3 = (thresh < 1.25**3).float().mean()
    rmse = torch.sqrt(((gt[mask] - pred[mask]) ** 2).mean())
    rmse_log = torch.sqrt((torch.log(gt[mask]) - torch.log(pred[mask])) ** 2).nanmean()
    abs_rel = (torch.abs(gt - pred)[mask] / gt[mask]).mean()
    sq_rel = ((gt - pred)[mask] ** 2 / gt[mask]).mean()
    return abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3


class NormalMetrics(nn.Module):
    """(mae, rmse, mean, med) of predicted and reference [B,C,H,W] normal maps: mean angular error over all pixels, RMSE
    and mean absolute error averaged per image, and the lower median absolute error over everything."""

    def __init__(self, **kwargs):
        super().__init__()

    @torch.no_grad()
    def forward(self, pred: Tensor, gt: Tensor):
        if pred.is_cuda:
            return _f32(normal_from_sums(normal_sums(pred, gt), pred.shape))
        return normal_torch(pred, gt)


def normal_torch(pred: Tensor, gt: Tensor) -> Tuple[Tensor, ...]:
    """NormalMetrics in plain torch on any device (the reference's code): the CPU route."""
    pred, gt = pred.float(), u8_as_float(gt)
    b, c, _, _ = gt.shape
    mae = mean_angular_error(pred, gt).mean()
    rmse = torch.sqrt(torch.mean(torch.square(gt - pred), dim=[1, 2, 3])).mean()
    mean_err = torch.mean(torch.abs(gt - pred), dim=[1, 2, 3]).mean()
    med_err = torch.median(torch.abs(gt.reshape(b, c, -1) - pred.reshape(b, c, -1))).mean()
    return mae, rmse, mean_err, med_err
