"""Depth / normal regularisation strategies with the reference's API
(/root/reference/dn_splatter/regularization_strategy.py): `DNRegularization(...)(pred_depth=, gt_depth=,
pred_normal=, gt_normal=, scales=, gt_img=)` and `AGSMeshRegularization`.

DNRegularization is the hot path: its depth term (EdgeAwareLogL1 / LogL1 / L1 / MSE over the gt>tol mask),
normal L1 + TV and min-scale term are evaluated by fused CUDA kernels (dnr_loss_fwd / dnr_loss_bwd /
dnr_scale_loss_*: one pass over the rendered maps each way instead of ~40 torch kernels and two boolean-mask
gathers with host syncs).  Loss types the kernels do not cover (Pearson, Huber, ...) run through the torch
modules of losses.py.  AGSMeshRegularization's depth and normal terms run in the same way on dnr_ags_loss_fwd /
dnr_ags_loss_bwd, with the step gates passed as flags; its configurations the kernels do not cover keep the torch ops
(step-gated, mask-indexed; SURVEY.md §2.1 #2).  The reference's quirks are reproduced, not fixed (SURVEY Appendix B6-B9).
"""
from __future__ import annotations

import ctypes as C
from abc import abstractmethod
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor

from . import _lib as L
from .losses import DepthLoss, DepthLossType, NormalLoss, NormalLossType
from .rasterize import _timed

_FUSED_DEPTH = {DepthLossType.EdgeAwareLogL1: 1, DepthLossType.LogL1: 2, DepthLossType.L1: 3, DepthLossType.MSE: 4}


def _shared_holder(*tensors):
    """The dn_rasterize holder shared by all the given rendered maps (None if any map is not a direct raster output or
    they come from different renders): only then can a loss hand its backward to dnr_raster_bwd."""
    from .rasterize import raster_holder

    hs = [raster_holder(t) for t in tensors if t is not None]
    if not hs or any(h is None for h in hs) or any(h is not hs[0] for h in hs):
        return None
    return hs[0]


class _FusedDNLoss(torch.autograd.Function):
    """(1+lambda) * depth_term + L1(normal) + TV(normal) on rendered maps; see include/dnr.h dnr_loss_*.

    `gt_normal` may be uint8 (value / 255, as get_gt_img does) and `edge_image` the uint8 photometric image (clamped
    below at 10/255 in the kernel, dn_model.py:633) instead of the fp32 `gt_img`.  With a raster `holder` the backward
    does not write gradient images: it leaves a spec for dnr_raster_bwd, whose prologue evaluates the same formulas
    per pixel (BASELINE north_star: the regularisers are fused into the backward kernel)."""

    @staticmethod
    def forward(ctx, pred_depth, pred_normal, gt_depth, gt_normal, gt_img, depth_type: int, depth_lambda: float,
                depth_tolerance: float, use_normal: bool, holder=None, edge_image=None):
        lib = L.load()
        ref = pred_depth if pred_depth is not None else pred_normal
        if ref.device.type != "cuda":
            raise L.DnrError("DNRegularization: the fused regulariser needs CUDA tensors (no CPU path)")
        if depth_type:
            H, W = pred_depth.shape[0], pred_depth.shape[1]
        else:
            H, W = pred_normal.shape[0], pred_normal.shape[1]
        dev = ref.device

        def prep(t, keep_u8=False):
            if t is None:
                return None
            if keep_u8 and t.dtype == torch.uint8:
                return t.detach().to(device=dev).contiguous()
            return t.detach().to(device=dev, dtype=torch.float32).contiguous()

        pd, pn, gd, gi = prep(pred_depth), prep(pred_normal), prep(gt_depth), prep(gt_img)
        gn = prep(gt_normal, keep_u8=True)
        ei = prep(edge_image, keep_u8=True)
        flags = 0
        if gn is not None and gn.dtype == torch.uint8:
            flags |= L.LOSS_NORMAL_U8
        if ei is not None:
            assert ei.dtype == torch.uint8, "edge_image is the raw uint8 image"
            flags |= L.LOSS_EDGE_FROM_IMAGE | L.LOSS_IMG_U8
        partials = torch.empty(12, dtype=torch.float32, device=dev)
        a = L.DnrArgs()
        a.width, a.height = W, H
        a.depth_loss_type, a.use_normal_loss = int(depth_type), int(bool(use_normal))
        a.depth_lambda, a.depth_tolerance = float(depth_lambda), float(depth_tolerance)
        a.loss_flags = flags
        for k, t in dict(out_depth=pd, out_normal=pn, gt_depth=gd, gt_normal=gn, gt_rgb=gi, gt_image=ei,
                         loss_partials=partials).items():
            setattr(a, k, None if t is None else t.data_ptr())
        L.check(_timed("loss_fwd", lib.dnr_loss_fwd, C.byref(a), L.stream()), "dnr_loss_fwd")
        ctx.keep = (pd, pn, gd, gn, gi, ei, partials)
        ctx.fwd_stream = torch.cuda.current_stream()
        ctx.cfg = (W, H, int(depth_type), int(bool(use_normal)), float(depth_lambda), float(depth_tolerance), flags)
        ctx.shapes = (None if pred_depth is None else pred_depth.shape, None if pred_normal is None else pred_normal.shape)
        ctx.holder = holder
        return partials[11].clone()

    @staticmethod
    def backward(ctx, v):
        with torch.cuda.stream(ctx.fwd_stream):
            return _FusedDNLoss._backward(ctx, v)

    @staticmethod
    def _backward(ctx, v):
        lib = L.load()
        pd, pn, gd, gn, gi, ei, partials = ctx.keep
        W, H, depth_type, use_normal, lam, tol, flags = ctx.cfg
        v = v.detach().to(torch.float32).contiguous()
        none9 = (None,) * 9
        if ctx.holder is not None:
            from .rasterize import zero_token

            ctx.holder.setdefault("deferred", {})["reg"] = dict(
                depth_type=depth_type, use_normal=use_normal, depth_lambda=lam, depth_tolerance=tol, gt_depth=gd,
                gt_normal=gn if use_normal else None, gt_rgb=gi, edge_image=ei, loss_partials=partials, v=v)
            vd = zero_token(pd.view(ctx.shapes[0])) if (depth_type and ctx.needs_input_grad[0]) else None
            vn = zero_token(pn.view(ctx.shapes[1])) if (use_normal and ctx.needs_input_grad[1]) else None
            return (vd, vn) + none9
        a = L.DnrArgs()
        a.width, a.height = W, H
        a.depth_loss_type, a.use_normal_loss, a.depth_lambda, a.depth_tolerance = depth_type, use_normal, lam, tol
        a.loss_flags = flags
        for k, t in dict(out_depth=pd, out_normal=pn, gt_depth=gd, gt_normal=gn, gt_rgb=gi, gt_image=ei,
                         loss_partials=partials, v_loss=v).items():
            setattr(a, k, None if t is None else t.data_ptr())
        vd = torch.empty(ctx.shapes[0], dtype=torch.float32, device=v.device) if (depth_type and ctx.needs_input_grad[0]) else None
        vn = torch.empty(ctx.shapes[1], dtype=torch.float32, device=v.device) if (use_normal and ctx.needs_input_grad[1]) else None
        if vd is not None or vn is not None:
            L.check(lib.dnr_loss_bwd(C.byref(a), None if vd is None else vd.data_ptr(),
                                     None if vn is None else vn.data_ptr(), L.stream()), "dnr_loss_bwd")
        return (vd, vn) + none9


class _FusedAGSLoss(torch.autograd.Function):
    """AGSMeshRegularization's depth + normal terms in one kernel each way (include/dnr.h dnr_ags_loss_*); differentiable
    w.r.t. `pred_depth` and `pred_normal`.  The surface normal is value-only (it comes from detached depth).

    `cfg` = (depth_type, depth_lambda, depth_tolerance, normal_lambda, flags): the step gates arrive already decided as
    flags (DNR_AGS_CONF_GATE, DNR_AGS_ANGLE_MASK) and as normal_lambda (0 while step <= 7000).  The normal maps are
    [H,W,3] in the [0,1] encoding (gt may be uint8) or, with AGS_SIGNED_CHW, fp32 [3,H,W] already signed.  `keep_mask`
    (uint8 [H,W]) receives the surface term's selection when given."""

    @staticmethod
    def forward(ctx, pred_depth, pred_normal, gt_depth, confidence, image, surf_normal, gt_normal, cfg, keep_mask=None):
        lib = L.load()
        depth_type, depth_lambda, tol, lam, flags = cfg
        if pred_normal.device.type != "cuda":
            raise L.DnrError("AGSMeshRegularization: the fused regulariser needs CUDA tensors (no CPU path)")
        dev = pred_normal.device
        chw = bool(flags & L.AGS_SIGNED_CHW)
        H, W = (pred_normal.shape[1], pred_normal.shape[2]) if chw else (pred_normal.shape[0], pred_normal.shape[1])

        def prep(t, n, keep_u8=False):
            if t is None:
                return None
            assert t.numel() == n, f"map of {t.numel()} values where {n} are expected"
            if keep_u8 and t.dtype == torch.uint8:
                return t.detach().to(device=dev).contiguous()
            return t.detach().to(device=dev, dtype=torch.float32).contiguous()

        pn, sn = prep(pred_normal, 3 * H * W), prep(surf_normal, 3 * H * W)
        gn = prep(gt_normal, 3 * H * W, keep_u8=not chw)
        pd = prep(pred_depth, H * W) if depth_type else None
        gd = prep(gt_depth, H * W) if depth_type else None
        conf = prep(confidence, H * W, keep_u8=bool(flags & L.AGS_CONF_RAW)) if depth_type else None
        im = prep(image, 3 * H * W, keep_u8=True) if depth_type == 1 else None
        if gn.dtype == torch.uint8:
            flags |= L.AGS_NORMAL_U8
        if im is not None and im.dtype == torch.uint8:
            flags |= L.AGS_IMG_U8
        if conf is not None and conf.dtype == torch.uint8:
            flags |= L.AGS_CONF_U8
        if not (flags & L.AGS_CONF_GATE):
            conf = None
        partials = torch.empty(16, dtype=torch.float32, device=dev)
        a = L.DnrAgsLoss()
        a.width, a.height, a.depth_loss_type, a.flags = W, H, int(depth_type), int(flags)
        a.depth_lambda, a.depth_tolerance, a.normal_lambda = float(depth_lambda), float(tol), float(lam)
        for k, t in dict(pred_depth=pd, gt_depth=gd, confidence=conf, image=im, surf_normal=sn, gt_normal=gn,
                         pred_normal=pn, partials=partials, keep_mask=keep_mask).items():
            setattr(a, k, None if t is None else t.data_ptr())
        L.check(_timed("ags_loss_fwd", lib.dnr_ags_loss_fwd, C.byref(a), L.stream()), "dnr_ags_loss_fwd")
        ctx.keep = (pd, gd, conf, im, sn, gn, pn, partials)
        ctx.args = a
        ctx.fwd_stream = torch.cuda.current_stream()
        ctx.shapes = (None if pred_depth is None else pred_depth.shape, pred_normal.shape)
        return partials[11].clone()

    @staticmethod
    def backward(ctx, v):
        with torch.cuda.stream(ctx.fwd_stream):
            lib = L.load()
            a = ctx.args
            v = v.detach().to(torch.float32).contiguous()
            a.v_loss = v.data_ptr()
            a.keep_mask = None
            dev = v.device
            vd = torch.empty(ctx.shapes[0], dtype=torch.float32, device=dev) if (a.depth_loss_type and ctx.needs_input_grad[0]) else None
            vn = torch.empty(ctx.shapes[1], dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
            if vd is not None or vn is not None:
                L.check(_timed("ags_loss_bwd", lib.dnr_ags_loss_bwd, C.byref(a), None if vd is None else vd.data_ptr(),
                               None if vn is None else vn.data_ptr(), L.stream()), "dnr_ags_loss_bwd")
            return (vd, vn) + (None,) * 7


class _ScaleLoss(torch.autograd.Function):
    """mean_i min_k exp(scales[i,k]) (reference regularization_strategy.py:195-199)."""

    @staticmethod
    def forward(ctx, scales):
        lib = L.load()
        if scales.device.type != "cuda":
            raise L.DnrError("scale loss: CUDA tensor required (no CPU path)")
        s = scales.detach().float().contiguous()
        out = torch.empty(1, dtype=torch.float32, device=s.device)
        L.check(_timed("scale_loss_fwd", lib.dnr_scale_loss_fwd, s.data_ptr(), s.shape[0], out.data_ptr(), L.stream()),
                "dnr_scale_loss_fwd")
        ctx.s = s
        ctx.fwd_stream = torch.cuda.current_stream()
        return out[0].clone()

    @staticmethod
    def backward(ctx, v):
        with torch.cuda.stream(ctx.fwd_stream):
            return _ScaleLoss._backward(ctx, v)

    @staticmethod
    def _backward(ctx, v):
        lib = L.load()
        s = ctx.s
        v = v.detach().float().contiguous()
        g = torch.empty_like(s)
        L.check(_timed("scale_loss_bwd", lib.dnr_scale_loss_bwd, s.data_ptr(), s.shape[0], v.data_ptr(), g.data_ptr(),
                       L.stream()), "dnr_scale_loss_bwd")
        return g


class FusedL1(torch.autograd.Function):
    """mean |pred - gt| with gt fp32 or uint8 (/255): the parent SplatfactoModel's photometric L1 in one pass each way.
    With a raster `holder` (pred is a direct dn_rasterize output) the backward is evaluated inside dnr_raster_bwd."""

    @staticmethod
    def forward(ctx, pred, gt, holder=None):
        lib = L.load()
        if pred.device.type != "cuda" or gt.device != pred.device:
            raise L.DnrError("FusedL1 needs CUDA tensors on one device (no CPU path)")
        p = pred.detach().float().contiguous()
        g = gt.detach().contiguous()
        if g.dtype != torch.uint8:
            g = g.float()
        assert g.numel() == p.numel(), "pred / gt size mismatch"
        out = torch.empty(1, dtype=torch.float32, device=p.device)
        L.check(lib.dnr_l1_fwd(p.data_ptr(), g.data_ptr(), p.numel(), int(g.dtype == torch.uint8), out.data_ptr(), L.stream()),
                "dnr_l1_fwd")
        ctx.keep = (p, g)
        ctx.shape = pred.shape
        ctx.fwd_stream = torch.cuda.current_stream()
        ctx.holder = holder
        return out[0].clone()

    @staticmethod
    def backward(ctx, v):
        with torch.cuda.stream(ctx.fwd_stream):
            return FusedL1._backward(ctx, v)

    @staticmethod
    def _backward(ctx, v):
        lib = L.load()
        p, g = ctx.keep
        v = v.detach().float().contiguous()
        if ctx.holder is not None:
            from .rasterize import zero_token

            ctx.holder.setdefault("deferred", {})["l1"] = dict(gt=g, v=v)
            return zero_token(p.view(ctx.shape)), None, None
        vp = torch.empty_like(p)
        L.check(lib.dnr_l1_bwd(p.data_ptr(), g.data_ptr(), p.numel(), int(g.dtype == torch.uint8), v.data_ptr(), vp.data_ptr(),
                               L.stream()), "dnr_l1_bwd")
        return vp.view(ctx.shape), None, None


class FusedSSIM(torch.autograd.Function):
    """Mean SSIM of two [H,W,C] CUDA images (torchmetrics semantics, see losses.ssim) in one kernel each way;
    differentiable w.r.t. `pred` only.  `gt` is fp32 or uint8 (read as value / 255, as get_gt_img converts it).  Default
    since round 2 (DNSplatterModelConfig.fused_ssim); losses.ssim() is its reference
    (tests/test_gpu_model.py::test_fused_ssim_matches_torch)."""

    @staticmethod
    def forward(ctx, pred, gt):
        lib = L.load()
        if pred.device.type != "cuda" or gt.device != pred.device:
            raise L.DnrError("FusedSSIM needs CUDA tensors on one device (no CPU path)")
        p = pred.detach().float().contiguous()
        g = gt.detach().contiguous()
        if g.dtype != torch.uint8:
            g = g.float()
        assert p.dim() == 3 and p.shape == g.shape, "pred / gt must both be [H,W,C]"
        H, W, Cn = p.shape
        dmaps = torch.empty((3, H, W, Cn), dtype=torch.float32, device=p.device)
        out = torch.empty(1, dtype=torch.float32, device=p.device)
        L.check(lib.dnr_ssim_fwd_ex(p.data_ptr(), g.data_ptr(), int(g.dtype == torch.uint8), H, W, Cn, dmaps.data_ptr(),
                                    out.data_ptr(), L.stream()), "dnr_ssim_fwd_ex")
        ctx.keep = (p, g, dmaps)
        ctx.fwd_stream = torch.cuda.current_stream()
        return out[0] / float((H - 10) * (W - 10) * Cn)

    @staticmethod
    def backward(ctx, v):
        with torch.cuda.stream(ctx.fwd_stream):
            lib = L.load()
            p, g, dmaps = ctx.keep
            v = v.detach().float().contiguous()
            vp = torch.empty_like(p)
            H, W, Cn = p.shape
            L.check(lib.dnr_ssim_bwd_ex(p.data_ptr(), g.data_ptr(), int(g.dtype == torch.uint8), H, W, Cn, dmaps.data_ptr(),
                                        v.data_ptr(), vp.data_ptr(), L.stream()), "dnr_ssim_bwd_ex")
            return vp, None


class FusedPhotometric(torch.autograd.Function):
    """main = (1 - ssim_lambda) * mean|pred - gt| + ssim_lambda * (1 - mean SSIM(pred, gt)): the parent
    SplatfactoModel's photometric loss (dn_model.py:624-628 -> [EXT]) in one kernel each way — the L1 sum rides on the
    SSIM kernel's loads and its sign gradient is written by the SSIM backward, so `pred` receives ONE gradient image and
    autograd has nothing to accumulate.  `gt`: [H,W,C] fp32 or uint8 (value / 255)."""

    @staticmethod
    def forward(ctx, pred, gt, ssim_lambda: float):
        lib = L.load()
        if pred.device.type != "cuda" or gt.device != pred.device:
            raise L.DnrError("FusedPhotometric needs CUDA tensors on one device (no CPU path)")
        p = pred.detach().float().contiguous()
        g = gt.detach().contiguous()
        if g.dtype != torch.uint8:
            g = g.float()
        assert p.dim() == 3 and p.shape == g.shape, "pred / gt must both be [H,W,C]"
        H, W, Cn = p.shape
        dmaps = torch.empty((3, H, W, Cn), dtype=torch.float32, device=p.device)
        out = torch.empty(3, dtype=torch.float32, device=p.device)
        L.check(_timed("photometric_fwd", lib.dnr_photometric_fwd, p.data_ptr(), g.data_ptr(), int(g.dtype == torch.uint8), H, W,
                       Cn, float(ssim_lambda), dmaps.data_ptr(), out.data_ptr(), L.stream()), "dnr_photometric_fwd")
        ctx.keep = (p, g, dmaps)
        ctx.lam = float(ssim_lambda)
        ctx.fwd_stream = torch.cuda.current_stream()
        return out[2].clone()

    @staticmethod
    def backward(ctx, v):
        with torch.cuda.stream(ctx.fwd_stream):
            lib = L.load()
            p, g, dmaps = ctx.keep
            v = v.detach().float().contiguous()
            vp = torch.empty_like(p)
            H, W, Cn = p.shape
            L.check(_timed("photometric_bwd", lib.dnr_photometric_bwd, p.data_ptr(), g.data_ptr(), int(g.dtype == torch.uint8), H,
                           W, Cn, ctx.lam, dmaps.data_ptr(), v.data_ptr(), vp.data_ptr(), L.stream()), "dnr_photometric_bwd")
            return vp, None, None


def u8_to_float(img: Tensor, divisor: float = 255.0, clamp_min: float = 0.0) -> Tensor:
    """uint8 CUDA image -> fp32 (/divisor, clamped from below) in one kernel (get_gt_img + clamp of the reference)."""
    src = img.contiguous()
    dst = torch.empty(src.shape, dtype=torch.float32, device=src.device)
    L.check(L.load().dnr_u8_to_f32(src.data_ptr(), src.numel(), float(divisor), float(clamp_min), dst.data_ptr(), L.stream()),
            "dnr_u8_to_f32")
    return dst


class RegularizationStrategy(nn.Module):
    """Depth and normal regularization super class (reference :99-118)."""

    def __init__(self, **kwargs):
        super().__init__()
        self.device_indicator_param = nn.Parameter(torch.empty(0))

    @property
    def device(self):
        return self.device_indicator_param.device

    @abstractmethod
    def get_loss(self, **kwargs):
        """Loss"""

    def forward(self, **kwargs):
        return self.get_loss(**kwargs)

    def get_scale_loss(self, scales):
        return _ScaleLoss.apply(scales)


class DNRegularization(RegularizationStrategy):
    """Regularization strategy of DN-Splatter (reference :121-199)."""

    def __init__(self, depth_tolerance: float = 0.1,
                 depth_loss_type: Optional[DepthLossType] = DepthLossType.EdgeAwareLogL1,
                 depth_lambda: float = 0.2, normal_lambda: float = 0.1):
        super().__init__()
        self.depth_tolerance = depth_tolerance
        self.depth_loss_type = depth_loss_type
        self.depth_loss = DepthLoss(self.depth_loss_type)
        self.depth_lambda = depth_lambda
        self.normal_loss_type = NormalLossType.L1
        self.normal_loss = NormalLoss(self.normal_loss_type)
        self.normal_smooth_loss_type = NormalLossType.Smooth
        self.normal_smooth_loss = NormalLoss(self.normal_smooth_loss_type)
        self.normal_lambda = normal_lambda  # unused by the reference too (quirk B7)

    def _fusable(self, with_depth: bool) -> bool:
        return (not with_depth) or self.depth_loss_type in _FUSED_DEPTH

    fuse_backward = True
    """Hand the backward of the fused terms to dnr_raster_bwd when the maps are direct raster outputs; DNSplatterModel sets
    it from DNSplatterModelConfig.fuse_loss_backward (False: dnr_loss_bwd writes gradient images)."""

    def get_loss(self, pred_depth, gt_depth, pred_normal, gt_normal, **kwargs):
        with_depth = self.depth_loss is not None
        with_normal = self.normal_loss is not None
        if self._fusable(with_depth) and (with_depth or with_normal):
            if with_depth and gt_depth is None:
                raise TypeError("use_depth_loss is set but the batch holds no depth (reference: '>' on NoneType)")
            dtype = _FUSED_DEPTH[self.depth_loss_type] if with_depth else 0
            gt_img = kwargs.get("gt_img") if dtype == 1 else None
            edge_image = None
            if dtype == 1 and gt_img is None:
                raise KeyError("gt_img")
            if gt_img is not None and gt_img.dtype == torch.uint8:  # raw image: clamped (10/255) inside the kernels
                gt_img, edge_image = None, gt_img
            pd, pn = (pred_depth if with_depth else None), (pred_normal if with_normal else None)
            holder = _shared_holder(pd, pn) if self.fuse_backward else None
            loss = _FusedDNLoss.apply(pd, pn, gt_depth if with_depth else None, gt_normal if with_normal else None, gt_img,
                                      dtype, self.depth_lambda, self.depth_tolerance, with_normal, holder, edge_image)
        else:
            if gt_normal is not None and gt_normal.dtype == torch.uint8:
                gt_normal = u8_to_float(gt_normal) if gt_normal.is_cuda else gt_normal.float() / 255.0
            if kwargs.get("gt_img") is not None and kwargs["gt_img"].dtype == torch.uint8:
                gi = kwargs["gt_img"]
                kwargs["gt_img"] = u8_to_float(gi, 255.0, 10 / 255.0) if gi.is_cuda else (gi.float() / 255.0).clamp(min=10 / 255.0)
            loss = 0.0
            if with_depth:
                loss = loss + self.get_depth_loss(pred_depth, gt_depth, **kwargs)
            if with_normal:
                loss = loss + self.get_normal_loss(pred_normal, gt_normal, **kwargs)
        return loss + self.get_scale_loss(scales=kwargs["scales"])

    # --- the reference's per-term methods, kept callable (torch path for non-fused depth types) ---
    def get_depth_loss(self, pred_depth, gt_depth, **kwargs):
        valid = gt_depth > self.depth_tolerance
        if self.depth_loss_type in _FUSED_DEPTH:
            gt_img = kwargs.get("gt_img") if self.depth_loss_type == DepthLossType.EdgeAwareLogL1 else None
            return _FusedDNLoss.apply(pred_depth, None, gt_depth, None, gt_img, _FUSED_DEPTH[self.depth_loss_type],
                                      self.depth_lambda, self.depth_tolerance, False)
        if self.depth_loss_type == DepthLossType.PearsonDepth:  # reference :167-176 (global + lambda * local Pearson)
            n_valid = valid.sum()
            glob = (self.depth_loss(pred_depth, gt_depth.float()) * n_valid) / n_valid
            local = (DepthLoss(DepthLossType.LocalPearsonDepthLoss)(pred_depth, gt_depth.float()) * n_valid) / n_valid
            d = glob + self.depth_lambda * local
            return d + self.depth_lambda * d  # quirk B6
        d = self.depth_loss(pred_depth[valid], gt_depth[valid].float())
        return d + self.depth_lambda * d  # quirk B6

    def get_normal_loss(self, pred_normal, gt_normal, **kwargs):
        return _FusedDNLoss.apply(None, pred_normal, None, gt_normal, None, 0, 0.0, self.depth_tolerance, True)


def mean_angular_error(pred: Tensor, gt: Tensor) -> Tensor:
    """[C,H,W] x2 -> [H,W] angle in radians (reference :11-27)."""
    return torch.arccos(torch.clip((gt * pred).sum(0), -1.0, 1.0))


def find_edges(im: Tensor, threshold: float = 0.01, dilation_itr: int = 1) -> Tensor:
    """Edge mask from the Laplacian of 1/(im + 1e-6), dilated by a 3x3 box (reference :40-96).  [C,H,W] -> bool."""
    c = im.shape[0]
    lap = torch.tensor([[0, 1, 0], [1, -4, 1], [0, 1, 0]], dtype=torch.float32, device=im.device)
    lap = lap[None, None].expand(c, 1, 3, 3).contiguous()
    box = torch.ones(c, 1, 3, 3, dtype=torch.float32, device=im.device)
    edges = (F.conv2d((1.0 / (im.float() + 1e-6))[None], lap, padding=1, groups=c) > threshold).float()
    dil = edges
    for _ in range(dilation_itr):
        # single-channel input compounds the dilation; the 3-channel branch of the reference re-dilates `edges`
        dil = F.conv2d(dil if c == 1 else edges, box, padding=1, groups=c)
    return dil[0] > 0.0


class AGSMeshRegularization(RegularizationStrategy):
    """AGS-Mesh filtering strategy (reference :202-327), step-gated.

    With `fused` (the default) and CUDA maps, a fused depth type (EdgeAwareLogL1 / LogL1 / L1 / MSE) and both losses
    configured, the depth and normal terms run in one kernel each way (_FusedAGSLoss) and the scale term in the min-scale
    kernels: no boolean-mask gathers, no host syncs, so a training step that uses it can be captured in a CUDA graph.
    Everything else runs the torch code below, which restates the reference line by line."""

    fused = True

    def __init__(self, depth_tolerance: float = 0.1,
                 depth_loss_type: Optional[DepthLossType] = DepthLossType.EdgeAwareLogL1, depth_lambda: float = 0.2,
                 normal_lambda: float = 0.1, normal_mask_steps: int = 15000, depth_mask_steps: int = 7000):
        super().__init__()
        self.depth_tolerance, self.depth_loss_type = depth_tolerance, depth_loss_type
        self.depth_loss = DepthLoss(self.depth_loss_type)
        self.depth_lambda = depth_lambda
        self.normal_loss_type = NormalLossType.L1
        self.normal_loss = NormalLoss(self.normal_loss_type)
        self.normal_smooth_loss_type = NormalLossType.Smooth
        self.normal_smooth_loss = NormalLoss(self.normal_smooth_loss_type)
        self.normal_lambda = normal_lambda
        self.normal_mask_steps, self.depth_mask_steps = normal_mask_steps, depth_mask_steps
        self.step = 0

    def _fusable(self) -> bool:
        return self.fused and self.depth_loss_type in _FUSED_DEPTH and self.depth_loss is not None and self.normal_loss is not None

    def _gates(self, step: int):
        """(flags, normal lambda) of the step: the confidence gate from 7000 on (hard-coded upstream, not depth_mask_steps),
        the normal terms from 7001 on, the angular mask instead of the edge mask from normal_mask_steps on."""
        flags = (L.AGS_CONF_GATE if step >= 7000 else 0) | (0 if step < self.normal_mask_steps else L.AGS_ANGLE_MASK)
        return flags, (self.normal_lambda if step > 7000 else 0.0)

    def _fused_ok(self, step, pred_depth, gt_depth, surf_normal, gt_normal, pred_normal, confidence_map, gt_img) -> bool:
        maps = (pred_depth, gt_depth, surf_normal, gt_normal, pred_normal)
        if not self._fusable() or any(t is None or not t.is_cuda or t.dtype != torch.float32 for t in maps):
            return False
        if surf_normal.requires_grad or gt_normal.dim() != 3 or gt_normal.shape[0] != 3:
            return False
        if step >= 7000 and (confidence_map is None or not confidence_map.is_cuda or confidence_map.dtype != torch.float32):
            return False
        if self.depth_loss_type == DepthLossType.EdgeAwareLogL1:
            return gt_img is not None and gt_img.is_cuda and gt_img.dtype == torch.float32 and gt_img.shape[-1] == 3
        return True

    def fused_loss(self, step, pred_depth, gt_depth, surf_normal, gt_normal, pred_normal, confidence, image, scales,
                   confidence_raw: bool = False, signed_chw: bool = False, keep_mask=None):
        """get_loss on the fused kernels.  Default layout: `surf_normal`, `gt_normal`, `pred_normal` are [H,W,3] in the
        [0,1] encoding the model holds (gt fp32 or uint8), `image` the uint8 image (clamped at 10/255 by the kernel) or
        the fp32 edge image; `confidence_raw`: `confidence` is the batch's map (uint8 or fp32), gated on
        1 - get_gt_img(c) / 255 > 0.  `signed_chw`: the normals are the signed [3,H,W] maps get_loss receives."""
        flags, lam = self._gates(step)
        if confidence_raw:
            flags |= L.AGS_CONF_RAW
        if signed_chw:
            flags |= L.AGS_SIGNED_CHW
        cfg = (_FUSED_DEPTH[self.depth_loss_type], self.depth_lambda, self.depth_tolerance, lam, flags)
        reg = _FusedAGSLoss.apply(pred_depth, pred_normal, gt_depth, confidence, image, surf_normal, gt_normal, cfg, keep_mask)
        return reg + _ScaleLoss.apply(scales)

    def get_loss(self, step, pred_depth, gt_depth, surf_normal, gt_normal, pred_normal, confidence_map, **kwargs):
        if self._fused_ok(step, pred_depth, gt_depth, surf_normal, gt_normal, pred_normal, confidence_map, kwargs.get("gt_img")):
            return self.fused_loss(step, pred_depth, gt_depth, surf_normal, gt_normal, pred_normal, confidence_map,
                                   kwargs.get("gt_img"), kwargs["scales"], signed_chw=True)
        d = self.get_depth_loss(step=step, pred_depth=pred_depth, gt_depth=gt_depth, confidence_map=confidence_map, **kwargs)
        n = self.get_normal_loss(step, surf_normal, gt_normal, pred_normal)
        return d + n + self.get_scale_loss(scales=kwargs["scales"])

    def get_scale_loss(self, scales):
        """Plain torch (this strategy is the torch-executed one; reference :322-327)."""
        return torch.min(torch.exp(scales), dim=1, keepdim=True)[0].mean()

    def get_depth_loss(self, step, pred_depth, gt_depth, confidence_map, **kwargs):
        if step >= 7000:  # hard-coded in the reference (:275), not depth_mask_steps
            gt_depth = torch.where(confidence_map > 0, gt_depth, torch.zeros_like(gt_depth))
        mask = gt_depth > self.depth_tolerance
        if self.depth_loss_type == DepthLossType.EdgeAwareLogL1:
            return self.depth_loss(pred_depth, gt_depth.float(), kwargs["gt_img"], mask) * self.depth_lambda
        return self.depth_loss(pred_depth[mask], gt_depth[mask]) * self.depth_lambda

    def get_normal_loss(self, step, surf_normal, gt_normal, pred_normal):
        lam = self.normal_lambda if step > 7000 else 0.0
        if step < self.normal_mask_steps:
            keep = ~find_edges(gt_normal)
            l1 = self.normal_loss(surf_normal[keep], gt_normal[keep]) * lam
        else:
            conf = ~(mean_angular_error(surf_normal, gt_normal) > 0.1)
            l1 = self.normal_loss(surf_normal[:, conf], gt_normal[:, conf]) * lam
        return l1 + self.normal_loss(pred_normal, gt_normal) * lam
