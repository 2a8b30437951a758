"""GPU tests of the DN-Splatter regulariser kernels against an fp64 reference.

The reference is oracle/dn_ref.py, whose loss code is pinned to the reference's by tests/golden: EdgeAwareLogL1 / LogL1 /
L1 / MSE over `gt > tolerance`, weighted (1 + lambda) (quirk B6), `l1_loss + tv_loss` of the normals and
`exp(scales).min(1).mean()`.  It is evaluated in float64 on the CPU and differentiated by fp64 autograd.  The inputs are
read exactly as the kernels read them: a uint8 normal map or image is `u8 * fp32(1/255)`, the edge image of
EdgeAwareLogL1 is additionally clamped below at fp32(10/255), and the tolerance is compared in fp32.

Covered here:
  * dnr_loss_fwd / dnr_loss_bwd through the C ABI: value and gradient maps, region by region (whole frame, interior,
    1-pixel border ring, last partial 32 x 8 CTA row / column), for every depth type, normal-map dtype, edge source,
    lambda, tolerance and upstream gradient, at degenerate and ragged shapes, on content with exact ties;
  * the same formulas evaluated in dnr_raster_bwd's prologue (the losses' deferred backward), against the same render's
    backward fed the kernel's gradient maps and the fp64 maps, one term at a time;
  * dnr_scale_loss_fwd / bwd with tied minima, dnr_l1_fwd / bwd and dnr_u8_to_f32 at full-frame sizes;
  * dnr_finalize_fwd (depth fill + surface normal) and dnr_normal_from_depth per pixel;
  * every route get_loss_dict has into these kernels, each asserting which backward ran.
"""
import ctypes as C
import math

import pytest
import torch

from tests.helpers import cuda_outputs, oracle_outputs, scene_and_camera

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

F32, F64 = torch.float32, torch.float64
INV255 = torch.tensor(1 / 255, dtype=F32)  # gt_normal_at / edge_weight: __fmul_rn((float)u8, 1.0f / 255.0f)
LO = torch.tensor(10 / 255, dtype=F32)  # edge_weight's clamp of the uint8 image (dn_model.py:633)
VS = (None, 1.0, -0.2, 3.7)  # upstream gradients of the loss; None is a null pointer, which means 1
LAMBDAS = (0.0, 0.2, 0.5)
TOLS = (0.0, 0.1, 2.5)
CTA_W, CTA_H = 32, 8  # image_ops.cu: img_grid
# Gradient maps, per region: |g - g64| <= MAP_RTOL |g64| + MAP_ATOL max|g64| pixel by pixel, and the region's norm-wise
# relative error <= MAP_NORM.  Measured on an H100 80GB HBM3 (700 W limit) over every case: at most 0.1 of the per-pixel
# bound (max |g - g64| = 2.7e-7 max|g64|) and a norm-wise error of 1.7e-7.
MAP_RTOL, MAP_ATOL, MAP_NORM = 2e-6, 1e-6, 1e-6
VALUE_RTOL = 2e-6  # sums of fp32 atomics up to 135 x 240 (measured: 5.0e-7)
VALUE_RTOL_1080P = 1e-5  # 1080p frames, 1M-6M Gaussians, 6.2M-element L1 (measured: 2.8e-6)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from dn_splatter_b200 import _lib as L

    return L, L.load()


def _next(x: float, toward: float) -> float:
    """The fp32 neighbour of fp32 `x` toward `toward`."""
    t = torch.tensor([x], dtype=F32)
    return float(torch.nextafter(t, torch.tensor([toward], dtype=F32)))


# ----------------------------------------------------------------------------------------------------- inputs
def _patches(t, H, W, b):
    return t.repeat_interleave(b, 0).repeat_interleave(b, 1)[:H, :W].contiguous()


def _inputs(kind, H, W, seed):
    """Maps for the loss kernels on the CPU: pd, gd [H,W,1]; pn, gn [H,W,3] fp32; gn8, img8 [H,W,3] uint8; rgb fp32.

    random    gt depth in (0.05, 5.05) (10 % zero), half the residuals 0.5 N(0,1), half 1e-4 N(0,1); random maps
    ties      4-pixel plateaus of normals (30 % background zeros) whose values are uint8 codes, pred == gt normal on a
              third of the pixels (both dtypes), pred depth == gt depth on a quarter, gt depth exactly at fp32(tol) and
              one ulp either side for every tolerance, a plateau image with codes 0..40 (below the 10/255 clamp too)
    last_col / last_row / none   valid gt depth only in the last column / the last row / nowhere
    """
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    n = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    gd = 0.05 + 5 * r(H, W, 1)
    gd[r(H, W, 1) < 0.1] = 0.0
    pd = gd + torch.where(r(H, W, 1) < 0.5, 0.5 * n(H, W, 1), 1e-4 * n(H, W, 1))
    pn, gn = r(H, W, 3), r(H, W, 3)
    gn8 = (r(H, W, 3) * 256).clamp(max=255).to(torch.uint8)
    img8 = (r(H, W, 3) * 256).clamp(max=255).to(torch.uint8)
    rgb = r(H, W, 3)
    if kind == "ties":
        bi, bj = -(-H // 4), -(-W // 4)
        codes = _patches((r(bi, bj, 3) * 256).clamp(max=255).to(torch.uint8), H, W, 4)
        codes[_patches(r(bi, bj, 1) < 0.3, H, W, 4).expand(H, W, 3)] = 0
        pn = codes.float() * INV255
        eq = (r(H, W, 1) < 1 / 3).expand(H, W, 3)
        gn8 = torch.where(eq, codes, gn8)
        gn = torch.where(eq, pn, gn)
        img8 = _patches((r(bi, bj, 3) * 41).to(torch.uint8), H, W, 4)
        rgb = img8.float() * INV255
        flat = torch.arange(H * W).view(H, W, 1)
        special = [v for tol in TOLS for t in [float(torch.tensor(tol, dtype=F32))]
                   for v in (t, _next(t, math.inf), _next(t, -math.inf))]
        for k, v in enumerate(special):  # every 37th pixel from k on: all nine values once the frame has 9 pixels
            gd = torch.where(flat % 37 == k, torch.tensor(v, dtype=F32), gd)
        pd = torch.where(flat % 4 == 3, gd, pd)
    elif kind in ("last_col", "last_row", "none"):
        keep = torch.zeros(H, W, 1, dtype=torch.bool)
        if kind == "last_col":
            keep[:, W - 1] = True
        elif kind == "last_row":
            keep[H - 1] = True
        gd = torch.where(keep, 3 + r(H, W, 1), torch.zeros(()))  # valid under every tolerance
    elif kind != "random":
        raise ValueError(kind)
    return dict(pd=pd.contiguous(), gd=gd.contiguous(), pn=pn.contiguous(), gn=gn.contiguous(), gn8=gn8.contiguous(),
                img8=img8.contiguous(), rgb=rgb.contiguous())


# ----------------------------------------------------------------------------------------------------- reference
def _edge_image(inp, edge_u8):
    return (inp["img8"].float() * INV255).clamp(min=LO) if edge_u8 else inp["rgb"]


def ref_depth(inp, depth_type, tol, edge_u8, dtype=F64):
    """(depth term before the (1 + lambda) weight, its gradient map [H,W,1]) of dn_ref in `dtype`."""
    from oracle import dn_ref

    pd = inp["pd"].to(dtype).requires_grad_(True)
    gd = inp["gd"].to(dtype)
    mask = inp["gd"] > torch.tensor(tol, dtype=F32)  # the kernels compare fp32 gt with fp32 tolerance
    if depth_type == 1:
        d = dn_ref.edge_aware_logl1(pd, gd, _edge_image(inp, edge_u8).to(dtype), mask)
    elif depth_type == 2:
        d = dn_ref.logl1_pp(pd[mask], gd[mask]).mean()
    elif depth_type == 3:
        d = (pd[mask] - gd[mask]).abs().mean()
    elif depth_type == 4:
        d = ((pd[mask] - gd[mask]) ** 2).mean()
    else:
        raise ValueError(depth_type)
    (gr,) = torch.autograd.grad(d, pd)
    return float(d.detach()), gr


def ref_normal(inp, gt_u8, dtype=F64):
    """(L1, TV, gradient map [H,W,3] of L1 + TV) of dn_ref in `dtype`."""
    from oracle import dn_ref

    pn = inp["pn"].to(dtype).requires_grad_(True)
    gn = (inp["gn8"].float() * INV255 if gt_u8 else inp["gn"]).to(dtype)
    l1, tv = dn_ref.l1_loss(pn, gn), dn_ref.tv_loss(pn)
    (gr,) = torch.autograd.grad(l1 + tv, pn)
    return float(l1.detach()), float(tv.detach()), gr


# ----------------------------------------------------------------------------------------------------- kernels
def _abi(dev, depth_type, normal, edge_u8, lam, tol, vs=VS):
    """dnr_loss_fwd then dnr_loss_bwd for every v: (partials [12], {v: (v_depth [H,W] | None, v_normal [H,W,3] | None)}).
    `normal`: None, "f32" or "u8"; the output maps start as NaN, so a pixel the kernel does not write fails."""
    L, lib = _lib()
    H, W = dev["pd"].shape[:2]
    a = L.DnrArgs()
    a.width, a.height = W, H
    a.depth_loss_type, a.use_normal_loss = depth_type, int(normal is not None)
    a.depth_lambda, a.depth_tolerance = lam, tol
    flags = 0
    ptrs = {}
    if depth_type:
        ptrs.update(out_depth=dev["pd"], gt_depth=dev["gd"])
        if depth_type == 1:
            if edge_u8:
                ptrs["gt_image"] = dev["img8"]
                flags |= L.LOSS_EDGE_FROM_IMAGE | L.LOSS_IMG_U8
            else:
                ptrs["gt_rgb"] = dev["rgb"]
    if normal is not None:
        ptrs.update(out_normal=dev["pn"], gt_normal=dev["gn8"] if normal == "u8" else dev["gn"])
        if normal == "u8":
            flags |= L.LOSS_NORMAL_U8
    a.loss_flags = flags
    partials = torch.full((12,), float("nan"), dtype=F32, device="cuda")
    ptrs["loss_partials"] = partials
    for k, t in ptrs.items():
        setattr(a, k, t.data_ptr())
    L.check(lib.dnr_loss_fwd(C.byref(a), _stream()), "dnr_loss_fwd")
    maps = {}
    for v in vs:
        vt = None if v is None else torch.tensor([v], dtype=F32, device="cuda")
        a.v_loss = None if vt is None else vt.data_ptr()
        vd = torch.full((H, W), float("nan"), dtype=F32, device="cuda") if depth_type else None
        vn = torch.full((H, W, 3), float("nan"), dtype=F32, device="cuda") if normal is not None else None
        L.check(lib.dnr_loss_bwd(C.byref(a), None if vd is None else vd.data_ptr(), None if vn is None else vn.data_ptr(),
                                 _stream()), "dnr_loss_bwd")
        maps[v] = (vd, vn)
    torch.cuda.synchronize()
    return partials.cpu(), {v: tuple(None if m is None else m.cpu() for m in mm) for v, mm in maps.items()}


# ----------------------------------------------------------------------------------------------------- checks
def _regions(H, W):
    """[(name, bool [H,W])]: whole frame, interior, 1-pixel border ring, last partial CTA row / column."""
    interior = torch.zeros(H, W, dtype=torch.bool)
    interior[1:H - 1, 1:W - 1] = True
    out = [("all", torch.ones(H, W, dtype=torch.bool)), ("interior", interior), ("border", ~interior)]
    if H % CTA_H:
        m = torch.zeros(H, W, dtype=torch.bool)
        m[H // CTA_H * CTA_H:] = True
        out.append(("last_cta_row", m))
    if W % CTA_W:
        m = torch.zeros(H, W, dtype=torch.bool)
        m[:, W // CTA_W * CTA_W:] = True
        out.append(("last_cta_col", m))
    return [(name, m) for name, m in out if bool(m.any())]  # no interior below 3 x 3


def map_errors(g, g64):
    """{region: (max over pixels of |g - g64| / (MAP_RTOL |g64| + MAP_ATOL max|g64|), norm-wise relative error)}."""
    g, g64 = g.double(), g64.double()
    H, W = g.shape[:2]
    scale = MAP_RTOL * g64.abs() + MAP_ATOL * float(g64.abs().max())
    diff = (g - g64).abs()
    ratio = torch.where(diff == 0, 0.0, torch.where(scale > 0, diff / scale.clamp(min=1e-300), math.inf))
    ratio = torch.nan_to_num(ratio, nan=math.inf)  # a NaN in the kernel's map
    if ratio.dim() == 3:
        ratio = ratio.amax(-1)
    out = {}
    for name, m in _regions(H, W):
        dn, wn = float((g - g64)[m].norm()), float(g64[m].norm())
        out[name] = (float(ratio[m].max()), dn / wn if wn > 0 else (0.0 if dn == 0 else math.inf))
    return out


def _check_map(g, g64, what):
    assert bool(torch.isfinite(g).all()), f"{what}: non-finite gradient at {torch.nonzero(~torch.isfinite(g))[:4].tolist()}"
    for name, (ratio, rel) in map_errors(g, g64).items():
        assert ratio <= 1.0, f"{what} [{name}]: per-pixel error {ratio:.2f} x the bound"
        assert rel <= MAP_NORM, f"{what} [{name}]: norm-wise relative error {rel:.3e} > {MAP_NORM:.0e}"


def value_error(got, want, allow=0.0, rtol=VALUE_RTOL):
    """|got - want| / (rtol |want| + allow); NaN must match NaN (0 when both are, inf when only one is)."""
    if math.isnan(want) or math.isnan(got):
        return 0.0 if (math.isnan(want) and math.isnan(got)) else math.inf
    err = abs(got - want)
    bound = rtol * abs(want) + allow
    return err / bound if bound > 0 else (0.0 if err == 0 else math.inf)


def _check_value(got, want, what, allow=0.0, rtol=VALUE_RTOL):
    e = value_error(got, want, allow, rtol)
    assert e <= 1.0, f"{what}: value {got!r} vs fp64 {want!r} ({e:.2f} x the bound)"


# ----------------------------------------------------------------------------------------------------- kernel cases
def _configs():
    """(depth type, normal map None / "f32" / "u8", uint8 edge image): every depth type with and without normals, both
    normal dtypes, both edge sources for EdgeAwareLogL1."""
    for t in range(5):
        for normal in (None, "f32", "u8"):
            if t == 0 and normal is None:
                continue
            for edge_u8 in ((False, True) if t == 1 else (False,)):
                yield t, normal, edge_u8


def _check_inputs(inp, what, configs, lambdas=LAMBDAS, tols=TOLS, value_rtol=VALUE_RTOL):
    dev = {k: v.cuda() for k, v in inp.items()}
    depth_refs, normal_refs = {}, {}
    for t, normal, edge_u8 in configs:
        for tol in tols:
            if t and (t, tol, edge_u8) not in depth_refs:
                d64, g64 = ref_depth(inp, t, tol, edge_u8)
                # LogL1 types: log(1 + |e|) of tiny residuals loses digits in any fp32 evaluation; the value may be off by
                # twice torch's own fp32 error
                d32 = ref_depth(inp, t, tol, edge_u8, F32)[0] if t in (1, 2) else d64
                depth_refs[(t, tol, edge_u8)] = (d64, d32, g64)
            if normal is not None and normal not in normal_refs:
                normal_refs[normal] = ref_normal(inp, normal == "u8")
            for lam in lambdas:
                name = f"{what} type={t} normal={normal} edge_u8={edge_u8} lambda={lam} tol={tol}"
                part, maps = _abi(dev, t, normal, edge_u8, lam, tol)
                want_d, allow = 0.0, 0.0
                if t:
                    d64, d32, g64 = depth_refs[(t, tol, edge_u8)]
                    want_d = d64 + lam * d64
                    allow = 2 * abs((d32 + lam * d32) - want_d) if not math.isnan(want_d) else 0.0
                    _check_value(float(part[8]), want_d, name + " depth", allow, value_rtol)
                else:
                    assert float(part[8]) == 0.0, name
                l1, tv = 0.0, 0.0
                if normal is not None:
                    l1, tv, gn64 = normal_refs[normal]
                    _check_value(float(part[9]), l1, name + " normal L1", rtol=value_rtol)
                    _check_value(float(part[10]), tv, name + " normal TV", rtol=value_rtol)
                else:
                    assert float(part[9]) == 0.0 and float(part[10]) == 0.0, name
                _check_value(float(part[11]), want_d + (l1 + tv), name + " total", allow, value_rtol)
                for v in VS[1:]:
                    vd, vn = maps[v]
                    if t:
                        _check_map(vd, v * (1 + lam) * g64[..., 0], f"{name} v={v} v_depth")
                    if normal is not None:
                        _check_map(vn, v * gn64, f"{name} v={v} v_normal")
                # a null upstream gradient is 1, bit for bit
                for m_null, m_one in zip(maps[None], maps[1.0]):
                    assert m_null is None or torch.equal(m_null, m_one), name + " v=null"


SHAPES = [(1, 37), (37, 1), (2, 2), (8, 32), (9, 33), (49, 81), (75, 53), (135, 240)]
KINDS = ["random", "ties", "last_col", "last_row", "none"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("hw", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_loss_kernels_match_fp64(hw, kind):
    """dnr_loss_fwd / dnr_loss_bwd against fp64 for depth types 0-4 x normals off / fp32 / uint8 x edge source x lambda x
    tolerance x upstream gradient.  1 x W and H x 1 have an empty TV axis: the value is NaN exactly where torch's mean of
    an empty tensor is, the gradient stays finite.  8 x 32 is one full CTA, 9 x 33 one CTA and a 1-pixel ragged row and
    column.  With no valid depth the depth value is NaN and its gradient zero; with valid depth only in the last column
    (row) EdgeAwareLogL1's x (y) count is zero."""
    H, W = hw
    inp = _inputs(kind, H, W, seed=H * 1000 + W + KINDS.index(kind))
    if kind == "ties" and H * W >= 9:  # the premises: exact ties and gt depth exactly at every fp32 tolerance
        assert bool((inp["pd"] == inp["gd"]).any())
        for tol in TOLS:
            assert bool((inp["gd"] == torch.tensor(tol, dtype=F32)).any()), tol
    _check_inputs(inp, f"{kind} {H}x{W}", list(_configs()))


def test_loss_kernels_match_fp64_at_1080p():
    """The training frame: ~8k CTAs adding into the partial sums."""
    inp = _inputs("random", 1080, 1920, seed=1080)
    configs = [(1, "u8", True), (1, "f32", False), (2, "f32", False), (3, None, False), (4, "u8", False), (0, "u8", False)]
    _check_inputs(inp, "1080p", configs, lambdas=(0.2,), tols=(0.1,), value_rtol=VALUE_RTOL_1080P)


# ----------------------------------------------------------------------------------------------------- raster prologue
RASTER_HW = (53, 75)  # ragged against the 16-pixel raster tile and the 32 x 8 loss CTA
V_ROUTE = -0.2
# Norm-wise, on top of 4 x the atomics' noise floor: the prologue against dnr_loss_bwd's maps (the same fp32 formulas),
# and the fp64 maps rounded to fp32 against dnr_loss_bwd's maps.  One sample of the floor understates the atomics' noise
# (measured on an H100: floor up to 1.0e-6 |g|, differences up to 2.6e-6 |g| and 3.4e-6 |g| respectively); a fault in
# the prologue's edge mask moves these gradients by more than 1e-2 |g|.
ROUTE_REL_KERNEL, ROUTE_REL_FP64 = 1e-5, 1e-5
PARAM_KEYS = ("means", "quats", "scales", "opacities", "features_dc", "features_rest")


def _raster_grads(out, p, outputs, grad_maps):
    gs = torch.autograd.grad(outputs, [p[k] for k in PARAM_KEYS], grad_outputs=grad_maps, retain_graph=True,
                             allow_unused=True)
    res = {k: (torch.zeros_like(p[k]) if g is None else g).detach().clone() for k, g in zip(PARAM_KEYS, gs)}
    res["absgrad"] = out.means2d.absgrad.clone()
    return res


def _depth_target(out, region, seed):
    """gt depth near the render inside `region`, 0 (below every tolerance) outside it."""
    H, W = out.depth.shape[:2]
    g = torch.Generator().manual_seed(seed)
    d = out.depth.detach().cpu() * (1 + 0.2 * torch.randn(H, W, 1, generator=g))
    keep = torch.zeros(H, W, 1, dtype=torch.bool)
    if region == "all":
        keep[:] = torch.rand(H, W, 1, generator=g) >= 0.1
    elif region == "last_col":
        keep[:, W - 1] = True
    elif region == "last_row":
        keep[H - 1] = True
    elif region == "border":
        keep[:] = True
        keep[1:H - 1, 1:W - 1] = False
    return torch.where(keep, d.clamp(min=0.5), torch.zeros(())).contiguous()


TERMS = [("l1", "u8"), ("l1", "f32"), ("normal", "u8"), ("normal", "f32")] + [
    ("depth", (t, edge, region)) for t, edge in ((1, True), (1, False), (2, False), (3, False), (4, False))
    for region in ("all", "last_col", "last_row", "border")]


@pytest.mark.parametrize("term,opt", TERMS, ids=[f"{t}-{o}" if t != "depth" else f"depth{o[0]}-{'u8' if o[1] else 'f32'}-{o[2]}"
                                                 for t, o in TERMS])
def test_raster_prologue_matches_the_gradient_map_route(term, opt):
    """One term at a time on one render (classic, normals on): the backward evaluated in dnr_raster_bwd's prologue (the
    loss Functions given the raster holder) against the same render's backward fed explicit gradient maps, (a) the fp64
    reference maps in fp32 and (b) the maps dnr_loss_bwd / dnr_l1_bwd write.  All go through the same lists and raster
    kernel; only the prologue and the order of float atomics differ, and the bound is set from the atomics' noise floor
    (the map route run twice).  A depth term confined to the last column, last row or border ring is not diluted."""
    from dn_splatter_b200.regularization_strategy import FusedL1, _FusedDNLoss

    H, W = RASTER_HW
    params, cam = scene_and_camera(400, W, H, view=2)
    p, out = cuda_outputs(params, cam, requires_grad=True)
    holder = out.info
    g = torch.Generator().manual_seed(TERMS.index((term, opt)))
    v = torch.tensor(V_ROUTE, device="cuda")
    if term == "l1":
        gt8 = (torch.rand(H, W, 3, generator=g) * 256).clamp(max=255).to(torch.uint8)
        gt = (gt8 if opt == "u8" else gt8.float() * INV255 + 1e-3 * torch.rand(H, W, 3, generator=g)).cuda()
        fused = lambda: FusedL1.apply(out.rgb, gt, holder)  # noqa: E731
        x = out.rgb.detach().clone().requires_grad_(True)
        (kmap,) = torch.autograd.grad(v * FusedL1.apply(x, gt), x)
        gt_read = (gt.cpu().float() * INV255 if gt.dtype == torch.uint8 else gt.cpu()).double()
        xr = out.rgb.detach().cpu().double().requires_grad_(True)
        (rmap,) = torch.autograd.grad(V_ROUTE * (xr - gt_read).abs().mean(), xr)
        outputs, maps_b, maps_a = [out.rgb], [kmap], [rmap.float().cuda()]
    else:
        if term == "normal":
            depth_type, edge_u8, use_normal, gd = 0, False, True, None
        else:
            depth_type, edge_u8, region = opt
            use_normal = False
            gd = _depth_target(out, region, seed=depth_type)
        gn8 = (torch.rand(H, W, 3, generator=g) * 256).clamp(max=255).to(torch.uint8)
        gn = gn8 if opt == "u8" else torch.rand(H, W, 3, generator=g)
        img8 = (torch.rand(H, W, 3, generator=g) * 256).clamp(max=255).to(torch.uint8)
        rgb = torch.rand(H, W, 3, generator=g)
        lam, tol = 0.2, 0.1
        pd_ = out.depth if depth_type else None
        pn_ = out.normal if use_normal else None
        gd_c = None if gd is None else gd.cuda()
        gn_c = gn.cuda() if use_normal else None
        gi = rgb.cuda() if depth_type == 1 and not edge_u8 else None
        ei = img8.cuda() if depth_type == 1 and edge_u8 else None
        fused = lambda: _FusedDNLoss.apply(pd_, pn_, gd_c, gn_c, gi, depth_type, lam, tol, use_normal, holder, ei)  # noqa
        xd = None if pd_ is None else pd_.detach().clone().requires_grad_(True)
        xn = None if pn_ is None else pn_.detach().clone().requires_grad_(True)
        kl = _FusedDNLoss.apply(xd, xn, gd_c, gn_c, gi, depth_type, lam, tol, use_normal, None, ei)
        maps_b = list(torch.autograd.grad(v * kl, [x for x in (xd, xn) if x is not None]))
        inp = dict(pd=out.depth.detach().cpu(), gd=gd, pn=out.normal.detach().cpu(), gn=gn.float() if opt != "u8" else gn,
                   gn8=gn8, img8=img8, rgb=rgb)
        maps_a = []
        if depth_type:
            maps_a.append((V_ROUTE * (1 + lam) * ref_depth(inp, depth_type, tol, edge_u8)[1]).float().cuda())
        if use_normal:
            maps_a.append((V_ROUTE * ref_normal(inp, opt == "u8")[2]).float().cuda())
        outputs = [o for o in (pd_, pn_) if o is not None]
    b1 = _raster_grads(out, p, outputs, maps_b)
    b2 = _raster_grads(out, p, outputs, maps_b)
    ra = _raster_grads(out, p, outputs, maps_a)
    loss = fused()
    gs = torch.autograd.grad(v * loss, [p[k] for k in PARAM_KEYS], retain_graph=True, allow_unused=True)
    assert "deferred" not in holder, "the raster backward did not consume the deferred loss"
    fz = {k: (torch.zeros_like(p[k]) if gg is None else gg) for k, gg in zip(PARAM_KEYS, gs)}
    fz["absgrad"] = out.means2d.absgrad.clone()
    assert float(b1["means"].norm()) > 0, "the term must reach the Gaussians"
    for k, want in b1.items():
        for name, got, rel in (("prologue", fz[k], ROUTE_REL_KERNEL), ("fp64 maps", ra[k], ROUTE_REL_FP64)):
            assert bool(torch.isfinite(got).all()), f"{term} {opt} {name} {k}: non-finite"
            e = route_error(got, want, b2[k], rel)
            assert e <= 1.0, f"{term} {opt} {name} {k}: {e:.2f} x the bound (noise floor x 4 + {rel:.0e} |g|)"


def route_error(got, want, again, rel):
    """||got - want|| / (4 ||again - want|| + rel ||want||): `again` is the map route run a second time, whose difference
    from `want` is the noise of the raster backward's float atomics."""
    err, floor, n = float((got - want).norm()), float((again - want).norm()), float(want.norm())
    bound = 4 * floor + rel * n
    return err / bound if bound > 0 else (0.0 if err == 0 else math.inf)


# ----------------------------------------------------------------------------------------------------- scale loss
def _scales(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        return 2 * torch.randn(n, 3, generator=g) - 3
    if kind == "tie3":  # every Gaussian at initialisation: log(avg_dist).repeat(1, 3)
        return (torch.randn(n, 1, generator=g) - 4).repeat(1, 3).contiguous()
    if kind == "tie2":  # two equal minima at random columns, the third larger
        s = (torch.randn(n, 1, generator=g) - 4).repeat(1, 3)
        col = torch.randint(0, 3, (n,), generator=g)
        s[torch.arange(n), col] += 0.5 + torch.rand(n, generator=g)
        return s.contiguous()
    if kind == "exp_tie":
        # distinct log-scales one ulp apart whose exp rounds to one fp32 value (|s| < 0.1: an ulp of s is under a tenth
        # of an ulp of exp(s)): the smaller log-scale comes after its twin, so torch's first index of the minimal exp is
        # not the argmin of s
        x = 0.2 * (torch.rand(n, generator=g) - 0.5)
        lo = torch.nextafter(x, torch.full_like(x, -1.0))
        big = x + 0.3
        rows = [torch.stack(c, 1) for c in ((x, lo, big), (big, x, lo), (x, big, lo))]
        pick = torch.randint(0, 3, (n,), generator=g)
        return torch.where(pick[:, None] == 0, rows[0], torch.where(pick[:, None] == 1, rows[1], rows[2])).contiguous()
    raise ValueError(kind)


def _scale_abi(s, v):
    L, lib = _lib()
    n = s.shape[0]
    out = torch.full((1,), float("nan"), dtype=F32, device="cuda")
    L.check(lib.dnr_scale_loss_fwd(s.data_ptr(), n, out.data_ptr(), _stream()), "dnr_scale_loss_fwd")
    grads = {}
    for vv in v:
        vt = None if vv is None else torch.tensor([vv], dtype=F32, device="cuda")
        gs = torch.full_like(s, float("nan"))
        L.check(lib.dnr_scale_loss_bwd(s.data_ptr(), n, None if vt is None else vt.data_ptr(), gs.data_ptr(), _stream()),
                "dnr_scale_loss_bwd")
        grads[vv] = gs
    torch.cuda.synchronize()
    return float(out), grads


SCALE_NS = [1, 255, 256, 257, 100_003, 1_000_000, 6_000_000]


@pytest.mark.parametrize("kind", ["random", "tie3", "tie2", "exp_tie"])
@pytest.mark.parametrize("n", SCALE_NS)
def test_scale_loss_matches_fp64_and_torch_tie_index(n, kind):
    """mean_i min_k exp(s_ik): the value against fp64, and a gradient with exactly one non-zero per row, at the index
    torch's `exp(scales).min(1)` reports (the first minimal exp, evaluated on the device as the reference trains), with
    value v exp(s) / n."""
    s = _scales(kind, n, seed=n % 9973 + len(kind))
    sd = s.cuda()
    got, grads = _scale_abi(sd, VS)
    s64 = s.double()
    want = float(torch.exp(s64).min(1)[0].mean())
    _check_value(got, want, f"n={n} {kind}", rtol=VALUE_RTOL if n < 100_000 else VALUE_RTOL_1080P)
    idx = torch.exp(sd).min(1)[1].cpu()
    if kind == "exp_tie" and n >= 255:  # the premise: most rows are fp32 ties whose first index is not the argmin of s
        assert float((idx != s.argmin(1)).float().mean()) > 0.5
    rows = torch.arange(n)
    for v in VS[1:]:
        gv = grads[v].cpu()
        assert bool(((gv != 0).sum(1) == 1).all()), f"n={n} {kind} v={v}: rows without exactly one non-zero"
        assert torch.equal(gv.abs().argmax(1), idx), f"n={n} {kind} v={v}: gradient on another axis than torch's index"
        want_g = v * torch.exp(s64[rows, idx]) / n
        torch.testing.assert_close(gv[rows, idx].double(), want_g, rtol=1e-6, atol=0.0, msg=f"n={n} {kind} v={v}")
    assert torch.equal(grads[None], grads[1.0])


# ----------------------------------------------------------------------------------------------------- L1 / uint8
def _l1_abi(pred, gt, v):
    L, lib = _lib()
    n = pred.numel()
    u8 = int(gt.dtype == torch.uint8)
    out = torch.full((1,), float("nan"), dtype=F32, device="cuda")
    L.check(lib.dnr_l1_fwd(pred.data_ptr(), gt.data_ptr(), n, u8, out.data_ptr(), _stream()), "dnr_l1_fwd")
    vt = None if v is None else torch.tensor([v], dtype=F32, device="cuda")
    vp = torch.full_like(pred, float("nan"))
    L.check(lib.dnr_l1_bwd(pred.data_ptr(), gt.data_ptr(), n, u8, None if vt is None else vt.data_ptr(), vp.data_ptr(),
                           _stream()), "dnr_l1_bwd")
    torch.cuda.synchronize()
    return float(out), vp


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("n", [1, 1023, 1025, 1_000_003, 1080 * 1920 * 3])
def test_l1_kernels_match_fp64(n, u8):
    """dnr_l1_fwd / bwd: grid-stride loops capped at 8 CTAs per SM (~20 strides at 1080p) and sizes that are not a multiple
    of the 1024 elements a CTA covers per stride.  The gradient is sgn(pred - gt) fp32(v / n) bit for bit (0 where
    pred == gt), the value the fp64 mean."""
    g = torch.Generator().manual_seed(n % 1000 + u8)
    gt8 = (torch.rand(n, generator=g) * 256).clamp(max=255).to(torch.uint8)
    gt_read = gt8.float() * INV255 if u8 else torch.rand(n, generator=g)
    pred = torch.where(torch.rand(n, generator=g) < 0.1, gt_read, torch.rand(n, generator=g))
    gt = gt8 if u8 else gt_read
    for v in VS:
        got, vp = _l1_abi(pred.cuda(), gt.cuda(), v)
        want = float((pred.double() - gt_read.double()).abs().mean())
        _check_value(got, want, f"n={n} u8={u8}", rtol=VALUE_RTOL if n < 100_000 else VALUE_RTOL_1080P)
        vf = torch.tensor(1.0 if v is None else v, dtype=F32)
        s = vf / torch.tensor(float(n), dtype=F32)
        assert torch.equal(vp.cpu(), torch.sign(pred - gt_read) * s), f"n={n} u8={u8} v={v}"


@pytest.mark.parametrize("shape", [(256,), (1080, 1920, 3), (1000, 1001)], ids=["codes", "1080p", "1001000"])
def test_u8_to_f32_is_torch_bit_for_bit(shape):
    """dnr_u8_to_f32 is torch's device `x.float() / 255` and its `.clamp(min=10/255)` bit for bit."""
    from dn_splatter_b200.regularization_strategy import u8_to_float

    if shape == (256,):
        x = torch.arange(256, dtype=torch.int32).to(torch.uint8).cuda()
    else:
        g = torch.Generator().manual_seed(sum(shape))
        x = (torch.rand(shape, generator=g) * 256).clamp(max=255).to(torch.uint8).cuda()
    assert torch.equal(u8_to_float(x), x.float() / 255.0)
    assert torch.equal(u8_to_float(x, 255.0, 10 / 255.0), (x.float() / 255.0).clamp(min=10 / 255.0))


# ----------------------------------------------------------------------------------------------------- depth-derived maps
INTR = (71.5, 64.25, 3.25, -2.5)  # fx != fy; principal point offset from the centre by (3.25, -2.5) pixels
SN_ATOL = 3e-5  # per component (measured on an H100: 1.5e-5, next to the factor-2 depth steps of normal_from_depth)


def sn_error(got, want):
    return float((got.double() - want).abs().max())


def _depth_alpha(H, W, kind, seed):
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(H, dtype=F32)[:, None, None]
    j = torch.arange(W, dtype=F32)[None, :, None]
    depth = (2 + 0.02 * i + 0.01 * j + 0.05 * torch.rand(H, W, 1, generator=g)).contiguous()
    alpha = 0.2 + 0.8 * torch.rand(H, W, 1, generator=g)
    if kind == "holes":
        alpha[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
        for y, x in ((0, W // 2), (H - 1, W // 3), (H // 2, 0), (H // 3, W - 1), (1, W // 2), (H - 2, 2), (H // 2, W // 2)):
            if 0 <= y < H and 0 <= x < W:
                alpha[y, x] = 0.0
        depth[alpha == 0] = 123.0  # the stored value at a hole must be ignored by its neighbours
    elif kind == "empty":
        alpha.zero_()
        depth.zero_()
    return depth.contiguous(), alpha.contiguous()


def _intrinsics(H, W):
    fx, fy, dx, dy = INTR
    return fx, fy, W / 2 + dx, H / 2 + dy


def _camera_args(a, L, H, W, host, keep):
    fx, fy, cx, cy = _intrinsics(H, W)
    if host:
        a.flags = L.FLAG_HOST_CAMERA
        a.host_cam[16], a.host_cam[17], a.host_cam[18], a.host_cam[19] = fx, fy, cx, cy
    else:
        K = torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=F32, device="cuda")
        keep.append(K)
        a.K = K.data_ptr()


DA_SHAPES = [(1, 9), (2, 40), (40, 2), (3, 3), (9, 33), (53, 75), (135, 240)]


@pytest.mark.parametrize("host", [False, True], ids=["device_K", "host_camera"])
@pytest.mark.parametrize("kind", ["holes", "empty", "full"])
@pytest.mark.parametrize("hw", DA_SHAPES, ids=[f"{h}x{w}" for h, w in DA_SHAPES])
def test_finalize_fwd_matches_fp64(hw, kind, host):
    """dnr_finalize_fwd: pixels with alpha == 0 take the frame max bit for bit (0 in an empty frame), the others keep their
    depth; the surface normal of the filled depth matches dn_ref.surface_normal_output per pixel, and the 1-pixel border
    (every pixel when H or W < 3) is exactly 0.5."""
    from oracle import dn_ref

    L, lib = _lib()
    H, W = hw
    depth, alpha = _depth_alpha(H, W, kind, seed=H * 7 + W)
    dmax = float(torch.where(alpha > 0, depth, torch.zeros(())).max()) if kind != "empty" else 0.0
    filled = torch.where(alpha > 0, depth, torch.tensor(dmax, dtype=F32))
    d, al = depth.cuda(), alpha.cuda()
    dm = torch.tensor([dmax], dtype=F32).view(torch.int32).cuda()
    sn = torch.full((H, W, 3), float("nan"), dtype=F32, device="cuda")
    a = L.DnrArgs()
    a.width, a.height = W, H
    keep = []
    _camera_args(a, L, H, W, host, keep)
    a.out_depth, a.out_alpha, a.depth_max, a.out_surface_normal = d.data_ptr(), al.data_ptr(), dm.data_ptr(), sn.data_ptr()
    L.check(lib.dnr_finalize_fwd(C.byref(a), _stream()), "dnr_finalize_fwd")
    torch.cuda.synchronize()
    assert torch.equal(d.cpu(), filled)
    fx, fy, cx, cy = _intrinsics(H, W)
    want = dn_ref.surface_normal_output(filled.double(), fx, fy, cx, cy, W, H)
    got = sn.cpu()
    border = torch.ones(H, W, dtype=torch.bool)
    border[1:H - 1, 1:W - 1] = False
    assert bool((got[border] == 0.5).all())
    err = sn_error(got, want)
    assert err <= SN_ATOL, f"surface normal: max error {err:.3e} > {SN_ATOL:.0e}"
    if kind == "empty":
        assert bool((got == 0.5).all())


@pytest.mark.parametrize("host", [False, True], ids=["device_K", "host_camera"])
@pytest.mark.parametrize("hw", DA_SHAPES, ids=[f"{h}x{w}" for h, w in DA_SHAPES])
def test_normal_from_depth_matches_fp64(hw, host):
    """dnr_normal_from_depth (normal_supervision="depth") against dn_ref.normal_from_depth_image per pixel, on a depth map
    with jumps; the border (everything when H or W < 3) is exactly 0."""
    from oracle import dn_ref

    L, lib = _lib()
    H, W = hw
    depth, alpha = _depth_alpha(H, W, "holes", seed=H + W)
    depth = torch.where(alpha > 0, depth, 2 * depth.amin()).contiguous()  # steps of a factor 2 around the holes
    d = depth.cuda()
    out = torch.full((H, W, 3), float("nan"), dtype=F32, device="cuda")
    a = L.DnrArgs()
    a.width, a.height = W, H
    keep = []
    _camera_args(a, L, H, W, host, keep)
    a.out_depth, a.out_surface_normal = d.data_ptr(), out.data_ptr()
    L.check(lib.dnr_normal_from_depth(C.byref(a), _stream()), "dnr_normal_from_depth")
    torch.cuda.synchronize()
    fx, fy, cx, cy = _intrinsics(H, W)
    want = dn_ref.normal_from_depth_image(depth.double(), fx, fy, cx, cy, W, H)
    got = out.cpu()
    border = torch.ones(H, W, dtype=torch.bool)
    border[1:H - 1, 1:W - 1] = False
    assert bool((got[border] == 0.0).all())
    err = sn_error(got, want)
    assert err <= SN_ATOL, f"normal from depth: max error {err:.3e} > {SN_ATOL:.0e}"


# ----------------------------------------------------------------------------------------------------- model routes
ROUTES = {
    # name: (config, batch transform, dnr_loss_bwd calls, reg deferred into raster_bwd)
    "default": (dict(), None, 0, True),
    "unfused": (dict(fuse_loss_backward=False), None, 1, False),
    "host_batch": (dict(), "host", 0, True),
    "mask": (dict(), "mask", 1, False),
    "antialiased": (dict(rasterize_mode="antialiased"), None, 1, False),
    "normal_from_depth": (dict(normal_supervision="depth"), None, 0, True),
    "depth_only": (dict(use_normal_loss=False), None, 0, True),
    "normals_only": (dict(use_depth_loss=False), None, 0, True),
    "sensor_depth": (dict(), "sensor", 0, True),
}


def _count_calls(monkeypatch, lib, name, record):
    orig = getattr(lib, name)

    def call(*args):
        record(args)
        return orig(*args)

    monkeypatch.setitem(lib.__dict__, name, call)


def _route_oracle(params, cam, batch, cfg, depth_key, mask):
    """get_loss_dict's main loss for the route in fp64 (ssim_lambda = 0): the photometric L1 (of gt * mask and pred * mask
    with a mask, nerfstudio's semantics) plus DNRegularization of the (masked) maps, the min-scale term included."""
    from oracle import dn_ref

    rmode = cfg.get("rasterize_mode", "classic")
    p, ref = oracle_outputs(params, cam, dtype=F64, requires_grad=True, rasterize_mode=rmode, predict_normals=True)
    gt_img = batch["image"].double() / 255.0
    rgb, gt = ref["rgb"], gt_img
    depth, normal = ref["depth"], ref["normal"]
    gdepth = batch[depth_key].double() if depth_key else None
    if cfg.get("normal_supervision") == "depth":
        gnormal = None
    else:
        gnormal = batch["normal"].double() / 255.0
    if mask is not None:
        m = mask.double()
        rgb, gt = rgb * m, gt * m
        depth, normal, gnormal = depth * m, normal * m, gnormal * m
        gdepth = gdepth * m
    if gnormal is None:  # dn_model.py:669-686: normals of the detached rendered depth, mapped to [0, 1]
        gnormal = dn_ref.surface_normal_output(depth.detach(), cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["width"],
                                               cam["height"])
    loss = (gt - rgb).abs().mean()
    use_depth, use_normal = cfg.get("use_depth_loss", True), cfg.get("use_normal_loss", True)
    loss = loss + dn_ref.dn_regularization(depth, gdepth, normal, gnormal, p["scales"], gt_img.clamp(min=10 / 255.0),
                                           depth_lambda=0.2, depth_loss_type="EdgeAwareLogL1" if use_depth else None,
                                           use_normal_loss=use_normal)
    loss.backward()
    return float(loss.detach()), p


@pytest.mark.parametrize("route", list(ROUTES))
def test_model_route_matches_fp64_and_runs_the_backward_it_claims(route, monkeypatch):
    """Each route get_loss_dict has into the regulariser: the main loss and Gaussian-parameter gradients against the fp64
    oracle, and the backward that actually ran: dnr_loss_bwd writing gradient images, or the loss specs deferred into
    dnr_raster_bwd's prologue (and consumed there)."""
    from dn_splatter_b200.losses import DepthLossType
    from tests.test_gpu_model import _camera, _model

    cfg, transform, want_loss_bwd, want_deferred = ROUTES[route]
    H, W = 49, 81
    params, cam = scene_and_camera(500, W, H, view=2)
    g = torch.Generator().manual_seed(len(route))
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    depth[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
    depth_key = "sensor_depth" if transform == "sensor" else "mono_depth"
    raw = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), depth_key: depth,
           "normal": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8)}
    mask = None
    if transform == "mask":
        mask = torch.rand(H, W, 1, generator=g) >= 0.2
        raw["mask"] = mask
    kw = dict(use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType.EdgeAwareLogL1, ssim_lambda=0.0,
              predict_normals=True)
    kw.update(cfg)
    L, lib = _lib()
    loss_bwd, raster_bwd = [], []
    _count_calls(monkeypatch, lib, "dnr_loss_bwd", loss_bwd.append)
    _count_calls(monkeypatch, lib, "dnr_raster_bwd", lambda args: raster_bwd.append(
        (args[0]._obj.loss_flags, args[0]._obj.depth_loss_type, args[0]._obj.use_normal_loss)))
    m = _model(params, **kw)
    batch = {k: (v if transform == "host" else v.cuda()) for k, v in raw.items()}
    out = m.get_outputs(_camera(cam))
    ld = m.get_loss_dict(out, batch)
    ld["main_loss"].backward()
    torch.cuda.synchronize()
    assert "deferred" not in m.raster_out.info, "a deferred loss was left undelivered"
    assert len(loss_bwd) == want_loss_bwd, (route, len(loss_bwd))
    reg = [r for r in raster_bwd if r[1] or r[2]]
    if want_deferred:
        want_type = 1 if kw["use_depth_loss"] else 0
        assert len(reg) == 1 and reg[0][1:] == (want_type, int(kw.get("use_normal_loss", True))), (route, raster_bwd)
        assert reg[0][0] & L.LOSS_FUSED_BWD
        u8_maps = transform != "host"
        assert bool(reg[0][0] & L.LOSS_EDGE_FROM_IMAGE) == (u8_maps and want_type == 1), (route, reg)
        normal_u8 = u8_maps and kw.get("normal_supervision", "mono") == "mono" and kw.get("use_normal_loss", True)
        assert bool(reg[0][0] & L.LOSS_NORMAL_U8) == normal_u8, (route, reg)
    else:
        assert not reg, (route, raster_bwd)
    want, p = _route_oracle(params, cam, raw, kw, depth_key if kw["use_depth_loss"] else None, mask)
    got = float(ld["main_loss"])
    assert abs(got - want) <= 2e-4 * max(1.0, abs(want)), (got, want)
    errs = {k: float((m.gauss_params[k].grad.cpu().double() - p[k].grad).norm() / p[k].grad.norm()) for k in PARAM_KEYS}
    bad = {k: f"{v:.3e}" for k, v in errs.items() if not v <= 1e-3}
    assert not bad, f"relative gradient error above 1e-3: {bad}"
