"""GPU tests of the photometric loss kernels (csrc/ssim.cu) against an fp64 reference.

The reference is losses.ssim (torchmetrics semantics: reflect pad, 11x11 Gaussian window with sigma 1.5, crop) and
`(1 - l) mean|x - y| + l (1 - SSIM)`, evaluated in float64 on the CPU; its gradient comes from fp64 autograd.  A uint8
target is read as `u8 * fp32(1/255)`, the product the kernels form.  Every case checks the loss value and, region by
region (interior band, 5-pixel border ring, ragged last tile row / column, whole image), the gradient for several
upstream gradients `v`: a fault confined to the border or to a partial tile is not diluted by the rest of the image.
The model-level tests take the three routes get_loss_dict has into these kernels: FusedPhotometric with an fp32
image, FusedSSIM with a mask (upstream gradient -ssim_lambda), and FusedPhotometric under a scaled backward."""
import ctypes as C

import pytest
import torch

from tests.helpers import oracle_outputs, scene_and_camera

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

INV255 = torch.tensor(1 / 255, dtype=torch.float32)  # ld_gt<true>: __fmul_rn((float)u8, 1.0f / 255.0f)
TILE = 16
VS = (1.0, -0.2, 3.7)  # upstream gradients of the loss
ENTRIES = (("ssim", None), ("photometric", 0.0), ("photometric", 0.2), ("photometric", 1.0))
# Gradient bounds per region: (norm-wise relative error, per-pixel error as a fraction of the region's max |g64|).
# Measured on an H100 80GB HBM3 (400 W limit), the kernels stay below 1.5e-6 and 1.7e-6 on every case held to them.
TOL = (1e-5, 1e-5)
VALUE_ATOL = 1e-6  # up to 128 x 128 (measured: 3.2e-7); the sums are fp32 atomics of per-CTA partials


# ----------------------------------------------------------------------------------------------------- inputs
def _content(kind, H, W, C, u8, seed):
    """(pred [H,W,C] fp32 on the device, target [H,W,C] fp32 or uint8 on the device)."""
    g = torch.Generator().manual_seed(seed)
    rand = lambda: torch.rand(H, W, C, generator=g)  # noqa: E731
    if kind == "noise":
        x, y = rand(), rand()
    elif kind == "correlated":
        x = rand()
        y = 0.6 * x + 0.4 * rand()
    elif kind == "ramp":  # smooth ramps: tiny local variance, every window cancellation-bound
        i = torch.arange(H, dtype=torch.float32)[:, None, None] / H
        j = torch.arange(W, dtype=torch.float32)[None, :, None] / W
        c = torch.arange(C, dtype=torch.float32)[None, None, :] / (4 * C)
        x = (0.3 + 0.4 * i + 0.1 * j + c).expand(H, W, C).contiguous()
        y = (0.25 + 0.45 * i + 0.05 * j + c).expand(H, W, C).contiguous()
    elif kind == "constant":  # 20x20 constant patches: windows inside one patch have sigma = 0
        bi, bj = -(-H // 20), -(-W // 20)
        up = lambda t: t.repeat_interleave(20, 0).repeat_interleave(20, 1)[:H, :W].contiguous()  # noqa: E731
        x = up(torch.rand(bi, bj, C, generator=g))
        y = up(torch.rand(bi, bj, C, generator=g))
    elif kind == "extremes":  # a third of the pixels at 0, a third at 1
        def ext():
            r = rand()
            return torch.where(r < 1 / 3, 0.0, torch.where(r < 2 / 3, 1.0, rand()))
        x, y = ext(), ext()
    elif kind == "equal":
        y = rand()
        x = y.clone()
    else:
        raise ValueError(kind)
    if u8:
        y8 = (y * 255).round().to(torch.uint8)
        if kind == "extremes":
            r = rand()
            y8 = torch.where(r < 1 / 3, 0, torch.where(r < 2 / 3, 255, y8.int())).to(torch.uint8)
        y8 = y8.cuda()
        if kind == "equal":  # built on the device, exactly as the kernel reads the target
            return y8.float() * INV255.cuda(), y8
        return x.cuda(), y8
    return x.cuda(), y.cuda()


def _target_as_read(y):
    """The target as the kernels read it, on the CPU in fp32."""
    y = y.cpu()
    return y.float() * INV255 if y.dtype == torch.uint8 else y


# ----------------------------------------------------------------------------------------------------- reference
def _reference(x, y, dtype=torch.float64):
    """(mean SSIM, its gradient, mean |x - y|, its gradient) w.r.t. x on the CPU in `dtype`."""
    from dn_splatter_b200.losses import ssim

    xr = x.detach().cpu().to(dtype).requires_grad_(True)
    yr = _target_as_read(y).to(dtype)
    s = ssim(yr.permute(2, 0, 1)[None], xr.permute(2, 0, 1)[None])
    (gs,) = torch.autograd.grad(s, xr)
    xr = xr.detach().requires_grad_(True)
    l1 = (xr - yr).abs().mean()
    (gl,) = torch.autograd.grad(l1, xr)  # torch.abs: subgradient 0 where x == y
    return float(s.detach()), gs, float(l1.detach()), gl


def _combine(ref, entry, lam):
    """(value, gradient) of the entry point from the parts `_reference` returns."""
    s, gs, l1, gl = ref
    if entry == "ssim":
        return s, gs
    return (1 - lam) * l1 + lam * (1 - s), (1 - lam) * gl - lam * gs


# ----------------------------------------------------------------------------------------------------- kernels
def _fused(entry, lam, x, y, vs=VS):
    """Value and {v: d(v * value)/dx} through the autograd Functions get_loss_dict uses."""
    from dn_splatter_b200.regularization_strategy import FusedPhotometric, FusedSSIM

    xg = x.detach().clone().requires_grad_(True)
    out = FusedSSIM.apply(xg, y) if entry == "ssim" else FusedPhotometric.apply(xg, y, lam)
    grads = {v: torch.autograd.grad(v * out, xg, retain_graph=True)[0] for v in vs}
    return float(out.detach()), grads


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _abi_fwd(entry, lam, x, y):
    """(out, dmaps) of dnr_ssim_fwd_ex (out: [SSIM sum]) or dnr_photometric_fwd (out: [SSIM sum, L1 sum, main])."""
    from dn_splatter_b200 import _lib as L

    lib = L.load()
    H, W, Cn = x.shape
    dmaps = torch.empty((3, H, W, Cn), dtype=torch.float32, device=x.device)
    u8 = int(y.dtype == torch.uint8)
    if entry == "ssim":
        out = torch.empty(1, dtype=torch.float32, device=x.device)
        L.check(lib.dnr_ssim_fwd_ex(x.data_ptr(), y.data_ptr(), u8, H, W, Cn, dmaps.data_ptr(), out.data_ptr(), _stream()),
                "dnr_ssim_fwd_ex")
    else:
        out = torch.empty(3, dtype=torch.float32, device=x.device)
        L.check(lib.dnr_photometric_fwd(x.data_ptr(), y.data_ptr(), u8, H, W, Cn, float(lam), dmaps.data_ptr(),
                                        out.data_ptr(), _stream()), "dnr_photometric_fwd")
    return out, dmaps


def _abi_bwd(entry, lam, x, y, dmaps, v):
    """Gradient image of dnr_ssim_bwd_ex / dnr_photometric_bwd; `v` None passes a null upstream-gradient pointer."""
    from dn_splatter_b200 import _lib as L

    lib = L.load()
    H, W, Cn = x.shape
    vp = torch.empty_like(x)
    vt = None if v is None else torch.tensor([v], dtype=torch.float32, device=x.device)
    vptr = None if vt is None else vt.data_ptr()
    u8 = int(y.dtype == torch.uint8)
    if entry == "ssim":
        rc = lib.dnr_ssim_bwd_ex(x.data_ptr(), y.data_ptr(), u8, H, W, Cn, dmaps.data_ptr(), vptr, vp.data_ptr(), _stream())
    else:
        rc = lib.dnr_photometric_bwd(x.data_ptr(), y.data_ptr(), u8, H, W, Cn, float(lam), dmaps.data_ptr(), vptr,
                                     vp.data_ptr(), _stream())
    L.check(rc, entry + " backward")
    torch.cuda.synchronize()
    return vp


# ----------------------------------------------------------------------------------------------------- checks
def _regions(H, W):
    """[(name, bool [H,W])]: whole image, interior band, border ring, and the last tile row / column when partial."""
    interior = torch.zeros(H, W, dtype=torch.bool)
    interior[5:H - 5, 5:W - 5] = True
    out = [("all", torch.ones(H, W, dtype=torch.bool)), ("interior", interior), ("border", ~interior)]
    if H % TILE:
        m = torch.zeros(H, W, dtype=torch.bool)
        m[H // TILE * TILE:] = True
        out.append(("last_tile_row", m))
    if W % TILE:
        m = torch.zeros(H, W, dtype=torch.bool)
        m[:, W // TILE * TILE:] = True
        out.append(("last_tile_col", m))
    return out


def _check_value(got, want, atol, what):
    err = abs(got - want)
    assert err <= atol, f"{what}: value {got!r} vs fp64 {want!r} (error {err:.3e} > {atol:.1e})"


def _check_grad(g, g64, tol, what):
    """Per region: ||g - g64|| <= tol[0] ||g64|| and max |g - g64| <= tol[1] max |g64|."""
    g = g.detach().cpu().double()
    for name, m in _regions(*g.shape[:2]):
        d, w = (g - g64)[m], g64[m]
        rel = float(d.norm() / w.norm())
        pix = float(d.abs().max() / w.abs().max())
        assert rel <= tol[0], f"{what} [{name}]: norm-wise relative gradient error {rel:.3e} > {tol[0]:.0e}"
        assert pix <= tol[1], f"{what} [{name}]: per-pixel gradient error {pix:.3e} of max|g64| > {tol[1]:.0e}"


def _check_grad_vs_fp32(g, g64, g32, what):
    """Cancellation-bound content: per region, the kernel's gradient may be no less accurate than torch's own fp32
    evaluation of the same reference, ||g - g64|| <= 2 ||g32 - g64|| + 1e-6 ||g64||."""
    g = g.detach().cpu().double()
    for name, m in _regions(*g.shape[:2]):
        e, e32, n64 = float((g - g64)[m].norm()), float((g32 - g64)[m].norm()), float(g64[m].norm())
        assert e <= 2 * e32 + 1e-6 * n64, \
            f"{what} [{name}]: gradient error {e:.3e} > 2 x fp32 torch's {e32:.3e} + 1e-6 x {n64:.3e}"


def _check_case(x, y, what, entries=ENTRIES, fp32_criterion=False, value_atol=VALUE_ATOL):
    """Value and per-region gradient of every entry point, for every upstream gradient in VS, against fp64.  With
    `fp32_criterion` the value may also be off by twice torch's fp32 error, and the gradient is held to
    _check_grad_vs_fp32 instead of TOL."""
    ref = _reference(x, y)
    ref32 = _reference(x, y, torch.float32) if fp32_criterion else None
    for entry, lam in entries:
        want, g64 = _combine(ref, entry, lam)
        got, grads = _fused(entry, lam, x, y)
        name = f"{what} {entry} lambda={lam}"
        atol = value_atol + (2 * abs(_combine(ref32, entry, lam)[0] - want) if fp32_criterion else 0.0)
        _check_value(got, want, atol, name)
        if entry == "photometric" and lam == 0.0:
            # pure L1: the sign gradient is the reference's up to the fp32 rounding of (1 - l) / (H W C), and exactly
            # zero where pred == target
            for v, g in grads.items():
                torch.testing.assert_close(g.cpu().double(), v * g64, rtol=1e-6, atol=0.0, msg=f"{name} v={v}")
            continue
        for v, g in grads.items():
            if fp32_criterion:
                _check_grad_vs_fp32(g, v * g64, v * _combine(ref32, entry, lam)[1].double(), f"{name} v={v}")
            else:
                _check_grad(g, v * g64, TOL, f"{name} v={v}")


# ----------------------------------------------------------------------------------------------------- kernel cases
SHAPES = [(11, 11), (11, 200), (200, 11), (12, 13), (16, 16), (17, 33), (26, 27), (31, 47), (49, 81), (75, 53), (64, 80)]


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("hw", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_photometric_kernels_match_fp64_at_edge_shapes(hw, u8):
    """11x11 has one interior pixel; 11xW and Hx11 one interior row / column; the rest are ragged in one or both
    directions or exact multiples of the 16-pixel tile.  fp32 targets correlated with pred, uint8 targets noise."""
    H, W = hw
    x, y = _content("noise" if u8 else "correlated", H, W, 3, u8, seed=H * 1000 + W)
    _check_case(x, y, f"{H}x{W}")


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("hw", [(17, 33), (31, 47)], ids=["17x33", "31x47"])
@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 6, 7])
def test_photometric_kernels_match_fp64_for_every_channel_group(C, hw, u8):
    """Channels go to the kernels in groups of three: C = 1..7 runs groups 1, 2, 3, 3+1, 3+2, 3+3, 3+3+1, so every
    compile-time channel count with and without a uint8 target."""
    H, W = hw
    x, y = _content("correlated", H, W, C, u8, seed=C * 7 + H)
    _check_case(x, y, f"{H}x{W}x{C}")


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("hw", [(26, 27), (75, 53)], ids=["26x27", "75x53"])
@pytest.mark.parametrize("kind", ["noise", "correlated", "extremes", "ramp", "constant", "equal"])
def test_photometric_kernels_match_fp64_on_edge_content(kind, hw, u8):
    """Noise, correlated pairs and images with many pixels at exactly 0 and 1 (uint8: 0 and 255) against the fixed
    bounds.  Smooth ramps, constant patches and pred == target are dominated by the fp32 E[x^2] - mu^2 cancellation in
    any fp32 evaluation (torch's own fp32 path is off by up to 1e-3 on the ramps): there the kernel has to be at least
    as accurate as torch's fp32 path of the reference."""
    H, W = hw
    x, y = _content(kind, H, W, 3, u8, seed=len(kind) * 100 + H)
    if kind == "equal":
        # the premise: the kernel sees pred and target as equal (its L1 sum is exactly zero) ...
        out, _ = _abi_fwd("photometric", 0.2, x, y)
        assert float(out[1]) == 0.0, float(out[1])
        # ... so the L1 part of the gradient (all of it at lambda = 0) is exactly zero everywhere, as torch.abs gives
        for v in VS:
            _, grads = _fused("photometric", 0.0, x, y, vs=(v,))
            assert int(torch.count_nonzero(grads[v])) == 0, v
    fp32_criterion = kind in ("ramp", "constant", "equal")
    _check_case(x, y, f"{kind} {H}x{W}", fp32_criterion=fp32_criterion)


def test_photometric_kernels_match_fp64_at_1080p():
    """The bench frame: 1080x1920x3, uint8 target, ~8k CTAs adding into one fp32 sum; both entry points."""
    x, y = _content("correlated", 1080, 1920, 3, True, seed=1080)
    _check_case(x, y, "1080p", entries=(("ssim", None), ("photometric", 0.2)), value_atol=1e-5)  # measured: 1.6e-6


@pytest.mark.parametrize("entry,lam", ENTRIES, ids=["ssim", "photometric0", "photometric0.2", "photometric1"])
def test_null_upstream_gradient_is_one(entry, lam):
    """A null `v` pointer through the C ABI means v = 1: bit-identical to an explicit 1, and equal to fp64."""
    x, y = _content("correlated", 31, 47, 3, True, seed=4)
    _, dmaps = _abi_fwd(entry, lam, x, y)
    g_null = _abi_bwd(entry, lam, x, y, dmaps, None)
    assert torch.equal(g_null, _abi_bwd(entry, lam, x, y, dmaps, 1.0))
    want = _combine(_reference(x, y), entry, lam)[1]
    _check_grad(g_null, want, TOL, f"{entry} lambda={lam} v=null")


@pytest.mark.parametrize("C", [2, 3, 7])
@pytest.mark.parametrize("entry,lam", [("ssim", None), ("photometric", 0.2)], ids=["ssim", "photometric"])
def test_uint8_target_equals_its_fp32_image(entry, lam, C):
    """A uint8 target and the fp32 image u8 * fp32(1/255) are the same input: same derivative maps and gradient bit for
    bit, and the same sums up to the order of the fp32 atomics."""
    x, y8 = _content("correlated", 37, 45, C, True, seed=C)
    yf = y8.float() * INV255.cuda()
    o8, d8 = _abi_fwd(entry, lam, x, y8)
    of, df = _abi_fwd(entry, lam, x, yf)
    assert torch.equal(d8, df)
    torch.testing.assert_close(o8, of, rtol=1e-6, atol=0.0)
    for v in VS:
        assert torch.equal(_abi_bwd(entry, lam, x, y8, d8, v), _abi_bwd(entry, lam, x, yf, df, v)), v
    (va, ga), (vb, gb) = _fused(entry, lam, x, y8), _fused(entry, lam, x, yf)
    assert abs(va - vb) <= 1e-6 * abs(vb), (va, vb)
    for v in VS:
        assert torch.equal(ga[v], gb[v]), v


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
def test_photometric_at_lambda_one_is_minus_ssim(u8):
    """dnr_photometric_bwd at l = 1 runs launch_ssim_bwd with weights (-1, 0): minus dnr_ssim_bwd_ex bit for bit (zeros
    may differ in sign).  Both forwards write the same derivative maps."""
    x, y = _content("correlated", 41, 39, 5, u8, seed=41)
    _, dp = _abi_fwd("photometric", 1.0, x, y)
    _, ds = _abi_fwd("ssim", None, x, y)
    assert torch.equal(dp, ds)
    for v in (None,) + VS:
        assert torch.equal(_abi_bwd("photometric", 1.0, x, y, dp, v), -_abi_bwd("ssim", None, x, y, ds, v)), v


@pytest.mark.parametrize("entry,lam", [("ssim", None), ("photometric", 0.2)], ids=["ssim", "photometric"])
def test_photometric_gradient_is_deterministic(entry, lam):
    """The backward has no atomics: two runs give the same gradient bit for bit.  Only the forward sums are added by
    atomics, so only they may differ, and only in the last bits."""
    x, y = _content("noise", 270, 480, 3, True, seed=9)
    runs = [_fused(entry, lam, x, y) for _ in range(2)]
    assert abs(runs[0][0] - runs[1][0]) <= 1e-6, (runs[0][0], runs[1][0])
    for v in VS:
        assert torch.equal(runs[0][1][v], runs[1][1][v]), v
    (_, d1), (_, d2) = _abi_fwd(entry, lam, x, y), _abi_fwd(entry, lam, x, y)
    assert torch.equal(d1, d2)


# ----------------------------------------------------------------------------------------------------- model routes
def _model_route(hw, ssim_lambda, image, mask=None, scale=1.0):
    """get_loss_dict's main loss and Gaussian-parameter gradients of one view against an fp64 oracle with the
    regularisers off, so that only the photometric term (and the min-scale term every config has) remains.  With a
    mask the oracle follows nerfstudio: gt * mask and pred * mask, L1 mean, then SSIM of the masked pair."""
    from dn_splatter_b200.losses import ssim
    from oracle import dn_ref
    from tests.test_gpu_model import _camera, _model

    H, W = hw
    params, cam = scene_and_camera(500, W, H, view=2)
    # a mask multiplies the normal map (quirk B11) and predict_normals=False leaves that map on the CPU (quirk B13), so
    # the mask route renders normals; with use_normal_loss=False they do not enter the loss either way
    normals = mask is not None
    m = _model(params, ssim_lambda=ssim_lambda, use_depth_loss=False, predict_normals=normals, use_normal_loss=False)
    batch = {"image": image.cuda()}
    if mask is not None:
        batch["mask"] = mask.cuda()
    ld = m.get_loss_dict(m.get_outputs(_camera(cam)), batch)
    (scale * ld["main_loss"]).backward()
    p, ref = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True, predict_normals=normals)
    gt = image.double() / 255.0 if image.dtype == torch.uint8 else image.double()
    pred = ref["rgb"]
    if mask is not None:
        gt, pred = gt * mask.double(), pred * mask.double()
    loss = (1 - ssim_lambda) * (gt - pred).abs().mean()
    loss = loss + ssim_lambda * (1 - ssim(gt.permute(2, 0, 1)[None], pred.permute(2, 0, 1)[None]))
    loss = loss + dn_ref.dn_regularization(ref["depth"], None, ref["normal"], None, p["scales"], None,
                                           depth_loss_type=None, use_normal_loss=False)
    (scale * loss).backward()
    want = float(loss.detach())
    assert abs(float(ld["main_loss"]) - want) <= 2e-4 * max(1.0, abs(want)), (float(ld["main_loss"]), want)
    errs = {k: float((m.gauss_params[k].grad.cpu().double() - p[k].grad).norm() / p[k].grad.norm())
            for k in ("means", "quats", "scales", "opacities", "features_dc", "features_rest")}
    bad = {k: f"{v:.3e}" for k, v in errs.items() if not v <= 1e-3}
    assert not bad, f"relative gradient error above 1e-3: {bad}"


MODEL_SHAPES = [(49, 81), (53, 75)]
MODEL_IDS = ["81x49", "75x53"]


@pytest.mark.parametrize("hw", MODEL_SHAPES, ids=MODEL_IDS)
def test_model_fused_route_with_fp32_image(hw):
    """A datamanager that hands over float images: FusedPhotometric with an fp32 target."""
    H, W = hw
    g = torch.Generator().manual_seed(H + W)
    _model_route(hw, 0.2, torch.rand(H, W, 3, generator=g))


@pytest.mark.parametrize("ssim_lambda", [0.2, 0.8])
@pytest.mark.parametrize("as_bool", [False, True], ids=["float_mask", "bool_mask"])
@pytest.mark.parametrize("hw", MODEL_SHAPES, ids=MODEL_IDS)
def test_model_mask_route(hw, as_bool, ssim_lambda):
    """A batch with a mask takes the unfused L1 and FusedSSIM of the masked pair, whose upstream gradient is -l."""
    H, W = hw
    g = torch.Generator().manual_seed(H * W)
    image = (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8)
    mask = torch.rand(H, W, 1, generator=g) >= 0.2
    _model_route(hw, ssim_lambda, image, mask=mask if as_bool else mask.float())


@pytest.mark.parametrize("hw", MODEL_SHAPES, ids=MODEL_IDS)
def test_model_fused_route_scaled_backward(hw):
    """uint8 image, FusedPhotometric, and a backward from 3.7 x main_loss: the kernel must apply the upstream gradient."""
    H, W = hw
    g = torch.Generator().manual_seed(H - W)
    _model_route(hw, 0.2, (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), scale=3.7)
