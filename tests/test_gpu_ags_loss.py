"""GPU tests of the fused AGS-Mesh regulariser (csrc/ags_loss.cu) against the fp64 oracle (oracle/ags_ref.py), against
the torch path on the same CUDA inputs, and through the model, the captured training step and the Trainer.

Rules (through the C ABI):
  * keep mask: equal to the oracle's on every element outside the decision band (Laplacian margin within EDGE_BAND of
    the sum of |terms|, angle within ANGLE_BAND of 0.1); an in-band element may take either outcome, and the count of
    in-band elements is printed;
  * value: within VALUE_RTOL of the fp64 value evaluated with the kernel's own mask (NaN exactly where the oracle's
    selection or depth mask is empty);
  * v_depth: per pixel |g - g64| <= MAP_RTOL |g64| + MAP_ATOL max|g64| and norm-wise <= MAP_NORM (the rule of
    test_gpu_regularizer.py); v_normal: within 1 ulp of sgn(d) * fp32((v * lam * 2) / (3HW)).
"""
import ctypes as C
import math

import pytest
import torch

from oracle import ags_ref
from tests.ags_cases import STEPS, TOL, make_case

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

F32, F64 = torch.float32, torch.float64
MAP_RTOL, MAP_ATOL, MAP_NORM = 2e-6, 1e-6, 1e-6
VALUE_RTOL, VALUE_RTOL_1080P = 2e-6, 1e-5
EDGE_BAND = 2e-6  # relative to sum |terms|: 5 fp32 additions of the Laplacian
ANGLE_BAND = 2e-5  # radians: an fp32 dot of unit vectors near 0.1 rad, through acosf
LAMBDA, NORMAL_LAMBDA = 0.2, 0.1
VS = (None, 1.0, -0.2, 3.7)
SHAPES = [(1, 1), (1, 5), (2, 3), (3, 2), (3, 40), (2, 33), (81, 49), (135, 240)]
DTYPES = [(False, False, True), (True, True, True), (True, False, False), (False, True, False)]  # normal, conf, img u8


def _lib():
    from dn_splatter_b200 import _lib as L

    return L, L.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _kernel(case, step, depth_type, v, normal_mask_steps=15000):
    """dnr_ags_loss_fwd / bwd through the C ABI on the [0,1] maps with the raw confidence map."""
    L, lib = _lib()
    d = {k: t.cuda().contiguous() for k, t in case.items()}
    H, W = d["pn"].shape[:2]
    flags = L.AGS_CONF_RAW
    flags |= L.AGS_CONF_GATE if step >= 7000 else 0
    flags |= 0 if step < normal_mask_steps else L.AGS_ANGLE_MASK
    flags |= L.AGS_NORMAL_U8 if d["gn"].dtype == torch.uint8 else 0
    flags |= L.AGS_CONF_U8 if d["conf"].dtype == torch.uint8 else 0
    flags |= L.AGS_IMG_U8 if d["img"].dtype == torch.uint8 else 0
    partials = torch.empty(16, device="cuda")
    keep = torch.full((H, W), 255, dtype=torch.uint8, device="cuda")
    vt = None if v is None else torch.tensor([v], dtype=F32, device="cuda")
    a = L.DnrAgsLoss()
    a.width, a.height, a.depth_loss_type, a.flags = W, H, depth_type, flags
    a.depth_lambda, a.depth_tolerance, a.normal_lambda = LAMBDA, TOL, (NORMAL_LAMBDA if step > 7000 else 0.0)
    for k, t in dict(pred_depth=d["pd"], gt_depth=d["gd"], confidence=d["conf"], image=d["img"], surf_normal=d["sn"],
                     gt_normal=d["gn"], pred_normal=d["pn"], partials=partials, keep_mask=keep, v_loss=vt).items():
        setattr(a, k, None if t is None else t.data_ptr())
    L.check(lib.dnr_ags_loss_fwd(C.byref(a), _stream()), "dnr_ags_loss_fwd")
    vd = torch.empty(H, W, device="cuda")
    vn = torch.empty(H, W, 3, device="cuda")
    L.check(lib.dnr_ags_loss_bwd(C.byref(a), vd.data_ptr(), vn.data_ptr(), _stream()), "dnr_ags_loss_bwd")
    torch.cuda.synchronize()
    bits = keep.cpu().to(torch.int64)
    kmask = torch.stack([(bits >> c) & 1 for c in range(3)]).bool()
    assert int(bits.max()) <= 7
    return dict(value=float(partials[11]), partials=partials.cpu(), keep=kmask, vd=vd.cpu(), vn=vn.cpu())


def _map_ok(g, ref, what):
    ref = ref.to(F64)
    g = g.to(F64).reshape(ref.shape)
    scale = float(ref.abs().max()) if ref.numel() else 0.0
    err = (g - ref).abs()
    bound = MAP_RTOL * ref.abs() + MAP_ATOL * scale
    assert bool((err <= bound).all()), (what, float((err - bound).max()), scale)
    if scale > 0:
        assert float(err.norm() / ref.norm()) <= MAP_NORM, (what, float(err.norm() / ref.norm()))


def _check(case, step, depth_type, v, value_rtol=VALUE_RTOL):
    k = _kernel(case, step, depth_type, v)
    H, W = case["pn"].shape[:2]
    ref = ags_ref.ags_loss(case["pd"], case["gd"], case["conf"], case["img"], case["sn"], case["gn"], case["pn"],
                           depth_type=depth_type, depth_lambda=LAMBDA, tol=TOL, normal_lambda=NORMAL_LAMBDA, step=step)
    # keep mask: the oracle's outside the decision band
    if step < 15000:
        lap_margin = ags_ref.laplacian_r(ags_ref.signed(case["gn"]))
        near = ((lap_margin[0] - ags_ref.EDGE_T).abs() <= EDGE_BAND * lap_margin[1])
        band = ags_ref.dilate(near)  # a pixel whose dilation window holds an in-band Laplacian
    else:
        band = (ref["margin"].abs() <= ANGLE_BAND)[None].expand(3, -1, -1)
    n_band = int(band.sum())
    mism = (k["keep"] != ref["keep"]) & ~band
    print(f"[ags] {H}x{W} step {step} type {depth_type}: {n_band} in-band elements, {int((k['keep'] != ref['keep']).sum())} differ")
    assert not bool(mism.any()), (int(mism.sum()), "keep-mask elements differ outside the band")
    # value at the kernel's own mask
    own = ags_ref.ags_loss(case["pd"], case["gd"], case["conf"], case["img"], case["sn"], case["gn"], case["pn"],
                           depth_type=depth_type, depth_lambda=LAMBDA, tol=TOL, normal_lambda=NORMAL_LAMBDA, step=step,
                           keep=k["keep"])
    want = float(own["value"])
    if math.isnan(want):
        assert math.isnan(k["value"]), (k["value"], want)
    else:
        assert abs(k["value"] - want) <= value_rtol * max(abs(want), 1e-30) + 1e-30, (k["value"], want)
    vv = 1.0 if v is None else v
    if not math.isnan(want) or depth_type == 0 or math.isfinite(float(own["depth"])):
        _map_ok(k["vd"], own["v_depth"] * vv, "v_depth")
    # v_normal: 1 ulp of the fp32 expression
    lam = NORMAL_LAMBDA if step > 7000 else 0.0
    kf = (torch.tensor(vv, dtype=F32) * torch.tensor(lam, dtype=F32) * 2) / torch.tensor(3.0 * H * W, dtype=F32)
    d = (ags_ref.signed(case["pn"]) - ags_ref.signed(case["gn"])).permute(1, 2, 0)
    expect = torch.sign(d) * kf
    ulp = (torch.nextafter(expect.abs(), torch.tensor(math.inf)) - expect.abs())
    assert bool(((k["vn"] - expect).abs() <= ulp).all())


@pytest.mark.parametrize("hw", SHAPES)
@pytest.mark.parametrize("depth_type", [0, 1, 2, 3, 4])
def test_ags_kernel_matches_fp64(hw, depth_type):
    H, W = hw
    for si, step in enumerate(STEPS):
        nu8, cu8, iu8 = DTYPES[(si + depth_type) % len(DTYPES)]
        case = make_case(H, W, seed=H * 131 + W + 7 * si + depth_type, normal_u8=nu8, conf_u8=cu8, img_u8=iu8)
        _check(case, step, depth_type, VS[(si + depth_type) % len(VS)])


def test_ags_kernel_matches_fp64_at_1080p():
    case = make_case(1080, 1920, seed=3, normal_u8=True, conf_u8=True, img_u8=True)
    for step, v in ((8000, None), (16000, 3.7)):
        _check(case, step, 1, v, value_rtol=VALUE_RTOL_1080P)


def test_ags_empty_selection_is_nan():
    """Every element an edge (random gt normals) and every depth invalid: NaN, as the reference's mean of nothing."""
    H, W = 16, 40
    g = torch.Generator().manual_seed(1)
    case = make_case(H, W, seed=2)
    case["gn"] = torch.rand(H, W, 3, generator=g)
    k = _kernel(case, 100, 3, None)
    if not bool(k["keep"].any()):
        assert math.isnan(k["value"])
    case["gd"] = torch.zeros_like(case["gd"])
    k = _kernel(case, 16000, 3, None)
    assert math.isnan(k["value"]) and bool((k["vd"] == 0).all())


def test_ags_argument_errors():
    L, lib = _lib()
    a = L.DnrAgsLoss()
    assert lib.dnr_ags_loss_fwd(None, None) == -1
    assert lib.dnr_ags_loss_fwd(C.byref(a), None) == -2
    a.width, a.height, a.depth_loss_type = 8, 8, 5
    assert lib.dnr_ags_loss_fwd(C.byref(a), None) == -3
    a.depth_loss_type, a.flags = 1, 1 << 9
    assert lib.dnr_ags_loss_fwd(C.byref(a), None) == -3
    a.flags = 0
    assert lib.dnr_ags_loss_fwd(C.byref(a), None) == -1
    assert lib.dnr_ags_loss_bwd(C.byref(a), None, None, None) == -1


# ------------------------------------------------------------------------------------------- against the torch path
@pytest.mark.parametrize("step", STEPS)
def test_ags_fused_matches_torch_path(step):
    from dn_splatter_b200.regularization_strategy import AGSMeshRegularization

    H, W = 81, 49
    for seed in range(step, step + 100):  # the first content whose decision band is empty
        case = make_case(H, W, seed=seed, normal_u8=False, conf_u8=False, img_u8=False)
        km = ags_ref.keep_mask(ags_ref.signed(case["sn"]), ags_ref.signed(case["gn"]), angle=step >= 15000)
        band = km["margin"].abs() <= (EDGE_BAND if step < 15000 else ANGLE_BAND)
        if not bool(band.any()):
            break
    assert not bool(band.any()), "content with an empty decision band"
    conf = ags_ref.gate_map(case["conf"], raw=True)
    res = {}
    for fused in (True, False):
        ags = AGSMeshRegularization().cuda()
        ags.fused = fused
        pd = case["pd"].cuda().requires_grad_(True)
        pn = case["pn"].cuda().requires_grad_(True)
        scales = torch.randn(50, 3, generator=torch.Generator().manual_seed(1)).cuda().requires_grad_(True)
        loss = ags(step=step, pred_depth=pd, gt_depth=case["gd"].cuda(), surf_normal=(2 * case["sn"].cuda() - 1).permute(2, 0, 1),
                   gt_normal=(2 * case["gn"].cuda() - 1).permute(2, 0, 1), pred_normal=(2 * pn - 1).permute(2, 0, 1),
                   confidence_map=conf.cuda(), scales=scales, gt_img=case["img"].cuda())
        loss.backward()
        res[fused] = (float(loss.detach()), pd.grad.cpu(), pn.grad.cpu(), scales.grad.cpu())
    (lf, gdf, gnf, gsf), (lt, gdt, gnt, gst) = res[True], res[False]
    if math.isnan(lt):
        assert math.isnan(lf)
    else:
        assert abs(lf - lt) <= 1e-5 * max(1.0, abs(lt)), (lf, lt)
    _map_ok(gdf, gdt, "v_depth vs torch")
    _map_ok(gnf, gnt, "v_normal vs torch")
    _map_ok(gsf, gst, "v_scales vs torch")


# ------------------------------------------------------------------------------------------------ model level
def _ags_model(params, fused=True, **kw):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.losses import DepthLossType

    cfg = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", regularization_strategy="ags-mesh",
                                use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType.EdgeAwareLogL1, **kw)
    m = cfg.setup(device="cuda")
    m.load_gaussians(params)
    m.regularization_strategy.fused = fused
    m.train()
    return m


def _ags_batch(m, cam, seed=5):
    """uint8 image and confidence, the render's own depth (10 % zeroed) and, as mono normals, its surface normal in uint8,
    so both normal selections keep a part of the frame (a random normal map is all edges: NaN, as upstream)."""
    with torch.no_grad():
        out = m.get_outputs(cam)
    H, W = out["depth"].shape[:2]
    g = torch.Generator().manual_seed(seed)
    depth = out["depth"].cpu() * (1 + 0.05 * torch.randn(H, W, 1, generator=g))
    depth[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
    conf = (torch.rand(H, W, 1, generator=g) * 255).to(torch.uint8)
    normal = (out["surface_normal"].cpu() * 255).round().to(torch.uint8)
    batch = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), "mono_depth": depth, "normal": normal,
             "confidence": conf}
    return {k: v.cuda() for k, v in batch.items()}


@pytest.mark.parametrize("step", [100, 7000, 7001, 15000])
def test_ags_model_fused_matches_torch(step):
    from dn_splatter_b200 import regularization_strategy as RS
    from tests.helpers import scene_and_camera
    from tests.test_gpu_model import _camera

    params, cam = scene_and_camera(3000, 112, 96)
    batch = _ags_batch(_ags_model(params), _camera(cam))
    out = {}
    for fused in (True, False):
        m = _ags_model(params, fused=fused, ssim_lambda=0.2)
        m.step = step
        calls = []
        orig = RS._FusedAGSLoss.apply
        RS._FusedAGSLoss.apply = lambda *a: (calls.append(1), orig(*a))[1]
        try:
            ld = m.get_loss_dict(m.get_outputs(_camera(cam)), dict(batch))
        finally:
            RS._FusedAGSLoss.apply = orig
        assert bool(calls) == fused, "the fused route runs exactly when fused is set"
        (ld["main_loss"] + ld["scale_reg"]).backward()
        out[fused] = (float(ld["main_loss"]),
                      {k: p.grad.detach().clone() for k, p in m.gauss_params.items() if p.grad is not None})
    lf, lt = out[True][0], out[False][0]
    assert math.isfinite(lt), lt
    assert abs(lf - lt) <= 1e-5 * max(1.0, abs(lt)), (lf, lt)
    assert set(out[True][1]) == set(out[False][1]) and out[False][1]
    for k, gt in out[False][1].items():
        gf = out[True][1][k]
        rel = float((gf - gt).norm() / (gt.norm() + 1e-30))
        assert rel <= 1e-5, (k, rel)


def test_ags_captured_step_matches_eager_and_guards_gates():
    with torch.cuda.stream(torch.cuda.Stream()):  # a capture cannot use the legacy default stream (graph_step.py)
        _captured_step_body()


def _captured_step_body():
    from dn_splatter_b200.graph_step import GraphedTrainStep
    from dn_splatter_b200.synthetic import ring_cameras
    from tests.helpers import scene_and_camera
    from tests.test_gpu_model import _camera

    params, _ = scene_and_camera(4000, 160, 128)
    cams = [_camera(c) for c in ring_cameras(6, 160, 128)]
    for c in cams:
        c.camera_to_worlds = c.camera_to_worlds.cpu()
    m = _ags_model(params, ssim_lambda=0.2, sync_free=True)
    batch = _ags_batch(m, cams[0])
    m.step = 6999
    bucket = m.enable_flat_grads()

    def eager(i):
        bucket.zero_()
        ld = m.get_loss_dict(m.get_outputs(cams[i]), dict(batch))
        (ld["main_loss"] + ld["scale_reg"]).backward()
        return float(ld["main_loss"] + ld["scale_reg"]), bucket.flat.clone()

    for i in (0, 1, 2):
        eager(i)
    step = GraphedTrainStep(m, bucket, cams[0], batch, n_slots=1)

    def rel(a, b):
        return float((a - b).norm() / (b.norm() + 1e-30))

    def replay_matches(i):
        """A replay equals the eager fused step within 1e-6 relative, or within 4x the step's own run-to-run spread when
        that is larger: the raster backward accumulates per-Gaussian gradients with float atomics, whose order varies."""
        want, again = eager(i), eager(i)
        assert math.isfinite(want[0]), want[0]
        loss = step(cams[i], 0)
        torch.cuda.synchronize()
        got = (float(loss), bucket.flat.clone())
        d_loss, spread_loss = abs(got[0] - want[0]), abs(again[0] - want[0])
        d_flat, spread_flat = rel(got[1], want[1]), rel(again[1], want[1])
        print(f"[ags graph] step {m.step} view {i}: loss {got[0]!r} eager {want[0]!r} (again {again[0]!r}); bucket rel "
              f"{d_flat:.3g}, eager run-to-run {spread_flat:.3g}")
        assert d_loss <= max(1e-6 * max(1.0, abs(want[0])), 4 * spread_loss), (got[0], want[0], again[0])
        assert d_flat <= max(1e-6, 4 * spread_flat), (d_flat, spread_flat)

    replay_matches(1)
    for nxt in (7000, 7001, 15000):
        m.step = nxt - 1
        step.recapture()
        replay_matches(2)
        m.step = nxt
        with pytest.raises(RuntimeError, match="recapture"):
            step(cams[1], 0)
        step.recapture()
        replay_matches(1)


def test_ags_trainer_runs_finite():
    from dn_splatter_b200.trainer import Trainer
    from dn_splatter_b200.synthetic import ring_cameras
    from tests.helpers import scene_and_camera
    from tests.test_gpu_model import _camera

    params, _ = scene_and_camera(2000, 96, 64)
    cams = [_camera(c) for c in ring_cameras(4, 96, 64)]
    m = _ags_model(params, ssim_lambda=0.2)
    batch = _ags_batch(m, cams[0])
    m.num_train_data = 4
    tr = Trainer(m, lambda s: (cams[s % 4], dict(batch)), max_steps=20, fused_adam=True)
    for _ in range(10):
        out = tr.train_iteration()
        assert torch.isfinite(out["loss"])
