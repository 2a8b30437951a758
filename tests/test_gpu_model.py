"""GPU tests of the reference-facing surface: DNSplatterModel.get_outputs / get_loss_dict and
DNRegularization against the oracle (whose loss code is pinned to the reference's by tests/golden)."""
import pytest
import torch

from tests.helpers import frac_close, oracle_outputs, scene_and_camera

pytestmark = pytest.mark.gpu
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")


def _model(params, **cfg_kw):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig

    cfg = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", **cfg_kw)
    m = cfg.setup(device="cuda")
    m.load_gaussians(params)
    m.background_color = torch.tensor([0.1490, 0.1647, 0.2157])
    m.step = 30000
    m.train()
    return m


def _camera(cam):
    from dn_splatter_b200.cameras import Cameras

    return Cameras(cam["c2w"][None].cuda(), cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["width"], cam["height"],
                   metadata={"cam_idx": 7})


def _batch(H, W, seed=5):
    g = torch.Generator().manual_seed(seed)
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    depth[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
    return {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), "mono_depth": depth,
            "normal": torch.rand(H, W, 3, generator=g)}


@needs_cuda
def test_get_outputs_keys_shapes_and_side_outputs():
    params, cam = scene_and_camera(800, 112, 96)
    m = _model(params)
    out = m.get_outputs(_camera(cam))
    assert set(out) == {"rgb", "depth", "normal", "surface_normal", "accumulation", "background"}
    H, W = 96, 112
    assert out["rgb"].shape == (H, W, 3) and out["depth"].shape == (H, W, 1) and out["normal"].shape == (H, W, 3)
    assert out["surface_normal"].shape == (H, W, 3) and out["accumulation"].shape == (H, W, 1)
    assert m.xys.shape == (1, 800, 2) and m.radii.shape == (800,) and m.radii.dtype == torch.int32
    assert m.depths.shape == (1, 800) and m.conics.shape == (1, 800, 3) and m.num_tiles_hit.shape == (1, 800)
    assert m.last_size == (H, W) and m.camera_idx == 7
    assert torch.equal(m.vis_indices, torch.where(m.radii > 0)[0])
    assert m.get_outputs("not a camera") == {}
    _, ref = oracle_outputs(params, cam)
    for k, kk in (("rgb", "rgb"), ("normal", "normal"), ("accumulation", "accumulation")):
        frac, mx = frac_close(out[k], ref[kk], atol=1e-4)
        assert frac > 0.999, (k, frac, mx)
    torch.testing.assert_close(m.normals.detach().cpu(), ref["gauss_normals"], rtol=1e-4, atol=1e-5)


@needs_cuda
@pytest.mark.parametrize("depth_type", ["EdgeAwareLogL1", "LogL1", "L1", "MSE"])
def test_loss_dict_matches_oracle_and_gradients_flow(depth_type):
    from dn_splatter_b200.losses import DepthLossType
    from oracle import dn_ref

    params, cam = scene_and_camera(900, 128, 80, view=2)
    H, W = 80, 128
    batch = _batch(H, W)
    m = _model(params, use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType(depth_type if depth_type != "MSE" else "mse"),
               ssim_lambda=0.0)
    out = m.get_outputs(_camera(cam))
    ld = m.get_loss_dict(out, dict(batch))
    assert set(ld) == {"main_loss", "scale_reg"}
    ld["main_loss"].backward()
    # oracle
    p, ref = oracle_outputs(params, cam, requires_grad=True)
    gt_img = (batch["image"].float() / 255.0)
    rgb_loss = (gt_img - ref["rgb"]).abs().mean()
    reg = dn_ref.dn_regularization(ref["depth"], batch["mono_depth"], ref["normal"], batch["normal"], p["scales"],
                                   gt_img.clamp(min=10 / 255.0), depth_lambda=0.2, depth_loss_type=depth_type)
    want = rgb_loss + reg
    want.backward()
    assert abs(float(ld["main_loss"]) - float(want)) <= 2e-4 * max(1.0, abs(float(want))), (float(ld["main_loss"]), float(want))
    for k in ("means", "quats", "scales", "opacities", "features_dc", "features_rest"):
        got, w = m.gauss_params[k].grad.cpu(), p[k].grad
        rel = float((got - w).norm() / (w.norm() + 1e-20))
        assert rel < 5e-3, f"{k}: {rel:.3e}"
    assert m.xys_flat.absgrad is not None and m.xys_flat.grad is not None


def _fp64_oracle_loss(params, cam, batch, depth_type, ssim_lambda, **oracle_kw):
    """The reference's loss for the same view in fp64: (1 - l) L1 + l (1 - SSIM) + DNRegularization, with the uint8 image
    and normal maps read as value / 255 (the image clamped at 10/255 for the regulariser, quirk B10)."""
    from dn_splatter_b200.dn_model import ssim
    from oracle import dn_ref

    p, ref = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True, **oracle_kw)
    gt_img = batch["image"].double() / 255.0
    loss = (1 - ssim_lambda) * (gt_img - ref["rgb"]).abs().mean()
    if ssim_lambda > 0:
        loss = loss + ssim_lambda * (1 - ssim(gt_img.permute(2, 0, 1)[None], ref["rgb"].permute(2, 0, 1)[None]))
    loss = loss + dn_ref.dn_regularization(ref["depth"], batch["mono_depth"].double(), ref["normal"],
                                           batch["normal"].double() / 255.0, p["scales"], gt_img.clamp(min=10 / 255.0),
                                           depth_lambda=0.2, depth_loss_type=depth_type)
    loss.backward()
    return float(loss.detach()), p


def _check_loss_dict_against_fp64_oracle(hw, depth_type, ssim_lambda, **cfg_kw):
    from dn_splatter_b200.losses import DepthLossType

    H, W = hw
    params, cam = scene_and_camera(500, W, H, view=2)
    g = torch.Generator().manual_seed(H * 100 + W)
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    depth[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
    batch = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), "mono_depth": depth,
             "normal": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8)}
    m = _model(params, use_depth_loss=True, depth_lambda=0.2, ssim_lambda=ssim_lambda,
               depth_loss_type=DepthLossType(depth_type if depth_type != "MSE" else "mse"), **cfg_kw)
    ld = m.get_loss_dict(m.get_outputs(_camera(cam)), {k: v.cuda() for k, v in batch.items()})
    ld["main_loss"].backward()
    want, p = _fp64_oracle_loss(params, cam, batch, depth_type, ssim_lambda,
                                rasterize_mode=cfg_kw.get("rasterize_mode", "classic"))
    assert abs(float(ld["main_loss"]) - want) <= 2e-4 * max(1.0, abs(want)), (float(ld["main_loss"]), want)
    errs = {k: float((m.gauss_params[k].grad.cpu().double() - p[k].grad).norm() / p[k].grad.norm())
            for k in ("means", "quats", "scales", "opacities", "features_dc", "features_rest")}
    bad = {k: f"{v:.3e}" for k, v in errs.items() if not v <= 1e-3}
    assert not bad, f"relative gradient error above 1e-3: {bad}"


@needs_cuda
@pytest.mark.parametrize("ssim_lambda", [0.0, 0.2])
@pytest.mark.parametrize("depth_type", ["EdgeAwareLogL1", "LogL1", "L1", "MSE"])
@pytest.mark.parametrize("hw", [(49, 81), (53, 75)], ids=["81x49", "75x53"])
def test_loss_dict_gradients_match_fp64_oracle_at_ragged_sizes(hw, depth_type, ssim_lambda):
    """get_loss_dict's gradients at frame sizes that are not multiples of the tile: the fused photometric loss
    (FusedPhotometric with SSIM, or FusedL1) and the regularisers evaluated in raster_bwd's prologue read neighbours
    through clamped indices along the ragged edge.  uint8 image and normal supervision."""
    _check_loss_dict_against_fp64_oracle(hw, depth_type, ssim_lambda)


@needs_cuda
@pytest.mark.parametrize("ssim_lambda", [0.0, 0.2])
@pytest.mark.parametrize("hw", [(49, 81), (80, 128)], ids=["81x49", "128x80"])
def test_antialiased_two_pass_loss_dict_matches_fp64_oracle(hw, ssim_lambda):
    """rasterize_mode="antialiased" with normals renders twice (colour / depth with opacity x compensation, normals
    with the plain opacity) and sums both passes' gradients."""
    _check_loss_dict_against_fp64_oracle(hw, "EdgeAwareLogL1", ssim_lambda, rasterize_mode="antialiased",
                                         predict_normals=True)


@needs_cuda
def test_flat_grad_bucket_equals_autograd_path():
    params, cam = scene_and_camera(700, 96, 96, view=1)
    batch = _batch(96, 96)
    from dn_splatter_b200.losses import DepthLossType

    kw = dict(use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType.EdgeAwareLogL1, ssim_lambda=0.2)
    a, b = _model(params, **kw), _model(params, **kw)
    bucket = b.enable_flat_grads()
    bucket.zero_()
    for m in (a, b):
        out = m.get_outputs(_camera(cam))
        ld = m.get_loss_dict(out, dict(batch))
        (ld["main_loss"] + ld["scale_reg"]).backward()
    for k in ("means", "quats", "scales", "opacities", "features_dc", "features_rest"):
        ga, gb = a.gauss_params[k].grad, b.gauss_params[k].grad  # float atomics: run-to-run order noise only
        assert float((ga - gb).norm() / (ga.norm() + 1e-30)) < 1e-4, k
        assert b.gauss_params[k].grad.data_ptr() == bucket.views[k].data_ptr()


@needs_cuda
def test_normal_from_depth_image_matches_reference_goldens(golden_dir):
    import glob
    import os

    import numpy as np

    from dn_splatter_b200.utils.normal_utils import normal_from_depth_image

    for f in sorted(glob.glob(os.path.join(golden_dir, "dn_reference_[ab].npz"))):
        z = np.load(f)
        d = torch.from_numpy(z["in_pred_depth"]).cuda()
        fx, fy, cx, cy = [float(v) for v in z["in_intr"]]
        H, W, _ = d.shape
        n = normal_from_depth_image(d, fx, fy, cx, cy, (W, H), torch.eye(4).cuda(), d.device)
        torch.testing.assert_close(n.cpu(), torch.from_numpy(z["out_normal_from_depth"]), rtol=1e-4, atol=2e-5)


@needs_cuda
def test_dn_regularization_matches_reference_goldens(golden_dir):
    import glob
    import os

    import numpy as np

    from dn_splatter_b200.losses import DepthLoss, DepthLossType
    from dn_splatter_b200.regularization_strategy import DNRegularization

    for f in sorted(glob.glob(os.path.join(golden_dir, "dn_reference_[ab].npz"))):
        z = {k: torch.from_numpy(v).cuda() for k, v in np.load(f).items()}
        for key, lam, t in (("dn_reg_lambda0.2", 0.2, None), ("dn_reg_lambda0.5", 0.5, None),
                            ("dn_reg_LogL1", 0.2, DepthLossType.LogL1), ("dn_reg_L1", 0.2, DepthLossType.L1),
                            ("dn_reg_mse", 0.2, DepthLossType.MSE), ("dn_reg_nodepth", 0.2, "none")):
            reg = DNRegularization(depth_lambda=lam).cuda()
            if t == "none":
                reg.depth_loss = None
            elif t is not None:
                reg.depth_loss_type, reg.depth_loss = t, DepthLoss(t)
            pd = z["in_pred_depth"].clone().requires_grad_(True)
            pn = z["in_pred_normal"].clone().requires_grad_(True)
            sc = z["in_scales"].clone().requires_grad_(True)
            v = reg(pred_depth=pd, gt_depth=z["in_gt_depth"], pred_normal=pn, gt_normal=z["in_gt_normal"], scales=sc,
                    gt_img=z["in_gt_img"])
            torch.testing.assert_close(v, z["out_" + key], rtol=2e-5, atol=1e-6)
            if key == "dn_reg_lambda0.2":
                v.backward()
                torch.testing.assert_close(pd.grad, z["out_grad_pred_depth"], rtol=1e-4, atol=1e-8)
                torch.testing.assert_close(pn.grad, z["out_grad_pred_normal"], rtol=1e-4, atol=1e-8)
                torch.testing.assert_close(sc.grad, z["out_grad_scales"], rtol=1e-4, atol=1e-8)


@needs_cuda
def test_fused_l1_and_u8_conversion_match_torch():
    from dn_splatter_b200.regularization_strategy import FusedL1, u8_to_float

    g = torch.Generator().manual_seed(3)
    pred = torch.rand(37, 53, 3, generator=g).cuda().requires_grad_(True)
    gt8 = (torch.rand(37, 53, 3, generator=g) * 255).to(torch.uint8).cuda()
    gtf = gt8.float() / 255.0
    for gt in (gt8, gtf):
        pred.grad = None
        loss = FusedL1.apply(pred, gt)
        (loss * 3.0).backward()
        ref_p = pred.detach().clone().requires_grad_(True)
        ref = (gtf - ref_p).abs().mean()
        (ref * 3.0).backward()
        torch.testing.assert_close(loss, ref, rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(pred.grad, ref_p.grad, rtol=1e-6, atol=1e-9)
    assert torch.equal(u8_to_float(gt8), gtf)
    assert torch.equal(u8_to_float(gt8, 255.0, 10 / 255.0), gtf.clamp(min=10 / 255.0))


@needs_cuda
def test_cuda_graph_step_matches_eager_step():
    """One captured training view (zero grads -> get_outputs -> get_loss_dict -> backward) replayed for two different
    cameras must reproduce the eager loss and gradients of those cameras."""
    # the whole loop lives on a non-default stream: the legacy stream cannot take part in a capture, and autograd
    # remembers the stream each parameter's gradient accumulator was created on (see graph_step.py)
    with torch.cuda.stream(torch.cuda.Stream()):
        _graph_step_body()


@needs_cuda
def test_graphed_train_step_overflow_is_loud_and_recoverable():
    """A training graph captured with far fewer intersection slots than the view needs: the truncated replay is reported
    by check_capacity (DnrCapacityError), and after recapture() the replays reproduce the eager loss and gradients."""
    with torch.cuda.stream(torch.cuda.Stream()):
        _graph_step_body(n_gauss=12000, capacity=4096)


@needs_cuda
@pytest.mark.parametrize("overflow", [False, True], ids=["fits", "overflow_recapture"])
def test_cuda_graph_step_with_ssim_matches_eager_step(overflow):
    """The captured step bench.py times: ssim_lambda = 0.2, so the photometric term is FusedPhotometric inside the
    graph.  Replays (after an overflow and recapture too) must reproduce the eager loss and gradients."""
    kw = dict(n_gauss=12000, capacity=4096) if overflow else {}
    with torch.cuda.stream(torch.cuda.Stream()):
        _graph_step_body(ssim_lambda=0.2, **kw)


def _graph_step_body(n_gauss=4000, capacity=None, ssim_lambda=0.0):
    from dn_splatter_b200.graph_step import GraphedTrainStep
    from dn_splatter_b200.losses import DepthLossType
    from dn_splatter_b200.rasterize import DnrCapacityError
    from dn_splatter_b200.synthetic import ring_cameras

    params, _ = scene_and_camera(n_gauss, 160, 128)
    cams = [_camera(c) for c in ring_cameras(6, 160, 128)]
    for c in cams:
        c.camera_to_worlds = c.camera_to_worlds.cpu()
    batch = {k: v.cuda() for k, v in _batch(128, 160).items()}
    kw = dict(use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType.EdgeAwareLogL1,
              ssim_lambda=ssim_lambda, sync_free=True)
    m = _model(params, **kw)
    bucket = m.enable_flat_grads()
    eager, counts = {}, {}
    for i in (0, 1, 2, 4):  # also seeds the intersection-capacity statistics the capture needs
        bucket.zero_()
        ld = m.get_loss_dict(m.get_outputs(cams[i]), dict(batch))
        (ld["main_loss"] + ld["scale_reg"]).backward()
        eager[i] = (float(ld["main_loss"] + ld["scale_reg"]), bucket.flat.clone())
        counts[i] = int(m.raster_out.info["n_isects_dev"])
    del ld  # a live autograd graph would pin AccumulateGrad nodes created on the default stream (see graph_step.py)
    step = GraphedTrainStep(m, bucket, cams[0], batch, n_slots=2, capacity=capacity)
    if capacity is not None:
        assert min(counts.values()) > 2 * capacity, ("the test scene must overflow the captured capacity", counts)
        worst = max(counts, key=counts.get)  # recapture() then has room for every view below
        step(cams[worst], 0)
        with pytest.raises(DnrCapacityError):
            step.check_capacity(wait=True)
        assert step.max_count == counts[worst]
        step.recapture()
        assert step.capacity > counts[worst]
    for i, slot in ((4, 0), (1, 1), (2, 0)):
        for k, v in batch.items():
            step.batches[slot][k].copy_(v)
        loss = step(cams[i], slot)
        torch.cuda.synchronize()
        step.check_capacity(wait=True)
        assert abs(float(loss) - eager[i][0]) <= 1e-5 * max(1.0, abs(eager[i][0])), (i, float(loss), eager[i][0])
        rel = float((bucket.flat - eager[i][1]).norm() / (eager[i][1].norm() + 1e-30))
        assert rel < 1e-4, (i, rel)


@needs_cuda
@pytest.mark.parametrize("hw", [(64, 80), (37, 53), (128, 160), (11, 200)])
def test_fused_ssim_matches_torch(hw):
    """csrc/ssim.cu (value + gradient) against dn_model.ssim() — the torchmetrics restatement the default path uses."""
    from dn_splatter_b200.dn_model import ssim
    from dn_splatter_b200.regularization_strategy import FusedSSIM

    H, W = hw
    g = torch.Generator().manual_seed(H * 1000 + W)
    x = torch.rand(H, W, 3, generator=g).cuda().requires_grad_(True)
    y = (x.detach().cpu() * 0.6 + 0.4 * torch.rand(H, W, 3, generator=g)).cuda()
    if H <= 10 or W <= 10:
        with pytest.raises(Exception):
            FusedSSIM.apply(x, y)
        return
    ref = ssim(y.permute(2, 0, 1)[None], x.permute(2, 0, 1)[None])
    (gref,) = torch.autograd.grad(ref, x)
    out = FusedSSIM.apply(x, y)
    (gout,) = torch.autograd.grad(out, x)
    assert abs(float(out) - float(ref)) < 2e-5
    assert float((gout - gref).norm() / gref.norm()) < 1e-4
    # uint8 target read as stored (value / 255), 1 and 4 channels (more than one channel group per CTA)
    for C in (1, 3, 4):
        xc = torch.rand(H, W, C, generator=g).cuda().requires_grad_(True)
        y8 = (torch.rand(H, W, C, generator=g) * 255).to(torch.uint8).cuda()
        yf = y8.float() / 255.0
        ref = ssim(yf.permute(2, 0, 1)[None], xc.permute(2, 0, 1)[None])
        (gref,) = torch.autograd.grad(ref, xc)
        out = FusedSSIM.apply(xc, y8)
        (gout,) = torch.autograd.grad(out, xc)
        assert abs(float(out) - float(ref)) < 2e-5, C
        # uncorrelated noise images are the worst case for the fp32 E[x^2] - mx^2 cancellation (in the torch reference too)
        assert float((gout - gref).norm() / gref.norm()) < 1e-3, C


@needs_cuda
def test_fused_adam_matches_torch_adam():
    """optim.FusedAdam (one dnr_adam_step launch) against one torch.optim.Adam per group over 20 steps, odd sizes
    (scalar tail, unaligned views) included."""
    from dn_splatter_b200.optim import FusedAdam

    g = torch.Generator().manual_seed(11)
    shapes = {"means": (1001, 3), "quats": (1001, 4), "features_rest": (1001, 15, 3), "opacities": (1001, 1), "odd": (7,)}
    lrs = {"means": 1.6e-4, "quats": 1e-3, "features_rest": 1.25e-4, "opacities": 5e-2, "odd": 1e-2}
    a = {k: torch.nn.Parameter(torch.randn(*s, generator=g).cuda()) for k, s in shapes.items()}
    b = {k: torch.nn.Parameter(v.detach().clone()) for k, v in a.items()}
    fused = FusedAdam([{"params": [p], "lr": lrs[k], "eps": 1e-15, "name": k} for k, p in a.items()])
    ref = {k: torch.optim.Adam([p], lr=lrs[k], eps=1e-15) for k, p in b.items()}
    for step in range(20):
        for k in a:
            grad = (torch.randn(shapes[k], generator=g) * 10.0 ** (-(len(k) % 5))).cuda()
            a[k].grad, b[k].grad = grad.clone(), grad.clone()
        fused.step()
        for o in ref.values():
            o.step()
    for k in a:
        for x, y in ((fused.state[a[k]]["exp_avg"], ref[k].state[b[k]]["exp_avg"]),
                     (fused.state[a[k]]["exp_avg_sq"], ref[k].state[b[k]]["exp_avg_sq"]), (a[k].data, b[k].data)):
            assert float((x - y).abs().max()) <= 1e-5 * float(y.abs().max()), k


@needs_cuda
@pytest.mark.parametrize("depth_type,ssim_lambda", [("EdgeAwareLogL1", 0.0), ("EdgeAwareLogL1", 0.2), ("LogL1", 0.0),
                                                     ("L1", 0.2), ("mse", 0.0)])
def test_loss_gradients_fused_into_raster_bwd_match_the_gradient_image_path(depth_type, ssim_lambda, monkeypatch):
    """BASELINE north_star: the Depth / Normal / TV regularisers (and the photometric L1) are differentiated inside
    dnr_raster_bwd.  The same step with the losses' own backward kernels writing gradient images (fuse_loss_backward =
    False: dnr_loss_bwd runs, and only there) and with host-resident float maps (the generic torch path of get_loss_dict)
    must give the same loss and the same parameter gradients."""
    from dn_splatter_b200 import _lib as L
    from dn_splatter_b200.losses import DepthLossType

    lib = L.load()
    loss_bwd_calls = []
    orig = lib.dnr_loss_bwd
    monkeypatch.setitem(lib.__dict__, "dnr_loss_bwd", lambda *args: loss_bwd_calls.append(1) or orig(*args))
    params, cam = scene_and_camera(1200, 144, 112, view=2)
    H, W = 112, 144
    g = torch.Generator().manual_seed(11)
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    depth[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
    raw = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), "mono_depth": depth,
           "normal": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8)}
    kw = dict(use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType(depth_type), ssim_lambda=ssim_lambda)
    runs = {}
    for name, fuse, dev in (("fused", True, "cuda"), ("images", False, "cuda"), ("host", True, "cpu")):
        m = _model(params, fuse_loss_backward=fuse, **kw)
        batch = {k: v.to(dev) for k, v in raw.items()}
        out = m.get_outputs(_camera(cam))
        ld = m.get_loss_dict(out, batch)
        loss_bwd_calls.clear()
        (ld["main_loss"] + ld["scale_reg"]).backward()
        assert len(loss_bwd_calls) == (1 if name == "images" else 0), (name, len(loss_bwd_calls))
        runs[name] = (float(ld["main_loss"]), {k: m.gauss_params[k].grad.clone() for k in
                                                ("means", "quats", "scales", "opacities", "features_dc", "features_rest")},
                      m.xys_flat.absgrad.clone())
        if name == "fused":  # nothing was left undelivered, and the deferred specs were consumed by the raster backward
            assert "deferred" not in m.raster_out.info
    for other in ("images", "host"):
        assert abs(runs["fused"][0] - runs[other][0]) <= 2e-6 * max(1.0, abs(runs[other][0])), other
        for k, want in runs[other][1].items():
            rel = float((runs["fused"][1][k] - want).norm() / (want.norm() + 1e-30))
            assert rel < 2e-4, (other, k, rel)
        ab = runs[other][2]
        assert float((runs["fused"][2] - ab).abs().max()) <= 2e-4 * float(ab.abs().max() + 1e-30)


@needs_cuda
def test_render_service_equals_get_outputs_for_camera_and_survives_overflow():
    """SURVEY §8f-1: the captured-forward render service hands out, in order, exactly the maps of
    model.get_outputs_for_camera (device maps and pinned host copies), and a view that does not fit the captured
    intersection capacity is re-rendered after a re-capture instead of being delivered truncated."""
    from dn_splatter_b200.render_service import ViewRenderer, _ForwardGraphs
    from dn_splatter_b200.synthetic import ring_cameras

    params, _ = scene_and_camera(4000, 160, 112)
    m = _model(params)
    W, H = 160, 112
    cams = [_camera(c) for c in ring_cameras(7, W, H)]
    keys = ("rgb", "depth", "normal", "surface_normal", "accumulation")
    want = []
    m.eval()
    for c in cams:
        out = m.get_outputs_for_camera(c)
        want.append({k: out[k].clone() for k in keys})
    m.train()
    for to_host in (False, True):
        r = ViewRenderer(m, keys=keys, to_host=to_host)
        got = [(i, {k: v.clone() for k, v in d.items()}) for i, d in r.render(cams)]
        assert [i for i, _ in got] == list(range(len(cams)))
        for (i, d), w in zip(got, want):
            for k in keys:
                assert torch.equal(d[k].to("cuda"), w[k]), (to_host, i, k)
        assert r.recaptures == 0 and m.training
        # again through the same captured graphs (steady state)
        for (i, d), w in zip(r.render(cams), want):
            assert torch.equal(d["rgb"].to("cuda"), w["rgb"])
    r = ViewRenderer(m, keys=keys, to_host=True)
    r._graphs[(W, H)] = _ForwardGraphs(m, cams[0], keys, r.n_slots, capacity=4096)  # far too small: every view overflows it
    got = [(i, {k: v.clone() for k, v in d.items()}) for i, d in r.render(cams)]
    assert r.recaptures >= 1 and [i for i, _ in got] == list(range(len(cams)))
    for (i, d), w in zip(got, want):
        for k in keys:
            assert torch.equal(d[k].to("cuda"), w[k]), (i, k)
