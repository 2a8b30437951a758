"""Camera optimisation on the GPU: the view-matrix gradient that dnr_project_bwd returns (DnrArgs.v_viewmat) against
the fp64 oracle's autograd, the pose gradient end to end through DNSplatterModel, a 1M-Gaussian / 1080p invariance
check, the captured training step, and pose recovery from perturbed cameras."""
import math

import pytest
import torch

from dn_splatter_b200.camera_opt import CameraOptimizerConfig, compose, exp_map_SE3, exp_map_SO3xR3
from dn_splatter_b200.rasterize import get_viewmat
from dn_splatter_b200.synthetic import BACKGROUND, make_scene, ring_cameras
from oracle import dn_ref
from oracle import gsplat_ref as G
from tests.test_gpu_backward_edges import region_mask, rel_err, route_loss

pytestmark = pytest.mark.gpu
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")

TOL = 1e-3
XI = torch.tensor([0.08, -0.05, 0.1, 0.02, -0.015, 0.01], dtype=torch.float64)  # viewmat differs from the normals' c2w


def oracle_render(p, cam, viewmat, c2w, rasterize_mode="classic", sh_degree=3):
    """dn_ref.get_outputs with the world->camera matrix given separately (the optimised pose) while the normals use the
    un-optimised c2w, as DNSplatterModel.get_outputs does with camera optimisation on."""
    dt = p["means"].dtype
    colors = torch.cat([p["features_dc"][:, None, :], p["features_rest"]], dim=1)
    render, alpha, info = G.rasterization(
        p["means"], p["quats"] / p["quats"].norm(dim=-1, keepdim=True), torch.exp(p["scales"]),
        torch.sigmoid(p["opacities"]).squeeze(-1), colors, viewmat, dn_ref.intrinsics(cam["fx"], cam["fy"], cam["cx"],
                                                                                       cam["cy"], dt),
        cam["width"], cam["height"], 16, near_plane=0.01, far_plane=1e10, sh_degree=sh_degree,
        rasterize_mode=rasterize_mode)
    bg = torch.tensor(BACKGROUND, dtype=dt)
    rgb = torch.clamp(render[..., :3] + (1 - alpha) * bg, 0.0, 1.0)
    d = render[..., 3:4]
    depth = torch.where(alpha > 0, d, d.detach().max())
    _, n_cam = dn_ref.gaussian_normals(p["quats"], p["scales"], p["means"], c2w.to(dt))
    nim = G.rasterize_gaussians_legacy(info["means2d"].detach(), info["conics"], n_cam,
                                       torch.sigmoid(p["opacities"]).squeeze(-1), cam["height"], cam["width"], 16,
                                       info["isect_offsets"], info["flatten_ids"])
    nim = nim / nim.norm(dim=-1, keepdim=True)
    return {"rgb": rgb, "depth": depth, "normal": (nim + 1) / 2, "accumulation": alpha}


def perturbed_viewmat(c2w, xi=XI):
    return get_viewmat(compose(c2w.double()[None], exp_map_SE3(xi[None]))[0])


class ViewmatOracle:
    """One fp64 oracle forward with a viewmat that requires grad, differentiated once per route (graph kept)."""

    def __init__(self, params, cam, mode, sh_degree):
        self.vm = perturbed_viewmat(cam["c2w"]).requires_grad_(True)
        self.p = {k: v.detach().double() for k, v in params.items()}
        self.out = oracle_render(self.p, cam, self.vm, cam["c2w"].double(), mode, sh_degree)

    def grad(self, route, mask, use_normal):
        self.vm.grad = None
        o = self.out
        route_loss(o["rgb"], o["depth"], o["normal"], o["accumulation"], route, mask,
                   use_normal=use_normal).backward(retain_graph=True)
        return self.vm.grad.clone()


_ORACLES: dict = {}


def _raw_cases():
    out = []
    for mode in ("classic", "antialiased"):
        for sh in (0, 3):
            for cam_on in ("device", "host"):
                for route in ("rgb", "depth", "normal", "alpha", "all"):
                    if mode == "antialiased" and route == "normal":
                        continue  # one antialiased pass composites normals with the compensated opacity (see below)
                    out.append((mode, sh, cam_on, route))
    return out


@needs_cuda
@pytest.mark.parametrize("mode,sh,cam_on,route", _raw_cases(),
                         ids=[f"{m}-sh{s}-{c}cam-{r}" for m, s, c, r in _raw_cases()])
def test_viewmat_gradient_matches_fp64_oracle(mode, sh, cam_on, route):
    """Raw d(loss)/d(viewmat) at a ragged 81x49 frame, with the viewmat on the device or on the host (then the camera
    reaches the kernels by value: DNR_FLAG_HOST_CAMERA).  The single-pass antialiased render composites the normal image
    with the compensated opacity while the reference's normal pass uses the plain one, so its normal route is left out
    (the model's two-pass mode is covered end to end below)."""
    from dn_splatter_b200 import dn_rasterize

    W, H = 81, 49
    params = make_scene(400, seed=0)
    cam = ring_cameras(5, W, H)[0]
    key = (mode, sh)
    if key not in _ORACLES:
        _ORACLES.clear()
        _ORACLES[key] = ViewmatOracle(params, cam, mode, sh)
    orc = _ORACLES[key]
    mask = region_mask(H, W, "all")
    use_normal = mode == "classic"
    want = orc.grad(route, mask, use_normal)
    assert float(want[:3, :3].norm()) > 0 and float(want[:3, 3].norm()) > 0, "rotation and translation must get a gradient"
    p = {k: v.cuda().requires_grad_(True) for k, v in params.items()}
    c2w = cam["c2w"].cuda()
    K = torch.tensor([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], dtype=torch.float32, device="cuda")
    vm = orc.vm.detach().float().to("cuda" if cam_on == "device" else "cpu").requires_grad_(True)
    out = dn_rasterize(p["means"], p["quats"], p["scales"], p["opacities"], p["features_dc"], p["features_rest"], vm, K, W,
                       H, sh_degree=sh, background=BACKGROUND, c2w=c2w, antialiased=mode == "antialiased")
    route_loss(out.rgb, out.depth, out.normal, out.alpha, route, mask, use_normal=use_normal).backward()
    assert vm.grad.device == vm.device
    got = vm.grad.cpu()
    assert not bool(got[3].any()), "row 3 of the viewmat gets no gradient"
    err = rel_err(got[:3], want[:3])
    assert err <= TOL, f"viewmat gradient rel err {err:.3e} (rotation {rel_err(got[:3, :3], want[:3, :3]):.3e}, " \
                       f"translation {rel_err(got[:3, 3], want[:3, 3]):.3e})"
    # a viewmat that does not require grad: no pose gradient, the same parameter gradients
    g1 = {k: v.grad.clone() for k, v in p.items()}
    for v in p.values():
        v.grad = None
    out = dn_rasterize(p["means"], p["quats"], p["scales"], p["opacities"], p["features_dc"], p["features_rest"],
                       vm.detach(), K, W, H, sh_degree=sh, background=BACKGROUND, c2w=c2w,
                       antialiased=mode == "antialiased")
    route_loss(out.rgb, out.depth, out.normal, out.alpha, route, mask, use_normal=use_normal).backward()
    for k in p:
        assert rel_err(p[k].grad, g1[k]) <= 1e-5, k


def _model(params, mode, n_cams, **cfg_kw):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig

    cfg = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black",
                                camera_optimizer=CameraOptimizerConfig(mode=mode), **cfg_kw)
    m = cfg.setup(device="cuda", num_train_data=n_cams)
    m.load_gaussians(params)
    m.step = 30000
    m.train()
    return m


def _camera(cam, idx):
    from dn_splatter_b200.cameras import Cameras

    return Cameras(cam["c2w"][None], cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["width"], cam["height"],
                   metadata={"cam_idx": idx})


@needs_cuda
@pytest.mark.parametrize("rasterize_mode", ["classic", "antialiased"])
@pytest.mark.parametrize("mode", ["SO3xR3", "SE3"])
def test_pose_gradient_through_the_model_matches_fp64_oracle(mode, rasterize_mode):
    """pose_adjustment.grad through get_outputs / get_loss_dict (default losses: 0.8 L1 + 0.2 SSIM, DN regulariser with
    EdgeAwareLogL1 depth and normal terms) at 81x49, against the same loss on the fp64 oracle with the pose map in fp64.
    Antialiased + normals renders twice; both passes' pose gradients add up."""
    from dn_splatter_b200.dn_model import ssim
    from dn_splatter_b200.losses import DepthLossType

    H, W, idx = 49, 81, 2
    params = make_scene(500, seed=0)
    cam = ring_cameras(5, W, H)[2]
    g = torch.Generator().manual_seed(H * 100 + W)
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    depth[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
    batch = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), "mono_depth": depth,
             "normal": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8)}
    m = _model(params, mode, 4, use_depth_loss=True, depth_lambda=0.2, ssim_lambda=0.2,
               depth_loss_type=DepthLossType.EdgeAwareLogL1, rasterize_mode=rasterize_mode)
    xi = XI.float() * 0.5
    with torch.no_grad():
        m.camera_optimizer.pose_adjustment[idx] = xi.cuda()
    ld = m.get_loss_dict(m.get_outputs(_camera(cam, idx)), {k: v.cuda() for k, v in batch.items()})
    (ld["main_loss"] + ld["scale_reg"]).backward()
    got = m.camera_optimizer.pose_adjustment.grad.cpu().double()
    assert not bool(got[[0, 1, 3]].any())
    # fp64 oracle: the same pose map, the reference's losses
    xi64 = xi.double()[None].requires_grad_(True)
    c2w64 = cam["c2w"].double()
    exp_map = exp_map_SO3xR3 if mode == "SO3xR3" else exp_map_SE3
    vm = get_viewmat(compose(c2w64[None], exp_map(xi64))[0])
    p = {k: v.detach().double().requires_grad_(True) for k, v in params.items()}
    ref = oracle_render(p, cam, vm, c2w64, rasterize_mode)
    gt_img = batch["image"].double() / 255.0
    loss = 0.8 * (gt_img - ref["rgb"]).abs().mean() + 0.2 * (1 - ssim(gt_img.permute(2, 0, 1)[None],
                                                                      ref["rgb"].permute(2, 0, 1)[None]))
    loss = loss + dn_ref.dn_regularization(ref["depth"], batch["mono_depth"].double(), ref["normal"],
                                           batch["normal"].double() / 255.0, p["scales"], gt_img.clamp(min=10 / 255.0),
                                           depth_lambda=0.2, depth_loss_type="EdgeAwareLogL1")
    loss.backward()
    want = xi64.grad[0]
    assert float(want[:3].norm()) > 0 and float(want[3:].norm()) > 0
    err = rel_err(got[idx], want)
    assert err <= TOL, f"pose gradient rel err {err:.3e}: got {got[idx].tolist()} want {want.tolist()}"


@needs_cuda
def test_full_size_translation_gradient_equals_the_sum_of_mean_gradients():
    """1M Gaussians at 1080p, where the oracle is too slow.  For a loss on rgb, depth and alpha (normals rendered, not in
    the loss), moving the camera rigidly is moving every mean the other way: W^T v_t = sum_i v_means_i exactly."""
    from dn_splatter_b200 import dn_rasterize

    W, H = 1920, 1080
    params = make_scene(1_000_000, seed=0)
    cam = ring_cameras(200, W, H)[17]
    p = {k: v.cuda().requires_grad_(True) for k, v in params.items()}
    c2w = cam["c2w"].cuda()
    K = torch.tensor([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], dtype=torch.float32, device="cuda")
    vm = get_viewmat(c2w).detach().requires_grad_(True)
    out = dn_rasterize(p["means"], p["quats"], p["scales"], p["opacities"], p["features_dc"], p["features_rest"], vm, K, W,
                       H, background=BACKGROUND, c2w=c2w)
    g = torch.Generator().manual_seed(1)
    wr, wd, wa = (torch.rand(H, W, c, generator=g).cuda() for c in (3, 1, 1))
    ((out.rgb * wr).sum() + 0.1 * (out.depth * wd).sum() + (out.alpha * wa).sum()).backward()
    Wm = vm.detach().double()[:3, :3]
    lhs = Wm.T @ vm.grad.double()[:3, 3]
    rhs = p["means"].grad.double().sum(0)
    spread = float(p["means"].grad.double().norm(dim=1).sum() / rhs.norm())  # cancellation: sum of |terms| / |sum|
    err = float((lhs - rhs).norm() / rhs.norm())
    print(f"full size: rel err {err:.3e}, sum |v_means_i| / |sum v_means_i| = {spread:.1f}, touched "
          f"{int((p['means'].grad.abs().sum(1) > 0).sum())}")
    assert err <= TOL, (err, spread)


@needs_cuda
def test_captured_step_with_camera_opt_matches_eager_step():
    """GraphedTrainStep with camera optimisation, replayed for views with different cam_idx: the loss, the gradient
    bucket and the pose gradient equal the eager step's."""
    with torch.cuda.stream(torch.cuda.Stream()):
        _captured_body()


def _captured_body():
    from dn_splatter_b200.graph_step import GraphedTrainStep
    from dn_splatter_b200.losses import DepthLossType

    W, H, n_cams = 160, 128, 6
    params = make_scene(4000, seed=0)
    cams = [_camera(c, i) for i, c in enumerate(ring_cameras(n_cams, W, H))]
    g = torch.Generator().manual_seed(5)
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    batch = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda(), "mono_depth": depth.cuda(),
             "normal": torch.rand(H, W, 3, generator=g).cuda()}
    m = _model(params, "SO3xR3", n_cams, use_depth_loss=True, depth_lambda=0.2,
               depth_loss_type=DepthLossType.EdgeAwareLogL1, ssim_lambda=0.0, sync_free=True)
    with torch.no_grad():
        m.camera_optimizer.pose_adjustment.copy_(0.02 * torch.randn(n_cams, 6, generator=g).cuda())
    bucket = m.enable_flat_grads()
    pa = m.camera_optimizer.pose_adjustment
    eager = {}
    for i in (0, 1, 2, 4):
        bucket.zero_()
        pa.grad = None
        ld = m.get_loss_dict(m.get_outputs(cams[i]), dict(batch))
        (ld["main_loss"] + ld["scale_reg"]).backward()
        eager[i] = (float(ld["main_loss"] + ld["scale_reg"]), bucket.flat.clone(), pa.grad.clone())
    del ld
    pa.grad = None
    step = GraphedTrainStep(m, bucket, cams[0], batch, n_slots=2)
    assert pa.grad is not None and not bool(pa.grad.any()), "capture must leave the accumulated pose gradient as it was"
    grad_ptr = pa.grad.data_ptr()
    for i, slot in ((4, 0), (1, 1), (2, 0)):
        pa.grad.zero_()
        loss = step(cams[i], slot)
        torch.cuda.synchronize()
        step.check_capacity(wait=True)
        assert pa.grad.data_ptr() == grad_ptr
        assert abs(float(loss) - eager[i][0]) <= 1e-5 * max(1.0, abs(eager[i][0])), (i, float(loss), eager[i][0])
        rel = float((bucket.flat - eager[i][1]).norm() / (eager[i][1].norm() + 1e-30))
        assert rel < 1e-4, (i, rel)
        rel = float((pa.grad - eager[i][2]).norm() / eager[i][2].norm())
        assert rel < 1e-4 and bool(pa.grad[i].abs().gt(0).all()), (i, rel)
    # replays accumulate into the same buffer, as eager backwards do
    step(cams[1], 1)
    torch.cuda.synchronize()
    rel = float((pa.grad - eager[2][2] - eager[1][2]).norm() / (eager[1][2] + eager[2][2]).norm())
    assert rel < 1e-4, rel
    from dn_splatter_b200.cameras import Cameras

    c = ring_cameras(n_cams, W, H)[3]
    with pytest.raises(ValueError, match="cam_idx"):
        step(Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H), 0)


def _rotation_angle(R):
    return float(torch.arccos(((torch.trace(R) - 1) / 2).clamp(-1.0, 1.0)))


RECOVERY_STEPS = 800


@needs_cuda
def test_pose_recovery_from_perturbed_cameras():
    """Targets rendered from the true poses; four training cameras start about 1 degree and 2 % of the scene radius off.
    With the Gaussians frozen, Adam on the poses alone (lr 1e-3, no accumulation) brings every view's rotation and
    translation error below a quarter of its start value within RECOVERY_STEPS steps."""
    W, H, n_cams = 160, 128, 4
    params = make_scene(20000, seed=0)
    ring = ring_cameras(n_cams, W, H)
    m = _model(params, "SO3xR3", n_cams)
    for t in m.gauss_params.values():
        t.requires_grad_(False)
    gen = torch.Generator().manual_seed(11)
    true_c2w, cams, targets = [], [], []
    radius = 5.0  # make_scene: means in [-5, 5]^3
    for i, c in enumerate(ring):
        true_c2w.append(c["c2w"].double())
        m.eval()
        with torch.no_grad():
            o = m.get_outputs(_camera(c, i))
        targets.append((o["rgb"].detach().clone(), o["depth"].detach().clone()))
        axis = torch.randn(3, generator=gen, dtype=torch.float64)
        tdir = torch.randn(3, generator=gen, dtype=torch.float64)
        delta = torch.cat([tdir / tdir.norm() * 0.02 * radius, axis / axis.norm() * math.radians(1.0)])
        bad = compose(c["c2w"].double()[None], exp_map_SE3(delta[None]))[0].float()
        cams.append(_camera(dict(c, c2w=bad), i))
    m.train()
    opt = torch.optim.Adam(m.camera_optimizer.parameters(), lr=1e-3, eps=1e-15)

    def errors():
        out = []
        with torch.no_grad():
            adj = m.camera_optimizer(slice(0, n_cams)).double().cpu()
            for i in range(n_cams):
                est = compose(cams[i].camera_to_worlds.double(), adj[i:i + 1])[0]
                out.append((_rotation_angle(est[:, :3].T @ true_c2w[i][:, :3]), float((est[:, 3] - true_c2w[i][:, 3]).norm())))
        return out

    start, trace = errors(), []
    for s in range(RECOVERY_STEPS):
        if s % 100 == 0:
            trace.append((s, max(e[0] / e0[0] for e, e0 in zip(errors(), start)),
                          max(e[1] / e0[1] for e, e0 in zip(errors(), start))))
        i = s % n_cams
        opt.zero_grad(set_to_none=False)
        out = m.get_outputs(cams[i])
        loss = (out["rgb"] - targets[i][0]).abs().mean() + 0.1 * (out["depth"] - targets[i][1]).abs().mean()
        loss.backward()
        opt.step()
    end = errors()
    print("pose recovery (rotation rad, translation) start", start, "end", end)
    print("pose recovery: (step, worst rotation error / start, worst translation error / start)", trace)
    for (r0, t0), (r1, t1) in zip(start, end):
        assert r1 < 0.25 * r0 and t1 < 0.25 * t0, (start, end)
