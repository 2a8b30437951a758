"""BASELINE.json configs[0]: 1k Gaussians, one 128x128 view — the reference's pure-PyTorch projection + compositing +
depth/normal regularisers on the CPU (plumbing, no GPU).  Checks the oracle itself: finite outputs and loss, fp32 vs
fp64 agreement, integer outputs independent of precision, and a finite-difference check of the fp64 gradient."""
import pytest
import torch

from tests.helpers import oracle_outputs, scene_and_camera

from oracle import dn_ref


def _loss(out, p, gt_depth, gt_normal, gt_img):
    reg = dn_ref.dn_regularization(out["depth"], gt_depth, out["normal"], gt_normal, p["scales"], gt_img, depth_lambda=0.2)
    return (out["rgb"] - gt_img).abs().mean() + reg


def test_c1_oracle_forward_backward_is_finite_and_precision_consistent():
    params, cam = scene_and_camera(1000, 128, 128, view=1)
    g = torch.Generator().manual_seed(7)
    gt_img = torch.rand(128, 128, 3, generator=g).clamp(min=10 / 255.0)
    gt_depth = 2 + 6 * torch.rand(128, 128, 1, generator=g)
    gt_normal = torch.rand(128, 128, 3, generator=g)
    p32, o32 = oracle_outputs(params, cam, requires_grad=True)
    p64, o64 = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True)
    for k in ("rgb", "depth", "normal", "surface_normal", "accumulation"):
        assert torch.isfinite(o32[k]).all(), k
        frac = ((o32[k].double() - o64[k]).abs() <= 1e-4 + 1e-4 * o64[k].abs()).double().mean()
        assert frac > 0.999, (k, float(frac))
    # integer outputs do not depend on the precision except for ceil() flips on the radius (none expected at this size)
    assert (o32["info"]["radii"] != o64["info"]["radii"]).float().mean() < 2e-3
    l32 = _loss(o32, p32, gt_depth, gt_normal, gt_img)
    l64 = _loss(o64, p64, gt_depth.double(), gt_normal.double(), gt_img.double())
    assert torch.isfinite(l32) and abs(float(l32) - float(l64)) < 1e-4 * max(1.0, abs(float(l64)))
    l32.backward()
    l64.backward()
    for k in p32:
        assert torch.isfinite(p32[k].grad).all(), k
        rel = (p32[k].grad.double() - p64[k].grad).norm() / (p64[k].grad.norm() + 1e-30)
        assert rel < 5e-3, (k, float(rel))


@pytest.mark.parametrize("name,idx", [("means", (10, 2)), ("scales", (3, 0)), ("opacities", (7, 0)), ("features_dc", (5, 1))])
def test_c1_oracle_fp64_gradient_matches_finite_differences(name, idx):
    params, cam = scene_and_camera(60, 48, 40, view=2)
    # pick a Gaussian that is visible so the derivative is not trivially zero
    _, probe = oracle_outputs(params, cam, dtype=torch.float64)
    vis = torch.nonzero(probe["info"]["radii"] > 0).flatten()
    gi = int(vis[idx[0] % len(vis)])
    w = torch.rand(40, 48, 3, generator=torch.Generator().manual_seed(1)).double()
    # empty pixels carry depth.detach().max() (quirk B4): the reference detaches it, a finite difference would not
    covered = (probe["accumulation"] > 0).double()

    # the normal pass sees DETACHED means2d (quirk B3, dn_model.py:562): its dependence on `means` is real but carries no
    # gradient in the reference, so it is left out of the objective when differentiating w.r.t. means
    with_normal = name != "means"

    def total(o):
        t = (o["rgb"] * w).sum() + 0.1 * (o["depth"] * covered).sum() + o["accumulation"].sum()
        return t + (o["normal"] * w).sum() if with_normal else t

    def f(delta):
        q = {k: v.clone().double() for k, v in params.items()}
        q[name][gi, idx[1]] += delta
        _, o = oracle_outputs(q, cam, dtype=torch.float64)
        return float(total(o))

    p, o = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True)
    total(o).backward()
    analytic = float(p[name].grad[gi, idx[1]])
    h = 1e-5
    numeric = (f(h) - f(-h)) / (2 * h)
    assert abs(analytic - numeric) <= 1e-4 * max(1.0, abs(numeric)) + 1e-6, (analytic, numeric)


def _fd_check(params, cam, name, gi, comp, h=1e-5, **kw):
    """fp64 autograd of the oracle vs a central difference, for parameter entry params[name][(gi,) + comp]; the
    objective weights every output (rgb, covered depth, alpha, and the normal image except for `means`, quirk B3)."""
    H, W = cam["height"], cam["width"]
    _, probe = oracle_outputs(params, cam, dtype=torch.float64, **kw)
    w = torch.rand(H, W, 3, generator=torch.Generator().manual_seed(1)).double()
    covered = (probe["accumulation"] > 0).double()
    with_normal = name != "means"

    def total(o):
        t = (o["rgb"] * w).sum() + 0.1 * (o["depth"] * covered).sum() + o["accumulation"].sum()
        return t + (o["normal"] * w).sum() if with_normal else t

    def f(delta):
        q = {k: v.clone().double() for k, v in params.items()}
        q[name][(gi,) + comp] += delta
        return float(total(oracle_outputs(q, cam, dtype=torch.float64, **kw)[1]))

    p, o = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True, **kw)
    total(o).backward()
    analytic = float(p[name].grad[(gi,) + comp])
    numeric = (f(h) - f(-h)) / (2 * h)
    assert numeric != 0.0, "the entry must influence the objective"
    assert abs(analytic - numeric) <= 1e-4 * max(1.0, abs(numeric)) + 1e-6, (analytic, numeric)


def _visible(params, cam, k, **kw):
    _, probe = oracle_outputs(params, cam, dtype=torch.float64, **kw)
    vis = torch.nonzero(probe["info"]["radii"] > 0).flatten()
    return int(vis[k % len(vis)])


@pytest.mark.parametrize("name,k,comp", [("opacities", 7, (0,)), ("scales", 3, (1,)), ("quats", 10, (2,)), ("quats", 4, (0,))])
def test_oracle_antialiased_gradient_matches_finite_differences(name, k, comp):
    """rasterize_mode="antialiased": opacity x compensation, compensation = sqrt(det(cov) / det(cov + 0.3 I))."""
    params, cam = scene_and_camera(60, 48, 40, view=2)
    gi = _visible(params, cam, k, rasterize_mode="antialiased")
    _fd_check(params, cam, name, gi, comp, rasterize_mode="antialiased")


@pytest.mark.parametrize("degree", [1, 2])
@pytest.mark.parametrize("name", ["means", "features_rest"])
def test_oracle_low_sh_degree_gradient_matches_finite_differences(degree, name):
    """Active SH degree 1 and 2 with all 16 bases stored (the first 3000 training steps)."""
    params, cam = scene_and_camera(60, 48, 40, view=2)
    gi = _visible(params, cam, 5, sh_degree=degree)
    comp = (1,) if name == "means" else ((degree + 1) ** 2 - 2, 0)  # the highest active basis
    _fd_check(params, cam, name, gi, comp, sh_degree=degree)


def test_oracle_opacity_gradient_of_alpha_clamped_gaussian_matches_finite_differences():
    """The nearest visible Gaussian, moved to project onto a pixel centre at opacity 0.9995: its alpha clamps to 0.999
    at that pixel (no opacity gradient there) and not elsewhere.  The step is chosen so that no pixel's opacity x vis
    crosses 0.999 or 1/255."""
    from oracle import dn_ref, gsplat_ref as G

    params, cam = scene_and_camera(60, 48, 40, view=2)
    _, probe = oracle_outputs(params, cam, dtype=torch.float64)
    info = probe["info"]
    vis = torch.nonzero(info["radii"] > 0).flatten()
    gi = int(vis[torch.argmin(info["depths"][vis])])
    vm = dn_ref.get_viewmat(cam["c2w"].double())
    xc = params["means"][gi].double() @ vm[:3, :3].T + vm[:3, 3]
    u = (cam["fx"] * xc[0] / xc[2] + cam["cx"]).clamp(1, cam["width"] - 2)
    v = (cam["fy"] * xc[1] / xc[2] + cam["cy"]).clamp(1, cam["height"] - 2)
    xc[0] = (u.floor() + 0.5 - cam["cx"]) * xc[2] / cam["fx"]
    xc[1] = (v.floor() + 0.5 - cam["cy"]) * xc[2] / cam["fy"]
    params = {k: t.clone() for k, t in params.items()}
    params["means"][gi] = ((xc - vm[:3, 3]) @ vm[:3, :3]).float()
    op = 0.9995
    params["opacities"][gi] = torch.logit(torch.tensor(op, dtype=torch.float64)).float()
    op = float(torch.sigmoid(params["opacities"][gi].double()))
    # opacity x vis of this Gaussian at every pixel centre
    _, probe = oracle_outputs(params, cam, dtype=torch.float64)
    info = probe["info"]
    ys, xs = torch.meshgrid(torch.arange(cam["height"], dtype=torch.float64) + 0.5,
                            torch.arange(cam["width"], dtype=torch.float64) + 0.5, indexing="ij")
    dx, dy = info["means2d"][gi, 0] - xs, info["means2d"][gi, 1] - ys
    a, b, c = info["conics"][gi]
    ov = op * torch.exp(-(0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy))
    centre = (int(info["means2d"][gi, 1]), int(info["means2d"][gi, 0]))
    assert float(ov[centre]) > G.ALPHA_MAX, "the centre pixel must clamp"
    assert float(probe["accumulation"][centre]) >= G.ALPHA_MAX, "the centre pixel must composite the clamped alpha"
    # d(ov) = ov (1 - op) d(logit): keep it well inside the distance to both kinks
    margin = float(torch.minimum((ov - G.ALPHA_MAX).abs(), (ov - G.ALPHA_MIN).abs()).min())
    h = min(1e-5, 0.1 * margin / (1.0 - op))
    assert h >= 1e-8, f"a pixel sits {margin:.2e} from a kink: no usable step"
    _fd_check(params, cam, "opacities", gi, (0,), h=h)
