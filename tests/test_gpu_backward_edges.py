"""The rasterizer backward against the fp64 oracle on the branches the easy-path parity test
(test_gpu_parity.py::test_backward_matches_fp64_oracle) never reaches: ragged frames (odd row counts in the last tile
split a lane's pixel pair), alpha-clamped pixels, the antialiased compensation, active SH degrees below the stored one,
Jacobian-clamped Gaussians, lists several chunks deep, off-centre intrinsics and the activated-input path.

Each case differentiates one output route (rgb, depth, normal, alpha or their sum) over one pixel region (the whole
frame, the last partial tile row / column, or the rest) and bounds the norm-wise relative error of every parameter
group and of means2d.absgrad by 1e-3, the bound of the easy-path test.  Each case also asserts that its scene really
takes the branch it is named for: a scene that does not checks nothing."""
import pytest
import torch

from oracle import gsplat_ref as G
from tests.helpers import cuda_outputs, frac_close, oracle_outputs, scene_and_camera

pytestmark = pytest.mark.gpu
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")

GROUPS = ("means", "quats", "scales", "opacities", "features_dc", "features_rest")
ROUTES = ("rgb", "depth", "normal", "alpha", "all")
TOL = 1e-3
TILE = 16


def region_mask(H, W, region):
    """`edge`: the pixels of the last partial tile row and column; `interior`: the others."""
    edge = torch.zeros(H, W, dtype=torch.bool)
    if H % TILE:
        edge[H - H % TILE:, :] = True
    if W % TILE:
        edge[:, W - W % TILE:] = True
    return {"all": torch.ones_like(edge), "edge": edge, "interior": ~edge}[region]


def route_loss(rgb, depth, normal, alpha, route, mask, seed=0, use_normal=True):
    """Seeded random-weight sum of one output over the pixels of `mask` ("all": every output, depth weighted 0.1;
    without the normal image when `use_normal` is False)."""
    g = torch.Generator().manual_seed(seed)
    H, W = mask.shape
    w = {"rgb": torch.rand(H, W, 3, generator=g), "depth": torch.rand(H, W, 1, generator=g),
         "normal": torch.rand(H, W, 3, generator=g), "alpha": torch.rand(H, W, 1, generator=g)}
    m = mask[..., None]
    terms = {k: (x * (w[k] * m).to(x)).sum() for k, x in (("rgb", rgb), ("depth", depth), ("normal", normal),
                                                          ("alpha", alpha))}
    if route == "all":
        return terms["rgb"] + 0.1 * terms["depth"] + (terms["normal"] if use_normal else 0.0) + terms["alpha"]
    return terms[route]


def rel_err(got, want):
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    den = float(want.norm())
    return float((got - want).norm()) / den if den > 0 else float(got.norm())


class Oracle:
    """One fp64 oracle forward, differentiated once per (route, region): the graph is kept."""

    def __init__(self, params, cam, **kw):
        self.params, self.cam = params, cam
        self.p, self.out = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True, collect_absgrad=True, **kw)

    def grads(self, route, mask, use_normal=True):
        for t in self.p.values():
            t.grad = None
        for h in self.out["info"]["hooks"]:
            h[1].grad = None
        o = self.out
        route_loss(o["rgb"], o["depth"], o["normal"], o["accumulation"], route, mask,
                   use_normal=use_normal).backward(retain_graph=True)
        info = o["info"]
        g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in self.p.items()}
        g["absgrad"] = G.absgrad_from_hooks(info["hooks"], info["conics"], info["opacities"], self.p["means"].shape[0])
        return g


_ORACLES: dict = {}


def oracle_for(key, params, cam, **kw) -> Oracle:
    """The oracle of scene `key`, kept for the other routes / regions / list settings of the same scene."""
    if key not in _ORACLES:
        if len(_ORACLES) >= 4:
            _ORACLES.pop(next(iter(_ORACLES)))
        _ORACLES[key] = Oracle(params, cam, **kw)
    return _ORACLES[key]


def cuda_grads(params, cam, route, mask, use_normal=True, **kw):
    p, out = cuda_outputs(params, cam, requires_grad=True, **kw)
    route_loss(out.rgb, out.depth, out.normal, out.alpha, route, mask, use_normal=use_normal).backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).cpu() for k, v in p.items()}
    g["absgrad"] = out.means2d.absgrad.cpu()
    return g, out


def compare(oracle: Oracle, route, region, rows=None, groups=GROUPS + ("absgrad",), use_normal=True, **cuda_kw):
    """Per-group norm-wise relative error of the CUDA gradients of `route` over `region` (restricted to the Gaussian
    indices `rows` if given) against the fp64 oracle.  Returns (errors, oracle gradients, cuda gradients, cuda output)."""
    H, W = oracle.cam["height"], oracle.cam["width"]
    mask = region_mask(H, W, region)
    want = oracle.grads(route, mask, use_normal)
    got, out = cuda_grads(oracle.params, oracle.cam, route, mask, use_normal, **cuda_kw)
    sel = (lambda t: t) if rows is None else (lambda t: t[rows])
    errs = {k: rel_err(sel(got[k]), sel(want[k])) for k in groups}
    return errs, want, got, out


def assert_within(errs, tol=TOL, what=""):
    bad = {k: f"{v:.3e}" for k, v in errs.items() if not v <= tol}
    assert not bad, f"{what}: relative gradient error above {tol:g}: {bad}"


def assert_nontrivial(want, route, groups=("means", "opacities")):
    """The loss must actually reach the parameters: a zero oracle gradient compares nothing."""
    for k in groups:
        assert float(want[k].norm()) > 0, f"{route}: the oracle gradient of {k} is zero"


# ---------------------------------------------------------------------------------------------------- ragged frames

RAGGED = [(81, 49), (75, 53), (13, 7)]  # (W, H): 1-px last tile column and row; 11 x 5; smaller than one tile
LISTS = {"shift0": dict(list_shift=0), "shift2": dict(list_shift=2), "shift3": dict(list_shift=3),
         "exact": dict(exact_lists=True)}
RAGGED_CASES = [(wh, region) for wh in RAGGED for region in ("edge", "interior") if min(wh) >= TILE or region == "edge"]


@needs_cuda
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("lists", list(LISTS))
@pytest.mark.parametrize("wh,region", RAGGED_CASES, ids=[f"{w}x{h}-{r}" for (w, h), r in RAGGED_CASES])
def test_ragged_frames(wh, region, lists, route):
    """raster_bwd evaluates rows ly + {0, 2} and ly + {4, 6} of a lane as two pixel pairs: with an odd row count in the
    last tile one pixel of a pair is inside the image and its partner is not (clamped loads, masked contributions)."""
    W, H = wh
    params, cam = scene_and_camera(400, W, H, view=0)
    assert (H % TILE) % 2 == 1, "the last tile row must hold an odd number of rows"
    orc = oracle_for(("ragged", W, H), params, cam, predict_normals=True)
    mask = region_mask(H, W, region)
    covered = orc.out["accumulation"][..., 0].detach() > 0
    assert int((covered & mask).sum()) >= min(20, int(mask.sum())), "the region must receive splats"
    errs, want, _, _ = compare(orc, route, region, render_normals=True, **LISTS[lists])
    assert_nontrivial(want, route)
    assert_within(errs, what=f"{W}x{H} {region} {lists} {route}")


# ---------------------------------------------------------------------------------------------------- alpha clamp


def clamp_scene(n=1000, W=96, H=80, seed=4):
    """Every other Gaussian at opacity in [0.9992, 0.9999], its mean moved along its camera ray's plane so that it
    projects onto a pixel centre: alpha = min(opacity * vis, 0.999) then clamps at that pixel (vis = 1 there, and at most
    1 - 0.999 / 0.9992 below 1 is needed).  Small Gaussians leave enough of them unoccluded."""
    from oracle import dn_ref

    params, cam = scene_and_camera(n, W, H, view=1, seed=seed, scale_mult=0.3)
    g = torch.Generator().manual_seed(seed + 100)
    hi = torch.arange(0, n, 2)
    params["opacities"][hi] = torch.logit(0.9992 + 0.0007 * torch.rand(hi.numel(), 1, generator=g, dtype=torch.float64)).float()
    vm = dn_ref.get_viewmat(cam["c2w"].double())
    xc = params["means"].double() @ vm[:3, :3].T + vm[:3, 3]
    u = cam["fx"] * xc[:, 0] / xc[:, 2] + cam["cx"]
    v = cam["fy"] * xc[:, 1] / xc[:, 2] + cam["cy"]
    xc[:, 0] = (u.floor() + 0.5 - cam["cx"]) * xc[:, 2] / cam["fx"]
    xc[:, 1] = (v.floor() + 0.5 - cam["cy"]) * xc[:, 2] / cam["fy"]
    params["means"][hi] = ((xc - vm[:3, 3]) @ vm[:3, :3])[hi].float()
    return params, cam, hi


def tile_splats(out, W, H):
    """For each 16x16 tile of the oracle's render: (rows, cols, list positions, sigma[P, L], opacity * vis[P, L]) of every
    pixel against every entry of the tile's sorted list, and the pixels' last_ids [P, 1]."""
    info = out["info"]
    offs = info["isect_offsets"].tolist() + [info["flatten_ids"].shape[0]]
    m2, con, op = info["means2d"].detach(), info["conics"].detach(), info["opacities"].detach()
    last = info["last_ids"].long()
    tw = (W + TILE - 1) // TILE
    for t in range(len(offs) - 1):
        lo, hi = offs[t], offs[t + 1]
        if hi <= lo:
            continue
        y0, x0 = (t // tw) * TILE, (t % tw) * TILE
        y1, x1 = min(y0 + TILE, H), min(x0 + TILE, W)
        ys, xs = torch.meshgrid(torch.arange(y0, y1, dtype=m2.dtype) + 0.5, torch.arange(x0, x1, dtype=m2.dtype) + 0.5,
                                indexing="ij")
        g = info["flatten_ids"][lo:hi].long()
        dx = m2[g, 0][None] - xs.reshape(-1, 1)
        dy = m2[g, 1][None] - ys.reshape(-1, 1)
        sigma = 0.5 * (con[g, 0][None] * dx * dx + con[g, 2][None] * dy * dy) + con[g, 1][None] * dx * dy
        yield (slice(y0, y1), slice(x0, x1), torch.arange(lo, hi)[None], sigma, op[g][None] * torch.exp(-sigma),
               last[y0:y1, x0:x1].reshape(-1, 1))


def clamped_pixels(out, W, H):
    """Pixels that composited a splat with opacity * vis > 0.999, from the oracle's lists and last_ids."""
    hit = torch.zeros(H, W, dtype=torch.bool)
    for rows, cols, pos, sigma, ov, last in tile_splats(out, W, H):
        used = (pos <= last) & (sigma >= 0) & (ov > G.ALPHA_MAX)
        hit[rows, cols] = used.any(1).reshape(hit[rows, cols].shape)
    return hit


def stopped_pixels(out, W, H):
    """Pixels that stopped under the T * (1 - alpha) <= 1e-4 rule: the first entry after the pixel's last composited one
    that would have been valid there (sigma >= 0, alpha >= 1/255) would have taken the final transmittance to 1e-4 or
    below.  Returns [H, W] int64: the number of list entries left behind such a stop, -1 where the pixel did not stop."""
    left = torch.full((H, W), -1, dtype=torch.int64)
    T_final = 1.0 - out["accumulation"][..., 0].detach()
    for rows, cols, pos, sigma, ov, last in tile_splats(out, W, H):
        alpha = torch.clamp(ov, max=G.ALPHA_MAX)
        later = (pos > last) & (sigma >= 0) & (alpha >= G.ALPHA_MIN)
        first = torch.argmax(later.to(torch.int8), dim=1, keepdim=True)
        a_next = torch.gather(alpha, 1, first)[:, 0]
        stop = later.any(1) & (T_final[rows, cols].reshape(-1) * (1.0 - a_next) <= G.T_STOP)
        n_left = pos[0, -1] - last[:, 0]
        left[rows, cols] = torch.where(stop, n_left, torch.full_like(n_left, -1)).reshape(left[rows, cols].shape)
    return left


@needs_cuda
@pytest.mark.parametrize("route", ["rgb", "alpha", "all"])
def test_alpha_clamp(route):
    """alpha = min(opacity * vis, 0.999): a clamped pixel passes no gradient to sigma or opacity (the `slow` fix-up of
    raster_bwd) while its transmittance still uses 0.999."""
    params, cam, hi = clamp_scene()
    orc = oracle_for(("clamp",), params, cam, predict_normals=True)
    n_clamped = int(clamped_pixels(orc.out, cam["width"], cam["height"]).sum())
    assert n_clamped >= 100, f"only {n_clamped} pixels composite a clamped alpha"
    errs, want, _, _ = compare(orc, route, "all", rows=hi)
    assert_nontrivial({k: v[hi] for k, v in want.items()}, route)
    assert_within(errs, what=f"clamped Gaussians, {route}")
    errs, _, _, _ = compare(orc, route, "all")
    assert_within(errs, what=f"all Gaussians, {route}")


# ---------------------------------------------------------------------------------------------------- antialiased


@needs_cuda
@pytest.mark.parametrize("normals", [True, False])
@pytest.mark.parametrize("route", ["rgb", "depth", "alpha", "all"])
def test_antialiased(normals, route):
    """rasterize_mode="antialiased": opacity x compensation, and the hand-derived compensation gradient.  With normals on,
    one dn_rasterize pass composites the normal image with the compensated opacity too, whereas the reference's normal
    pass uses the plain opacity (the model renders twice for that: tests/test_gpu_model.py); so the normal image is
    left out of the loss here and the NORMALS kernels are checked on the colour / depth / alpha routes."""
    params, cam = scene_and_camera(1000, 96, 80, view=1)
    orc = oracle_for(("aa", normals), params, cam, predict_normals=normals, rasterize_mode="antialiased")
    _, out = cuda_outputs(params, cam, antialiased=True, render_normals=normals, exact_lists=True)
    ref_info = orc.out["info"]
    vis = (out.radii.cpu() > 0) & (ref_info["radii"] > 0)
    comp_ref = ref_info["compensations"].detach()[vis]
    comp = out.info["compensations"].cpu().double()[vis]
    assert float((comp_ref < 0.99).double().mean()) > 0.5, "compensations must be well below 1 on visible Gaussians"
    assert rel_err(comp, comp_ref) <= 1e-5, f"compensations: {rel_err(comp, comp_ref):.3e}"
    o = orc.out
    for name, got, want in (("rgb", out.rgb, o["rgb"]), ("alpha", out.alpha, o["accumulation"])):
        frac, mx = frac_close(got, want, atol=1e-4)
        assert frac >= 0.999 and mx <= 2e-2, f"{name}: {frac:.5f} of pixels within 1e-4, max err {mx:.3e}"
    frac, mx = frac_close(out.depth, o["depth"], atol=1e-4, rtol=1e-4)
    assert frac >= 0.999, f"depth: {frac:.5f} within tol, max err {mx:.3e}"
    errs, want, _, _ = compare(orc, route, "all", use_normal=False, antialiased=True, render_normals=normals)
    assert_nontrivial(want, route)
    assert_within(errs, what=f"antialiased normals={normals} {route}")


# ---------------------------------------------------------------------------------------------------- SH degrees


@needs_cuda
@pytest.mark.parametrize("route", ["rgb", "all"])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_active_sh_degree_below_stored(degree, route):
    """Training runs at active degree 0, 1, 2 for its first 3000 steps with all 16 bases stored: the bases above the
    active degree take no part in the colour and must receive exactly zero gradient."""
    params, cam = scene_and_camera(1000, 128, 80, view=2)
    assert params["features_rest"].shape[1] == 15
    orc = oracle_for(("sh", degree), params, cam, sh_degree=degree, predict_normals=True)
    errs, want, got, _ = compare(orc, route, "all", sh_degree=degree)
    assert_nontrivial(want, route, groups=("means", "features_dc"))
    k = (degree + 1) ** 2 - 1
    assert float(got["features_rest"][:, k:].abs().sum()) == 0.0, "inactive SH bases received a gradient"
    if degree > 0:
        assert float(want["features_rest"][:, :k].norm()) > 0
    assert_within(errs, what=f"sh degree {degree} {route}")


# ---------------------------------------------------------------------------------------------------- Jacobian clamp


def inside_camera(W=96, H=80):
    from dn_splatter_b200.synthetic import look_at_c2w

    c2w = look_at_c2w(torch.tensor([3.0, 0.0, 0.5]), torch.zeros(3), torch.tensor([0.0, 0.0, 1.0]))
    return {"c2w": c2w, "fx": 0.9 * W, "fy": 0.9 * W, "cx": W / 2.0, "cy": H / 2.0, "width": W, "height": H}


@needs_cuda
@pytest.mark.parametrize("route", ["rgb", "depth", "all"])
def test_jacobian_clamp(route):
    """A camera inside the cloud: Gaussians beyond 1.3 tan(fov) off axis are still visible, and their projection
    Jacobian uses the clamped mean, whose derivative goes to the camera-space depth instead of x / y."""
    from dn_splatter_b200.synthetic import make_scene
    from oracle import dn_ref

    params = make_scene(3000, seed=1)
    cam = inside_camera()
    orc = oracle_for(("jac",), params, cam, predict_normals=True)
    vm = dn_ref.get_viewmat(cam["c2w"].double())
    xc = params["means"].double() @ vm[:3, :3].T + vm[:3, 3]
    lim_x = 1.3 * 0.5 * cam["width"] / cam["fx"]
    lim_y = 1.3 * 0.5 * cam["height"] / cam["fy"]
    clamped = ((xc[:, 0] / xc[:, 2]).abs() > lim_x) | ((xc[:, 1] / xc[:, 2]).abs() > lim_y)
    want = orc.grads(route, region_mask(cam["height"], cam["width"], "all"))
    live = clamped & (orc.out["info"]["radii"] > 0) & (want["means"].abs().sum(-1) > 0)
    rows = torch.nonzero(live).flatten()
    assert rows.numel() >= 20, f"only {rows.numel()} visible Jacobian-clamped Gaussians receive a gradient"
    errs, _, _, _ = compare(orc, route, "all", rows=rows, groups=("means", "scales", "quats"))
    assert_within(errs, what=f"Jacobian-clamped Gaussians, {route}")
    errs, _, _, _ = compare(orc, route, "all")
    assert_within(errs, what=f"all Gaussians, {route}")


# ---------------------------------------------------------------------------------------------------- deep lists


@needs_cuda
@pytest.mark.parametrize("route", ROUTES)
def test_deep_lists(route):
    """Per-tile lists several 128-entry chunks deep, walked back to front, with pixels that stop under the
    T * (1 - alpha) <= 1e-4 rule more than one chunk before the end of their list."""
    params, cam = scene_and_camera(8000, 96, 80, view=1)
    orc = oracle_for(("deep",), params, cam, predict_normals=True)
    errs, want, _, out = compare(orc, route, "all", exact_lists=True)
    info = orc.out["info"]
    for who, offs, total in (("cuda", out.info["tile_offsets"].cpu().long()[:-1], out.info["n_isects"]),
                             ("oracle", info["isect_offsets"].long(), info["flatten_ids"].shape[0])):
        longest = int(torch.diff(offs, append=torch.tensor([total])).max())
        assert longest > 3 * 128, f"{who}: longest per-tile list {longest}"
    left = stopped_pixels(orc.out, cam["width"], cam["height"])
    assert int((left > 128).sum()) >= 100, "pixels must stop compositing more than one chunk before the end of their list"
    assert_nontrivial(want, route)
    assert_within(errs, what=f"deep lists {route}")


# ---------------------------------------------------------------------------------------------------- intrinsics


@needs_cuda
@pytest.mark.parametrize("route", ROUTES)
def test_off_centre_intrinsics(route):
    """fx != fy and a principal point away from the frame centre."""
    params, cam = scene_and_camera(1000, 96, 80, view=3)
    cam = dict(cam, fx=1.1 * cam["fx"], fy=0.8 * cam["fy"], cx=0.37 * cam["width"], cy=0.62 * cam["height"])
    orc = oracle_for(("intr",), params, cam, predict_normals=True)
    errs, want, _, _ = compare(orc, route, "all")
    assert_nontrivial(want, route)
    assert_within(errs, what=f"off-centre intrinsics {route}")


# ---------------------------------------------------------------------------------------------------- activated inputs


@needs_cuda
@pytest.mark.parametrize("normals", [True, False])
def test_activated_inputs_match_raw_through_the_chain_rule(normals):
    """DNR_FLAG_ACTIVATED takes exp(scales) and sigmoid(opacities) as given: its gradients, pushed through the
    activations, are the raw path's gradients."""
    params, cam = scene_and_camera(1000, 96, 80, view=1)
    mask = region_mask(cam["height"], cam["width"], "all")
    raw, _ = cuda_grads(params, cam, "all", mask, render_normals=normals)
    act_params = dict(params, scales=torch.exp(params["scales"]), opacities=torch.sigmoid(params["opacities"]))
    act, _ = cuda_grads(act_params, cam, "all", mask, render_normals=normals, activated=True)
    sig = torch.sigmoid(params["opacities"])
    chained = dict(act, scales=act["scales"] * torch.exp(params["scales"]), opacities=act["opacities"] * sig * (1 - sig))
    errs = {k: rel_err(chained[k], raw[k]) for k in GROUPS + ("absgrad",)}
    assert_within(errs, tol=1e-5, what=f"activated vs raw, normals={normals}")
