"""GPU parity tests: libdnr_b200.so (through the C ABI / dn_rasterize) against the CPU oracle on the same
seeded scenes.  Tolerances (SURVEY.md §8c):
  * radii, tiles_per_gauss, sorted (tile, depth, id) lists, tile offsets: BIT-EXACT (activated-input path,
    where both sides see identical fp32 inputs);
  * per-Gaussian floats: <= 1e-5 relative;
  * images: <= 1e-4 abs for all but a handful of pixels whose alpha sits on the 1/255 or T<=1e-4 thresholds
    (`__expf` vs torch.exp flips the branch; a flip changes a pixel by at most ~1/255) — at least 99.9 % of
    pixels within 1e-4 and every pixel within 2e-2;
  * gradients: <= 1e-3 relative (norm-wise) against the fp64 oracle.
"""
import pytest
import torch

from tests.helpers import cuda_outputs, frac_close, oracle_outputs, scene_and_camera

pytestmark = pytest.mark.gpu

needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")

CASES = [
    dict(n=1000, width=128, height=128, view=1),  # BASELINE config C1 shape
    dict(n=3000, width=200, height=136, view=3),  # width not a multiple of 16
    dict(n=400, width=75, height=53, view=0),  # ragged both ways
]


def _activated(params):
    p = dict(params)
    p["quats"] = params["quats"] / params["quats"].norm(dim=-1, keepdim=True)
    p["scales"] = torch.exp(params["scales"])
    p["opacities"] = torch.sigmoid(params["opacities"])
    return p


@needs_cuda
@pytest.mark.parametrize("case", CASES)
def test_projection_and_binning_bit_exact(case):
    from oracle import dn_ref, gsplat_ref as G

    params, cam = scene_and_camera(**case)
    act = _activated(params)
    W, H = cam["width"], cam["height"]
    vm = dn_ref.get_viewmat(cam["c2w"])
    K = dn_ref.intrinsics(cam["fx"], cam["fy"], cam["cx"], cam["cy"])
    proj = G.project_gaussians(act["means"], act["quats"], act["scales"], vm, K, W, H)
    tpg, isect_ids, flat, offs, _ = G.isect_tiles(proj["means2d"], proj["radii"], proj["depths"], 16, W, H)

    _, out = cuda_outputs(act, cam, activated=True, viewmat=vm, exact_lists=True)
    assert torch.equal(out.radii.cpu(), proj["radii"]), "radii must be bit-exact"
    assert torch.equal(out.tiles_per_gauss.cpu(), tpg), "tiles_per_gauss must be bit-exact"
    for name, got, want in (("means2d", out.means2d, proj["means2d"]), ("depths", out.depths, proj["depths"]),
                            ("conics", out.conics, proj["conics"])):
        torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-6, msg=lambda m: f"{name}: {m}")
    assert out.info["n_isects"] == flat.shape[0]
    assert torch.equal(out.info["flatten_ids"].cpu(), flat), "sorted intersection list must be bit-exact"
    assert torch.equal(out.info["tile_offsets"].cpu()[:-1], offs), "tile offsets must be bit-exact"
    assert int(out.info["tile_offsets"][-1]) == flat.shape[0]
    # the (tile, depth-bits, id) keys gsplat would have produced, reconstructed from our outputs
    to = out.info["tile_offsets"].cpu().long()
    tile_of = torch.repeat_interleave(torch.arange(to.numel() - 1), to[1:] - to[:-1])
    dbits = out.depths.cpu().view(torch.int32).long()[out.info["flatten_ids"].cpu().long()]
    assert torch.equal((tile_of << 32) | dbits, isect_ids)


@needs_cuda
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("normals", [True, False])
def test_forward_images_match_oracle(case, normals):
    params, cam = scene_and_camera(**case)
    _, ref = oracle_outputs(params, cam, predict_normals=normals)
    _, out = cuda_outputs(params, cam, render_normals=normals, exact_lists=True)  # last_ids index gsplat's full lists
    # raw-parameter path: expf on the GPU vs torch.exp on the CPU may move a radius across an integer
    mism = (out.radii.cpu() != ref["info"]["radii"]).float().mean().item()
    assert mism <= 2e-3, f"radii mismatch fraction {mism}"
    checks = [("rgb", out.rgb, ref["rgb"]), ("alpha", out.alpha, ref["accumulation"])]
    if normals:
        checks.append(("normal", out.normal, ref["normal"]))
    for name, got, want in checks:
        frac, mx = frac_close(got, want, atol=1e-4)
        assert frac >= 0.999 and mx <= 2e-2, f"{name}: {frac:.5f} of pixels within 1e-4, max err {mx:.3e}"
    frac, mx = frac_close(out.depth, ref["depth"], atol=1e-4, rtol=1e-4)
    assert frac >= 0.999, f"depth: {frac:.5f} within tol, max err {mx:.3e}"
    frac, mx = frac_close(out.surface_normal, ref["surface_normal"], atol=2e-3)
    assert frac >= 0.995, f"surface_normal: {frac:.5f} within 2e-3, max err {mx:.3e}"
    if normals:
        torch.testing.assert_close(out.normals_world.cpu(), ref["gauss_normals"], rtol=1e-4, atol=1e-5)
    assert torch.equal(out.info["last_ids"].cpu(), ref["info"]["last_ids"]) or \
        (out.info["last_ids"].cpu() != ref["info"]["last_ids"]).float().mean() < 2e-3


def _loss(out_rgb, out_depth, out_normal, out_alpha, seed=0):
    g = torch.Generator().manual_seed(seed)
    H, W, _ = out_rgb.shape
    w_rgb = torch.rand(H, W, 3, generator=g).to(out_rgb)
    w_d = torch.rand(H, W, 1, generator=g).to(out_rgb)
    w_n = torch.rand(H, W, 3, generator=g).to(out_rgb)
    w_a = torch.rand(H, W, 1, generator=g).to(out_rgb)
    return (out_rgb * w_rgb).sum() + 0.1 * (out_depth * w_d).sum() + (out_normal * w_n).sum() + (out_alpha * w_a).sum()


@needs_cuda
@pytest.mark.parametrize("case", CASES[:2])
@pytest.mark.parametrize("normals", [True, False])
def test_backward_matches_fp64_oracle(case, normals):
    params, cam = scene_and_camera(**case)
    p64, ref = oracle_outputs(params, cam, dtype=torch.float64, requires_grad=True, predict_normals=normals,
                              collect_absgrad=True)
    ref["info"]["means2d"].retain_grad()
    _loss(ref["rgb"], ref["depth"], ref["normal"], ref["accumulation"]).backward()
    pc, out = cuda_outputs(params, cam, requires_grad=True, render_normals=normals)
    _loss(out.rgb, out.depth, out.normal, out.alpha).backward()
    for k in ("means", "quats", "scales", "opacities", "features_dc", "features_rest"):
        got, want = pc[k].grad.cpu().double(), p64[k].grad
        rel = (got - want).norm() / (want.norm() + 1e-30)
        assert rel <= 1e-3, f"grad {k}: relative error {rel:.3e} (|want|={want.norm():.3e})"
    # means2d.grad and .absgrad (what densification consumes, dn_model.py:512)
    from oracle import gsplat_ref as G

    info = ref["info"]
    want_abs = G.absgrad_from_hooks(info["hooks"], info["conics"], info["opacities"], params["means"].shape[0])
    for name, got, want in (("grad", out.means2d.grad, info["means2d"].grad), ("absgrad", out.means2d.absgrad, want_abs)):
        rel = (got.cpu().double() - want).norm() / (want.norm() + 1e-30)
        assert rel <= 1e-3, f"means2d.{name}: relative error {rel:.3e} (|want|={want.norm():.3e})"


@needs_cuda
def test_all_culled_and_single_gaussian():
    params, cam = scene_and_camera(50, 64, 48)
    far = {k: v.clone() for k, v in params.items()}
    far["means"] = far["means"] + torch.tensor([1000.0, 0.0, 0.0])  # behind / outside every frustum
    _, out = cuda_outputs(far, cam)
    assert int((out.radii > 0).sum()) == 0 and out.info["n_isects"] == 0
    assert float(out.alpha.abs().max()) == 0.0
    bg = torch.tensor([0.1490, 0.1647, 0.2157])
    torch.testing.assert_close(out.rgb.cpu(), bg.expand(48, 64, 3), rtol=0, atol=1e-6)
    assert float(out.depth.abs().max()) == 0.0  # max over an empty render is 0
    one = {k: v[:1].clone() for k, v in params.items()}
    one["means"][:] = 0.0
    _, ref = oracle_outputs(one, cam)
    _, out = cuda_outputs(one, cam)
    frac, mx = frac_close(out.rgb, ref["rgb"], atol=1e-4)
    assert frac >= 0.999, (frac, mx)


@needs_cuda
@pytest.mark.parametrize("case", CASES + [dict(n=20000, width=320, height=240, view=2)])
def test_precise_hit_lists_render_bit_identical_images(case):
    """The default emission drops (tile, Gaussian) pairs that no pixel of the tile can reach; that must not change
    a single bit of any output, and the kept list must be an order-preserving sub-list of gsplat's."""
    params, cam = scene_and_camera(**case)
    _, full = cuda_outputs(params, cam, exact_lists=True)
    _, cut = cuda_outputs(params, cam, list_shift=0)
    for name in ("rgb", "depth", "normal", "alpha", "surface_normal"):
        assert torch.equal(getattr(full, name), getattr(cut, name)), f"{name} differs between exact and precise-hit lists"
    assert torch.equal(full.tiles_per_gauss, cut.tiles_per_gauss)  # API output stays gsplat's bbox count
    assert cut.info["n_isects"] < full.info["n_isects"]
    fo, co = full.info["tile_offsets"].cpu().tolist(), cut.info["tile_offsets"].cpu().tolist()
    ff, cf = full.info["flatten_ids"].cpu().tolist(), cut.info["flatten_ids"].cpu().tolist()
    for t in range(len(fo) - 1):
        it = iter(ff[fo[t]:fo[t + 1]])
        assert all(g in it for g in cf[co[t]:co[t + 1]]), f"tile {t}: kept list is not a sub-sequence"


@needs_cuda
@pytest.mark.parametrize("case", CASES + [dict(n=20000, width=320, height=240, view=2)])
def test_supertile_lists_render_bit_identical_images(case):
    """Lists kept per 32/64/128-pixel supertile (each 16x16 tile filters its supertile's list inside the raster kernels)
    must not change a single bit of any output; the backward must agree with the per-tile-list backward up to the order
    of its float atomics."""
    params, cam = scene_and_camera(**case)
    _, full = cuda_outputs(params, cam, exact_lists=True)
    pr, ref = cuda_outputs(params, cam, requires_grad=True, list_shift=0)
    _loss(ref.rgb, ref.depth, ref.normal, ref.alpha).backward()
    seen = []
    for shift in (1, 2, 3):
        stats = torch.zeros(4, dtype=torch.int64, device="cuda")
        p, out = cuda_outputs(params, cam, requires_grad=True, list_shift=shift, stats=stats)
        for name in ("rgb", "depth", "normal", "alpha", "surface_normal"):
            assert torch.equal(getattr(full, name), getattr(out, name)), f"{name}: list_shift={shift}"
        assert out.info["list_tile"] == 16 << shift
        _loss(out.rgb, out.depth, out.normal, out.alpha).backward()
        for k in p:
            rel = float((p[k].grad - pr[k].grad).norm() / (pr[k].grad.norm() + 1e-30))
            assert rel < 1e-4, (k, rel, shift)
        ab = ref.means2d.absgrad
        assert float((out.means2d.absgrad - ab).abs().max()) <= 1e-4 * float(ab.abs().max() + 1e-30)
        walked_f, kept_f, walked_b, kept_b = stats.tolist()
        assert 0 < kept_f <= walked_f and 0 < kept_b <= walked_b and kept_b <= kept_f
        seen.append((shift, out.info["n_isects"]))
    by_shift = dict(seen)
    assert by_shift[3] <= by_shift[2] <= by_shift[1] <= ref.info["n_isects"]  # coarser lists hold fewer pairs


@needs_cuda
def test_capacity_overflow_is_loud_and_recoverable():
    """sync-free sizing: a view that needs more slots than 1.15 x the largest count seen so far must never hand out
    gradients — its backward raises DnrCapacityError, the capacity grows, and the repeated view is exact."""
    import dn_splatter_b200.rasterize as R

    small, cam = scene_and_camera(4000, 208, 160, view=1, scale_mult=0.3)
    big, _ = scene_and_camera(4000, 208, 160, view=1, scale_mult=3.0)
    for _ in range(3):  # two seeding views (synchronous), then sync-free
        cuda_outputs(small, cam, sync_free=True)
    _, ref = cuda_outputs(big, cam)
    p, out = cuda_outputs(big, cam, requires_grad=True, sync_free=True)
    assert int(out.info["n_isects_dev"]) > out.info["n_isects"], "the test scene must overflow the seeded capacity"
    with pytest.raises(R.DnrCapacityError):
        _loss(out.rgb, out.depth, out.normal, out.alpha).backward()
    assert all(v.grad is None for v in p.values())
    p, out = cuda_outputs(big, cam, requires_grad=True, sync_free=True)  # capacity was raised: exact now
    for name in ("rgb", "depth", "normal", "alpha"):
        assert torch.equal(getattr(out, name), getattr(ref, name))
    _loss(out.rgb, out.depth, out.normal, out.alpha).backward()
    # a truncated no-grad render is reported by the next call instead
    R._CAPACITY.clear()
    for _ in range(3):
        cuda_outputs(small, cam, sync_free=True)
    with torch.no_grad():
        cuda_outputs(big, cam, sync_free=True)
        torch.cuda.synchronize()
        with pytest.raises(R.DnrCapacityError):
            cuda_outputs(big, cam, sync_free=True)
        _, again = cuda_outputs(big, cam, sync_free=True)
    assert torch.equal(again.rgb, ref.rgb)
    R._CAPACITY.clear()


@needs_cuda
def test_sync_free_capacity_mode_matches_sync_mode():
    import dn_splatter_b200.rasterize as R

    params, cam = scene_and_camera(5000, 256, 192, view=1)
    _, ref = cuda_outputs(params, cam)
    outs = [cuda_outputs(params, cam, sync_free=True)[1] for _ in range(4)]  # 2 seeding views, then sync-free
    for o in outs:
        for name in ("rgb", "depth", "normal", "alpha"):
            assert torch.equal(getattr(o, name), getattr(ref, name))
    assert int(outs[-1].info["n_isects_dev"]) == ref.info["n_isects"]
    assert outs[-1].info["n_isects"] >= ref.info["n_isects"]  # capacity, not count
    rep = R.capacity_report()
    assert all(over == 0 for _, over in rep.values())
    # backward through a capacity-sized list
    p, o = cuda_outputs(params, cam, requires_grad=True, sync_free=True)
    pr, r = cuda_outputs(params, cam, requires_grad=True)
    _loss(o.rgb, o.depth, o.normal, o.alpha).backward()
    _loss(r.rgb, r.depth, r.normal, r.alpha).backward()
    for k in p:  # same kernels, same lists: only the order of the float atomics differs between two runs
        rel = float((p[k].grad - pr[k].grad).norm() / (pr[k].grad.norm() + 1e-30))
        assert rel < 1e-4, (k, rel)
