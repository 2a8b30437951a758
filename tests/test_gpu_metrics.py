"""GPU tests of the render-metric kernels (csrc/ssim.cu dnr_rgb_metrics, csrc/metrics.cu dnr_depth_metrics /
dnr_normal_metrics) against the fp64 oracle (oracle/metrics_ref.py, itself pinned to the reference by
tests/test_metrics_cpu.py), and of the model / pipeline routes into them.

Bounds: a1..a3 and every count equal; the median bit-equal; PSNR within 1e-4 dB; SSIM within 1e-6; every other sum
within 2e-6 relative; inf / NaN cases equal.  One exception, as in tests/test_gpu_photometric.py: on constant patches
every fp32 SSIM is dominated by the E[x^2] - mu^2 cancellation, so there the kernel may also be off by twice torch's
own fp32 evaluation of the same formula, or by 1e-5 (the measured error is stated at the check)."""
import math

import pytest
import torch

from oracle import metrics_ref as R

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

SHAPES = [(11, 11), (37, 53), (80, 96), (1080, 1920)]
INV255 = torch.tensor(1 / 255, dtype=torch.float32)


def _images(kind, B, H, W, u8, seed):
    """(pred [B,H,W,3] fp32, target [B,H,W,3] fp32 or uint8), on the CPU."""
    g = torch.Generator().manual_seed(seed)
    rand = lambda: torch.rand(B, H, W, 3, generator=g)  # noqa: E731
    if kind == "noise":
        x, y = rand(), rand()
    elif kind == "correlated":
        x = rand()
        y = 0.6 * x + 0.4 * rand()
    elif kind == "constant":
        up = lambda t: t.repeat_interleave(20, 1).repeat_interleave(20, 2)[:, :H, :W].contiguous()  # noqa: E731
        x = up(torch.rand(B, -(-H // 20), -(-W // 20), 3, generator=g))
        y = up(torch.rand(B, -(-H // 20), -(-W // 20), 3, generator=g))
    elif kind == "equal":
        y = rand()
        x = y.clone()
    else:
        raise ValueError(kind)
    if u8:
        y8 = (y * 255).round().to(torch.uint8)
        return (y8.float() * INV255 if kind == "equal" else x), y8
    return x, y


def _bchw(t):
    return t.cuda().permute(0, 3, 1, 2)  # a [B,C,H,W] view of channels-last images, as the model passes them


def _rel(got, want, rtol, what):
    got, want = float(got), float(want)
    if math.isnan(want) or math.isinf(want):
        assert (math.isnan(got) and math.isnan(want)) or got == want, f"{what}: {got} vs {want}"
        return
    assert abs(got - want) <= rtol * abs(want) + 1e-300, f"{what}: {got!r} vs {want!r} (rel {abs(got - want) / abs(want):.2e})"


# ---------------------------------------------------------------------------------------------------------- RGB
CASES = [(hw, B, u8, kind) for hw in SHAPES for B in (1, 3) for u8 in (False, True)
         for kind in (("correlated", "equal") if hw == (1080, 1920) else ("noise", "correlated", "constant", "equal"))]


@pytest.mark.parametrize("hw,B,u8,kind", CASES, ids=[f"{h}x{w}-B{b}-{'u8' if u else 'f32'}-{k}" for (h, w), b, u, k in CASES])
def test_rgb_metrics_match_fp64(hw, B, u8, kind):
    from dn_splatter_b200 import metrics as MT

    H, W = hw
    x, y = _images(kind, B, H, W, u8, seed=H * 7 + W + B + 100 * u8 + len(kind))
    s = MT.rgb_sums(_bchw(x), _bchw(y))
    mse, psnr, ssim = MT.rgb_from_sums(s, (B, 3, H, W))
    ref = R.rgb(x, y)
    for b in range(B):
        _rel(s[b, 1], ref["sse"][b], 2e-6, f"sse[{b}]")
    ssim_atol = 1e-6
    if kind == "constant":
        from dn_splatter_b200.losses import ssim as ssim_fn

        yr = R.target_as_read(y)
        s32 = torch.stack([ssim_fn(yr[b].permute(2, 0, 1)[None], x[b].permute(2, 0, 1)[None]) for b in range(B)]).mean()
        # windows inside one patch have sigma = 0: every pixel's fp32 E[x^2] - mu^2 rounds to a few ulp against C2 = 9e-4.
        # Measured on an H100 80GB HBM3 (700 W): 6.3e-6 at 80x96 fp32, where torch's fp32 path is off by 1.9e-6.
        ssim_atol += max(2 * abs(float(s32) - float(ref["ssim"])), 1e-5)
    assert abs(float(ssim) - float(ref["ssim"])) <= ssim_atol, (float(ssim), float(ref["ssim"]))
    if kind == "equal":
        assert float(s[:, 1].sum()) == 0.0 and math.isinf(float(psnr)) and abs(float(ssim) - 1.0) <= 1e-6
    else:
        assert abs(float(psnr) - float(ref["psnr"])) <= 1e-4, (float(psnr), float(ref["psnr"]))
        _rel(mse, ref["mse"], 2e-6, "mse")
    # the public class returns the same values
    p2, s2, lp = MT.RGBMetrics()(_bchw(x), _bchw(y))
    assert lp is None and float(p2) == float(psnr.float()) and float(s2) == float(ssim.float())


# ---------------------------------------------------------------------------------------------------------- depth
def _depth_case(kind, shape, seed):
    g = torch.Generator().manual_seed(seed)
    p = 0.5 + 4 * torch.rand(*shape, generator=g)
    t = 0.05 + 4 * torch.rand(*shape, generator=g)
    if kind == "masked":
        t.view(-1)[::7] = 0.1  # exactly the tolerance: excluded
        t.view(-1)[1::11] = 0.0
        p.view(-1)[2::13] = 0.0  # pred 0 on valid pixels: misses for a1..a3, rmse_log inf
        p.view(-1)[3::17] = -1.0  # negative: the log term is NaN and left out of rmse_log
    elif kind == "empty":
        t = 0.1 * torch.rand(*shape, generator=g)
    elif kind == "close":  # ratios near the 1.25^k thresholds
        p = 1 + torch.rand(*shape, generator=g)
        t = p * torch.tensor([1.25, 1.5625, 1.953125, 1 / 1.25])[torch.randint(0, 4, shape, generator=g)]
        t = t * (1 + 1e-7 * (torch.rand(*shape, generator=g) - 0.5))
    return p, t


DEPTH = [(k, s) for k in ("noise", "masked", "close", "empty") for s in ((1, 11, 11), (1, 37, 53), (3, 80, 96), (1, 1080, 1920))]


@pytest.mark.parametrize("kind,shape", DEPTH, ids=[f"{k}-{'x'.join(map(str, s))}" for k, s in DEPTH])
def test_depth_metrics_match_fp64(kind, shape):
    from dn_splatter_b200 import metrics as MT

    p, t = _depth_case(kind, shape, seed=sum(shape) + len(kind))
    s = MT.depth_sums(p.cuda(), t.cuda(), 0.1)
    ref = R.depth(p, t, 0.1)
    for i in (0, 1, 2, 3, 8):
        assert float(s[i]) == float(ref["sums"][i]), (i, float(s[i]), float(ref["sums"][i]))
    for i in (4, 5, 6, 7):
        _rel(s[i], ref["sums"][i], 2e-6, f"sum[{i}]")
    got = MT.depth_from_sums(s)
    for v, k in zip(got, ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")):
        if k in ("a1", "a2", "a3"):
            assert float(v) == float(ref[k]) or (math.isnan(float(v)) and math.isnan(float(ref[k]))), k
        else:
            _rel(v, ref[k], 2e-6, k)
    if kind == "masked":
        assert math.isinf(float(got[3]))
    if kind == "empty":
        assert all(math.isnan(float(v)) for v in got)
        assert all(math.isnan(float(v)) for v in MT.DepthMetrics()(p.cuda(), t.cuda()))


# ---------------------------------------------------------------------------------------------------------- normal
NORMAL = [(B, H, W, u8) for B, H, W in ((1, 11, 11), (3, 11, 11), (1, 37, 53), (1, 80, 96), (3, 37, 53), (3, 1080, 1920))
          for u8 in (False, True)]


@pytest.mark.parametrize("B,H,W,u8", NORMAL, ids=[f"B{b}-{h}x{w}-{'u8' if u else 'f32'}" for b, h, w, u in NORMAL])
def test_normal_metrics_match_fp64(B, H, W, u8):
    """3BHW is odd for (1|3, 11, 11) and (1|3, 37, 53), even otherwise; uint8 targets give many ties."""
    from dn_splatter_b200 import metrics as MT

    g = torch.Generator().manual_seed(B * 1000 + H + W + u8)
    p = torch.rand(B, H, W, 3, generator=g)
    t = torch.rand(B, H, W, 3, generator=g)
    if u8:
        t = (t * 255).round().to(torch.uint8)
    s = MT.normal_sums(_bchw(p), _bchw(t))
    ref = R.normal(p, t)
    a = R.normal_abs_err(p, t).reshape(-1)
    assert float(s[3 * B]) == float(ref["med_err"]), (float(s[3 * B]), float(ref["med_err"]))
    assert float(torch.median(a)) == float(ref["med_err"])  # the lower median torch.median returns
    for b in range(B):
        _rel(s[3 * b], ref["acos_sum"][b], 2e-6, f"acos[{b}]")
        _rel(s[3 * b + 1], ref["sq_sum"][b], 2e-6, f"sq[{b}]")
        _rel(s[3 * b + 2], ref["abs_sum"][b], 2e-6, f"abs[{b}]")
    for v, k in zip(MT.normal_from_sums(s, (B, 3, H, W)), ("mae", "rmse", "mean_err", "med_err")):
        _rel(v, ref[k], 2e-6, k)


def test_normal_median_of_constant_and_two_valued_maps():
    """All |g - p| equal, and exactly half of them one value: the selection lands on the lower one."""
    from dn_splatter_b200 import metrics as MT

    p = torch.full((1, 8, 8, 3), 0.25)
    t = torch.full((1, 8, 8, 3), 0.75)
    assert float(MT.normal_sums(_bchw(p), _bchw(t))[3]) == 0.5
    t2 = t.clone()
    t2.view(-1)[::2] = 1.0
    assert float(MT.normal_sums(_bchw(p), _bchw(t2))[3]) == 0.5


# ---------------------------------------------------------------------------------------------------------- model
def _models(n_gauss=400):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.synthetic import make_scene

    params = make_scene(n_gauss, seed=5)
    out = []
    for dev in ("cuda", "cpu"):
        m = DNSplatterModelConfig(random_init=True, num_random=16, use_depth_loss=True, depth_lambda=0.2,
                                  predict_normals=True).setup(device=dev)
        m.load_gaussians(params)
        m.step = 30000
        m.eval()
        m.lpips = lambda a, b: (a - b).abs().mean() + 0.25 * a.mean()
        out.append(m)
    return out


def _ring(n, W, H):
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.synthetic import ring_cameras

    cams = ring_cameras(n, W, H)
    return Cameras(torch.stack([c["c2w"] for c in cams]), [c["fx"] for c in cams], [c["fy"] for c in cams],
                   [c["cx"] for c in cams], [c["cy"] for c in cams], W, H)


def _batches(n, W, H, u8=True, mask=False):
    g = torch.Generator().manual_seed(n + W)
    out = []
    for _ in range(n):
        d = 2 + 6 * torch.rand(H, W, 1, generator=g)
        d[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
        img = torch.rand(H, W, 3, generator=g)
        b = {"image": (img * 255).to(torch.uint8) if u8 else img, "sensor_depth": d,
             "normal": torch.rand(H, W, 3, generator=g)}
        if mask:
            b["mask"] = (torch.rand(H, W, 1, generator=g) > 0.2).float()
        out.append(b)
    return out


def _same(gpu, cpu, ssim64, what):
    """`ssim64`: the fp64 SSIM of the same pair.  The CPU route's SSIM is torch's fp32 conv formulation, which on renders
    with flat background is cancellation-bound (see test_gpu_photometric.py), so the GPU route's SSIM has to be within
    1e-6 of fp64 or at least as accurate as the CPU route."""
    assert list(gpu) == list(cpu), (what, list(gpu), list(cpu))
    for k in gpu:
        a, b = float(gpu[k]), float(cpu[k])
        if k == "rgb_psnr":
            assert abs(a - b) <= 1e-4, (what, k, a, b)
        elif k == "rgb_ssim":
            assert abs(a - ssim64) <= 1e-6 + 2 * abs(b - ssim64), (what, k, a, b, ssim64)
        elif math.isnan(b) or math.isinf(b):
            assert (math.isnan(a) and math.isnan(b)) or a == b, (what, k, a, b)
        else:
            # the CPU route evaluates in fp32 (the reference's own code): fp32 accuracy
            assert abs(a - b) <= 2e-6 * max(abs(b), 1.0), (what, k, a, b)


@pytest.mark.parametrize("u8,mask", [(True, False), (False, False), (False, True)], ids=["u8", "f32", "f32-mask"])
def test_model_gpu_route_equals_cpu_route(u8, mask):
    mg, mc = _models()
    cams = _ring(2, 96, 80)
    for i, batch in enumerate(_batches(2, 96, 80, u8=u8, mask=mask)):
        outputs = mg.get_outputs_for_camera(cams[i:i + 1])
        cpu_out = {k: v.detach().cpu() for k, v in outputs.items()}
        bg = {k: v.cuda() for k, v in batch.items()}
        gt = R.target_as_read(batch["image"])
        if not mask:
            s64 = float(R.rgb(cpu_out["rgb"][None], gt[None])["ssim"])
            _same(mg.get_metrics_dict(outputs, bg), mc.get_metrics_dict(cpu_out, batch), s64, f"metrics view {i}")
        m = batch.get("mask", torch.ones(1))
        s64 = float(R.rgb((cpu_out["rgb"] * m)[None], (gt * m)[None])["ssim"])
        rg, ig = mg.get_image_metrics_and_images(outputs, bg)
        rc, ic = mc.get_image_metrics_and_images(cpu_out, batch)
        _same(rg, rc, s64, f"image metrics view {i}")
        for k in ig:
            torch.testing.assert_close(ig[k].cpu(), ic[k], rtol=0, atol=1e-6)


def test_pipeline_average_over_a_ring_of_views():
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.dn_pipeline import DNSplatterPipelineConfig
    from dn_splatter_b200.synthetic import make_scene

    class DS:
        def __init__(self, cameras):
            self.cameras = cameras

        def __len__(self):
            return int(self.cameras.shape[0])

    class DM:
        def __init__(self, cameras, batches):
            self.train_dataset, self.eval_dataset, self.cached_eval = DS(cameras), DS(cameras), batches

    n, W, H = 6, 128, 96
    cams = _ring(n, W, H)
    batches = [{k: v.cuda() for k, v in b.items()} for b in _batches(n, W, H)]
    cfg = DNSplatterPipelineConfig(datamanager=DM(cams, batches),
                                   model=DNSplatterModelConfig(random_init=True, num_random=16, predict_normals=True))
    p = cfg.setup(device="cuda")
    p.model.load_gaussians(make_scene(2000, seed=6))
    p.model.step = 30000
    p.train()
    avg = p.get_average_eval_image_metrics(get_std=True)
    assert p.model.training
    p.eval()
    per = [p.model.get_image_metrics_and_images(p.model.get_outputs_for_camera(cams[i:i + 1]), batches[i])[0]
           for i in range(n)]
    p.train()
    keys = list(per[0]) + ["num_rays_per_sec", "fps"]
    assert set(avg) == set(keys) | {k + "_std" for k in keys}
    for k in per[0]:
        std, mean = torch.std_mean(torch.tensor([d[k] for d in per]))
        assert abs(avg[k] - float(mean)) <= 1e-6 * max(1.0, abs(float(mean))), k
        assert abs(avg[k + "_std"] - float(std)) <= 1e-5 * max(1.0, abs(float(std))), k
    assert avg["num_rays_per_sec"] > 0 and avg["fps"] > 0
