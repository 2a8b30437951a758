"""CPU tests of the render metrics (dn_splatter_b200/metrics.py, the model's get_metrics_dict /
get_image_metrics_and_images, the pipeline's get_average_eval_image_metrics) and of the fp64 oracle.

tests/golden/dn_metrics.npz holds the reference's own DepthMetrics / NormalMetrics / mean_angular_error and its own
model methods (with PSNR / SSIM from the oracle and a deterministic LPIPS stand-in), made by
tests/golden/make_golden_metrics.py."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from dn_splatter_b200 import _lib as L
from dn_splatter_b200 import metrics as MT
from oracle import metrics_ref as R

GOLD = os.path.join(os.path.dirname(__file__), "golden", "dn_metrics.npz")
DEPTH_CASES = ("noise", "masked", "close", "empty")
NORMAL_CASES = ("b1", "b3", "odd")
DEPTH_KEYS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _close(got, want, rtol, what):
    """Equal where NaN / inf, else within rtol (relative, absolute below 1)."""
    got, want = float(got), float(want)
    if math.isnan(want) or math.isinf(want):
        assert (math.isnan(got) and math.isnan(want)) or got == want, f"{what}: {got} vs {want}"
        return
    assert abs(got - want) <= rtol * max(1.0, abs(want)), f"{what}: {got!r} vs {want!r}"


def lpips_stub(a, b):
    """The golden run's LPIPS stand-in (tests/golden/make_golden_metrics.py)."""
    return (a - b).abs().mean() + 0.25 * a[:, 0].mean() + 0.125 * b[:, 2].mean()


# ------------------------------------------------------------------------------------------------ oracle and CPU route
@pytest.mark.parametrize("case", DEPTH_CASES)
def test_depth_oracle_and_cpu_route_equal_the_reference(gold, case):
    """The reference evaluates in fp32; the oracle's fp64 sums agree to fp32 accuracy, its ratio tests and counts
    exactly (a1..a3 as count ratios), and the NaN / inf cases are the same."""
    p, g = torch.from_numpy(gold[f"depth_{case}_pred"]), torch.from_numpy(gold[f"depth_{case}_gt"])
    want = gold[f"depth_{case}_out"]
    ref = R.depth(p, g)
    cpu = MT.DepthMetrics()(p, g)
    for i, k in enumerate(DEPTH_KEYS):
        if k in ("a1", "a2", "a3"):  # count / count: the reference's fp32 mean is the same ratio rounded to fp32
            _close(np.float32(float(ref[k])), want[i], 0.0, f"oracle {case} {k}")
        else:
            _close(ref[k], want[i], 2e-6, f"oracle {case} {k}")
        _close(cpu[i], want[i], 0.0, f"cpu route {case} {k}")
    if case == "masked":
        assert math.isinf(want[3]) and float(ref["sums"][0]) < p.numel()
    if case == "empty":
        assert all(math.isnan(v) for v in want)


@pytest.mark.parametrize("case", NORMAL_CASES)
def test_normal_oracle_and_cpu_route_equal_the_reference(gold, case):
    """Median bit-equal (the lower median of the fp32 |g - p|), the rest to fp32 accuracy."""
    p, g = torch.from_numpy(gold[f"normal_{case}_pred"]), torch.from_numpy(gold[f"normal_{case}_gt"])
    want = gold[f"normal_{case}_out"]
    ref = R.normal(p.permute(0, 2, 3, 1), g.permute(0, 2, 3, 1))
    cpu = MT.NormalMetrics()(p, g)
    for i, k in enumerate(("mae", "rmse", "mean_err", "med_err")):
        _close(ref[k], want[i], 0.0 if k == "med_err" else 2e-6, f"oracle {case} {k}")
        _close(cpu[i], want[i], 0.0, f"cpu route {case} {k}")
    assert torch.equal(MT.mean_angular_error(p, g), torch.from_numpy(gold[f"normal_{case}_mae_map"]))


def test_oracle_psnr_ssim_follow_torchmetrics_pooling():
    """PSNR pools the MSE over the batch; SSIM is the mean of per-image means; identical images give inf and 1."""
    g = torch.Generator().manual_seed(3)
    x, y = torch.rand(3, 20, 24, 3, generator=g), torch.rand(3, 20, 24, 3, generator=g)
    r = R.rgb(x, y)
    mse = ((x.double() - y.double()) ** 2).mean()
    assert abs(float(r["psnr"]) - 10 * math.log10(1 / float(mse))) < 1e-12
    per = [float(R.rgb(x[b:b + 1], y[b:b + 1])["ssim"]) for b in range(3)]
    assert abs(float(r["ssim"]) - sum(per) / 3) < 1e-12
    same = R.rgb(x, x)
    assert math.isinf(float(same["psnr"])) and abs(float(same["ssim"]) - 1.0) < 1e-12


def test_cpu_rgb_route_equals_the_oracle():
    g = torch.Generator().manual_seed(4)
    x = torch.rand(2, 23, 31, 3, generator=g)
    y = (0.6 * x + 0.4 * torch.rand(2, 23, 31, 3, generator=g))
    for tgt in (y, (y * 255).round().to(torch.uint8)):
        mse, psnr, ssim = MT.rgb_metrics(x.permute(0, 3, 1, 2), tgt.permute(0, 3, 1, 2))
        r = R.rgb(x, tgt)
        assert abs(float(psnr) - float(r["psnr"])) <= 1e-4
        assert abs(float(ssim) - float(r["ssim"])) <= 1e-6
        _close(mse, r["mse"], 2e-6, "mse")


def test_tf_resize_equals_torchvision():
    TF = pytest.importorskip("torchvision.transforms.functional")
    g = torch.Generator().manual_seed(5)
    for t in (torch.rand(3, 37, 53, generator=g), (torch.rand(3, 37, 53, generator=g) * 255).to(torch.uint8),
              torch.rand(1, 40, 56, generator=g, dtype=torch.float64)):
        for size in ((18, 26), (20, 28), (41, 60), (37, 53)):
            want = TF.resize(t, list(size), antialias=None)
            got = MT.tf_resize(t, size)
            assert got.dtype == want.dtype and torch.equal(got, want), (t.dtype, size)


# ------------------------------------------------------------------------------------------------ model glue
def _model(scales, **cfg_kw):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig

    cfg = DNSplatterModelConfig(random_init=True, num_random=16, **cfg_kw)
    m = cfg.setup(device="cpu")
    n = scales.shape[0]
    m.load_gaussians({"means": torch.zeros(n, 3), "scales": scales, "quats": torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1),
                      "features_dc": torch.zeros(n, 3), "features_rest": torch.zeros(n, 15, 3),
                      "opacities": torch.zeros(n, 1)})
    return m


def _golden_inputs(gold, tag):
    outputs = {k: torch.from_numpy(gold[f"{tag}_out_{k}"]) for k in ("rgb", "depth", "normal")}
    batch = {k: torch.from_numpy(gold[f"{tag}_batch_{k}"]) for k in ("image", "sensor_depth", "normal")
             if f"{tag}_batch_{k}" in gold}
    return outputs, batch


def _golden_model(gold, tag):
    cfg = eval(str(gold[f"{tag}_cfg"]))  # a repr of a dict of literals written by make_golden_metrics.py
    m = _model(torch.from_numpy(gold["model_scales"]), use_depth_loss=True, depth_lambda=0.2,
               num_downscales=1 if cfg.get("d", 1) > 1 else 0)
    m.step = 0
    m.train(cfg.get("d", 1) > 1)
    m.lpips = lpips_stub
    return m, cfg


def check_against_golden(res, gold, tag, route):
    keys = [str(k) for k in gold[f"{tag}_keys"]]
    assert list(res.keys()) == keys, (route, tag, list(res.keys()), keys)
    for k, want in zip(keys, gold[f"{tag}_values"]):
        if k == "rgb_psnr":
            assert abs(float(res[k]) - want) <= 1e-4, (route, tag, k, float(res[k]), want)
        elif k == "rgb_ssim":
            assert abs(float(res[k]) - want) <= 1e-6, (route, tag, k, float(res[k]), want)
        elif k in ("depth_a1", "depth_a2", "depth_a3"):
            assert abs(float(res[k]) - want) <= 1e-7, (route, tag, k, float(res[k]), want)  # fp32 count / count
        else:
            _close(res[k], want, 2e-6, f"{route} {tag} {k}")


@pytest.mark.parametrize("tag", ["md_full", "md_half", "md_nodepth"])
def test_get_metrics_dict_equals_the_reference(gold, tag):
    m, _ = _golden_model(gold, tag)
    outputs, batch = _golden_inputs(gold, tag)
    check_against_golden(m.get_metrics_dict(outputs, batch), gold, tag, "cpu")


@pytest.mark.parametrize("tag", ["im_full", "im_resize", "im_rgb_only"])
def test_get_image_metrics_and_images_equals_the_reference(gold, tag):
    m, _ = _golden_model(gold, tag)
    outputs, batch = _golden_inputs(gold, tag)
    res, images = m.get_image_metrics_and_images(outputs, batch)
    check_against_golden(res, gold, tag, "cpu")
    for k in ("img", "depth", "normal"):
        want = torch.from_numpy(gold[f"{tag}_images_{k}"])
        assert images[k].shape == want.shape and torch.allclose(images[k], want, rtol=0, atol=1e-6), k


def test_lpips_only_with_a_user_callable():
    m = _model(torch.zeros(4, 3))
    m.eval()
    g = torch.Generator().manual_seed(6)
    outputs = {"rgb": torch.rand(16, 20, 3, generator=g), "depth": torch.rand(16, 20, 1, generator=g),
               "normal": torch.rand(16, 20, 3, generator=g)}
    batch = {"image": (torch.rand(16, 20, 3, generator=g) * 255).to(torch.uint8)}
    assert m.lpips is None
    assert "rgb_lpips" not in m.get_metrics_dict(outputs, batch)
    assert "rgb_lpips" not in m.get_image_metrics_and_images(outputs, batch)[0]
    calls = []

    def stub(a, b):
        calls.append((a.clone(), b.clone()))
        return torch.tensor(0.25)

    m.lpips = stub
    for fn in (m.get_metrics_dict, lambda o, b: m.get_image_metrics_and_images(o, b)[0]):
        calls.clear()
        res = fn(outputs, batch)
        assert res["rgb_lpips"] == 0.25 and len(calls) == 1
        a, b = calls[0]
        assert torch.equal(a, MT.u8_as_float(batch["image"]).permute(2, 0, 1)[None])  # (gt, pred) as upstream
        assert torch.equal(b, outputs["rgb"].permute(2, 0, 1)[None])


def test_mask_applies_per_pixel_to_images_and_depths():
    """The reference's mask product fails for any real image; here both images and both depths are masked per
    pixel, and the result equals the oracle on the masked inputs."""
    m = _model(torch.zeros(4, 3))
    m.eval()
    g = torch.Generator().manual_seed(7)
    H, W = 24, 30
    outputs = {"rgb": torch.rand(H, W, 3, generator=g), "depth": 1 + torch.rand(H, W, 1, generator=g),
               "normal": torch.rand(H, W, 3, generator=g)}
    batch = {"image": torch.rand(H, W, 3, generator=g), "sensor_depth": 1 + torch.rand(H, W, 1, generator=g),
             "mask": (torch.rand(H, W, 1, generator=g) > 0.3).float()}
    res, images = m.get_image_metrics_and_images(outputs, batch)
    mask = batch["mask"]
    r = R.rgb((outputs["rgb"] * mask)[None], (batch["image"] * mask)[None])
    assert abs(res["rgb_psnr"] - float(r["psnr"])) <= 1e-4 and abs(res["rgb_ssim"] - float(r["ssim"])) <= 1e-6
    d = R.depth(outputs["depth"] * mask, batch["sensor_depth"] * mask)
    assert float(d["sums"][0]) == float((mask > 0).sum())
    for k in DEPTH_KEYS:
        _close(res["depth_" + k], d[k], 2e-6, k)
    assert torch.equal(images["depth"], torch.cat([batch["sensor_depth"] * mask, outputs["depth"] * mask], dim=1))


def test_rgba_target_is_composited_with_the_background():
    m = _model(torch.zeros(4, 3), background_color="white")
    m.eval()
    g = torch.Generator().manual_seed(8)
    rgba = torch.rand(16, 16, 4, generator=g)
    outputs = {"rgb": torch.rand(16, 16, 3, generator=g), "depth": torch.rand(16, 16, 1, generator=g),
               "normal": torch.rand(16, 16, 3, generator=g), "background": torch.ones(3)}
    res, images = m.get_image_metrics_and_images(outputs, {"image": rgba})
    comp = rgba[..., 3:] * rgba[..., :3] + (1 - rgba[..., 3:]) * 1.0
    assert torch.allclose(images["img"][:, :16], comp, atol=1e-7)
    assert abs(res["rgb_psnr"] - float(R.rgb(outputs["rgb"][None], comp[None])["psnr"])) <= 1e-4


# ------------------------------------------------------------------------------------------------ pipeline
class _EvalDataset:
    def __init__(self, cameras):
        self.cameras = cameras

    def __len__(self):
        return int(self.cameras.shape[0])


class _DataManager:
    def __init__(self, cameras, batches):
        self.train_dataset = _EvalDataset(cameras)
        self.eval_dataset = _EvalDataset(cameras)
        self.cached_eval = batches


def _pipeline(n_views, W=40, H=32):
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.dn_pipeline import DNSplatterPipelineConfig
    from dn_splatter_b200.synthetic import make_scene, ring_cameras

    cams = ring_cameras(n_views, W, H)
    cameras = Cameras(torch.stack([c["c2w"] for c in cams]), [c["fx"] for c in cams], [c["fy"] for c in cams],
                      [c["cx"] for c in cams], [c["cy"] for c in cams], W, H)
    g = torch.Generator().manual_seed(9)
    batches = []
    for _ in range(n_views):
        d = 2 + 6 * torch.rand(H, W, 1, generator=g)
        d[torch.rand(H, W, 1, generator=g) < 0.1] = 0.0
        batches.append({"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8), "sensor_depth": d,
                        "normal": torch.rand(H, W, 3, generator=g)})
    cfg = DNSplatterPipelineConfig(datamanager=_DataManager(cameras, batches),
                                   model=DNSplatterModelConfig(random_init=True, num_random=16, predict_normals=True))
    p = cfg.setup(device="cpu")
    p.model.load_gaussians(make_scene(200, seed=3))
    p.model.step = 30000
    return p, cameras, batches


def test_pipeline_average_over_eval_views():
    from tests.cpu_proxy import cpu_proxy

    p, cameras, batches = _pipeline(3)
    with cpu_proxy():
        p.train()
        avg = p.get_average_eval_image_metrics(get_std=True)
        assert p.model.training
        p.eval()
        per = [p.model.get_image_metrics_and_images(p.model.get_outputs_for_camera(cameras[i:i + 1]), batches[i])[0]
               for i in range(3)]
        p.train()
    keys = list(per[0].keys()) + ["num_rays_per_sec", "fps"]
    assert set(avg) == set(keys) | {k + "_std" for k in keys}
    for k in per[0]:
        vals = torch.tensor([d[k] for d in per])
        s, mu = torch.std_mean(vals)
        _close(avg[k], mu, 1e-6, k)
        _close(avg[k + "_std"], s, 1e-5, k + "_std")
    assert avg["num_rays_per_sec"] > 0 and abs(avg["fps"] * 32 * 40 - avg["num_rays_per_sec"]) <= 1e-6 * avg[
        "num_rays_per_sec"] * 3
    with cpu_proxy():
        plain = p.get_average_eval_image_metrics()
    assert set(plain) == set(keys)
    for k in per[0]:
        _close(plain[k], avg[k], 1e-6, k)


def test_pipeline_single_view_std_is_nan_and_unsupported_modes_raise():
    from tests.cpu_proxy import cpu_proxy

    p, _, _ = _pipeline(1)
    with cpu_proxy():
        avg = p.get_average_eval_image_metrics(get_std=True)
    assert math.isnan(avg["rgb_psnr_std"]) and not math.isnan(avg["rgb_psnr"])
    with pytest.raises(NotImplementedError):
        p.get_average_eval_image_metrics(output_path="renders")
    p.config.skip_point_metrics = False
    with pytest.raises(NotImplementedError):
        p.get_average_eval_image_metrics()
    p.config.skip_point_metrics = True

    class MushroomDataParser:
        pass

    p.datamanager.dataparser = MushroomDataParser()
    with pytest.raises(NotImplementedError):
        p.get_average_eval_image_metrics()


def test_no_module_imports_torchmetrics_or_lpips():
    import dn_splatter_b200.dn_model  # noqa: F401
    import dn_splatter_b200.dn_pipeline  # noqa: F401
    import sys

    assert not any(n.split(".")[0] in ("torchmetrics", "lpips") for n in sys.modules)


# ------------------------------------------------------------------------------------------------ C ABI
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        from dn_splatter_b200.build import build

        build()
    return L.load()


def test_metric_entry_argument_errors_are_negative_codes(lib):
    one = C.c_void_p(16)  # a non-NULL dummy: the checks come first, nothing is dereferenced
    assert lib.dnr_rgb_metrics(None, one, 0, 1, 11, 11, 3, one, None) == -1
    assert lib.dnr_rgb_metrics(one, None, 0, 1, 11, 11, 3, one, None) == -1
    assert lib.dnr_rgb_metrics(one, one, 0, 1, 11, 11, 3, None, None) == -1
    assert lib.dnr_rgb_metrics(one, one, 0, 1, 10, 11, 3, one, None) == -2
    assert lib.dnr_rgb_metrics(one, one, 0, 1, 11, 10, 3, one, None) == -2
    assert lib.dnr_rgb_metrics(one, one, 1, 0, 11, 11, 3, one, None) == -2
    assert lib.dnr_rgb_metrics(one, one, 0, 1, 11, 11, 0, one, None) == -2
    assert lib.dnr_depth_metrics(None, one, 10, 0.1, one, None) == -1
    assert lib.dnr_depth_metrics(one, one, 10, 0.1, None, None) == -1
    assert lib.dnr_depth_metrics(one, one, 0, 0.1, one, None) == -2
    assert lib.dnr_normal_metrics_workspace_bytes(0, 4, 4) == -2
    ws = lib.dnr_normal_metrics_workspace_bytes(2, 4, 4)
    assert ws > 256 * 8
    assert lib.dnr_normal_metrics(None, one, 0, 2, 4, 4, one, ws, one, None) == -1
    assert lib.dnr_normal_metrics(one, one, 0, 2, 4, 4, None, ws, one, None) == -1
    assert lib.dnr_normal_metrics(one, one, 0, 2, 4, 4, one, ws, None, None) == -1
    assert lib.dnr_normal_metrics(one, one, 0, 0, 4, 4, one, ws, one, None) == -2
    assert lib.dnr_normal_metrics(one, one, 0, 2, 0, 4, one, ws, one, None) == -2
    assert lib.dnr_normal_metrics(one, one, 0, 2, 4, 4, one, ws - 1, one, None) == -5
