"""Generates tests/golden/dn_metrics.npz by executing the REFERENCE's own render metrics, unmodified, imported from
where they lie:

  * dn_splatter/metrics.py's mean_angular_error, DepthMetrics and NormalMetrics on metric-level cases;
  * dn_model.py's DNSplatterModel.get_metrics_dict (:731-807) and get_image_metrics_and_images (:809-926), unbound, on
    a bare model object with the stubs of make_golden_model.py.

torchmetrics is absent: its PSNR and SSIM are the fp64 oracle (oracle/metrics_ref.py), its LPIPS a deterministic
stand-in that is not symmetric in its arguments (so the goldens pin the argument order and shapes as well as the key
names).  make_golden_model.py stubs torchvision; the real torchvision.transforms.functional is imported first, so
TF.resize is torchvision's own.

Run only where /root/reference exists:   python tests/golden/make_golden_metrics.py
"""
import os
import sys
import types

import numpy as np
import torch
import torchvision.transforms.functional  # noqa: F401  (the real module, before the stubs are installed)

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))
sys.path.insert(0, ROOT)
sys.path.insert(0, OUT)

import make_golden_model as MGM  # noqa: E402
from oracle import metrics_ref as R  # noqa: E402


def lpips_stub(a, b):
    """Deterministic LPIPS stand-in: depends on the order and the [1,3,H,W] layout of its arguments."""
    assert a.dim() == 4 and a.shape[:2] == (1, 3) and a.shape == b.shape
    return (a - b).abs().mean() + 0.25 * a[:, 0].mean() + 0.125 * b[:, 2].mean()


class _Fn(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f = f

    def forward(self, *a):
        return self.f(*a)


def _psnr(a, b):
    return R.rgb(b.permute(0, 2, 3, 1), a.permute(0, 2, 3, 1))["psnr"].float()


def _ssim(a, b):
    return R.rgb(b.permute(0, 2, 3, 1), a.permute(0, 2, 3, 1))["ssim"].float()


def metric_cases(Mt, z):
    g = torch.Generator().manual_seed(11)
    rand = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    depth_cases = {}
    p, t = 0.5 + 4 * rand(1, 37, 53), 0.5 + 4 * rand(1, 37, 53)
    depth_cases["noise"] = (p, t)
    p, t = 0.5 + 4 * rand(3, 20, 30), 0.05 + 4 * rand(3, 20, 30)
    t[:, :2] = 0.1  # exactly the tolerance: excluded
    p[:, 5:7] = 0.0  # pred 0 where gt is valid: rmse_log inf, a1 counts them as misses
    t[:, 7:9] = 0.0
    depth_cases["masked"] = (p, t)
    p = 1 + rand(1, 16, 16)
    depth_cases["close"] = (p, p * (1 + 0.3 * (rand(1, 16, 16) - 0.5)))
    depth_cases["empty"] = (1 + rand(1, 12, 12), 0.05 * rand(1, 12, 12))
    dm = Mt.DepthMetrics()
    for k, (p, t) in depth_cases.items():
        out = dm(p, t)
        z[f"depth_{k}_pred"], z[f"depth_{k}_gt"] = p.numpy(), t.numpy()
        z[f"depth_{k}_out"] = np.array([float(v) for v in out], dtype=np.float64)
    normal_cases = {"b1": (1, 21, 17), "b3": (3, 16, 12), "odd": (1, 9, 11)}
    nm = Mt.NormalMetrics()
    for k, (b, h, w) in normal_cases.items():
        p, t = rand(b, 3, h, w), rand(b, 3, h, w)
        out = nm(p, t)
        z[f"normal_{k}_pred"], z[f"normal_{k}_gt"] = p.numpy(), t.numpy()
        z[f"normal_{k}_out"] = np.array([float(v) for v in out], dtype=np.float64)
        z[f"normal_{k}_mae_map"] = Mt.mean_angular_error(p, t).numpy()


def bare_model(M, cfg_kw, scales, training=False, step=0):
    cfg = M.DNSplatterModelConfig(**cfg_kw)
    m = M.DNSplatterModel.__new__(M.DNSplatterModel)
    torch.nn.Module.__init__(m)
    m.config, m.step = cfg, step
    m.gauss_params = {"means": torch.zeros(scales.shape[0], 3), "scales": scales}
    Mt = sys.modules["dn_splatter.metrics"]
    m.rgb_metrics = Mt.RGBMetrics()
    m.rgb_metrics.psnr, m.rgb_metrics.ssim, m.rgb_metrics.lpips = _Fn(_psnr), _Fn(_ssim), _Fn(lpips_stub)
    m.psnr, m.ssim, m.lpips = _Fn(_psnr), _Fn(_ssim), _Fn(lpips_stub)
    m.depth_metrics, m.normal_metrics = Mt.DepthMetrics(), Mt.NormalMetrics()
    m.mse_loss = torch.nn.MSELoss()
    m.train(training)
    return m


def model_cases(M, z):
    MGM.SplatfactoModel.num_points = property(lambda self: self.means.shape[0])
    g = torch.Generator().manual_seed(23)
    rand = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    scales = torch.log(0.01 + 0.1 * rand(50, 3))
    z["model_scales"] = scales.numpy()
    H, W = 40, 56
    cases = {
        # get_metrics_dict at full resolution (eval) and while training at half resolution (TF.resize of the targets)
        "md_full": dict(method="metrics", d=1, out_hw=(H, W), depth=True),
        "md_half": dict(method="metrics", d=2, out_hw=(H // 2, W // 2), depth=True),
        "md_nodepth": dict(method="metrics", d=1, out_hw=(H, W), depth=False),
        # get_image_metrics_and_images; depth and normal rendered at another size than the targets
        "im_full": dict(method="images", out_hw=(H, W), depth=True, normal=True),
        "im_resize": dict(method="images", out_hw=(H, W), depth_hw=(H // 2, W // 2), normal_hw=(H // 2 + 3, W // 2 - 1),
                          depth=True, normal=True),
        "im_rgb_only": dict(method="images", out_hw=(H, W), depth=False, normal=False),
    }
    for tag, c in cases.items():
        oh, ow = c["out_hw"]
        dh, dw = c.get("depth_hw", (oh, ow))
        nh, nw = c.get("normal_hw", (oh, ow))
        outputs = {"rgb": rand(oh, ow, 3), "depth": 0.5 + 3 * rand(dh, dw, 1), "normal": rand(nh, nw, 3)}
        batch = {"image": rand(H, W, 3)}
        if c["depth"]:
            d = 0.5 + 3 * rand(H, W, 1)
            d[rand(H, W, 1) < 0.1] = 0.0
            batch["sensor_depth"] = d
        if c.get("normal"):
            batch["normal"] = rand(H, W, 3)
        if c["method"] == "metrics":
            # num_downscales = 1 with step 0: _get_downscale_factor() = 2 while training
            m = bare_model(M, dict(use_depth_loss=True, num_downscales=1 if c["d"] > 1 else 0), scales,
                           training=c["d"] > 1)
            res = M.DNSplatterModel.get_metrics_dict(m, outputs, batch)
            images = {}
        else:
            m = bare_model(M, dict(use_depth_loss=True), scales)
            res, images = M.DNSplatterModel.get_image_metrics_and_images(m, outputs, batch)
        z[f"{tag}_cfg"] = np.array(repr(c))
        z.update({f"{tag}_out_{k}": v.numpy() for k, v in outputs.items()})
        z.update({f"{tag}_batch_{k}": v.numpy() for k, v in batch.items()})
        z[f"{tag}_keys"] = np.array(list(res.keys()))
        z[f"{tag}_values"] = np.array([float(v) for v in res.values()], dtype=np.float64)
        z.update({f"{tag}_images_{k}": v.detach().numpy() for k, v in images.items()})
        print(tag, {k: round(float(v), 5) for k, v in res.items()})


def main():
    M = MGM.install()
    Mt = sys.modules["dn_splatter.metrics"]
    assert isinstance(sys.modules["torchvision.transforms.functional"], types.ModuleType)
    assert hasattr(M.TF.resize, "__code__"), "TF.resize must be torchvision's own"
    z = {}
    metric_cases(Mt, z)
    model_cases(M, z)
    np.savez_compressed(os.path.join(OUT, "dn_metrics.npz"), **z)


if __name__ == "__main__":
    main()
