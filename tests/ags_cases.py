"""Inputs of the AGS-Mesh regulariser tests (tests/test_gpu_ags_loss.py, tests/test_ags_ref_cpu.py), on the CPU.

Normals are 4-pixel plateaus of random unit vectors in the [0,1] encoding, so the gt normal has flat regions (no edge)
and plateau borders (edges); the surface normal equals the gt normal on a third of the pixels, is a small perturbation
of it on another third (angles around 0.1) and random on the rest.  The gt depth has exact-threshold pixels (fp32(tol)
and one ulp either side), the float confidence map the codes 255 (dropped from step 7000 on) and 254 (kept).
"""
import torch

F32 = torch.float32
TOL = 0.1
STEPS = (100, 6999, 7000, 7001, 14999, 15000, 30000)


def _patches(t, H, W, b):
    return t.repeat_interleave(b, 0).repeat_interleave(b, 1)[:H, :W].contiguous()


def _unit(v):
    return v / v.norm(dim=-1, keepdim=True).clamp(min=1e-6)


def make_case(H, W, seed, normal_u8=False, conf_u8=False, img_u8=True):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    nrm = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    gn_s = _patches(_unit(nrm((H + 3) // 4, (W + 3) // 4, 3)), H, W, 4)
    pick = r(H, W, 1)
    sn_s = torch.where(pick < 1 / 3, gn_s, torch.where(pick < 2 / 3, _unit(gn_s + 0.1 * nrm(H, W, 3)), _unit(nrm(H, W, 3))))
    gn = (gn_s + 1) / 2
    if normal_u8:
        gn = (gn * 255).round().to(torch.uint8)
    sn = ((sn_s + 1) / 2).to(F32)
    pn = (r(H, W, 3)).to(F32)
    gd = 0.05 + 5 * r(H, W, 1)
    gd[r(H, W, 1) < 0.1] = 0.0
    t = torch.tensor(TOL, dtype=F32)
    ties = r(H, W, 1)
    gd[ties < 0.05] = t
    gd[(ties >= 0.05) & (ties < 0.08)] = torch.nextafter(t, torch.tensor(1.0))
    gd[(ties >= 0.08) & (ties < 0.11)] = torch.nextafter(t, torch.tensor(0.0))
    pd = gd + torch.where(r(H, W, 1) < 0.5, 0.5 * nrm(H, W, 1), 1e-4 * nrm(H, W, 1))
    codes = torch.randint(0, 256, (H, W, 1), generator=g)
    codes[r(H, W, 1) < 0.2] = 255
    codes[r(H, W, 1) < 0.1] = 254
    conf = codes.to(torch.uint8) if conf_u8 else codes.to(F32)
    img = (_patches(r((H + 1) // 2, (W + 1) // 2, 3), H, W, 2) * 255).round()
    img = img.to(torch.uint8) if img_u8 else (img / 255).to(F32)
    return dict(pd=pd.to(F32), gd=gd.to(F32), conf=conf, img=img, sn=sn, gn=gn, pn=pn)
