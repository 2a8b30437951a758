"""The fp64 AGS-Mesh oracle (oracle/ags_ref.py) against the reference's goldens and the torch strategy, and the slips it
must catch: each plausible mistake in the kernel's rule moves the result past the GPU test's tolerance on the GPU test's
own cases (tests/ags_cases.py), by the printed factor."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import ags_ref
from tests.ags_cases import TOL, make_case

F32, F64 = torch.float32, torch.float64
GOLD_TOL = dict(rtol=1e-5, atol=1e-6)
VALUE_RTOL = 2e-6  # tests/test_gpu_ags_loss.py
MAP_NORM = 1e-6
EDGE_BAND = 2e-6


@pytest.fixture(scope="module")
def z(golden_dir):
    d = np.load(os.path.join(golden_dir, "dn_reference_modules.npz"))
    return {k: torch.from_numpy(d[k]) for k in d.files}


def test_oracle_reproduces_the_reference_goldens(z):
    sn, gn, pn = z["in_sn"], z["in_gn"], z["in_pn"]
    lap, scale = ags_ref.laplacian_r(gn)
    band = ags_ref.dilate((lap - ags_ref.EDGE_T).abs() <= EDGE_BAND * scale)
    got = ags_ref.find_edges(gn)
    want = z["out_find_edges_3"].bool()
    print(f"find_edges: {int(band.sum())} in-band elements")
    assert torch.equal(got[~band], want[~band])
    torch.testing.assert_close(ags_ref.mean_angular_error(sn, gn).float(), z["out_mean_angular_error"], **GOLD_TOL)
    for step in (100, 8000, 16000):
        torch.testing.assert_close(ags_ref.normal_loss_signed(step, sn, gn, pn).float(), z[f"out_ags_normal_{step}"], **GOLD_TOL)
    d = ags_ref.depth_loss_signed(100, z["in_pd"], z["in_gd"], z["in_conf"], z["in_img"])
    torch.testing.assert_close(d.float(), z["out_ags_depth_100"], **GOLD_TOL)
    scale_term = torch.exp(z["in_scales"].to(F64)).min(1)[0].mean()
    tot = d + ags_ref.normal_loss_signed(100, sn, gn, pn) + scale_term
    torch.testing.assert_close(tot.float(), z["out_ags_total_100"], **GOLD_TOL)


@pytest.mark.parametrize("step", [100, 7000, 8000, 16000])
def test_oracle_matches_torch_strategy_on_random_content(step):
    from dn_splatter_b200.regularization_strategy import AGSMeshRegularization

    case = make_case(40, 56, seed=step, img_u8=False)
    s, g, n = ags_ref.signed(case["sn"]), ags_ref.signed(case["gn"]), ags_ref.signed(case["pn"])
    conf = ags_ref.gate_map(case["conf"], raw=True)
    ags = AGSMeshRegularization()
    got = ags.get_depth_loss(step=step, pred_depth=case["pd"], gt_depth=case["gd"], confidence_map=conf, gt_img=case["img"])
    got = got + ags.get_normal_loss(step, s, g, n)
    want = ags_ref.ags_loss(case["pd"], case["gd"], case["conf"], case["img"], case["sn"], case["gn"], case["pn"],
                            depth_type=1, depth_lambda=0.2, tol=TOL, normal_lambda=0.1, step=step)["value"]
    torch.testing.assert_close(got.double(), want, rtol=1e-5, atol=1e-7)


def _ref(case, step, **kw):
    args = dict(depth_type=1, depth_lambda=0.2, tol=TOL, normal_lambda=0.1, step=step)
    args.update(kw)
    return ags_ref.ags_loss(case["pd"], case["gd"], case["conf"], case["img"], case["sn"], case["gn"], case["pn"], **args)


def _factor(a, b):
    return abs(float(a) - float(b)) / (VALUE_RTOL * max(abs(float(b)), 1e-30))


def _mask_slip(case, step, slip):
    """The surface term with the selection computed by a slipped rule (edge mode)."""
    g = ags_ref.signed(case["gn"])
    if slip == "pad_g":  # zero padding of g, not of r: r = 1 / (0 + 1e-6) outside the image
        gp = torch.nn.functional.pad(g.to(F32), (1, 1, 1, 1))
        r = (1.0 / (gp + torch.tensor(1e-6, dtype=F32))).to(F64)
        lap = r[:, :-2, 1:-1] + r[:, 2:, 1:-1] + r[:, 1:-1, :-2] + r[:, 1:-1, 2:] - 4 * r[:, 1:-1, 1:-1]
        keep = ~ags_ref.dilate(lap > ags_ref.EDGE_T)
    else:
        lap, _ = ags_ref.laplacian_r(g)
        e = lap > ags_ref.EDGE_T
        if slip == "no_dilation":
            keep = ~e
        else:  # dilation across channels
            keep = ~ags_ref.dilate(e.any(0, keepdim=True)).expand(3, -1, -1)
    return _ref(case, step, keep=keep)["value"]


def test_slips_leave_the_gpu_rule():
    case = make_case(81, 49, seed=81 * 131 + 49 + 7 * 6 + 1, img_u8=True)
    factors = {}
    right = _ref(case, 8000)
    d = _ref(case, 8000)["depth"]
    factors["(1 + lambda) depth weight"] = _factor(right["value"] - d + (1 + 0.2) * (d / 0.2), right["value"])
    at = _ref(case, 7000)
    no_gate = ags_ref.ags_loss(case["pd"], case["gd"], case["conf"], case["img"], case["sn"], case["gn"], case["pn"],
                               depth_type=1, depth_lambda=0.2, tol=TOL, normal_lambda=0.1, step=6999)
    factors["confidence gate at step > 7000"] = _factor(no_gate["depth"], at["depth"])
    lam_early = _ref(case, 7000, normal_lambda=0.1)
    with_lam = lam_early["depth"] + (_ref(case, 7001)["surface"] + _ref(case, 7001)["pred"])
    factors["lam at step >= 7000"] = _factor(with_lam, at["value"])
    for slip in ("pad_g", "no_dilation", "across_channels"):
        factors[slip] = _factor(_mask_slip(case, 8000, slip), right["value"])
    surf_3hw = right["surface"] * right["keep"].sum() / right["keep"].numel()
    factors["surface term over 3HW"] = _factor(right["depth"] + surf_3hw + right["pred"], right["value"])
    vn = right["v_normal"]
    factors["pred-normal gradient without its 2"] = float((vn / 2 - vn).norm() / vn.norm()) / MAP_NORM
    for k, f in factors.items():
        print(f"slip {k}: {f:.3g} x the tolerance")
    assert all(f > 1 and math.isfinite(f) for f in factors.values()), factors
