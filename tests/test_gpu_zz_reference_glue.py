"""CUDA path against the glue goldens: outputs, loss dict and parameter gradients that the REFERENCE's own
get_outputs / get_loss_dict code produced (tests/golden/make_golden_model.py; gsplat served by the restatement).
Runs last in the GPU suite (file name) — it was written after round 1's GPU budget was spent, so its tolerances are
the ones the CUDA-vs-oracle tests of tests/test_gpu_model.py already meet on the same kind of scene."""
import os

import pytest
import torch

from tests.helpers import frac_close
from tests.test_oracle_glue_golden import FILES, PARAMS, load, model_from_golden

pytestmark = pytest.mark.gpu
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")


@needs_cuda
@pytest.mark.parametrize("f", FILES, ids=[os.path.basename(f) for f in FILES])
def test_model_matches_reference_glue_goldens(f):
    z = load(f)
    m, cam, batch = model_from_golden(z, device="cuda")
    if bool(z["eval"]):
        m.eval()
    out = m.get_outputs(cam)
    m.train()
    for k in ("rgb", "normal", "surface_normal", "accumulation"):
        frac, mx = frac_close(out[k], z["out_" + k], atol=2e-4)
        assert frac > 0.995, (k, frac, mx)
    covered = z["out_accumulation"] > 0
    d_got, d_want = out["depth"].detach().cpu()[covered], z["out_depth"][covered]
    assert float(((d_got - d_want).abs() <= 1e-3 * d_want.abs() + 1e-4).float().mean()) > 0.995
    # integer radii: identical up to ceil() flips caused by the view matrix being rounded differently on the way in
    assert float((m.radii.cpu() != z["out_radii"]).float().mean()) < 0.01
    ld = m.get_loss_dict(out, batch)
    want = float(z["out_main_loss"])
    assert abs(float(ld["main_loss"]) - want) <= 1e-3 * max(1.0, abs(want)), (float(ld["main_loss"]), want)
    assert abs(float(ld["scale_reg"]) - float(z["out_scale_reg"])) <= 1e-5 * max(1.0, float(z["out_scale_reg"]))
    (ld["main_loss"] + ld["scale_reg"]).backward()
    for k in PARAMS:
        got, w = m.gauss_params[k].grad.cpu(), z["grad_" + k]
        rel = float((got - w).norm() / (w.norm() + 1e-30))
        assert rel < 1e-2, (k, rel)
    torch.testing.assert_close(m.normals.detach().cpu(), z["out_gauss_normals"], rtol=1e-4, atol=1e-5)
