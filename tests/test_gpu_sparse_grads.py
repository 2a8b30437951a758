"""The flat gradient bucket's sparse mode: the rasterizer flags every Gaussian whose gradient rows it writes, the flags
accumulate until `FlatGradBucket.zero_()`, which then clears only the flagged rows (plus the dense `scales` segment and
the flags), and FusedAdam.step() reads only the flagged gradient rows.  These tests pin the invariants that make that
exact: after zero_() the bucket, its flags and the rasterizer's grad_records workspace are all zero; every non-zero row
is flagged; the sparse Adam step equals the dense one bit for bit; and a bucket whose flags do not cover its rows is
handled densely."""
import pytest
import torch

from tests.helpers import scene_and_camera

pytestmark = pytest.mark.gpu
needs_cuda = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")

H, W = 112, 144


def _model(params, step=30000, **cfg_kw):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.losses import DepthLossType

    kw = dict(use_depth_loss=True, depth_lambda=0.2, depth_loss_type=DepthLossType.EdgeAwareLogL1, ssim_lambda=0.2,
              sync_free=True)
    kw.update(cfg_kw)
    cfg = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", **kw)
    m = cfg.setup(device="cuda")
    m.load_gaussians(params)
    m.background_color = torch.tensor([0.1490, 0.1647, 0.2157])
    m.step = step
    m.train()
    return m


def _cameras(n=6):
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.synthetic import ring_cameras

    return [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], c["width"], c["height"], metadata={"cam_idx": i})
            for i, c in enumerate(ring_cameras(n, W, H))]


def _batch(seed=5):
    g = torch.Generator().manual_seed(seed)
    depth = 2 + 6 * torch.rand(H, W, 1, generator=g)
    return {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda(), "mono_depth": depth.cuda(),
            "normal": torch.rand(H, W, 3, generator=g).cuda()}


def _backward(m, cam, batch):
    ld = m.get_loss_dict(m.get_outputs(cam), dict(batch))
    (ld["main_loss"] + ld["scale_reg"]).backward()


def _assert_flags_cover_rows(bucket):
    """Every non-zero gradient row outside the dense segments belongs to a flagged Gaussian; grad_records is all zero."""
    assert bucket.flags_valid
    flagged = bucket.touched != 0
    assert 0 < int(flagged.sum()) < bucket.n_gauss
    for name, v in bucket.views.items():
        if name in bucket.dense_params:
            continue
        nz = (v.reshape(bucket.n_gauss, -1) != 0).any(dim=1)
        assert int(nz.sum()) > 0, name
        assert not bool((nz & ~flagged).any()), (name, int((nz & ~flagged).sum()))
    assert not bool(bucket.grad_records.any())


def _assert_all_zero(bucket):
    assert not bool(bucket.flat.any()), int((bucket.flat != 0).sum())
    assert not bool(bucket.touched.any())
    assert not bool(bucket.grad_records.any())


CONFIGS = {
    "default": dict(),
    "antialiased_two_pass": dict(rasterize_mode="antialiased", predict_normals=True),
    "normals_off": dict(predict_normals=False, use_normal_loss=False),
    "sh_degree_1": dict(step=1000),
    "LogL1": dict(depth_loss_type="LogL1"),
    "L1": dict(depth_loss_type="L1"),
    "mse": dict(depth_loss_type="mse"),
}


@needs_cuda
@pytest.mark.parametrize("name", list(CONFIGS))
def test_zero_clears_bucket_flags_and_records_after_eager_and_graphed_steps(name):
    with torch.cuda.stream(torch.cuda.Stream()):  # a capture cannot use the legacy default stream (graph_step.py)
        _zero_body(dict(CONFIGS[name]))


def _zero_body(kw):
    from dn_splatter_b200.graph_step import GraphedTrainStep
    from dn_splatter_b200.losses import DepthLossType
    from dn_splatter_b200.optim import FusedAdam

    if "depth_loss_type" in kw:
        kw["depth_loss_type"] = DepthLossType(kw["depth_loss_type"])
    params, _ = scene_and_camera(3000, W, H)
    m = _model(params, **kw)
    bucket = m.enable_flat_grads()
    opt = FusedAdam.for_model(m)
    cams, batch = _cameras(), _batch()
    for c in cams:
        c.camera_to_worlds = c.camera_to_worlds.cpu()
    for i in range(4):
        bucket.zero_()
        if i > 0:  # the first zero_() of a fresh bucket is dense; every later one is sparse
            _assert_all_zero(bucket)
        _backward(m, cams[i], batch)
        _assert_flags_cover_rows(bucket)
        opt.step()
    step = GraphedTrainStep(m, bucket, cams[0], batch, n_slots=1)
    for i in (1, 3):
        step(cams[i], 0)
        torch.cuda.synchronize()
        step.check_capacity(wait=True)
        _assert_flags_cover_rows(bucket)
        opt.step()
    bucket.zero_()
    _assert_all_zero(bucket)


@needs_cuda
def test_zero_after_densification():
    """Densification re-creates the bucket: the new one starts dense, then goes sparse with the same invariants."""
    from dn_splatter_b200.densify import _replace_params
    from dn_splatter_b200.optim import FusedAdam

    params, _ = scene_and_camera(3000, W, H)
    m = _model(params)
    bucket = m.enable_flat_grads()
    opt = FusedAdam.for_model(m)
    cams, batch = _cameras(), _batch()
    for i in range(2):
        bucket.zero_()
        _backward(m, cams[i], batch)
        opt.step()
    extra = 257
    new = {k: torch.cat([p.detach(), p.detach()[:extra] * 1.01]) for k, p in m.gauss_params.items()}
    _replace_params(m, opt.as_dict(m), new, lambda t: torch.cat([t, torch.zeros_like(t[:extra])]))
    bucket = m._bucket
    assert bucket.n_gauss == 3000 + extra and not bucket.flags_valid
    for i in range(2, 5):
        bucket.zero_()
        _assert_all_zero(bucket)
        _backward(m, cams[i], batch)
        _assert_flags_cover_rows(bucket)
        opt.step()
    bucket.zero_()
    _assert_all_zero(bucket)


@needs_cuda
def test_sparse_adam_is_bit_identical_to_dense_adam(monkeypatch):
    """On the same gradients, FusedAdam.step() over a bucket with valid flags (sparse gradient reads) and over plain
    copies of those gradients (dnr_adam_step) give bit-identical parameters and moments, step after step."""
    from dn_splatter_b200.optim import FusedAdam

    params, _ = scene_and_camera(3000, W, H)
    m = _model(params)
    bucket = m.enable_flat_grads()
    opt = FusedAdam.for_model(m)
    names = bucket.names
    twin = {k: torch.nn.Parameter(m.gauss_params[k].detach().clone()) for k in names}
    twin_opt = FusedAdam([{"params": [twin[g["name"]]], "lr": g["lr"], "eps": g["eps"], "name": g["name"]}
                          for g in opt.param_groups if g["name"] in twin])
    sparse_calls = []
    launch = FusedAdam._launch_reduce
    monkeypatch.setattr(FusedAdam, "_launch_reduce", staticmethod(lambda *a: (sparse_calls.append(1), launch(*a))[1]))
    cams, batch = _cameras(), _batch()
    for i in range(5):
        bucket.zero_()
        _backward(m, cams[i], batch)
        assert bucket.flags_valid
        for k in names:
            twin[k].grad = bucket.views[k].clone()
        opt.step()
        twin_opt.step()
        for k in names:
            p, q = m.gauss_params[k], twin[k]
            assert torch.equal(p.detach(), q.detach()), (i, k)
            assert torch.equal(opt.state[p]["exp_avg"], twin_opt.state[q]["exp_avg"]), (i, k)
            assert torch.equal(opt.state[p]["exp_avg_sq"], twin_opt.state[q]["exp_avg_sq"]), (i, k)
    assert len(sparse_calls) == 5  # every step of the bucket took the sparse path, none of the twin's


@needs_cuda
def test_bucket_filled_by_other_means_is_zeroed_and_stepped_densely(monkeypatch):
    from dn_splatter_b200 import dn_rasterize, get_viewmat
    from dn_splatter_b200.optim import FusedAdam
    from dn_splatter_b200.parallel import FlatGradBucket

    sparse_calls = []
    launch = FusedAdam._launch_reduce
    monkeypatch.setattr(FusedAdam, "_launch_reduce", staticmethod(lambda *a: (sparse_calls.append(1), launch(*a))[1]))
    params, _ = scene_and_camera(3000, W, H)
    leaf = {k: torch.nn.Parameter(v.cuda()) for k, v in params.items()}
    bucket = FlatGradBucket(leaf)
    opt = FusedAdam([{"params": [leaf[k]], "lr": 1e-3, "eps": 1e-15, "name": k} for k in bucket.names])

    def backward():
        cam = scene_and_camera(1, W, H, view=1)[1]
        c2w = cam["c2w"].cuda()
        K = torch.tensor([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], dtype=torch.float32, device="cuda")
        out = dn_rasterize(leaf["means"], leaf["quats"], leaf["scales"], leaf["opacities"], leaf["features_dc"],
                           leaf["features_rest"], get_viewmat(c2w), K, W, H, c2w=c2w, grad_sink=bucket.sink())
        (out.rgb.sum() + out.depth.sum()).backward()

    # a fresh bucket filled by other means (a copy, as the multi-GPU test's shadow replica is) is dense
    bucket.flat.copy_(torch.rand_like(bucket.flat))
    opt.step()
    assert not bucket.flags_valid and not sparse_calls
    bucket.zero_()  # dense: also the rows the copy filled
    _assert_all_zero(bucket)
    backward()
    assert bucket.flags_valid
    opt.step()
    assert len(sparse_calls) == 1
    # configs with parameter-only loss terms besides min-scale never go sparse
    m = _model(params, use_scale_regularization=True)
    b2 = m.enable_flat_grads()
    b2.zero_()
    _backward(m, _cameras()[1], _batch())
    assert not b2.flags_valid
