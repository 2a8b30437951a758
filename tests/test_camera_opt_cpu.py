"""Camera optimisation on the host (CPU): the exponential maps against torch.linalg.matrix_exp, the CameraOptimizer
module and its model wiring, the Trainer's gradient accumulation, and the two-rank pose-gradient reduction (gloo).  The
CPU proxy (tests/cpu_proxy.py) renders with the oracle, whose autograd carries the viewmat gradient."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dn_splatter_b200.camera_opt import (TAYLOR_THETA2, CameraOptimizer, CameraOptimizerConfig, exp_map_SE3,
                                         exp_map_SO3xR3)


def _hat(w):
    return torch.tensor([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]], dtype=torch.float64)


def _tangents():
    """Seeded tangents on both sides of the Taylor switch (|omega|^2 below and above TAYLOR_THETA2), plus exact zero."""
    g = torch.Generator().manual_seed(5)
    out = [torch.zeros(6, dtype=torch.float64)]
    for scale in (1e-6, 1e-3, 0.05, 0.09, 0.11, 0.3, 1.0, 2.5):
        for _ in range(3):
            v = torch.randn(6, generator=g, dtype=torch.float64)
            v[3:] = v[3:] / v[3:].norm() * scale
            out.append(v)
    theta2 = torch.stack([(t[3:] ** 2).sum() for t in out])
    assert bool((theta2 < TAYLOR_THETA2).any()) and bool((theta2 > TAYLOR_THETA2).any())
    return out


def test_exp_maps_equal_matrix_exp_in_fp64():
    for xi in _tangents():
        v, w = xi[:3], xi[3:]
        twist = torch.zeros(4, 4, dtype=torch.float64)
        twist[:3, :3], twist[:3, 3] = _hat(w), v
        want_se3 = torch.linalg.matrix_exp(twist)[:3, :4]
        want_so3 = torch.cat([torch.linalg.matrix_exp(_hat(w)), v[:, None]], dim=1)
        assert float((exp_map_SE3(xi[None])[0] - want_se3).abs().max()) <= 1e-9, xi
        assert float((exp_map_SO3xR3(xi[None])[0] - want_so3).abs().max()) <= 1e-9, xi


def test_exp_maps_at_zero_are_identity_with_the_generators_as_jacobian():
    eye = torch.eye(4, dtype=torch.float64)[:3]
    gens = []
    for k in range(6):
        G = torch.zeros(3, 4, dtype=torch.float64)
        if k < 3:
            G[k, 3] = 1.0
        else:
            G[:3, :3] = _hat(torch.eye(3, dtype=torch.float64)[k - 3])
        gens.append(G)
    want = torch.stack(gens, dim=-1)  # [3,4,6]
    for fn in (exp_map_SE3, exp_map_SO3xR3):
        xi = torch.zeros(1, 6, dtype=torch.float64)
        assert torch.equal(fn(xi)[0], eye)
        jac = torch.autograd.functional.jacobian(lambda x: fn(x[None])[0], xi[0])
        assert bool(torch.isfinite(jac).all())
        torch.testing.assert_close(jac, want, rtol=0, atol=1e-12)
        # float32 too: the first training step runs there
        jac32 = torch.autograd.functional.jacobian(lambda x: fn(x[None])[0], torch.zeros(6))
        torch.testing.assert_close(jac32, want.float(), rtol=0, atol=1e-6)


def test_mode_off_adds_no_parameters_and_no_group():
    from dn_splatter_b200.dn_model import DNSplatterModelConfig

    opt = CameraOptimizerConfig(mode="off").setup(num_cameras=4, device="cpu")
    assert list(opt.parameters()) == [] and opt.state_dict() == {}
    cfg = DNSplatterModelConfig(random_init=True, num_random=16)
    m = cfg.setup(device="cpu", num_train_data=3)
    assert "camera_opt" not in m.get_param_groups()
    assert not any(k.startswith("camera_optimizer") for k in m.state_dict())
    on = DNSplatterModelConfig(random_init=True, num_random=16, camera_optimizer=CameraOptimizerConfig(mode="SO3xR3"))
    torch.manual_seed(0)
    m_off = cfg.setup(device="cpu", num_train_data=3)
    torch.manual_seed(0)
    m_on = on.setup(device="cpu", num_train_data=3)
    # the zero-initialised pose parameter draws nothing from the RNG: identical Gaussians
    for k in m_off.gauss_params:
        assert torch.equal(m_off.gauss_params[k], m_on.gauss_params[k])
    assert set(m_on.state_dict()) - set(m_off.state_dict()) == {"camera_optimizer.pose_adjustment"}
    pa = m_on.get_param_groups()["camera_opt"]
    assert len(pa) == 1 and pa[0].shape == (3, 6) and not bool(pa[0].any())


@pytest.mark.parametrize("mode", ["SO3xR3", "SE3"])
def test_apply_to_camera(mode):
    from dn_splatter_b200.cameras import Cameras

    opt = CameraOptimizerConfig(mode=mode).setup(num_cameras=3, device="cpu")
    c2w = torch.tensor([[1.0, 0, 0, 0.5], [0, 0, -1, 2.0], [0, 1, 0, -1.0]])
    plain = Cameras(c2w[None], 50.0, 50.0, 20.0, 16.0, 40, 32)
    assert opt.apply_to_camera(plain) is plain.camera_to_worlds  # no cam_idx: the pose as given
    cam = Cameras(c2w[None], 50.0, 50.0, 20.0, 16.0, 40, 32, metadata={"cam_idx": 2})
    torch.testing.assert_close(opt.apply_to_camera(cam), c2w[None])  # zero adjustment: identity
    with torch.no_grad():
        opt.pose_adjustment[2] = torch.tensor([0.1, -0.2, 0.05, 0.02, -0.01, 0.03])
    adj = torch.cat([opt(slice(2, 3))[0], torch.tensor([[0.0, 0, 0, 1]])])
    torch.testing.assert_close(opt.apply_to_camera(cam)[0], c2w @ adj)  # right-multiplication: camera-frame correction
    torch.testing.assert_close(opt(torch.tensor([2])), opt(slice(2, 3)))  # device-index form selects the same row


def _scene_and_views(n_views, W, H, seed=4):
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.synthetic import ring_cameras

    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H, metadata={"cam_idx": i})
            for i, c in enumerate(ring_cameras(n_views, W, H))]
    g = torch.Generator().manual_seed(3)
    batches = [{"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8),
                "mono_depth": 2 + 6 * torch.rand(H, W, 1, generator=g),
                "normal": torch.rand(H, W, 3, generator=g)} for _ in range(n_views)]
    return cams, batches


def _config(mode="SO3xR3", **kw):
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.losses import DepthLossType

    base = dict(random_init=True, num_random=16, background_color="black", use_depth_loss=True, depth_lambda=0.2,
                depth_loss_type=DepthLossType.LogL1, ssim_lambda=0.0, sh_degree_interval=1,
                camera_optimizer=CameraOptimizerConfig(mode=mode))
    base.update(kw)
    return DNSplatterModelConfig(**base)


def test_model_loss_dict_keys_and_errors_with_camera_opt_on():
    from dn_splatter_b200.synthetic import make_scene
    from tests.cpu_proxy import cpu_proxy

    cams, batches = _scene_and_views(3, 40, 32)
    with cpu_proxy():
        keys = {}
        for mode in ("off", "SE3"):
            m = _config(mode).setup(device="cpu", num_train_data=3)
            m.load_gaussians(make_scene(60, seed=4))
            m.step = 10
            m.train()
            ld = m.get_loss_dict(m.get_outputs(cams[1]), dict(batches[1]))
            keys[mode] = set(ld)
        assert keys["off"] == keys["SE3"] == {"main_loss", "scale_reg"}  # no camera_opt_regularizer (the reference drops it)
        (ld["main_loss"] + ld["scale_reg"]).backward()
        g = m.camera_optimizer.pose_adjustment.grad
        assert bool(g[1].abs().gt(0).all()) and not bool(g[0].any()) and not bool(g[2].any())
        m.num_train_data = 1
        with pytest.raises(ValueError, match="cam_idx"):
            m.get_outputs(cams[1])
        m.eval()  # evaluation renders with the pose as given: no index check, no pose gradient
        m.get_outputs(cams[1])


def test_trainer_accumulates_the_pose_gradient_and_steps_every_accum_steps():
    from dn_splatter_b200.synthetic import make_scene
    from dn_splatter_b200.trainer import Trainer
    from tests.cpu_proxy import cpu_proxy

    n_views, accum, n_steps = 3, 3, 8
    cams, batches = _scene_and_views(n_views, 40, 32)
    with cpu_proxy():
        m = _config(refine_every=1000, warmup_length=1000).setup(device="cpu", num_train_data=n_views)
        m.load_gaussians(make_scene(60, seed=4))
        tr = Trainer(m, lambda s: (cams[s % n_views], dict(batches[s % n_views])), max_steps=100, camera_opt_accum=accum)
        pa = m.camera_optimizer.pose_adjustment
        per_step, stepped_with = [], []
        pa.register_hook(lambda g: per_step.append(g.detach().clone()))
        real_step = tr.camera_opt.step

        def spy():
            stepped_with.append(pa.grad.detach().clone())
            return real_step()

        tr.camera_opt.step = spy
        moved = []
        for step in range(n_steps):
            before = pa.detach().clone()
            tr.train_iteration()
            moved.append(not torch.equal(before, pa.detach()))
    assert len(per_step) == n_steps
    assert [s for s in range(n_steps) if moved[s]] == [s for s in range(n_steps) if s % accum == accum - 1] == [2, 5]
    for k, got in enumerate(stepped_with):
        want = torch.stack(per_step[k * accum:(k + 1) * accum]).sum(0)
        torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-9)
        assert bool(got.abs().gt(0).any())


def _cam_opt_worker(rank, world, port, n_steps, accum, ret):
    from dn_splatter_b200.synthetic import make_scene
    from dn_splatter_b200.trainer import Trainer
    from tests.cpu_proxy import cpu_proxy

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    n_views = 4
    cams, batches = _scene_and_views(n_views, 40, 32)
    with cpu_proxy():
        m = _config(refine_every=1000, warmup_length=1000).setup(device="cpu", num_train_data=n_views)
        m.load_gaussians(make_scene(60, seed=4))

        def next_train(step):  # rank r renders views {i : i mod world == r}
            v = (step * world + rank) % n_views
            return cams[v], dict(batches[v])

        tr = Trainer(m, next_train, max_steps=100, world_size=world, camera_opt_accum=accum)
        for _ in range(n_steps):
            tr.train_iteration()
    pa = m.camera_optimizer.pose_adjustment.detach().clone()
    theirs = [torch.empty_like(pa) for _ in range(world)]
    dist.all_gather(theirs, pa)
    if rank == 0:
        ret.put((pa.numpy().copy(), all(torch.equal(t, pa) for t in theirs)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_trainer_keeps_poses_identical_and_equal_to_one_process_over_the_union():
    from dn_splatter_b200.densify import exponential_lr
    from dn_splatter_b200.synthetic import make_scene
    from dn_splatter_b200.trainer import Trainer
    from tests.cpu_proxy import cpu_proxy

    world, n_steps, accum, n_views = 2, 6, 2, 4
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_cam_opt_worker, args=(r, world, port, n_steps, accum, q)) for r in range(world)]
    for p in procs:
        p.start()
    got, same = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert same, "pose replicas diverged"
    # one process renders both ranks' views every step (the union), then the same optimiser schedule
    cams, batches = _scene_and_views(n_views, 40, 32)
    with cpu_proxy():
        m = _config(refine_every=1000, warmup_length=1000).setup(device="cpu", num_train_data=n_views)
        m.load_gaussians(make_scene(60, seed=4))
        tr = Trainer(m, None, max_steps=100, camera_opt_accum=accum)
        for step in range(n_steps):
            m.train()
            m.step_cb(step)
            tr.bucket.zero_()
            if step % accum == 0:
                tr.camera_opt.zero_grad(set_to_none=False)
            for r in range(world):
                v = (step * world + r) % n_views
                ld = m.get_loss_dict(m.get_outputs(cams[v]), dict(batches[v]))
                (ld["main_loss"] + ld["scale_reg"]).backward()
            for name, opt in tr.optimizers.items():
                g = tr.groups[name]
                if g.get("lr_final"):
                    for pg in opt.param_groups:
                        pg["lr"] = exponential_lr(g["lr"], g["lr_final"], step, g["max_steps"])
                opt.step()
            tr._camera_opt_step(step)
    want = m.camera_optimizer.pose_adjustment.detach()
    assert bool(want.abs().gt(0).all())  # every camera's pose moved
    torch.testing.assert_close(torch.from_numpy(got), want, rtol=1e-4, atol=1e-7)


def test_project_bwd_requires_touched_flags_and_accumulation():
    import ctypes as C

    from dn_splatter_b200 import _lib as L

    lib = L.load()
    a = L.DnrArgs()
    a.n_gauss, a.width, a.height, a.tile_size, a.sh_degree, a.sh_bases = 10, 32, 32, 16, 0, 1
    for name in ("viewmat", "K", "means", "quats", "scales", "opacities", "sh_dc", "radii", "grad_records", "v_means",
                 "v_quats", "v_scales", "v_opacities", "v_sh_dc", "v_viewmat"):
        setattr(a, name, 16)  # non-NULL dummies: the argument checks come first, nothing is dereferenced
    a.flags = L.FLAG_ACCUMULATE
    assert lib.dnr_project_bwd(C.byref(a), None) == -1  # DNR_E_NULL: no touched flags
    a.touched, a.flags = 16, 0
    assert lib.dnr_project_bwd(C.byref(a), None) == -3  # DNR_E_OPTION: the kernel only accumulates
