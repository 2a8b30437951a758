"""Times kernels around the hot path against the path each one replaces, so one GPU run decides which becomes the
default.

    python scripts/exp_bench.py [--n 1000000] [--reps 20] > exp_bench.jsonl

Rows (one JSON line each):
  ssim        FusedSSIM fwd+bwd  vs  dn_model.ssim (torch convs + autograd) at 1920x1080x3
  adam        FusedAdam (1 launch) vs  7 x torch.optim.Adam (default foreach) and fused=True, N Gaussians, SH degree 3
  camera_opt  project_bwd with vs without the view-matrix gradient (stage events), and the captured 1080p training step
              (GraphedTrainStep + FusedAdam) with camera optimisation off vs SO3xR3
  mesh        TSDF fusion of 200 ring views at 1920x1080 into a 512^3 grid over the scene cube (render + integrate, and
              integrate alone, from CUDA events), marching cubes of that volume, export_marching_cubes_mesh at 256^3
  poisson     export_dn_poisson_mesh on the same scene and views at depth 9 and 10 with CUDA-event stage times (render +
              back-project, sort + splat, solve and its cycle count, extract, trim + write), the multigrid's algorithmic
              bytes per cycle and the smoother's share of 3.35 TB/s (red-black kernels timed by torch.profiler in a
              separate solve), and export_gaussians_poisson_mesh at depth 9
  mesh_eval   the TSDF mesh of that scene against its depth-9 `dn` Poisson mesh, 200 ring views at 1080p: CUDA-event
              times of depth rendering, visibility counts, subdivision, sampling and nearest neighbours, and the fp64
              numpy oracle's visibility counts and cKDTree metrics on a subset for scale
  isooctree   export_isooctree_mesh's stages on the same scene, 200 ring views at 1080p, pixel_stride 6, max_depth 10:
              render into the frame buffers, hint cloud, octree + corners, isoFunc at the corners, dense fill, marching
              cubes (CUDA events), and the fp64 numpy oracle's isoFunc rate (point-frame evaluations per second) on a
              subset for scale
  depth_normals  DepthNormalConsistency's per-frame device work on a room frame (0.3-8 m, 5 % / 40 % holes in blobs) at
              1920x1440 and 1024x768, k = 200: back-projection, normals (k-NN + covariance + FastEigen3x3 + orientation)
              and the consistency pass (CUDA events), candidates examined per search (mean) and per surface pixel (mean,
              p99), and the fp64 numpy oracle's rate on a 64x48 crop for scale
Each row also checks agreement with the reference path (max abs / rel error), so a faster-but-wrong kernel is visible.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=1_000_000)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--only", default="")
args = ap.parse_args()


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def emit(row):
    print(json.dumps(row), flush=True)


def bench_ssim():
    from dn_splatter_b200.dn_model import ssim
    from dn_splatter_b200.regularization_strategy import FusedSSIM

    H, W = 1080, 1920
    g = torch.Generator().manual_seed(0)
    x = torch.rand(H, W, 3, generator=g).cuda().requires_grad_(True)
    y = (x.detach().cpu() * 0.7 + 0.3 * torch.rand(H, W, 3, generator=g)).cuda()

    def ref():
        s = ssim(y.permute(2, 0, 1)[None], x.permute(2, 0, 1)[None])
        return s, torch.autograd.grad(s, x)[0]

    def fused():
        s = FusedSSIM.apply(x, y)
        return s, torch.autograd.grad(s, x)[0]

    (sr, gr), (sf, gf) = ref(), fused()
    emit({"row": "ssim", "torch_ms": timed(ref, args.reps), "fused_ms": timed(fused, args.reps),
          "value_abs_err": abs(float(sr) - float(sf)), "grad_rel_err": float((gr - gf).norm() / gr.norm())})


def bench_adam():
    from dn_splatter_b200.optim import FusedAdam

    n = args.n
    shapes = {"means": (n, 3), "scales": (n, 3), "quats": (n, 4), "features_dc": (n, 3), "features_rest": (n, 15, 3),
              "opacities": (n, 1)}
    lrs = {"means": 1.6e-4, "scales": 5e-3, "quats": 1e-3, "features_dc": 2.5e-3, "features_rest": 1.25e-4, "opacities": 5e-2}
    g = torch.Generator(device="cuda").manual_seed(0)

    def make():
        torch.manual_seed(0)
        ps = {k: torch.nn.Parameter(torch.randn(*s, device="cuda", generator=g)) for k, s in shapes.items()}
        for p in ps.values():
            p.grad = torch.randn(p.shape, device="cuda", generator=g) * 1e-3
        return ps

    a = make()
    fused = FusedAdam([{"params": [p], "lr": lrs[k], "eps": 1e-15, "name": k} for k, p in a.items()])
    b = make()
    for k in a:
        b[k].data.copy_(a[k].data)
        b[k].grad.copy_(a[k].grad)
    ref = [torch.optim.Adam([p], lr=lrs[k], eps=1e-15) for k, p in b.items()]
    fused.step()
    for o in ref:
        o.step()
    err = max(float((a[k] - b[k]).abs().max()) for k in a)
    c = make()
    ref_fused = [torch.optim.Adam([p], lr=lrs[k], eps=1e-15, fused=True) for k, p in c.items()]
    floats = sum(p.numel() for p in a.values())
    t_f = timed(fused.step, args.reps)
    emit({"row": "adam", "n_gauss": n, "floats": floats, "fused_ms": t_f,
          "torch_foreach_ms": timed(lambda: [o.step() for o in ref], args.reps),
          "torch_fused_ms": timed(lambda: [o.step() for o in ref_fused], args.reps),
          "fused_GBps": floats * 28 / t_f / 1e6, "param_abs_err_after_1_step": err})


def bench_camera_opt():
    import dn_splatter_b200.rasterize as R
    from dn_splatter_b200 import dn_rasterize, get_viewmat
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import CameraOptimizerConfig, DNSplatterModelConfig
    from dn_splatter_b200.graph_step import GraphedTrainStep
    from dn_splatter_b200.losses import DepthLossType
    from dn_splatter_b200.optim import FusedAdam
    from dn_splatter_b200.synthetic import BACKGROUND, make_scene, ring_cameras

    W, H, n_views = 1920, 1080, 200
    ring = ring_cameras(n_views, W, H)
    row = {"row": "camera_opt", "n_gauss": args.n, "resolution": f"{W}x{H}"}
    # project_bwd alone: the same view, with and without a viewmat that requires grad
    cam = ring[3]
    K = torch.tensor([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], dtype=torch.float32, device="cuda")
    c2w = cam["c2w"].cuda()
    grads = {}
    for pose_grad in (False, True):
        p = {k: v.cuda().requires_grad_(True) for k, v in make_scene(args.n, seed=0).items()}
        vm = get_viewmat(c2w).detach().requires_grad_(pose_grad)
        out = dn_rasterize(p["means"], p["quats"], p["scales"], p["opacities"], p["features_dc"], p["features_rest"], vm, K, W,
                           H, background=BACKGROUND, c2w=c2w)
        loss = (out.rgb.sum() + out.depth.sum() * 0.1 + out.normal.sum()) * 1e-3
        inputs = list(p.values()) + ([vm] if pose_grad else [])
        R.STAGE_EVENTS = []
        for _ in range(args.reps):
            gr = torch.autograd.grad(loss, inputs, retain_graph=True)
        torch.cuda.synchronize()
        t = sorted(a.elapsed_time(b) for name, a, b in R.STAGE_EVENTS if name == "project_bwd")
        R.STAGE_EVENTS = None
        row["project_bwd_ms_pose_grad" if pose_grad else "project_bwd_ms"] = t[len(t) // 2]
        grads[pose_grad] = gr[:6]
    row["param_grad_rel_err"] = max(float((x - y).norm() / (x.norm() + 1e-30)) for x, y in zip(grads[False], grads[True]))
    # the captured training step (bench.py's loss configuration) over the camera ring, Adam included
    g = torch.Generator().manual_seed(1)
    batch = {"image": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda(),
             "mono_depth": (2 + 6 * torch.rand(H, W, 1, generator=g)).cuda(),
             "normal": (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).cuda()}
    for mode in ("off", "SO3xR3"):
        cfg = DNSplatterModelConfig(random_init=True, num_random=16, use_depth_loss=True, depth_lambda=0.2,
                                    depth_loss_type=DepthLossType.EdgeAwareLogL1, ssim_lambda=0.2, background_color="black",
                                    sync_free=True, camera_optimizer=CameraOptimizerConfig(mode=mode))
        m = cfg.setup(device="cuda", num_train_data=n_views)
        m.load_gaussians(make_scene(args.n, seed=0))
        m.step = 30000
        m.train()
        cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H, metadata={"cam_idx": i})
                for i, c in enumerate(ring)]
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            bucket = m.enable_flat_grads()
            opt = FusedAdam.for_model(m)
            for i in range(0, n_views, 25):  # sync-free capacity statistics for the capture
                bucket.zero_()
                ld = m.get_loss_dict(m.get_outputs(cams[i]), dict(batch))
                (ld["main_loss"] + ld["scale_reg"]).backward()
            del ld
            step = GraphedTrainStep(m, bucket, cams[0], batch, n_slots=1)

            def one(s=[0]):
                s[0] += 1
                step(cams[(37 * s[0]) % n_views], 0)
                opt.step()

            row[f"step_ms_{mode}"] = timed(one, args.reps)
            step.check_capacity(wait=True)
        del step, m, bucket, opt
        torch.cuda.empty_cache()
    emit(row)


def bench_knn():
    import time

    from dn_splatter_b200.sugar import KnnIndex
    from oracle import sugar_ref as S  # sklearn, the reference's backend: timed on the host as the baseline

    n, m = args.n, 200_000
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, 3, generator=g) * torch.tensor([3.0, 3.0, 0.5])
    y = x[torch.randint(0, n, (m,), generator=g)] + 0.01 * torch.randn(m, 3, generator=g)
    xc, yc = x.cuda(), y.cuda()
    t_build = timed(lambda: KnnIndex(xc), 5)
    index = KnnIndex(xc)
    t_query = timed(lambda: index.query(yc, 16), 5)
    t0 = time.time()
    want = S.knn_sk(x, y[:20_000], 16)
    t_sk = (time.time() - t0) * 1e3 * (m / 20_000)
    got = index.query(yc[:20_000], 16).cpu()
    emit({"row": "knn", "n_points": n, "n_queries": m, "build_ms": t_build, "query_ms": t_query,
          "sklearn_ms_extrapolated": t_sk, "index_agreement": float((got == want).float().mean())})


def bench_render_service():
    """SURVEY 8f-1: forward-only render-all-views loop (what gs-mesh / ns-eval do), maps kept on the device or copied
    to pinned host buffers."""
    import time

    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.render_service import ViewRenderer
    from dn_splatter_b200.synthetic import make_scene, ring_cameras

    W, H, n_views = 1920, 1080, 48
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", sync_free=True).setup(device="cuda")
    m.load_gaussians(make_scene(args.n, seed=0))
    m.step = 30000
    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H) for c in ring_cameras(n_views, W, H)]
    row = {"row": "render_service", "n_gauss": args.n, "views": n_views, "resolution": f"{W}x{H}"}
    for to_host in (False, True):
        r = ViewRenderer(m, to_host=to_host)
        for _ in r.render(cams[:8]):  # warm-up (also seeds the sync-free capacity)
            pass
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in r.render(cams):
            pass
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / n_views
        row["ms_per_view_host" if to_host else "ms_per_view_device"] = dt * 1e3
        row["mpix_s_host" if to_host else "mpix_s_device"] = W * H / 1e6 / dt
    emit(row)


def bench_mesh():
    """mesh.py on the bench scene.  Integrate's algorithmic bytes: a 16 B read + 16 B write per updated voxel plus its
    4 B depth and 12 B rgb gathers (the depth reads of in-frustum voxels that are not updated are not counted)."""
    import subprocess
    import tempfile
    import time

    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.mesh import TSDFVolume, export_marching_cubes_mesh
    from dn_splatter_b200.render_service import ViewRenderer
    from dn_splatter_b200.synthetic import make_scene, ring_cameras

    W, H, n_views, res = 1920, 1080, 200, 512
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", sync_free=True).setup(device="cuda")
    m.load_gaussians(make_scene(args.n, seed=0))
    m.step = 30000
    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H) for c in ring_cameras(n_views, W, H)]
    bounds, voxel = ((-5.0, -5.0, -5.0), (5.0, 5.0, 5.0)), 10.0 / res  # make_scene's means fill the cube [-5, 5]^3
    row = {"row": "mesh", "card": card, "n_gauss": args.n, "views": n_views, "resolution": f"{W}x{H}"}
    r = ViewRenderer(m, keys=("rgb", "depth"), to_host=False)
    vol = TSDFVolume(bounds, voxel_size=voxel, sdf_trunc=3 * voxel)
    row["grid"] = "x".join(map(str, vol.dims))
    for idx, maps in r.render(cams[:8]):  # warm-up: captures the forward graphs
        vol.integrate(maps["depth"], maps["rgb"], cams[idx])
    maps = next(iter(r.render(cams[:1])))[1]
    depth, rgb = maps["depth"].clone(), maps["rgb"].clone()
    vol.voxels.zero_()
    vol.integrate(depth, rgb, cams[0])
    updated = int((vol.voxels[:, 1] > 0).sum())
    t_int = timed(lambda: vol.integrate(depth, rgb, cams[0]), args.reps)
    row["integrate_ms"] = t_int
    row["integrate_updated_voxels"] = updated
    row["integrate_gb_s"] = updated * (32 + 16) / (t_int * 1e-3) / 1e9
    row["integrate_frac_of_3.35TB_s"] = row["integrate_gb_s"] / 3350.0
    vol.voxels.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for idx, maps in r.render(cams):
        vol.integrate(maps["depth"], maps["rgb"], cams[idx])
    e1.record()
    torch.cuda.synchronize()
    row["render_integrate_ms_per_view"] = e0.elapsed_time(e1) / n_views
    mesh = vol.extract_mesh()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        mesh = vol.extract_mesh()
    torch.cuda.synchronize()
    row["marching_cubes_ms"] = (time.perf_counter() - t0) / 3 * 1e3
    row["triangles"], row["vertices"] = int(mesh.faces.shape[0]), int(mesh.vertices.shape[0])
    del vol, mesh
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        export_marching_cubes_mesh(m, cams, tmp, resolution=64)  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mc = export_marching_cubes_mesh(m, cams, tmp, resolution=256)
        torch.cuda.synchronize()
        row["export_marching_cubes_256_s"] = time.perf_counter() - t0
        row["export_marching_cubes_256_triangles"] = int(mc.faces.shape[0])
    emit(row)


def multigrid_bytes(depth):
    """Algorithmic bytes of one V-cycle of dnr_poisson_solve, from the grid size: per node of every level but the 4^3
    coarsest, 2 + 2 red-black sweeps (each sweep reads chi once, b and S once and writes chi once: 20 B), the residual
    restriction (chi, b, S: 12 B, plus 1/8 node written), the coarse chi cleared and the prolongation (read chi, write
    chi, 1/8 node read: 8.5 B); plus the finest-level residual norm (12 B)."""
    R = 1 << depth
    levels = [(R >> l) ** 3 for l in range(depth - 2)]
    smooth = 4 * 20 * sum(levels)
    return {"smoother": smooth, "total": smooth + sum(n * (12 + 0.5 + 0.5 + 8.5) for n in levels) + 12 * levels[0]}


def bench_poisson():
    """poisson.py on the bench scene, the `dn` exporter's stages one after another as export_dn_poisson_mesh runs them."""
    import subprocess
    import tempfile

    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.mesh import marching_cubes, write_ply
    from dn_splatter_b200.poisson import (DEFAULT_POINT_WEIGHT, dn_point_cloud, export_gaussians_poisson_mesh, grid_sample,
                                          poisson_grid, poisson_solve, poisson_splat, trim_low_density)
    from dn_splatter_b200.synthetic import make_scene, ring_cameras

    W, H, n_views, total = 1920, 1080, 200, 2_000_000
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", sync_free=True).setup(device="cuda")
    m.load_gaussians(make_scene(args.n, seed=0))
    m.step = 30000
    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H) for c in ring_cameras(n_views, W, H)]
    dn_point_cloud(m, cams[:8], total_points=total // 25)  # warm-up: captures the forward graphs
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    with tempfile.TemporaryDirectory() as tmp:
        for depth in (9, 10):
            row = {"row": "poisson", "card": card, "n_gauss": args.n, "views": n_views, "resolution": f"{W}x{H}",
                   "exporter": "dn", "depth": depth, "total_points": total}
            e = [ev() for _ in range(6)]
            torch.cuda.synchronize()
            e[0].record()
            pts, nrm, col = dn_point_cloud(m, cams, total_points=total)
            e[1].record()
            grid = poisson_grid(pts, depth)
            sp = poisson_splat(pts, nrm, col, grid)
            e[2].record()
            sigma = DEFAULT_POINT_WEIGHT * float(sp["area_scale"])
            chi, hist = poisson_solve(grid, sp["screen"], sp["faces"], sigma)
            e[3].record()
            R, h, R4 = grid.R, grid.cell, grid.R // 4
            chi = chi.view(R, R, R)
            iso = float((grid_sample(chi, grid.origin, h, pts).double() * sp["weights"].double()).sum() / pts.shape[0])
            mesh = marching_cubes(chi, iso, [o + 0.5 * h for o in grid.origin], h)
            dens = grid_sample(sp["density"].view(R4, R4, R4), grid.origin, 4 * h, mesh.vertices)
            cw = grid_sample(sp["colors"].view(R4, R4, R4, 4), grid.origin, 4 * h, mesh.vertices)
            mesh = mesh._replace(colors=cw[:, :3] / cw[:, 3:].clamp_min(1e-30))
            e[4].record()
            write_ply(os.path.join(tmp, "dn.ply"), trim_low_density(mesh, dens))
            e[5].record()
            torch.cuda.synchronize()
            for k, name in enumerate(("render_backproject", "sort_splat", "solve", "extract", "trim_write")):
                row[f"{name}_ms"] = e[k].elapsed_time(e[k + 1])
            row["samples"], row["cycles"], row["residual"] = int(pts.shape[0]), len(hist) - 1, hist[-1]
            row["triangles"] = int(mesh.faces.shape[0])
            nbytes = multigrid_bytes(depth)
            row["bytes_per_cycle"], row["smoother_bytes_per_cycle"] = nbytes["total"], nbytes["smoother"]
            row["solve_gb_s"] = nbytes["total"] * row["cycles"] / (row["solve_ms"] * 1e-3) / 1e9
            del chi, mesh, dens, cw
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                _, hist2 = poisson_solve(grid, sp["screen"], sp["faces"], sigma)
                torch.cuda.synchronize()
            us = sum(getattr(k, "device_time_total", getattr(k, "cuda_time_total", 0.0))
                     for k in prof.key_averages() if "rbgs_kernel" in k.key)
            row["smoother_ms"] = us / 1e3
            row["smoother_gb_s"] = nbytes["smoother"] * (len(hist2) - 1) / (us * 1e-6) / 1e9 if us > 0 else None
            row["smoother_frac_of_3.35TB_s"] = None if us <= 0 else row["smoother_gb_s"] / 3350.0
            del sp, pts, nrm, col
            torch.cuda.empty_cache()
            emit(row)
        e0, e1 = ev(), ev()
        e0.record()
        g = export_gaussians_poisson_mesh(m, tmp, poisson_depth=9)[0]
        e1.record()
        torch.cuda.synchronize()
        emit({"row": "poisson", "card": card, "n_gauss": args.n, "exporter": "gaussians", "depth": 9,
              "total_ms": e0.elapsed_time(e1), "triangles": int(g.faces.shape[0])})


def bench_mesh_eval():
    """mesh_eval.py at a size users run: the bench scene's TSDF mesh (512^3 grid) as pred against its depth-9 `dn`
    Poisson mesh as gt, the 200 ring views at 1080p; CUDA-event stage times of one cull_mesh + compute_metrics pass
    (render, visibility, subdivision for both meshes; sampling and nearest neighbours), and the fp64 numpy oracle's
    visibility counts and cKDTree on a subset for scale."""
    import subprocess
    import time

    import numpy as np

    from dn_splatter_b200 import mesh_eval as ME
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.mesh import TSDFVolume, TriangleMesh
    from dn_splatter_b200.poisson import dn_point_cloud, poisson_reconstruct, trim_low_density
    from dn_splatter_b200.render_service import ViewRenderer
    from dn_splatter_b200.synthetic import make_scene, ring_cameras
    from oracle import mesh_eval_ref as R

    W, H, n_views, chunk = 1920, 1080, 200, 16
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", sync_free=True).setup(device="cuda")
    m.load_gaussians(make_scene(args.n, seed=0))
    m.step = 30000
    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H) for c in ring_cameras(n_views, W, H)]
    vol = TSDFVolume(((-5.0, -5.0, -5.0), (5.0, 5.0, 5.0)), voxel_size=10.0 / 512, sdf_trunc=3 * 10.0 / 512)
    for idx, maps in ViewRenderer(m, keys=("rgb", "depth"), to_host=False).render(cams):
        vol.integrate(maps["depth"], maps["rgb"], cams[idx])
    pred = vol.extract_mesh()
    del vol
    pts, nrm, col = dn_point_cloud(m, cams, total_points=2_000_000)
    gt, dens = poisson_reconstruct(pts, nrm, col, depth=9)
    gt = trim_low_density(gt, dens)
    del pts, nrm, col, dens, m
    torch.cuda.empty_cache()
    row = {"row": "mesh_eval", "card": card, "n_gauss": args.n, "views": n_views, "resolution": f"{W}x{H}",
           "pred_triangles": int(pred.faces.shape[0]), "gt_triangles": int(gt.faces.shape[0])}
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    ME.render_mesh_depth(pred, cams[:2])  # warm-up
    times = {"render_ms": 0.0, "visibility_ms": 0.0, "subdivide_ms": 0.0}
    culled = {}
    for tag, mesh in (("pred", pred), ("gt", gt)):
        e = [ev() for _ in range(2)]
        e[0].record()
        v, f = ME._mesh_on(mesh, "cuda", torch.float64)
        v, f = ME.remove_unreferenced(v, f)
        sub = ME.subdivide_to_size(TriangleMesh(v, f, None))
        e[1].record()
        torch.cuda.synchronize()
        times["subdivide_ms"] += e[0].elapsed_time(e[1])
        row[f"{tag}_subdivided_triangles"], row[f"{tag}_subdivided_vertices"] = int(sub.faces.shape[0]), int(sub.vertices.shape[0])
        v32, f32 = v.float().contiguous(), f.to(torch.int32).contiguous()
        cams32 = ME.camera_blocks(cams, torch.float32)
        obs = torch.zeros(sub.vertices.shape[0], dtype=torch.int32, device="cuda")
        inv = torch.zeros_like(obs)
        for c0 in range(0, n_views, chunk):
            c1 = min(c0 + chunk, n_views)
            e = [ev() for _ in range(3)]
            e[0].record()
            depth = ME._depth_call(v32, f32, cams32[c0:c1].contiguous(), W, H, 0.01, 10.0)
            e[1].record()
            o, i = ME.visibility_counts(sub.vertices, cams[c0:c1], depth, depth, chunk=c1 - c0)  # rendered depth as gt depth
            obs += o
            inv += i
            e[2].record()
            torch.cuda.synchronize()
            times["render_ms"] += e[0].elapsed_time(e[1])
            times["visibility_ms"] += e[1].elapsed_time(e[2])
        keep = ME.keep_faces(obs, inv, sub.faces)
        culled[tag] = TriangleMesh(*ME.remove_unreferenced(sub.vertices, sub.faces[keep]), None)
        row[f"{tag}_culled_triangles"] = int(keep.sum())
        if tag == "pred":  # the oracle's host path on the first views, for scale
            sv = sub.vertices.cpu().numpy()
            dm = depth.cpu().numpy()
            bl = [ME.camera_blocks(cams[k:k + 1], torch.float64)[0].cpu().numpy() for k in range(c0, c0 + 2)]
            t0 = time.perf_counter()
            ro, ri = R.visibility_counts(sv, bl, W, H, dm[:2], dm[:2])
            row["oracle_visibility_ms_per_view"] = (time.perf_counter() - t0) / 2 * 1e3
            o2, i2 = ME.visibility_counts(sub.vertices, cams[c0:c0 + 2], depth[:2], depth[:2])
            row["visibility_equals_oracle"] = bool(np.array_equal(o2.cpu().numpy(), ro) and np.array_equal(i2.cpu().numpy(), ri))
    row.update(times)
    g = torch.Generator(device="cuda").manual_seed(0)
    e = [ev() for _ in range(3)]
    e[0].record()
    n_p, n_g = int(ME.mesh_area(culled["pred"]) * 1e4), int(ME.mesh_area(culled["gt"]) * 1e4)
    pp, pn = ME.sample_surface(culled["pred"], n_p, g)
    gp, gn = ME.sample_surface(culled["gt"], n_g, g)
    e[1].record()
    met = ME.metrics_from_samples(pp, pn, gp, gn)
    e[2].record()
    torch.cuda.synchronize()
    row["sample_ms"], row["nn_metrics_ms"] = e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])
    row["pred_samples"], row["gt_samples"] = n_p, n_g
    row["nn_queries_per_s"] = (n_p + n_g) / (row["nn_metrics_ms"] * 1e-3)
    row["metrics"] = met
    sub_n = min(100_000, n_p, n_g)
    t0 = time.perf_counter()
    R.mesh_metrics(pp[:sub_n].cpu().numpy(), pn[:sub_n].cpu().numpy(), gp[:sub_n].cpu().numpy(), gn[:sub_n].cpu().numpy())
    row["oracle_ckdtree_metrics_s_per_100k"] = time.perf_counter() - t0
    emit(row)


def bench_isooctree():
    import subprocess
    import time

    import numpy as np

    from dn_splatter_b200 import isooctree as I
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.mesh import marching_cubes
    from dn_splatter_b200.synthetic import make_scene, ring_cameras
    from oracle import isooctree_ref as R

    W, H, n_views, stride, depth, thr = 1920, 1080, 200, 6, 10, 50
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    m = DNSplatterModelConfig(random_init=True, num_random=16, background_color="black", sync_free=True).setup(device="cuda")
    m.load_gaussians(make_scene(args.n, seed=0))
    m.step = 30000
    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], W, H) for c in ring_cameras(n_views, W, H)]
    row = {"row": "isooctree", "card": card, "n_gauss": args.n, "views": n_views, "resolution": f"{W}x{H}",
           "pixel_stride": stride, "max_depth": depth, "subdivision_threshold": thr}
    I.render_frames(m, cams[:4])  # warm-up: captures the forward graphs
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    e = [ev() for _ in range(7)]
    torch.cuda.synchronize()
    e[0].record()
    fs = I.render_frames(m, cams)
    e[1].record()
    hint, _ = I.hint_samples(fs, stride)
    e[2].record()
    tree = I.build_octree(hint, depth, thr)
    e[3].record()
    values = I.iso_eval(fs, tree.corner_points)
    e[4].record()
    field = I.fill_grid(tree, values)
    e[5].record()
    mesh = marching_cubes(field, 0.0, tree.origin, tree.cell)
    e[6].record()
    torch.cuda.synchronize()
    for k, name in enumerate(("render", "hint", "octree", "eval", "fill", "marching_cubes")):
        row[f"{name}_ms"] = e[k].elapsed_time(e[k + 1])
    row["hint_samples"], row["leaves"], row["corners"] = int(hint.shape[0]), int(tree.leaves.shape[0]), int(values.shape[0])
    row["triangles"] = int(mesh.faces.shape[0])
    row["eval_point_frames_per_s"] = values.shape[0] * n_views / (row["eval_ms"] * 1e-3)
    row["fill_gsamples_per_s"] = field.numel() / (row["fill_ms"] * 1e-3) / 1e9
    del field, mesh
    torch.cuda.empty_cache()
    nf, npt = 4, 20_000  # the oracle on a subset: its cost is linear in points x frames
    cam = R.CameraModel({"w": W, "h": H, "fl_x": float(cams[0].fx), "fl_y": float(cams[0].fy), "cx": float(cams[0].cx),
                         "cy": float(cams[0].cy)})
    frames = []
    for k in range(nf):
        c2w = np.eye(4)  # the pose row's c2w rotation and position; transform_matrix @ CAM_CONVENTION_CHANGE gives it back
        c2w[:3, :3], c2w[:3, 3] = fs._poses[k][12:21].reshape(3, 3), fs._poses[k][21:24]
        frames.append(R.Frame(cam, c2w @ R.CAM_CONVENTION_CHANGE, fs.depth[k].cpu().numpy(),
                              fs.normals[k].cpu().numpy().astype(np.uint8), True))
    pts = tree.corner_points[:npt].cpu().numpy()
    t0 = time.perf_counter()
    ref = R.iso_func(frames, pts)
    row["oracle_point_frames_per_s"] = npt * nf / (time.perf_counter() - t0)
    sub = I.FrameSet(fs.camera, nf, True)
    sub.depth.copy_(fs.depth[:nf])
    sub.normals.copy_(fs.normals[:nf])
    sub._poses[:] = fs._poses[:nf]
    got = I.iso_eval(sub, tree.corner_points[:npt]).cpu().numpy()
    row["eval_max_abs_err_vs_oracle"] = float(np.abs(got - ref).max())
    emit(row)


def bench_depth_normals():
    import subprocess
    import time

    import numpy as np

    from dn_splatter_b200 import depth_normals as DN
    from oracle import normals_ref as R

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]

    def room(w, h, share, seed=0):
        g = np.random.default_rng(seed)
        u, v = np.meshgrid(np.arange(w) / w, np.arange(h) / h)
        z = 0.3 + 7.7 * u ** 2 + 0.3 * np.sin(v * 6)  # 0.3-8 m across the frame
        hw, hh = w // 8, h // 8  # holes as blobs on a coarse grid, upsampled
        hu, hv = np.meshgrid(np.arange(hw), np.arange(hh))
        holes = np.zeros((hh, hw), bool)
        while holes.mean() < share:
            cx, cy, r = g.integers(0, hw), g.integers(0, hh), g.integers(1, max(2, hw // 20))
            holes |= (hu - cx) ** 2 + (hv - cy) ** 2 < r * r
        holes = np.repeat(np.repeat(holes, 8, 0), 8, 1)[:h, :w]
        return np.where(holes, 0, z).astype(np.float32)

    reps = 3
    for (w, h) in ((1920, 1440), (1024, 768)):
        for share in (0.05, 0.40):
            depth = room(w, h, share)
            intr = (0.73 * w, 0.73 * w, w / 2, h / 2)
            c2w = np.eye(4)
            mono = np.random.default_rng(1).integers(0, 256, (h * w, 3)).astype(np.uint8)
            n = w * h
            examined = torch.empty(n, dtype=torch.int32, device="cuda")
            stats = torch.zeros(2, dtype=torch.int64, device="cuda")
            ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
            pts = DN.backproject_depth(depth, *intr, c2w)  # warm-up
            DN.depth_normal_consistency(DN.estimate_normals(pts, 200, c2w[:3, 3]), mono, c2w)
            t = {"backproject": 0.0, "normals": 0.0, "consistency": 0.0}
            for r in range(reps):
                e = [ev() for _ in range(4)]
                torch.cuda.synchronize()
                e[0].record()
                pts = DN.backproject_depth(depth, *intr, c2w)
                e[1].record()
                nrm = DN.estimate_normals(pts, 200, c2w[:3, 3], stats=stats if r == 0 else None,
                                          examined=examined if r == 0 else None)
                e[2].record()
                DN.depth_normal_consistency(nrm, mono, c2w)
                e[3].record()
                torch.cuda.synchronize()
                for k, name in enumerate(t):
                    t[name] += e[k].elapsed_time(e[k + 1]) / reps
            s = stats.cpu().numpy()
            ex = examined.cpu().numpy()[depth.reshape(-1) > 0]
            row = {"row": "depth_normals", "card": card, "resolution": f"{w}x{h}", "holes": share, "k": 200,
                   "hole_share_measured": float((depth == 0).mean()), **{f"{k}_ms": v for k, v in t.items()},
                   "frame_ms": sum(t.values()), "searches": int(s[1]),
                   "candidates_per_search_mean": float(s[0] / s[1]),
                   "candidates_per_surface_pixel_mean": float(ex.mean()),
                   "candidates_per_surface_pixel_p99": float(np.percentile(ex, 99))}
            if (w, h) == (1024, 768) and share == 0.05:  # the oracle on a crop, for scale
                crop = pts.reshape(h, w, 3)[360:408, 480:544].reshape(-1, 3).cpu().numpy()
                t0 = time.perf_counter()
                ref, _ = R.estimate_normals(crop, 200)
                row["oracle_points_per_s"] = crop.shape[0] / (time.perf_counter() - t0)
                got = DN.estimate_normals(torch.from_numpy(crop).cuda(), 200).cpu().numpy()
                row["crop_max_abs_err_vs_oracle_up_to_sign"] = float(np.minimum(np.abs(got - ref).max(1),
                                                                               np.abs(got + ref).max(1)).max())
            emit(row)
            del pts, nrm, examined
            torch.cuda.empty_cache()


for name, fn in (("ssim", bench_ssim), ("adam", bench_adam), ("camera_opt", bench_camera_opt), ("knn", bench_knn),
                 ("render_service", bench_render_service), ("mesh", bench_mesh), ("poisson", bench_poisson),
                 ("mesh_eval", bench_mesh_eval), ("isooctree", bench_isooctree),
                 ("depth_normals", bench_depth_normals)):
    if args.only and name not in args.only.split(","):
        continue
    try:
        fn()
    except Exception as e:  # one broken experimental kernel must not hide the others
        emit({"row": name, "error": f"{type(e).__name__}: {e}"})
