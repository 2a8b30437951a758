"""Training-step time of the `ags-mesh` strategy: the torch regulariser, the fused kernels run eagerly, and the
CUDA-graph captured step, alternating in one process.

    python scripts/ags_step_bench.py [--n-gauss 1000000] [--width 1920] [--height 1080] [--steps 20] [--repeats 3]

Workload: bench.py's scene and cameras (1 M Gaussians at 1080p by default) with `regularization_strategy="ags-mesh"`,
EdgeAwareLogL1 depth, uint8 mono normals, a uint8 confidence map, at steps 8000 (edge mask) and 16000 (angular mask).
A step is bucket zero + get_outputs + get_loss_dict + backward (no optimiser), timed by a host clock around `--steps`
steps that end in a device synchronise.  Prints one JSON object: per step and arm the median ms/step over the repeats
and its spread (min, max), the mean device time of the ags_loss_fwd / ags_loss_bwd stages (CUDA events, a separate
untimed pass), and the card name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return f"nvidia-smi unavailable ({exc})"


def build(args, dev):
    from dn_splatter_b200.cameras import Cameras
    from dn_splatter_b200.dn_model import DNSplatterModelConfig
    from dn_splatter_b200.losses import DepthLossType
    from dn_splatter_b200.synthetic import make_scene, ring_cameras

    cfg = DNSplatterModelConfig(random_init=True, num_random=16, use_depth_loss=True, depth_lambda=0.2,
                                depth_loss_type=DepthLossType.EdgeAwareLogL1, predict_normals=True, use_normal_loss=True,
                                normal_supervision="mono", ssim_lambda=0.2, background_color="black", sync_free=True,
                                regularization_strategy="ags-mesh")
    model = cfg.setup(device=dev)
    model.load_gaussians(make_scene(args.n_gauss, seed=0))
    model.background_color = torch.tensor([0.1490, 0.1647, 0.2157])
    model.train()
    bucket = model.enable_flat_grads()
    cams = [Cameras(c["c2w"][None], c["fx"], c["fy"], c["cx"], c["cy"], c["width"], c["height"], metadata={"cam_idx": i})
            for i, c in enumerate(ring_cameras(args.views, args.width, args.height))]
    return model, bucket, cams


def make_sets(model, cams, args, dev):
    """bench.make_gt_sets' supervision (uint8 image, rendered depth, uint8 normals from it) plus a uint8 confidence map."""
    import bench

    ns = argparse.Namespace(height=args.height, width=args.width)
    sets = bench.make_gt_sets(model, cams, ns, True, args.gt_sets)
    g = torch.Generator().manual_seed(2)
    for b in sets:
        b["confidence"] = (torch.rand(args.height, args.width, 1, generator=g) * 255).to(torch.uint8)
    return [{k: v.to(dev) for k, v in b.items()} for b in sets]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-gauss", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--views", type=int, default=40)
    ap.add_argument("--gt-sets", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ags_step_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.cuda.set_stream(torch.cuda.Stream(device=dev))
    from dn_splatter_b200 import rasterize
    from dn_splatter_b200.graph_step import GraphedTrainStep

    model, bucket, cams = build(args, dev)
    sets = make_sets(model, cams, args, dev)
    rs = model.regularization_strategy

    def eager(s):
        bucket.zero_()
        ld = model.get_loss_dict(model.get_outputs(cams[s % len(cams)]), dict(sets[s % len(sets)]))
        (ld["main_loss"] + ld["scale_reg"]).backward()

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s in range(args.steps):
            fn(s)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0) / args.steps

    result = {"card": card(), "n_gauss": args.n_gauss, "width": args.width, "height": args.height, "steps": args.steps,
              "repeats": args.repeats, "arms": {}}
    for step in (8000, 16000):
        model.step = step
        for fused in (False, True):  # warm every shape of both eager arms (and the capacity statistics)
            rs.fused = fused
            for s in range(4):
                eager(s)
        rs.fused = True
        graphed = GraphedTrainStep(model, bucket, cams[0], sets[0], n_slots=1, warmup=2)

        def captured(s):
            for k, v in sets[s % len(sets)].items():
                graphed.batches[0][k].copy_(v, non_blocking=True)
            graphed(cams[s % len(cams)], 0)

        for s in range(3):
            captured(s)
        times = {"torch_eager": [], "fused_eager": [], "captured": []}
        for _ in range(args.repeats):
            rs.fused = False
            times["torch_eager"].append(timed(eager))
            rs.fused = True
            times["fused_eager"].append(timed(eager))
            times["captured"].append(timed(captured))
        graphed.check_capacity(wait=True)
        arms = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "all_ms": v}
                for k, v in times.items()}
        rs.fused = True
        rasterize.STAGE_EVENTS = []
        for s in range(args.steps):
            eager(s)
        torch.cuda.synchronize()
        stages = {}
        for name, e0, e1 in rasterize.STAGE_EVENTS:
            if name.startswith("ags_loss"):
                stages.setdefault(name, []).append(e0.elapsed_time(e1))
        rasterize.STAGE_EVENTS = None
        arms["stages_ms"] = {k: statistics.mean(v) for k, v in stages.items()}
        result["arms"][f"step_{step}"] = arms
        del graphed
    print(json.dumps(result))


if __name__ == "__main__":
    main()
