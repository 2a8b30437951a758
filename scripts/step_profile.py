"""Per-kernel device times of the captured training step (bench.py's flagship workload) under torch.profiler.

    python scripts/step_profile.py --out DIR [--replays N] [bench.py workload options...]

Builds the workload through bench.build_workload, captures it with GraphedTrainStep as bench.py does, replays N steps
(graph + eager Adam step, a different view and supervision set each step) with CUDA activities recorded, and writes
DIR/kernels.json (per kernel: calls, total and per-step device microseconds, sorted by time) and the Chrome trace
DIR/step_trace.json.  The card name and power limit are recorded beside the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return f"nvidia-smi unavailable ({exc})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for kernels.json and step_trace.json")
    ap.add_argument("--replays", type=int, default=20)
    own, rest = ap.parse_known_args()
    sys.argv = [sys.argv[0]] + rest
    args = bench.parse()
    assert torch.cuda.is_available(), "step_profile.py needs a GPU"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.cuda.set_stream(torch.cuda.Stream(device=dev))
    normals = not args.no_normals
    from dn_splatter_b200.graph_step import GraphedTrainStep
    from dn_splatter_b200.optim import FusedAdam

    model, bucket, cams = bench.build_workload(args, dev, normals)
    optimizer = FusedAdam.for_model(model)
    sets = [{k: v.to(dev) for k, v in b.items()} for b in bench.make_gt_sets(model, cams, args, normals, args.gt_sets)]
    views = list(range(len(cams)))
    with torch.no_grad():
        for v in views:
            model.get_outputs(cams[v])
    for s in range(max(3, args.warmup)):
        bench.run_step(model, bucket, cams[bench.view_of(s, views)], sets[s % len(sets)], optimizer=optimizer)
    graphed = GraphedTrainStep(model, bucket, cams[0], sets[0], n_slots=1, warmup=2)

    def step(s):
        for k, v in sets[s % len(sets)].items():
            graphed.batches[0][k].copy_(v, non_blocking=True)
        graphed(cams[bench.view_of(s, views)], 0)
        bucket.all_reduce()
        optimizer.step()

    for s in range(3):
        step(s)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(own.replays):
            step(s)
        torch.cuda.synchronize()
    graphed.check_capacity(wait=True)
    rows = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        r = rows.setdefault(e.name, {"calls": 0, "us": 0.0})
        r["calls"] += 1
        r["us"] += e.device_time
    kern = sorted(({"name": k, "calls": v["calls"], "us_total": v["us"], "us_per_step": v["us"] / own.replays}
                   for k, v in rows.items()), key=lambda r: -r["us_total"])
    os.makedirs(own.out, exist_ok=True)
    info = {"card": card(), "replays": own.replays, "width": args.width, "height": args.height, "n_gauss": args.n_gauss,
            "normals": normals, "device_us_per_step": sum(r["us_per_step"] for r in kern), "kernels": kern}
    with open(os.path.join(own.out, "kernels.json"), "w") as f:
        json.dump(info, f, indent=1)
    prof.export_chrome_trace(os.path.join(own.out, "step_trace.json"))
    print(info["card"])
    print(f"{'us/step':>9} {'calls':>6}  kernel   ({own.replays} replays)")
    for r in kern:
        print(f"{r['us_per_step']:9.1f} {r['calls']:6d}  {r['name'][:110]}")
    print(f"{info['device_us_per_step']:9.1f}         sum of device time per step")


if __name__ == "__main__":
    main()
