"""Times the render-metric entry points on one 1080p view (RGB with a uint8 target, depth, normals) with CUDA events,
next to the plain-torch formulation of the same metrics (the CPU route of metrics.py) applied to the same GPU tensors.

    python scripts/metrics_bench.py [--iters 200] [--warmup 20]

Prints the card name and power limit, the per-call times and the byte floor of each call computed from the shapes at
the H100 SXM data-sheet bandwidth (3.35 TB/s); the floors are bounds, not measurements.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dn_splatter_b200 import metrics as MT  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        limit = q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench.py needs a CUDA device")
    H, W = 1080, 1920
    g = torch.Generator(device="cuda").manual_seed(0)
    rgb = torch.rand(H, W, 3, device="cuda", generator=g)
    img = (torch.rand(H, W, 3, device="cuda", generator=g) * 255).to(torch.uint8)
    depth = 0.5 + 4 * torch.rand(H, W, 1, device="cuda", generator=g)
    sensor = 0.05 + 4 * torch.rand(H, W, 1, device="cuda", generator=g)
    normal = torch.rand(H, W, 3, device="cuda", generator=g)
    gt_normal = torch.rand(H, W, 3, device="cuda", generator=g)
    chw = lambda t: t.permute(2, 0, 1)[None]  # noqa: E731  (the model's [1,C,H,W] views)
    n = H * W
    floors = {  # bytes each call must read at least once
        "rgb": n * 3 * (4 + 1),  # fp32 render, uint8 target
        "rgb_f32_target": n * 3 * 8,
        "depth": n * 2 * 4,
        "normal": 4 * n * 3 * 8,  # four radix passes over fp32 maps
    }
    img_f = MT.u8_as_float(img)
    cases = {
        "rgb": (lambda: MT.rgb_sums(chw(rgb), chw(img)), lambda: [float(v) for v in MT.rgb_torch(chw(rgb), chw(img))]),
        "rgb_f32_target": (lambda: MT.rgb_sums(chw(rgb), chw(img_f)),
                           lambda: [float(v) for v in MT.rgb_torch(chw(rgb), chw(img_f))]),
        "depth": (lambda: MT.depth_sums(depth, sensor, 0.1), lambda: [float(v) for v in MT.depth_torch(depth, sensor)]),
        "normal": (lambda: MT.normal_sums(chw(normal), chw(gt_normal)),
                   lambda: [float(v) for v in MT.normal_torch(chw(normal), chw(gt_normal))]),
    }
    name, limit = card()
    print(json.dumps({"device": name, "power_limit_and_max_sm_clock": limit, "shape": [H, W], "iters": args.iters}))
    for k, (kern, ref) in cases.items():
        t_k = time_ms(kern, args.iters, args.warmup)
        t_t = time_ms(ref, args.iters, args.warmup)
        floor_us = floors[k] / HBM_BYTES_PER_S * 1e6
        print(json.dumps({"entry": k, "kernel_call_ms": round(t_k, 4), "torch_same_gpu_tensors_ms": round(t_t, 4),
                          "bytes_floor_MB": round(floors[k] / 1e6, 1), "datasheet_floor_us": round(floor_us, 1),
                          "note": "per call, including the one device-to-host read of the result"}))


if __name__ == "__main__":
    main()
