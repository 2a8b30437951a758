"""The fused photometric loss (dnr_photometric_fwd / _bwd) of two builds on the same seeded 1080p inputs.

    python scripts/photometric_ab.py dump DIR      # run this tree's library, write DIR/<case>_{out,v_pred}.npy + DIR/times.json
    python scripts/photometric_ab.py compare A B   # per case: v_pred bits that differ, and the two sums' difference

Run `dump` once from each tree (each imports the package and library of the tree it lives in), then `compare`.
A change to how the SSIM kernels are decomposed must leave every v_pred value bit-identical (each value is the same fp32
sequence of operations); only the SSIM and L1 sums may move, by their fp32 summation-order error.  `dump` also times
the forward and the backward call (CUDA events over 200 calls each after 20 warm-up calls) on the bench's case."""
import json
import os
import sys

import numpy as np

CASES = (("u8_c3", True, 3), ("f32_c3", False, 3), ("f32_c5", False, 5))  # u8_c3 is what bench.py's step runs
H, W, LAM, V = 1080, 1920, 0.2, 0.75


def _inputs(u8: bool, cn: int, dev):
    import torch

    g = torch.Generator().manual_seed(11 + cn + 100 * u8)
    x = torch.rand(H, W, cn, generator=g)
    y = torch.rand(H, W, cn, generator=g)
    y = (y * 255).to(torch.uint8) if u8 else (0.6 * x + 0.4 * y)  # fp32 targets correlated with pred: SSIM well away from 0
    return x.to(dev), y.to(dev)


def dump(out_dir: str) -> None:
    import ctypes as C

    import torch

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from dn_splatter_b200 import _lib as L

    lib = L.load()
    dev = torch.device("cuda:0")
    os.makedirs(out_dir, exist_ok=True)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    times = {"library": os.path.abspath(L.__file__), "device": torch.cuda.get_device_name(0)}
    for name, u8, cn in CASES:
        x, y = _inputs(u8, cn, dev)
        dmaps = torch.empty(3 * H * W * cn, dtype=torch.float32, device=dev)
        out = torch.empty(3, dtype=torch.float32, device=dev)
        vp = torch.empty_like(x)
        v = torch.tensor([V], dtype=torch.float32, device=dev)

        def fwd():
            L.check(lib.dnr_photometric_fwd(x.data_ptr(), y.data_ptr(), int(u8), H, W, cn, LAM, dmaps.data_ptr(), out.data_ptr(),
                                            st), "dnr_photometric_fwd")

        def bwd():
            L.check(lib.dnr_photometric_bwd(x.data_ptr(), y.data_ptr(), int(u8), H, W, cn, LAM, dmaps.data_ptr(), v.data_ptr(),
                                            vp.data_ptr(), st), "dnr_photometric_bwd")

        fwd()
        bwd()
        torch.cuda.synchronize()
        np.save(os.path.join(out_dir, name + "_out.npy"), out.cpu().numpy())
        np.save(os.path.join(out_dir, name + "_v_pred.npy"), vp.cpu().numpy())
        if name == CASES[0][0]:
            for label, fn in (("fwd", fwd), ("bwd", bwd)):
                for _ in range(20):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(200):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[f"{name}_{label}_us"] = 1e3 * e0.elapsed_time(e1) / 200
    with open(os.path.join(out_dir, "times.json"), "w") as f:
        json.dump(times, f, indent=1)
    print(json.dumps(times))


def compare(a: str, b: str) -> int:
    bad = 0
    for name, _, _ in CASES:
        va, vb = (np.load(os.path.join(d, name + "_v_pred.npy")) for d in (a, b))
        oa, ob = (np.load(os.path.join(d, name + "_out.npy")).astype(np.float64) for d in (a, b))
        diff = va.view(np.int32) != vb.view(np.int32)
        n = int(diff.sum())
        bad += n
        rel = np.abs(oa - ob) / np.maximum(np.abs(oa), 1e-30)
        print(f"{name}: v_pred values differing in any bit: {n} of {va.size}"
              + (f" (max |diff| {float(np.abs(va - vb).max()):.3e})" if n else "")
              + f"; SSIM sum {oa[0]:.9g} vs {ob[0]:.9g} (rel {rel[0]:.2e}), L1 sum {oa[1]:.9g} vs {ob[1]:.9g} "
              f"(rel {rel[1]:.2e}), main {oa[2]:.9g} vs {ob[2]:.9g}")
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "dump":
        dump(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
