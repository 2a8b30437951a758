"""One-launch Adam for the Gaussian parameter groups (SURVEY.md §8f-3).

The reference creates one torch.optim.Adam per parameter group (/root/reference/dn_splatter/dn_config.py:29-68: a
learning rate per group, eps 1e-15, an exponential schedule on `means`) and nerfstudio steps them in turn.
`FusedAdam` keeps that surface — it IS a torch.optim.Optimizer with one param_group per Gaussian group and the usual
`state[p] = {"step", "exp_avg", "exp_avg_sq"}`, so densification's moment surgery (densify._resize_adam_state) and
checkpointing work unchanged — but `step()` is a single `dnr_adam_step` launch over all groups.

The update rule is pinned against torch.optim.Adam on the CPU through `reference_step` (tests/test_fused_adam_cpu.py)
and the kernel against torch.optim.Adam on the GPU (tests/test_gpu_model.py).  The dense pass moves 28 B per float
(1.65 GB for 59 M floats: at least 0.49 ms at the H100 SXM data sheet's 3.35 TB/s).  When the gradients are views of a
parallel.FlatGradBucket whose `touched` flags are valid, `step()` reads only the flagged gradient rows (plus the dense
`scales` segment) through dnr_adam_step_reduce at world 1; results are bit-identical, because the other rows are exactly
zero.  `step_reduce(bucket)` is the multi-GPU form: the gradient sum over ranks happens inside the same kernel, read from
the peers' buckets over NVLink (parallel.PeerGradBucket, tests/test_gpu_multi.py).
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Iterable, Optional

import torch

from . import _lib as L
from .rasterize import _timed


def bias_corrections(step: int, beta1: float, beta2: float):
    """(1 - beta1^t, sqrt(1 - beta2^t)) in double precision, as torch's Adam computes them on the host."""
    return 1.0 - beta1 ** step, math.sqrt(1.0 - beta2 ** step)


class FusedAdam(torch.optim.Optimizer):
    """Adam (no weight decay, no amsgrad) over several parameter groups in one kernel launch.

    `params`: an iterable of param_group dicts `{"params": [p], "lr": ..., "eps": ..., "name": ...}`; use
    `FusedAdam.for_model(model)` to build the reference's groups."""

    def __init__(self, params: Iterable[Dict], lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-15):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))
        n = sum(len(g["params"]) for g in self.param_groups)
        if n > 16:
            raise ValueError("FusedAdam handles at most 16 tensors per launch (DNR_ADAM_MAX_SEGS)")

    @classmethod
    def for_model(cls, model, groups: Optional[Dict[str, Dict]] = None) -> "FusedAdam":
        from .dn_config import optimizer_groups

        groups = groups or optimizer_groups()
        pg = [{"params": [p], "lr": groups[name]["lr"], "eps": groups[name]["eps"], "name": name}
              for name, p in model.gauss_params.items() if name in groups]
        return cls(pg)

    def as_dict(self, model) -> Dict[str, "FusedAdam"]:
        """The `{group name: optimizer}` mapping densify.refinement_after expects (every name -> this optimizer)."""
        return {g["name"]: self for g in self.param_groups if "name" in g}

    def _segments(self):
        segs = []
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st["step"] = int(st["step"]) + 1
                bc1, bc2s = bias_corrections(st["step"], b1, b2)
                segs.append((p, p.grad, st["exp_avg"], st["exp_avg_sq"], float(group["lr"]), float(group["eps"]), bc1, bc2s,
                             b1, b2))
        return segs

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        segs = self._segments()
        if not segs:
            return loss
        if not all(s[0].is_cuda for s in segs):
            raise L.DnrError("FusedAdam needs CUDA parameters (no CPU path)")
        b1, b2 = segs[0][8], segs[0][9]
        assert all(s[8] == b1 and s[9] == b2 for s in segs), "one (beta1, beta2) pair per launch"
        bucket = self._flagged_bucket(segs)
        if bucket is not None:  # sparse gradient reads: the bucket's own flags are the mask, no peers, no barriers
            pr = L.DnrPeerReduce()
            pr.world, pr.rank, pr.n_gauss = 1, 0, bucket.n_gauss
            pr.peer_flat[0], pr.peer_touched[0] = bucket.flat.data_ptr(), bucket.touched.data_ptr()
            _timed("adam", self._launch_reduce, segs, bucket, pr)
            return loss
        arr = (L.DnrAdamSeg * len(segs))()
        for i, (p, g, m, v, lr, eps, bc1, bc2s, _, _) in enumerate(segs):
            assert p.is_contiguous() and g.is_contiguous() and m.is_contiguous() and v.is_contiguous()
            assert p.dtype == g.dtype == torch.float32
            arr[i].p, arr[i].g, arr[i].m, arr[i].v = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
            arr[i].n, arr[i].lr, arr[i].eps, arr[i].bc1, arr[i].bc2_sqrt = p.numel(), lr, eps, bc1, bc2s
        stream = L.stream()
        L.check(_timed("adam", L.load().dnr_adam_step, ctypes.cast(arr, ctypes.c_void_p), len(segs), b1, b2, stream),
                "dnr_adam_step")
        return loss

    @staticmethod
    def _flagged_bucket(segs):
        """The FlatGradBucket that every gradient of `segs` is a segment of, if its flags are valid; else None."""
        from .parallel import bucket_of

        bucket = bucket_of(segs[0][1])
        if bucket is None or not bucket.flags_valid:
            return None
        views = {v.data_ptr(): n for n, v in bucket.views.items()}
        for p, g, *_ in segs:
            name = views.get(g.data_ptr())
            if name is None or bucket.params[name] is not p:
                return None
        return bucket

    @torch.no_grad()
    def step_reduce(self, bucket):
        """Multi-GPU step: gradient reduction over NVLink peer memory fused into the Adam pass (dnr_adam_step_reduce).
        `bucket`: parallel.PeerGradBucket holding this model's gradients.  Equivalent to `bucket.all_reduce(); self.step()`
        up to the order of the floating-point sum over ranks (here: rank order, identical on every replica)."""
        segs = self._segments()
        if not segs:
            return
        pr = L.DnrPeerReduce()
        pr.world, pr.rank, pr.n_gauss = bucket.world, bucket.rank, bucket.n_gauss
        for k in range(bucket.world):
            pr.peer_flat[k], pr.peer_touched[k] = bucket.peer_flat[k], bucket.peer_touched[k]
        pr.mask = bucket.mask.data_ptr()
        bucket.barrier()  # every rank's backward has finished writing its bucket and flags
        self._launch_reduce(segs, bucket, pr)
        bucket.barrier()  # nobody zeroes its bucket while a peer still reads it

    @staticmethod
    def _launch_reduce(segs, bucket, pr) -> None:
        """dnr_adam_step_reduce over `segs`, whose gradients are segments of `bucket` (`pr`: the ranks' buckets and flags)."""
        b1, b2 = segs[0][8], segs[0][9]
        arr = (L.DnrAdamSeg * len(segs))()
        widths = (ctypes.c_int32 * len(segs))()
        lo, hi = bucket.flat.data_ptr(), bucket.flat.data_ptr() + bucket.flat.numel() * 4
        for i, (p, g, m, v, lr, eps, bc1, bc2s, _, _) in enumerate(segs):
            assert lo <= g.data_ptr() < hi, "parameter gradients must be views of the bucket"
            assert p.is_contiguous() and m.is_contiguous() and v.is_contiguous() and p.shape[0] == bucket.n_gauss
            arr[i].p, arr[i].g, arr[i].m, arr[i].v = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
            arr[i].n, arr[i].lr, arr[i].eps, arr[i].bc1, arr[i].bc2_sqrt = p.numel(), lr, eps, bc1, bc2s
            widths[i] = p.numel() // bucket.n_gauss
            arr[i].dense = int(any(bucket.params[name] is p for name in bucket.dense_params))
        stream = L.stream()
        L.check(L.load().dnr_adam_step_reduce(ctypes.cast(arr, ctypes.c_void_p), ctypes.cast(widths, ctypes.c_void_p), len(segs),
                                              b1, b2, ctypes.byref(pr), stream), "dnr_adam_step_reduce")

    @torch.no_grad()
    def reference_step(self):
        """The kernel's arithmetic restated in torch, operation for operation (csrc/adam.cu: adam_one) — used ONLY by the
        CPU tests that pin the update rule (against torch.optim.Adam, and the kernel against it bit for bit); never called
        by the product path."""
        for (p, g, m, v, lr, eps, bc1, bc2s, b1, b2) in self._segments():
            f = lambda x: torch.tensor(x, dtype=torch.float32)
            m.copy_(m + f(1.0 - b1) * (g - m))
            v.copy_(f(b2) * v + f(1.0 - b2) * g * g)
            # sqrtf is correctly rounded; torch's CPU float32 sqrt (a vector-math library) is not always (1 ulp off on
            # ~0.6 % of inputs with AVX-512).  The float64 sqrt rounded to float32 is: the double rounding of a square
            # root is harmless at 53 >= 2 * 24 + 2 bits.
            denom = v.double().sqrt().float() / f(bc2s) + f(eps)
            p.copy_(p - f(lr / bc1) * (m / denom))
