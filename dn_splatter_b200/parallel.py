"""Per-camera data parallelism (SURVEY.md §8e): Gaussian parameters are replicated, the views of a step are
sharded round-robin over the ranks (one process per GPU), every rank accumulates its views' per-Gaussian
gradients into ONE flat fp32 bucket that aliases the parameters' .grad tensors, and a single NCCL all-reduce
(sum) over NVLink/NVSwitch makes the gradients identical on all ranks.

The reference only wraps the model in DDP(find_unused_parameters=True) (dn_pipeline.py:123-128), which cannot
cope with densification re-creating parameters; this module is the working equivalent for the hot path."""
from __future__ import annotations

import ctypes
import weakref
from typing import Dict, Iterable, List, Optional

import torch
import torch.distributed as dist
from torch import Tensor

GRAD_PARAMS = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")

_BUCKETS: "weakref.WeakValueDictionary[int, FlatGradBucket]" = weakref.WeakValueDictionary()  # by flat.data_ptr()


def bucket_of(grad: Tensor) -> Optional["FlatGradBucket"]:
    """The live FlatGradBucket that `grad` is a view of, or None."""
    base = grad._base
    b = _BUCKETS.get(base.data_ptr()) if base is not None else None
    return b if b is not None and b.flat.data_ptr() == base.data_ptr() and b.flat.numel() == base.numel() else None


class FlatGradBucket:
    """One contiguous fp32 buffer holding the gradients of the six optimised gauss_params (59 floats per
    Gaussian at SH degree 3); `param.grad` are views into it, so autograd, the rasterizer's grad-sink path
    and the all-reduce all touch the same memory.

    The bucket also owns the rasterizer's per-Gaussian `touched` flags and its always-zero `grad_records` workspace
    (DNR_FLAG_PERSISTENT_WS).  The flags accumulate over every backward since the last `zero_()`.  While they cover every
    non-zero row (`flags_valid`), `zero_()` clears only the flagged rows and FusedAdam.step() reads only the flagged
    gradient rows: about 10 % of the bucket at 1 M Gaussians / 1080p."""

    def __init__(self, params: Dict[str, torch.nn.Parameter], names: Iterable[str] = GRAD_PARAMS):
        self.names = [n for n in names if n in params]
        self.params = {n: params[n] for n in self.names}
        total = sum(self._padded(p.numel()) for p in self.params.values())
        dev = next(iter(self.params.values())).device
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self.views: Dict[str, Tensor] = {}
        off = 0
        for n, p in self.params.items():
            v = self.flat[off:off + p.numel()].view_as(p)
            p.grad = v
            self.views[n] = v
            off += self._padded(p.numel())
        self.n_gauss = next(iter(self.params.values())).shape[0]
        self.touched = torch.zeros(self.n_gauss, dtype=torch.uint8, device=dev)
        self.grad_records = torch.zeros(self.n_gauss, 16, dtype=torch.float32, device=dev)  # DNR_GRAD_FLOATS
        # parameters whose gradient is non-zero for every Gaussian (a loss term that depends on the parameters alone:
        # DNRegularization's min-scale term on `scales`): never covered by the flags, zeroed and read in full
        self.dense_params = {"scales"} & set(self.params)
        # False for configs with other parameter-only loss terms (dn_model.enable_flat_grads)
        self.sparse_ok = True
        # flags_valid: every non-zero row outside the dense segments is flagged.  Only a backward through sink() after a
        # zero_() makes the flags valid; a fresh bucket may have been filled by other means.
        self.flags_valid, self._clean = False, False
        _BUCKETS[self.flat.data_ptr()] = self

    @staticmethod
    def _padded(n: int) -> int:
        """Segments start on 16-byte boundaries (float4 access in dnr_adam_step; the padding floats stay zero)."""
        return (n + 3) & ~3

    def zero_(self) -> None:
        if self.flags_valid:
            from . import _lib as L
            from .rasterize import _timed

            segs = (L.DnrGradSeg * len(self.names))()
            for i, n in enumerate(self.names):
                v = self.views[n]
                segs[i].g, segs[i].width, segs[i].dense = v.data_ptr(), v.numel() // self.n_gauss, int(n in self.dense_params)
            stream = L.stream()
            L.check(_timed("bucket_zero", L.load().dnr_grad_zero, ctypes.cast(segs, ctypes.c_void_p), len(segs),
                           self.touched.data_ptr(), self.n_gauss, stream), "dnr_grad_zero")
        else:
            self.flat.zero_()
            self.touched.zero_()
        self.flags_valid, self._clean = False, True
        for n, p in self.params.items():  # re-attach in case an optimizer set .grad = None
            if p.grad is None or p.grad.data_ptr() != self.views[n].data_ptr():
                p.grad = self.views[n]

    def note_backward(self) -> None:
        """Called by the rasterizer's backward after it wrote into sink(); it flags every row it writes.  The flags
        become valid with the first such backward after a zero_() and stay valid through the next ones."""
        self.flags_valid = self.sparse_ok and (self.flags_valid or self._clean)
        self._clean = False

    def sink(self) -> Dict[str, Tensor]:
        """Buffers for dn_rasterize(grad_sink=...)."""
        return dict(self.views, touched=self.touched, grad_records=self.grad_records, bucket=self)

    def all_reduce(self, group=None, async_op: bool = False):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        return None


class PeerGradBucket(FlatGradBucket):
    """FlatGradBucket whose buffer — together with the per-Gaussian `touched` flags dnr_raster_bwd writes — lives in
    NVLink-mapped symmetric memory (torch.distributed._symmetric_memory), so that every rank's kernels can read every
    other rank's gradient rows directly.  `optim.FusedAdam.step_reduce(bucket)` then replaces the
    `bucket.all_reduce(); optimizer.step()` pair with ONE pass that gathers, for each element, the rows of the ranks whose
    view touched the Gaussian (sum in rank order: bit-identical on all replicas) and applies the Adam update — the
    collective is fused into the consumer over peer memory instead of moving the dense 236 MB bucket through NCCL.

    One view per rank and step (the flags describe the last backward).  Needs one process per GPU on a single NVLink
    domain and an initialised NCCL process group."""

    def __init__(self, params: Dict[str, torch.nn.Parameter], names: Iterable[str] = GRAD_PARAMS, group=None):
        import torch.distributed._symmetric_memory as symm_mem

        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("PeerGradBucket needs an initialised process group")
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if self.world > 8:
            raise RuntimeError("PeerGradBucket: at most 8 ranks (one NVLink domain)")
        names = [n for n in names if n in params]
        ps = {n: params[n] for n in names}
        dev = next(iter(ps.values())).device
        n_gauss = next(iter(ps.values())).shape[0]
        total = sum(self._padded(p.numel()) for p in ps.values())
        # one symmetric allocation: [flat gradients | touched flags (padded to 16 B)]
        tbytes = (n_gauss + 15) // 16 * 16
        raw = symm_mem.empty(total * 4 + tbytes, dtype=torch.uint8, device=dev)
        self._handle = symm_mem.rendezvous(raw, self.group.group_name)
        self._raw = raw
        raw.zero_()
        self.names, self.params = names, ps
        self.flat = raw[: total * 4].view(torch.float32)
        self.touched = raw[total * 4: total * 4 + n_gauss]
        self.n_gauss, self._flat_bytes = n_gauss, total * 4
        self.views: Dict[str, Tensor] = {}
        off = 0
        for n, p in ps.items():
            v = self.flat[off:off + p.numel()].view_as(p)
            p.grad = v
            self.views[n] = v
            off += self._padded(p.numel())
        self.mask = torch.zeros(tbytes, dtype=torch.uint8, device=dev)
        # parameters whose gradient is non-zero for every Gaussian on every rank (a loss term that depends on the parameters
        # alone: DNRegularization's min-scale term on `scales`): their segment is gathered from all ranks, not by `touched`
        self.dense_params = {"scales"} & set(ps)
        # dense zero_() and per-backward flags (dnr_raster_bwd clears them): the sparse single-GPU path is not used here
        self.sparse_ok, self.flags_valid, self._clean = False, False, False
        base = [int(x) for x in self._handle.buffer_ptrs]
        self.peer_flat = base
        self.peer_touched = [b + self._flat_bytes for b in base]
        assert self.peer_flat[self.rank] == self.flat.data_ptr()

    def sink(self) -> Dict[str, Tensor]:
        out = dict(self.views)
        out["touched"] = self.touched  # dn_rasterize writes the flags straight into the symmetric buffer
        return out

    def barrier(self) -> None:
        """Cross-rank barrier on the current stream (device-side signal pads of the symmetric allocation)."""
        self._handle.barrier(channel=0)


def shard_views(n_views: int, rank: int, world_size: int) -> List[int]:
    """Round-robin view assignment: rank r renders {i : i mod world_size == r}."""
    return list(range(rank, n_views, world_size))


def all_reduce_densification_stats(xys_grad_norm: Optional[Tensor], vis_counts: Optional[Tensor],
                                   max_2Dsize: Optional[Tensor], group=None) -> None:
    """The extra small collectives needed only at refine_every boundaries (SURVEY §8e): sums and a max."""
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1):
        return
    if xys_grad_norm is not None:
        dist.all_reduce(xys_grad_norm, op=dist.ReduceOp.SUM, group=group)
    if vis_counts is not None:
        dist.all_reduce(vis_counts, op=dist.ReduceOp.SUM, group=group)
    if max_2Dsize is not None:
        dist.all_reduce(max_2Dsize, op=dist.ReduceOp.MAX, group=group)
