"""CUDA-graph capture of one whole training view: bucket.zero_ -> get_outputs -> get_loss_dict -> backward
(-> the caller's all-reduce / optimiser outside the graph).  ~46 kernel launches, ~60 allocations and ~1.3 ms of
Python per view collapse into one cudaGraphLaunch, which makes the step immune to host jitter and removes the
inter-kernel launch gaps.  render_service.py captures its forward with the same StaticCamera and capture_slots.

What makes the step capturable (see rasterize.py / dn_model.py):
  * `fixed_capacity`: intersection buffers sized once (1.15 x the largest count seen), no count read-back inside the
    graph; every replay's count goes to a rasterize.CountWatch, checked at the NEXT call (and by `check_capacity()`):
    a replay that needed more slots raises DnrCapacityError — call `recapture()` and redo;
  * the camera lives in a StaticCamera that `load_camera` refreshes with one small pinned H2D copy before each
    replay (resolution must not change between replays);
  * the supervision maps live in static device buffers that the caller fills (H2D or D2D) before each replay;
  * gradients go to the flat bucket (static addresses); the loss is a static 0-dim tensor.
Run the training loop on a non-default stream (`torch.cuda.set_stream(torch.cuda.Stream())`): the legacy default
stream cannot take part in a capture and autograd pins each parameter's gradient accumulator to the stream it was
first used on.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

from . import _lib as L
from .rasterize import GROWTH, CountWatch, get_viewmat, grow, suggested_capacity


class StaticCamera:
    """What get_outputs renders with while installed as the model's `_graph_cam`: the static device camera block
    [viewmat 16 | K 9 | c2w 12], read through `viewmat` / `K` / `c2w`, and the graph's fixed intersection `capacity`.
    With `num_cameras` (camera optimisation) also the view's metadata["cam_idx"] as a device int64 [1], `cam_idx`: the
    graph selects the view's pose_adjustment row with it."""

    def __init__(self, size: Tuple[int, int], device, capacity: int, num_cameras: Optional[int] = None):
        self.size, self.capacity = size, int(capacity)
        self.data = torch.zeros(37, device=device)
        self.viewmat, self.K, self.c2w = self.data[:16].view(4, 4), self.data[16:25].view(3, 3), self.data[25:].view(3, 4)
        self.num_cameras = num_cameras
        self.cam_idx = torch.zeros(1, dtype=torch.int64, device=device) if num_cameras is not None else None

    def load(self, camera) -> None:
        """Refreshes the block from a camera: ONE 148-byte async H2D copy from a per-camera pinned tensor
        (stream-ordered after the previous replay, so the host may run ahead)."""
        assert (int(camera.width.flatten()[0]), int(camera.height.flatten()[0])) == self.size, "resolution is baked in"
        pinned = camera.__dict__.get("_dnr_graph_cam")
        if pinned is None:
            c2w = camera.camera_to_worlds.reshape(-1, 3, 4)[0].detach().float().cpu()
            pinned = torch.cat([get_viewmat(c2w).reshape(-1), camera.get_intrinsics_matrices()[0].float().cpu().reshape(-1),
                                c2w.reshape(-1)]).contiguous().pin_memory()
            camera.__dict__["_dnr_graph_cam"] = pinned
        if self.cam_idx is not None:
            metadata = getattr(camera, "metadata", None)
            if not metadata or "cam_idx" not in metadata:
                raise ValueError("camera optimisation in a captured step needs metadata['cam_idx'] on every camera")
            if not 0 <= int(metadata["cam_idx"]) < self.num_cameras:
                raise ValueError(f"cam_idx {int(metadata['cam_idx'])} is not one of the {self.num_cameras} training cameras")
            idx = camera.__dict__.get("_dnr_graph_idx")
            if idx is None or int(idx[0]) != int(metadata["cam_idx"]):
                idx = torch.tensor([int(metadata["cam_idx"])], dtype=torch.int64).pin_memory()
                camera.__dict__["_dnr_graph_idx"] = idx
            self.cam_idx.copy_(idx, non_blocking=True)
        self.data.copy_(pinned, non_blocking=True)


def capture_slots(fn, n_slots: int, warmup: int, device) -> Tuple[List[torch.cuda.CUDAGraph], list]:
    """Runs `fn(0)` `warmup` times on a side stream (allocator pools, cub temp sizes), then captures `fn(slot)` once per
    slot into graphs that share one memory pool; returns the graphs and what each captured call returned."""
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn(0)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize(device)
    # thread-local capture mode: other threads of the process (NCCL's watchdog, the symmetric-memory runtime of a
    # multi-rank job) keep making CUDA API calls while we capture; in the default "global" mode any of them invalidates
    # the capture (cudaErrorStreamCaptureInvalidated, seen intermittently at 2 ranks)
    graphs, results, pool = [], [], None
    for slot in range(n_slots):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=pool, capture_error_mode="thread_local"):
            results.append(fn(slot))
        pool = g.pool()
        graphs.append(g)
    return graphs, results


class GraphedTrainStep:
    def __init__(self, model, bucket, example_camera, example_batch: Dict[str, Tensor], n_slots: int = 2,
                 capacity: Optional[int] = None, warmup: int = 3):
        assert model.training, "capture the training step in train() mode"
        if model.config.background_color == "random":
            raise ValueError("background_color='random' draws a new host-side colour every step; a captured graph would "
                             "freeze the first one.  Use 'black' / 'white' (or run eagerly).")
        self.model, self.bucket = model, bucket
        dev = self.device = model.device
        W, H = int(example_camera.width.flatten()[0]), int(example_camera.height.flatten()[0])
        if capacity is None:
            cfg = model.config
            capacity = suggested_capacity(model.num_points, W, H, cfg.predict_normals, cfg.exact_isect_lists, dev.index,
                                          cfg.list_shift)
        if capacity <= 0:
            raise ValueError("no intersection statistics yet: run a few sync_free views first or pass capacity=")
        cam_opt = model.config.camera_optimizer_mode != "off"
        self.cam = StaticCamera((W, H), dev, capacity, num_cameras=model.num_train_data if cam_opt else None)
        if cam_opt:
            # replays accumulate the pose gradient into a buffer whose address the graph baked in
            pa = model.camera_optimizer.pose_adjustment
            if pa.grad is None:
                pa.grad = torch.zeros_like(pa)
        self.batches: List[Dict[str, Tensor]] = [
            {k: torch.empty_like(v, device=dev) for k, v in example_batch.items()} for _ in range(n_slots)]
        self.losses = [torch.zeros((), device=dev) for _ in range(n_slots)]
        self._camera = example_camera
        self._n_slots, self._warmup = n_slots, warmup
        self._watch = CountWatch("Call recapture() and run the view again.")
        for b in self.batches:
            for k, v in example_batch.items():
                b[k].copy_(v)
        self.load_camera(example_camera)
        self._capture()

    @property
    def capacity(self) -> int:
        return self.cam.capacity

    @property
    def max_count(self) -> int:
        return self._watch.max_seen

    @staticmethod
    def _gates(m):
        """Host-side, step-dependent branches of get_outputs / get_loss_dict that a capture bakes in."""
        c = m.config
        gates = (min(m.step // c.sh_degree_interval, c.sh_degree), bool(c.use_scale_regularization and m.step % 10 == 0),
                 bool(c.use_binary_opacities and m.step > c.warmup_length), m._get_downscale_factor())
        if c.regularization_strategy == "ags-mesh":  # AGSMeshRegularization's confidence gate, normal weight, mask kind
            gates += (m.step >= 7000, m.step > 7000, m.step < m.regularization_strategy.normal_mask_steps)
        return gates

    def _capture(self) -> None:
        model = self.model
        self._captured_gates = self._gates(model)
        self.graphs = []
        # Autograd graphs of earlier eager steps keep the parameters' AccumulateGrad nodes alive, and those remember the
        # stream they were created on (usually the legacy default stream, which may not take part in a capture):
        # drop the model's cached outputs so the nodes are rebuilt on the warm-up / capture streams.
        import gc

        for name in ("raster_out", "xys", "xys_flat", "radii", "depths", "conics", "num_tiles_hit"):
            if name in model.__dict__:
                model.__dict__[name] = None
        gc.collect()
        # the warm-up runs add real pose gradients: keep the accumulation window's gradient as it was
        pa = model.camera_optimizer.pose_adjustment if self.cam.cam_idx is not None else None
        saved = pa.grad.clone() if pa is not None else None
        self.graphs, self._count_dev = capture_slots(self._eager, self._n_slots, self._warmup, self.device)
        if pa is not None:
            pa.grad.copy_(saved)

    def _eager(self, slot: int) -> Tensor:
        m = self.model
        m.__dict__["_graph_cam"] = self.cam
        try:
            self.bucket.zero_()  # sparse or dense as the bucket's flags allow when the graph is captured
            L.capture_ok("bucket zero")
            out = m.get_outputs(self._camera)
            L.capture_ok("get_outputs")
            ld = m.get_loss_dict(out, dict(self.batches[slot]))
            L.capture_ok("get_loss_dict")
            loss = ld["main_loss"] + ld["scale_reg"]
            loss.backward()
            L.capture_ok("backward")
            self.losses[slot].copy_(loss.detach())
            return m.raster_out.info["n_isects_dev"]  # the graph's own count tensor
        finally:
            m.__dict__["_graph_cam"] = None

    def load_camera(self, camera) -> None:
        """Refreshes the static camera block from a camera (StaticCamera.load)."""
        self.cam.load(camera)

    def __call__(self, camera, slot: int = 0) -> Tensor:
        """Replays the captured step for `camera` on the supervision maps currently in `self.batches[slot]`;
        returns the static loss tensor of that slot (read it asynchronously)."""
        if self._gates(self.model) != self._captured_gates:
            raise RuntimeError(f"step-dependent host decisions changed since capture ({self._captured_gates} -> "
                               f"{self._gates(self.model)}): call recapture()")
        self.check_capacity()
        self.load_camera(camera)
        self.graphs[slot].replay()
        self._watch.observe(self._count_dev[slot], self.capacity)
        return self.losses[slot]

    def check_capacity(self, wait: bool = False) -> None:
        """Raises DnrCapacityError if a finished replay needed more intersection slots than the graph was captured
        with (its gradients are truncated: discard them, `recapture()`, replay the view again)."""
        self._watch.poll(wait)
        self._watch.raise_unreported()

    def recapture(self, capacity: Optional[int] = None) -> None:
        """Re-captures the step with room for the largest count seen so far (grow(.., GROWTH)) or the given capacity."""
        self._watch.poll(wait=True)
        self._watch.unreported = None  # an overflow of the old graphs: the caller runs that view again
        need = int(capacity) if capacity else grow(self.max_count, GROWTH)
        self.cam.capacity = max(self.cam.capacity, need)
        torch.cuda.synchronize(self.device)
        self._capture()
