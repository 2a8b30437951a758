"""A minimal training loop standing in for nerfstudio's Trainer [EXT] around the hot path: per-group Adam with the
reference's learning rates (dn_config.py:29-68), the callback order of SURVEY §3.1 (step_cb -> forward -> losses ->
backward -> [all-reduce] -> optimizer step -> after_train -> refinement every `refine_every`), per-camera sharding
over ranks.  With camera optimisation on, the "camera_opt" group has its own torch.optim.Adam, stepped with nerfstudio's
gradient accumulation (TRAINER_DEFAULTS: every 100 steps).  Eager launches (the Gaussian count changes at refinements; capture a GraphedTrainStep between them if
wanted)."""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch

from .densify import build_optimizers, exponential_lr
from .dn_config import MAX_NUM_ITERATIONS, TRAINER_DEFAULTS, optimizer_groups


class Trainer:
    def __init__(self, model, next_train: Callable[[int], tuple], max_steps: int = MAX_NUM_ITERATIONS,
                 world_size: int = 1, seed: int = 0, fused_adam: bool = False, peer_reduce: bool = False,
                 camera_opt_accum: Optional[int] = None):
        self.model, self.next_train, self.max_steps = model, next_train, max_steps
        self.groups = optimizer_groups(max_steps)
        self.fused = None
        if fused_adam:  # all groups in one dnr_adam_step launch, see optim.py
            from .optim import FusedAdam

            self.fused = FusedAdam.for_model(model, self.groups)
            self.optimizers: Dict[str, torch.optim.Optimizer] = self.fused.as_dict(model)
        else:
            self.optimizers = build_optimizers(model, self.groups)
        # peer_reduce: the gradient sum over ranks happens inside the Adam kernel over NVLink peer memory
        # (optim.FusedAdam.step_reduce) instead of an NCCL all-reduce of the dense bucket followed by the step
        self.peer_reduce = bool(peer_reduce) and world_size > 1
        if self.peer_reduce and self.fused is None:
            raise ValueError("peer_reduce needs fused_adam=True (the reduction is part of dnr_adam_step_reduce)")
        self.bucket = model.enable_flat_grads(peer=self.peer_reduce)
        # camera poses: not part of FusedAdam (which steps every group every step).  nerfstudio's Trainer zeroes a group
        # with gradient_accumulation_steps = k at step % k == 0 and steps it at step % k == k - 1 [EXT]
        self.camera_opt: Optional[torch.optim.Optimizer] = None
        cam_params = model.get_param_groups().get("camera_opt")
        if cam_params:
            g = self.groups["camera_opt"]
            self.camera_opt = torch.optim.Adam(cam_params, lr=g["lr"], eps=g["eps"])
            for p in cam_params:  # every rank joins the all-reduce, also one whose views had no cam_idx
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
        self.camera_opt_accum = int(camera_opt_accum if camera_opt_accum is not None
                                    else TRAINER_DEFAULTS["gradient_accumulation_steps"]["camera_opt"])
        self.world_size = world_size
        self.generator = torch.Generator().manual_seed(seed)  # identical on every rank: identical split samples
        self.step = 0

    def train_iteration(self) -> Dict[str, float]:
        m, step = self.model, self.step
        m.train()
        m.step_cb(step)
        camera, batch = self.next_train(step)
        self.bucket = m._bucket or m.enable_flat_grads()
        self.bucket.zero_()
        if self.camera_opt is not None and step % self.camera_opt_accum == 0:
            self.camera_opt.zero_grad(set_to_none=False)  # keeps the gradient's address (a captured step accumulates there)
        outputs = m.get_outputs(camera)
        loss_dict = m.get_loss_dict(outputs, batch)
        loss = loss_dict["main_loss"] + loss_dict["scale_reg"]
        loss.backward()
        if self.world_size > 1 and not self.peer_reduce:
            self.bucket.all_reduce()
        for name, opt in self.optimizers.items():
            g = self.groups[name]
            if g.get("lr_final"):
                for pg in opt.param_groups:
                    if pg.get("name", name) == name:
                        pg["lr"] = exponential_lr(g["lr"], g["lr_final"], step, g["max_steps"])
            if self.fused is None:
                opt.step()
        if self.peer_reduce:
            self.fused.step_reduce(self.bucket)
        elif self.fused is not None:
            self.fused.step()
        if self.camera_opt is not None:
            self._camera_opt_step(step)
        m.after_train(step)
        info: Optional[Dict[str, int]] = None
        if step > 0 and step % m.config.refine_every == 0:
            st = m.__dict__.get("_densify_state")
            # Reduce ONLY when refinement_after will consume (and reset) the statistics: during warm-up it returns without
            # resetting them, and an in-place all-reduce there would be summed again at the next boundary (weight W^k).
            if self.world_size > 1 and st is not None:
                # identical statistics -> identical decisions (and identical split samples: same seed)
                st.all_reduce_before_refinement(step, m.config.warmup_length)
            info = m.refinement_after(self.optimizers, step, generator=self.generator)
        self.step += 1
        return {"loss": loss.detach(), "refine": info}

    def _camera_opt_step(self, step: int) -> None:
        g = self.groups["camera_opt"]
        for pg in self.camera_opt.param_groups:  # the scheduler advances every step
            pg["lr"] = exponential_lr(g["lr"], g["lr_final"], step, g["max_steps"])
        if step % self.camera_opt_accum != self.camera_opt_accum - 1:
            return
        if self.world_size > 1:  # every rank renders other cameras: sum the pose gradient once per accumulation window
            import torch.distributed as dist

            for pg in self.camera_opt.param_groups:
                for p in pg["params"]:
                    if p.grad is not None:
                        dist.all_reduce(p.grad, op=dist.ReduceOp.SUM)
        self.camera_opt.step()
