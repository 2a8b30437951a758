"""Camera-pose optimisation: stand-in for nerfstudio 1.1.3's `CameraOptimizerConfig` / `CameraOptimizer` and the two
exponential maps of `nerfstudio.cameras.lie_groups` [EXT], used when nerfstudio is not installed (with nerfstudio,
dn_model imports its classes and `config.camera_optimizer.setup(...)` builds nerfstudio's optimizer, as the reference
does at dn_model.py:245-247).

A pose correction is a tangent vector xi = (v, omega) per training camera (`pose_adjustment [num_cameras, 6]`,
zero-initialised).  `apply_to_camera` right-multiplies the camera-to-world matrix by exp(xi), so the correction is
expressed in the camera frame.  Only the projection / SH view sees the corrected pose: the rasterizer returns
d(loss)/d(viewmat) from its projection backward (dnr_project_bwd, DnrArgs.v_viewmat) and autograd carries it through
`get_viewmat` and the maps below to `pose_adjustment`.

Differences from nerfstudio's maps, all below fp32 resolution of the result: both maps here take their coefficients
from theta^2 = |omega|^2 with a Taylor branch for theta^2 < TAYLOR_THETA2 (nerfstudio clamps |omega|^2 at 1e-4 in
SO3xR3, and uses lower-order approximations near zero in SE3).  So both equal torch.linalg.matrix_exp of the twist to
fp64 rounding, and at xi = 0 exactly — where every training run starts — the Jacobian is finite and equals the six
generators (a norm-based formulation has an infinite derivative of |omega| there).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Literal, Type, Union

import torch
from torch import Tensor, nn

TAYLOR_THETA2 = 1e-2  # below: 4-term series (truncation < 3e-11 in every coefficient); above: closed forms


def _coefficients(theta2: Tensor):
    """A = sin(t)/t, B = (1 - cos t)/t^2, C = (t - sin t)/t^3 for t^2 = theta2 [b,1], finite with finite gradients at 0."""
    small = theta2 < TAYLOR_THETA2
    t2 = torch.where(small, torch.ones_like(theta2), theta2)  # the closed forms never see 0 (no inf / nan in backward)
    t = t2.sqrt()
    s, c = t.sin(), t.cos()
    a_big, b_big, c_big = s / t, (1.0 - c) / t2, (t - s) / (t2 * t)
    x = theta2
    a_small = 1.0 - x / 6.0 * (1.0 - x / 20.0 * (1.0 - x / 42.0))
    b_small = 0.5 - x / 24.0 * (1.0 - x / 30.0 * (1.0 - x / 56.0))
    c_small = 1.0 / 6.0 - x / 120.0 * (1.0 - x / 42.0 * (1.0 - x / 72.0))
    return (torch.where(small, a_small, a_big), torch.where(small, b_small, b_big), torch.where(small, c_small, c_big))


def _hat(w: Tensor) -> Tensor:
    """[b,3] -> skew-symmetric [b,3,3] with hat(w) x = w x x (device ops only)."""
    z = torch.zeros_like(w[:, 0])
    return torch.stack([torch.stack([z, -w[:, 2], w[:, 1]], -1),
                        torch.stack([w[:, 2], z, -w[:, 0]], -1),
                        torch.stack([-w[:, 1], w[:, 0], z], -1)], 1)


def _rotation(omega: Tensor):
    K = _hat(omega)
    K2 = K @ K
    A, B, C = _coefficients((omega * omega).sum(-1, keepdim=True))
    eye = torch.eye(3, dtype=omega.dtype, device=omega.device)
    return eye + A[:, :, None] * K + B[:, :, None] * K2, K, K2, B, C


def exp_map_SO3xR3(tangent_vector: Tensor) -> Tensor:
    """nerfstudio lie_groups.exp_map_SO3xR3 [EXT]: [b,6] (translation, axis-angle) -> [b,3,4] = [exp(hat(omega)) | v]."""
    R = _rotation(tangent_vector[:, 3:])[0]
    return torch.cat([R, tangent_vector[:, :3, None]], dim=2)


def exp_map_SE3(tangent_vector: Tensor) -> Tensor:
    """nerfstudio lie_groups.exp_map_SE3 [EXT]: [b,6] (v, omega) -> [b,3,4], the top rows of matrix_exp([[hat(omega), v],
    [0, 0]]) = [R | V v] with V = I + B hat(omega) + C hat(omega)^2."""
    R, K, K2, B, C = _rotation(tangent_vector[:, 3:])
    v = tangent_vector[:, :3, None]
    t = v + B[:, :, None] * (K @ v) + C[:, :, None] * (K2 @ v)
    return torch.cat([R, t], dim=2)


def compose(c2w: Tensor, adj: Tensor) -> Tensor:
    """c2w [b,3,4] @ [[adj], [0,0,0,1]] without a host-side constant (adj [b,3,4])."""
    R = c2w[:, :, :3]
    return torch.cat([R @ adj[:, :, :3], R @ adj[:, :, 3:] + c2w[:, :, 3:]], dim=2)


@dataclass
class CameraOptimizerConfig:
    """nerfstudio 1.1.3 CameraOptimizerConfig [EXT] (fields the model uses)."""

    _target: Type = field(default_factory=lambda: CameraOptimizer)
    mode: Literal["off", "SO3xR3", "SE3"] = "off"
    """Pose optimization strategy to use. If enabled, we recommend SO3xR3."""
    trans_l2_penalty: float = 1e-2
    """L2 penalty on translation parameters (only in get_loss_dict, which the model does not call)."""
    rot_l2_penalty: float = 1e-3
    """L2 penalty on rotation parameters (only in get_loss_dict, which the model does not call)."""

    def setup(self, **kwargs) -> "CameraOptimizer":
        return self._target(self, **kwargs)


class CameraOptimizer(nn.Module):
    """nerfstudio 1.1.3 CameraOptimizer [EXT]: one learnable pose correction per training camera."""

    config: CameraOptimizerConfig

    def __init__(self, config: CameraOptimizerConfig, num_cameras: int, device: Union[torch.device, str] = "cpu",
                 **kwargs) -> None:
        super().__init__()
        self.config = config
        self.num_cameras = num_cameras
        if config.mode in ("SO3xR3", "SE3"):
            # torch.zeros: no RNG draw, so the Gaussians' initialisation is the same with and without camera optimisation
            self.pose_adjustment = nn.Parameter(torch.zeros((num_cameras, 6), device=device))
        elif config.mode != "off":
            raise ValueError(f"unknown camera optimizer mode {config.mode!r}")

    def forward(self, indices) -> Tensor:
        """Pose corrections [b,3,4] of the cameras `indices` (a slice, a list, or an int64 index tensor on any device:
        a slice or a device tensor selects the rows without a host-to-device copy)."""
        if self.config.mode == "off":
            n = len(range(self.num_cameras)[indices]) if isinstance(indices, slice) else len(indices)
            return torch.eye(4, device=self._device())[None, :3, :4].tile(n, 1, 1)
        if isinstance(indices, Tensor):  # index_select: its backward (index_add_) is capturable and never syncs
            rows = self.pose_adjustment.index_select(0, indices.to(self.pose_adjustment.device).reshape(-1))
        else:
            rows = self.pose_adjustment[indices, :]
        return exp_map_SO3xR3(rows) if self.config.mode == "SO3xR3" else exp_map_SE3(rows)

    def _device(self):
        p = next(self.parameters(), None)
        return p.device if p is not None else torch.device("cpu")

    def apply_to_camera(self, camera) -> Tensor:
        """The optimised camera-to-world [1,3,4] of a one-camera batch (unchanged in mode "off" or without
        metadata["cam_idx"], e.g. evaluation cameras)."""
        c2w = camera.camera_to_worlds
        metadata = getattr(camera, "metadata", None)
        if self.config.mode == "off" or not metadata or "cam_idx" not in metadata:
            return c2w
        i = int(metadata["cam_idx"])
        adj = self(slice(i, i + 1))
        return compose(c2w.reshape(-1, 3, 4).to(adj), adj)

    def get_loss_dict(self, loss_dict: Dict) -> None:
        """nerfstudio's pose regulariser (API parity: DNSplatterModel.get_loss_dict does not add it, as the reference's
        does not)."""
        if self.config.mode != "off":
            loss_dict["camera_opt_regularizer"] = (
                self.pose_adjustment[:, :3].norm(dim=-1).mean() * self.config.trans_l2_penalty
                + self.pose_adjustment[:, 3:].norm(dim=-1).mean() * self.config.rot_l2_penalty)

    def get_metrics_dict(self, metrics_dict: Dict) -> None:
        if self.config.mode != "off":
            trans = self.pose_adjustment[:, :3].detach().norm(dim=-1)
            rot = torch.rad2deg(self.pose_adjustment[:, 3:].detach().norm(dim=-1))
            metrics_dict["camera_opt_translation_max"] = trans.max()
            metrics_dict["camera_opt_translation_mean"] = trans.mean()
            metrics_dict["camera_opt_rotation_mean"] = rot.mean()
            metrics_dict["camera_opt_rotation_max"] = rot.max()

    def get_param_groups(self, param_groups: Dict[str, List[nn.Parameter]]) -> None:
        params = list(self.parameters())
        if self.config.mode != "off":
            assert len(params) > 0
            param_groups["camera_opt"] = params
        else:
            assert len(params) == 0
