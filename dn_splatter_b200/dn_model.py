"""DNSplatterModel / DNSplatterModelConfig with the reference's public surface
(/root/reference/dn_splatter/dn_model.py:55-123 config, :126-265 init, :404-612 get_outputs,
:614-729 get_loss_dict), driving the H100 rasterizer instead of gsplat.

The class works standalone (nerfstudio is optional): cameras are duck-typed (cameras.Cameras or
nerfstudio's), parameters keep the reference's names so checkpoints stay interchangeable
(gauss_params: means, scales, quats, features_dc, features_rest, opacities, normals).
Evaluation (get_metrics_dict, get_image_metrics_and_images; reference :731-926) runs on the metric kernels of
metrics.py; LPIPS only through a user-set `model.lpips` callable.  What is deliberately NOT here: SuGaR density helpers,
crop boxes — outside the hot path (SURVEY.md §2.1 #1, §8f).  Camera optimisation (camera_opt.py) renders the
training views with the optimised pose; the projection backward returns the pose gradient.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Literal, Optional, Tuple, Type, Union

import torch
import torch.nn.functional as F
from torch import Tensor

from .camera_opt import compose as compose_pose
from .cameras import Cameras, is_camera
from .losses import DepthLoss, DepthLossType, TVLoss, ssim  # noqa: F401  (ssim re-exported)
from .metrics import DepthMetrics, NormalMetrics, rgb_metrics, tf_resize, u8_as_float
from .rasterize import dn_rasterize, get_viewmat, raster_holder, to_device_async
from .regularization_strategy import (AGSMeshRegularization, DNRegularization, FusedL1, FusedPhotometric, FusedSSIM,
                                      u8_to_float)
from .utils.normal_utils import normal_from_depth_image

SH_C0 = 0.28209479177387814


def num_sh_bases(degree: int) -> int:
    """gsplat.cuda_legacy._wrapper.num_sh_bases [EXT] (reference dn_model.py:35,139)."""
    return (degree + 1) ** 2


def RGB2SH(rgb: Tensor) -> Tensor:
    """nerfstudio.models.splatfacto.RGB2SH [EXT]."""
    return (rgb - 0.5) / SH_C0


def SH2RGB(sh: Tensor) -> Tensor:
    """reference dn_model.py:1512-1517."""
    return sh * SH_C0 + 0.5


def random_quat_tensor(N: int, **kwargs) -> Tensor:
    """Uniform random rotations as wxyz-slot quaternions (reference dn_model.py:1497-1509)."""
    u, v, w = (torch.rand(N, **kwargs) for _ in range(3))
    a, b = torch.sqrt(1 - u), torch.sqrt(u)
    return torch.stack([a * torch.sin(2 * math.pi * v), a * torch.cos(2 * math.pi * v),
                        b * torch.sin(2 * math.pi * w), b * torch.cos(2 * math.pi * w)], dim=-1)


def quat_to_rotmat(quat: Tensor) -> Tensor:
    """gsplat.cuda_legacy._torch_impl.quat_to_rotmat [EXT]: wxyz, normalised inside."""
    w, x, y, z = torch.unbind(F.normalize(quat, dim=-1), dim=-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1),
    ], dim=-2)


def rotation_between(v1: Tensor, v2: Tensor) -> Tensor:
    """Rotation matrices taking unit v1 onto unit v2, Rodrigues (reference rotate_vector_to_vector :1520-1552)."""
    u, t = F.normalize(v1, dim=-1), F.normalize(v2, dim=-1)
    c = (u * t).sum(-1, keepdim=True)
    Kx = t[:, :, None] * u[:, None, :] - u[:, :, None] * t[:, None, :]
    eye = torch.eye(3, device=v1.device).expand(len(u), 3, 3)
    R = eye + Kx + (Kx @ Kx) / (1 + c)[..., None]
    R = torch.where(((c - 1).abs() < 1e-10)[..., None], eye, R)
    return torch.where(((c + 1).abs() < 1e-10)[..., None], -eye, R)


def matrix_to_quaternion(M: Tensor) -> Tensor:
    """Rotation matrices [N,3,3] -> wxyz quaternions, vectorised (the reference loops on the host, :1555-1599)."""
    m = M.reshape(-1, 3, 3)
    tr = m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    cand = torch.stack([
        torch.stack([1 + tr, m[:, 2, 1] - m[:, 1, 2], m[:, 0, 2] - m[:, 2, 0], m[:, 1, 0] - m[:, 0, 1]], -1),
        torch.stack([m[:, 2, 1] - m[:, 1, 2], 1 + m[:, 0, 0] - m[:, 1, 1] - m[:, 2, 2], m[:, 0, 1] + m[:, 1, 0], m[:, 0, 2] + m[:, 2, 0]], -1),
        torch.stack([m[:, 0, 2] - m[:, 2, 0], m[:, 0, 1] + m[:, 1, 0], 1 + m[:, 1, 1] - m[:, 0, 0] - m[:, 2, 2], m[:, 1, 2] + m[:, 2, 1]], -1),
        torch.stack([m[:, 1, 0] - m[:, 0, 1], m[:, 0, 2] + m[:, 2, 0], m[:, 1, 2] + m[:, 2, 1], 1 + m[:, 2, 2] - m[:, 0, 0] - m[:, 1, 1]], -1),
    ], dim=1)  # [N,4 branches,4]
    branch = torch.where(tr > 0, 0, torch.where((m[:, 0, 0] > m[:, 1, 1]) & (m[:, 0, 0] > m[:, 2, 2]), 1,
                                                torch.where(m[:, 1, 1] > m[:, 2, 2], 2, 3)))
    q = cand[torch.arange(len(m)), branch]
    # q / S with S = 2 sqrt(d), d the branch's own diagonal term: a unit quaternion for a proper rotation, and — like
    # the reference, which does not renormalise — (0,0,0,0.7071) for the -I that rotation_between returns for
    # anti-parallel vectors (pinned by tests/test_init_golden.py)
    d = q[torch.arange(len(m)), branch]
    return q / (2.0 * torch.sqrt(d))[:, None]


try:  # nerfstudio is optional: with it the config / model classes below extend Splatfacto's, as the reference's do
    from nerfstudio.cameras.camera_optimizers import CameraOptimizerConfig  # type: ignore
    from nerfstudio.models.splatfacto import SplatfactoModel as _ModelBase  # type: ignore
    from nerfstudio.models.splatfacto import SplatfactoModelConfig as _ConfigBase  # type: ignore

    HAVE_NERFSTUDIO = True
except Exception:  # noqa: BLE001
    HAVE_NERFSTUDIO = False
    _ModelBase = torch.nn.Module
    from .camera_opt import CameraOptimizerConfig  # stand-in for nerfstudio's (camera_opt.py)

    @dataclass
    class _ConfigBase:  # no inherited fields: they are spelled out below with nerfstudio 1.1.3's defaults
        pass


@dataclass
class DNSplatterModelConfig(_ConfigBase):
    """Field names and defaults of the reference's DNSplatterModelConfig (dn_model.py:55-123) plus the
    inherited SplatfactoModelConfig fields [EXT] that the hot path reads.  Dead fields are kept for API
    compatibility and do nothing, exactly as in the reference (SURVEY.md §5)."""

    _target: Type = field(default_factory=lambda: DNSplatterModel)
    regularization_strategy: Literal["dn-splatter", "ags-mesh"] = "dn-splatter"
    use_depth_loss: bool = False
    depth_loss_type: DepthLossType = DepthLossType.EdgeAwareLogL1
    depth_tolerance: float = 0.1
    smooth_loss_type: DepthLossType = DepthLossType.TV
    depth_lambda: float = 0.0
    use_depth_smooth_loss: bool = False
    smooth_loss_lambda: float = 0.1
    predict_normals: bool = True
    use_normal_loss: bool = True
    use_normal_cosine_loss: bool = False
    use_normal_tv_loss: bool = True
    normal_supervision: Literal["mono", "depth"] = "mono"
    normal_lambda: float = 0.1
    use_sparse_loss: bool = False
    sparse_lambda: float = 0.1
    sparse_loss_steps: int = 10
    use_binary_opacities: bool = False
    binary_opacities_threshold: float = 0.9
    two_d_gaussians: bool = True
    warmup_length: int = 500
    num_downscales: int = 0
    use_scale_regularization: bool = False
    max_gauss_ratio: float = 5.0
    stop_split_at: int = 15000
    camera_optimizer: CameraOptimizerConfig = field(default_factory=lambda: CameraOptimizerConfig(mode="off"))
    """Config of the camera optimizer to use (reference dn_model.py:113-116): "off", "SO3xR3" or "SE3"."""
    output_depth_during_training: bool = True
    pearson_lambda: float = 0
    # ---- inherited splatfacto fields [EXT nerfstudio 1.1.3 defaults] ----
    sh_degree: int = 3
    sh_degree_interval: int = 1000
    rasterize_mode: Literal["classic", "antialiased"] = "classic"
    background_color: Literal["random", "black", "white"] = "random"
    ssim_lambda: float = 0.2
    random_init: bool = False
    num_random: int = 50000
    random_scale: float = 10.0
    refine_every: int = 100
    reset_alpha_every: int = 30
    resolution_schedule: int = 3000
    cull_alpha_thresh: float = 0.1
    cull_scale_thresh: float = 0.5
    cull_screen_size: float = 0.15
    split_screen_size: float = 0.05
    stop_screen_size_at: int = 4000
    densify_grad_thresh: float = 0.0008
    densify_size_thresh: float = 0.01
    n_split_samples: int = 2
    continue_cull_post_densification: bool = True
    # ---- dn_splatter_b200 options (not in the reference) ----
    exact_isect_lists: bool = False
    """Emit gsplat's full bbox tile lists instead of the precise-hit lists (parity debugging; images are identical)."""
    sync_free: bool = False
    """Size intersection buffers from earlier views instead of reading the count back (no host sync per view)."""
    fused_ssim: bool = True
    """Evaluate the SSIM term with csrc/ssim.cu (one kernel each way instead of the conv2d formulation, equal to
    1e-6); False keeps the plain-torch `ssim()` below, which is also what non-CUDA tensors use."""
    fuse_loss_backward: bool = True
    """The gradients of the photometric L1 and of DNRegularization's depth / normal terms are evaluated inside
    dnr_raster_bwd (no gradient images, no separate loss-backward launches) whenever the losses see the raster outputs
    directly (no mask, no downscale)."""
    list_shift: int = 2
    """Intersection lists per (16 << list_shift)-pixel supertile (see csrc/binning.cu); ignored with exact_isect_lists."""

    @property
    def camera_optimizer_mode(self) -> str:  # round-1 name of the field
        return getattr(self.camera_optimizer, "mode", "off")

    def setup(self, **kwargs):
        return self._target(self, **kwargs)


class DNSplatterModel(_ModelBase):
    """Depth + Normal splatter on the H100 rasterizer."""

    config: DNSplatterModelConfig

    def __init__(self, config: DNSplatterModelConfig, seed_points: Optional[Tuple[Tensor, ...]] = None,
                 num_train_data: int = 1, device: Union[str, torch.device] = "cuda", **kwargs):
        self._init_device = torch.device(device)
        self._bucket = None
        if HAVE_NERFSTUDIO:
            # SplatfactoModel.__init__ stores seed_points, Model.__init__ stores config / scene_box / num_train_data and
            # calls populate_modules() (ours); callbacks, param groups, metrics and the viewer hooks come from the base
            super().__init__(config, kwargs.pop("scene_box", None), num_train_data, seed_points=seed_points, **kwargs)
        else:
            super().__init__()
            self.config = config
            self.seed_points = seed_points
            self.num_train_data = num_train_data
            self.kwargs = kwargs
            self.populate_modules()
        self.to(self._init_device)

    def load_gaussians(self, params: Dict[str, Tensor]) -> None:
        """Replaces the Gaussian set (same parameter names); used by benchmarks / checkpoint import."""
        dev = self.device
        n = params["means"].shape[0]
        new = {k: torch.nn.Parameter(v.detach().to(dev).float().contiguous()) for k, v in params.items()}
        if "normals" not in new:
            new["normals"] = torch.nn.Parameter(torch.zeros(n, 3, device=dev))
        self.gauss_params = torch.nn.ParameterDict(new)
        self._bucket = None

    def enable_flat_grads(self, peer: bool = False, group=None):
        """Gradients of the six optimised parameter groups become views of ONE flat buffer that the
        rasterizer's backward accumulates into directly (no autograd copies) and that multi-GPU training
        all-reduces with a single NCCL call (parallel.FlatGradBucket) — or, with peer=True, that lives in NVLink-mapped
        symmetric memory so that optim.FusedAdam.step_reduce can gather the gradient rows straight from the peers
        (parallel.PeerGradBucket)."""
        from .parallel import FlatGradBucket, PeerGradBucket

        if peer and (self.config.use_scale_regularization or self.config.use_sparse_loss):
            raise NotImplementedError("peer-memory gradient reduction gathers only the rows of composited Gaussians, plus the "
                                      "`scales` segment (min-scale regulariser); other parameter-only loss terms make more "
                                      "segments dense: use peer=False (NCCL all-reduce)")
        self._bucket = PeerGradBucket(dict(self.gauss_params), group=group) if peer else FlatGradBucket(dict(self.gauss_params))
        if self.config.use_scale_regularization or self.config.use_sparse_loss:
            self._bucket.sparse_ok = False  # the same parameter-only terms: no sparse zero_() / Adam reads
        self._bucket_mode = (bool(peer), group)  # densification re-creates the bucket in the same mode (densify._replace_params)
        return self._bucket

    # ------------------------------------------------------------------ init (reference :131-265)
    def k_nearest_sklearn(self, x: Tensor, k: int):
        from sklearn.neighbors import NearestNeighbors

        xn = x.cpu().numpy()
        nn_model = NearestNeighbors(n_neighbors=k + 1, algorithm="auto", metric="euclidean").fit(xn)
        d, i = nn_model.kneighbors(xn)
        return d[:, 1:].astype("float32"), i[:, 1:].astype("float32")

    def populate_modules(self):
        cfg = self.config
        if self.seed_points is not None and not cfg.random_init:
            means = self.seed_points[0].float().cpu()
        else:
            means = (torch.rand((cfg.num_random if cfg.random_init else 500000, 3)) - 0.5) * (
                cfg.random_scale if cfg.random_init else 10)
        self.xys_grad_norm = None
        self.max_2Dsize = None
        dim_sh = num_sh_bases(cfg.sh_degree)
        n = means.shape[0]
        if self.seed_points is not None and not cfg.random_init:
            shs = torch.zeros((n, dim_sh, 3))
            rgb = self.seed_points[1].float().cpu() / 255
            shs[:, 0, :3] = RGB2SH(rgb) if cfg.sh_degree > 0 else torch.logit(rgb, eps=1e-10)
            features_dc, features_rest = shs[:, 0, :].clone(), shs[:, 1:, :].clone()
        else:
            features_dc, features_rest = torch.rand(n, 3), torch.zeros((n, dim_sh - 1, 3))
        opacities = torch.logit(0.1 * torch.ones(n, 1))
        self.step = 0
        self.crop_box = None
        if cfg.background_color == "random":
            self.background_color = torch.tensor([0.1490, 0.1647, 0.2157])  # reference :160-163
        else:
            self.background_color = torch.tensor({"black": [0.0, 0.0, 0.0], "white": [1.0, 1.0, 1.0]}[cfg.background_color])
        self.mse_loss = torch.nn.MSELoss()
        # LPIPS needs network weights: rgb_lpips is reported only when the user sets a callable lpips(gt, pred) here
        self.lpips = None
        self.depth_metrics = DepthMetrics()
        self.normal_metrics = NormalMetrics()
        if cfg.use_depth_loss:
            self.depth_loss = DepthLoss(cfg.depth_loss_type)
            assert cfg.depth_lambda > 0, "depth_lambda should be > 0"
        if cfg.use_depth_smooth_loss:
            self.smooth_loss = DepthLoss(DepthLossType.EdgeAwareTV if cfg.smooth_loss_type == DepthLossType.EdgeAwareTV
                                         else DepthLossType.TV)
        dist, _ = self.k_nearest_sklearn(means, 3)
        avg_dist = torch.from_numpy(dist).mean(dim=-1, keepdim=True)
        with torch.no_grad():
            if self.seed_points is not None and len(self.seed_points) == 3:
                normals = F.normalize(self.seed_points[-1].float().cpu(), dim=-1)
                scales = torch.log(avg_dist.repeat(1, 3))
                scales[:, 2] = torch.log((avg_dist / 10)[:, 0])
                z = torch.tensor([0.0, 0.0, 1.0]).repeat(n, 1)
                quats = matrix_to_quaternion(rotation_between(z, normals))
            else:
                scales = torch.log(avg_dist.repeat(1, 3))
                quats = random_quat_tensor(n)
                idx = torch.argmin(scales, dim=-1)
                normals = F.normalize(quat_to_rotmat(quats)[torch.arange(n), :, idx], dim=1)
        P = torch.nn.Parameter
        self.gauss_params = torch.nn.ParameterDict({
            "means": P(means), "scales": P(scales), "quats": P(quats), "features_dc": P(features_dc),
            "features_rest": P(features_rest), "opacities": P(opacities), "normals": P(normals.detach()),
        })
        self.camera_idx = 0
        self.camera = None
        if cfg.use_normal_tv_loss:
            self.tv_loss = TVLoss()
        if cfg.regularization_strategy == "dn-splatter":
            self.regularization_strategy = DNRegularization()
            self.regularization_strategy.fuse_backward = cfg.fuse_loss_backward
        elif cfg.regularization_strategy == "ags-mesh":
            self.regularization_strategy = AGSMeshRegularization()
        else:
            raise NotImplementedError
        rs = self.regularization_strategy
        if cfg.use_depth_loss:  # reference :256-262
            rs.depth_loss_type, rs.depth_loss, rs.depth_lambda = cfg.depth_loss_type, self.depth_loss, cfg.depth_lambda
        else:
            rs.depth_loss_type, rs.depth_loss = None, None
        if not cfg.use_normal_loss:
            rs.normal_loss = None
        # reference :245-247; moved to the model's device with the module.  No RNG draw (zero-initialised).
        self.camera_optimizer = cfg.camera_optimizer.setup(num_cameras=self.num_train_data, device="cpu")

    # ------------------------------------------------------------------ parameter views
    means = property(lambda self: self.gauss_params["means"])
    scales = property(lambda self: self.gauss_params["scales"])
    quats = property(lambda self: self.gauss_params["quats"])
    features_dc = property(lambda self: self.gauss_params["features_dc"])
    features_rest = property(lambda self: self.gauss_params["features_rest"])
    opacities = property(lambda self: self.gauss_params["opacities"])
    normals = property(lambda self: self.gauss_params["normals"])
    num_points = property(lambda self: self.gauss_params["means"].shape[0])
    colors = property(lambda self: SH2RGB(self.features_dc) if self.config.sh_degree > 0 else torch.sigmoid(self.features_dc))

    @property
    def device(self):
        return self.gauss_params["means"].device

    @property
    def vis_indices(self):
        """Indices of visible Gaussians (reference :531).  Lazy: torch.where synchronises the device."""
        return torch.where(self.radii > 0)[0]

    def get_gaussian_param_groups(self) -> Dict[str, List[torch.nn.Parameter]]:
        return {n: [self.gauss_params[n]] for n in ("means", "scales", "quats", "features_dc", "features_rest",
                                                     "opacities", "normals")}

    def get_param_groups(self):
        """SplatfactoModel.get_param_groups [EXT]: the Gaussian groups plus "camera_opt" unless the mode is "off"."""
        groups = self.get_gaussian_param_groups()
        self.camera_optimizer.get_param_groups(param_groups=groups)
        return groups

    # ------------------------------------------------------------------ helpers [EXT splatfacto]
    def _get_downscale_factor(self) -> int:
        if self.training:
            return 2 ** max(self.config.num_downscales - self.step // self.config.resolution_schedule, 0)
        return 1

    def _get_background_color(self) -> Tensor:
        if self.config.background_color == "random":
            return torch.rand(3) if self.training else self.background_color
        return self.background_color

    def _downscale_if_required(self, image: Tensor) -> Tensor:
        """nerfstudio 1.1.3 splatfacto `resize_image` [EXT]: d x d box filter (conv2d with uniform weights, stride d)."""
        d = self._get_downscale_factor()
        if d > 1:
            image = image.to(torch.float32)
            weight = (1.0 / (d * d)) * torch.ones((1, 1, d, d), dtype=torch.float32, device=image.device)
            return F.conv2d(image.permute(2, 0, 1)[:, None, ...], weight, stride=d).squeeze(1).permute(1, 2, 0)
        return image

    def get_gt_img(self, image: Tensor, clamp_min: float = 0.0) -> Tensor:
        """SplatfactoModel.get_gt_img [EXT]: uint8 -> float / 255, downscale, to the model's device; `clamp_min` is the
        reference's `.clamp(min=10 / 255)` applied AFTER the resize (dn_model.py:633)."""
        d = self._get_downscale_factor()
        if image.dtype == torch.uint8:
            if image.device.type == "cuda" and d == 1:
                return u8_to_float(image, 255.0, clamp_min).to(self.device)  # one kernel instead of float() / 255 / clamp
            image = image.float() / 255.0
        image = self._downscale_if_required(image).to(self.device)
        return image.clamp(min=clamp_min) if clamp_min > 0.0 else image

    def composite_with_background(self, image: Tensor, background: Tensor) -> Tensor:
        if image.shape[2] == 4:
            alpha = image[..., -1:].repeat(1, 1, 3)
            return alpha * image[..., :3] + (1 - alpha) * background.to(image)
        return image

    # ------------------------------------------------------------------ get_outputs (reference :404-612)
    def get_outputs(self, camera) -> Dict[str, Union[Tensor, List[Tensor]]]:
        if not is_camera(camera):
            print("Called get_outputs with not a camera")
            return {}
        cfg = self.config
        if self.training:
            assert camera.shape[0] == 1, "Only one camera at a time"
        # camera optimisation (reference :420-425): training views with metadata["cam_idx"] render with the optimised pose;
        # evaluation, mode "off" and views without an index use the pose as given
        cam_idx = None
        if self.training and cfg.camera_optimizer_mode != "off":
            meta = getattr(camera, "metadata", None)
            if meta and "cam_idx" in meta:
                cam_idx = int(meta["cam_idx"])
                if not 0 <= cam_idx < self.num_train_data:
                    raise ValueError(f"camera optimisation: cam_idx {cam_idx} is not one of the model's "
                                     f"{self.num_train_data} training cameras (num_train_data)")
        if cfg.use_binary_opacities and self.step > cfg.warmup_length:  # reference :427-437
            skip = cfg.reset_alpha_every * cfg.refine_every
            if self.step % skip != 0 and self.step % skip not in range(1, 201):
                self.gauss_params["opacities"].data = torch.where(
                    self.opacities >= cfg.binary_opacities_threshold, torch.ones_like(self.opacities),
                    torch.zeros_like(self.opacities))
        if self.crop_box is not None and not self.training:
            raise NotImplementedError("crop boxes are viewer-only and outside the hot path")
        if cfg.rasterize_mode not in ("antialiased", "classic"):
            raise ValueError("Unknown rasterize_mode: %s", cfg.rasterize_mode)
        if cfg.sh_degree <= 0:
            raise NotImplementedError("sh_degree == 0 (sigmoid colours) is broken upstream (SURVEY A1.4); not mirrored")
        scale_fac = self._get_downscale_factor()
        camera.rescale_output_resolution(1 / scale_fac)
        dev = self.device
        # Per-camera constants are cached on the camera object as HOST tensors and handed to the kernels by value:
        # the step issues no H2D copy and no device op for the camera (unless its pose is optimised, below).
        cache = camera.__dict__.setdefault("_dnr_cache", {})
        pose = camera.camera_to_worlds
        key = (scale_fac, pose.data_ptr(), pose._version)  # an in-place pose update invalidates the entry
        if key not in cache:
            cache.clear()
            c2w_host = pose.reshape(-1, 3, 4)[0].detach().float().cpu()
            cache[key] = (camera.get_intrinsics_matrices()[0].float().cpu(), int(camera.width.flatten()[0]),
                          int(camera.height.flatten()[0]), c2w_host, get_viewmat(c2w_host))
        K, W, H, c2w_fixed, viewmat = cache[key]
        if cam_idx is not None:  # the pose gradient needs a device viewmat: device copies of K and the un-optimised c2w
            dkey = (key, str(dev))
            if dkey not in cache:
                cache[dkey] = (to_device_async(K, dev), to_device_async(c2w_fixed, dev))
            K, c2w_fixed = cache[dkey]
        fixed_capacity = 0
        gc = self.__dict__.get("_graph_cam")
        if gc is not None:  # CUDA-graph mode: camera in static device buffers (refreshed before each replay), fixed capacity
            K, c2w_fixed, viewmat, fixed_capacity = gc.K, gc.c2w, gc.viewmat, gc.capacity
        if cam_idx is not None:
            # c2w @ exp(pose_adjustment[cam_idx]) on the device; in graph mode the row index is a device tensor too.  The
            # normals keep the un-optimised, detached c2w (reference :550-560).
            rows = gc.cam_idx if gc is not None else slice(cam_idx, cam_idx + 1)
            viewmat = get_viewmat(compose_pose(c2w_fixed.reshape(1, 3, 4), self.camera_optimizer(rows)))
        self.last_size = (H, W)
        camera.rescale_output_resolution(scale_fac)
        sh_degree_to_use = min(self.step // cfg.sh_degree_interval, cfg.sh_degree)
        background = self._get_background_color()

        # rasterize_mode="antialiased" with normals: the reference's colour pass uses opacity x compensation, its normal
        # pass (legacy rasterize_gaussians, :564-575) the plain opacity.  One fused pass cannot carry two alpha streams,
        # so this (non-default) mode renders twice, as the reference does: colour / depth antialiased, normals classic.
        dual = cfg.rasterize_mode == "antialiased" and cfg.predict_normals
        common = dict(sh_degree=sh_degree_to_use, near_plane=0.01, far_plane=1e10, background=background, c2w=c2w_fixed,
                      exact_lists=cfg.exact_isect_lists, sync_free=cfg.sync_free, fixed_capacity=fixed_capacity,
                      list_shift=cfg.list_shift, stats=self.__dict__.get("_raster_stats"))
        params = (self.means, self.quats, self.scales, self.opacities, self.features_dc, self.features_rest, viewmat, K, W, H)
        sink = self._bucket.sink() if (self._bucket is not None and torch.is_grad_enabled()) else None
        out = dn_rasterize(*params, antialiased=cfg.rasterize_mode == "antialiased",
                           render_normals=cfg.predict_normals and not dual, grad_sink=sink, **common)
        out_n = dn_rasterize(*params, antialiased=False, render_normals=True, surface_normal=False, grad_sink=sink,
                             **common) if dual else out
        self.raster_out = out
        self.xys = out.means2d[None]  # [1,N,2]; .grad / .absgrad live on out.means2d after backward
        self.xys_flat = out.means2d
        self.radii = out.radii
        self.depths = out.depths[None]
        self.conics = out.conics[None]
        self.num_tiles_hit = out.tiles_per_gauss[None]
        if cfg.predict_normals:
            self.gauss_params["normals"].data = out_n.normals_world  # reference :558 (same Parameter object)
            normals_im = out_n.normal
        else:
            normals_im = torch.full((1, H, W, 3), 0.0)  # quirk B13: CPU zeros
        if getattr(camera, "metadata", None) is not None and "cam_idx" in camera.metadata:
            self.camera_idx = camera.metadata["cam_idx"]
        self.camera = camera
        return {
            "rgb": out.rgb, "depth": out.depth, "normal": normals_im, "surface_normal": out.surface_normal,
            "accumulation": out.alpha, "background": self._background_on_device(background, dev),
        }

    def _background_on_device(self, background: Tensor, dev) -> Tensor:
        if background is self.background_color:  # fixed colour: upload once
            cached = self.__dict__.get("_bg_dev")
            if cached is None or cached.device != torch.device(dev):
                cached = to_device_async(background, dev)
                self.__dict__["_bg_dev"] = cached
            return cached
        return to_device_async(background, dev)

    def forward(self, camera):
        return self.get_outputs(camera)

    @torch.no_grad()
    def get_outputs_for_camera(self, camera, obb_box=None) -> Dict[str, Tensor]:
        assert camera is not None, "must provide camera to gaussian model"
        return self.get_outputs(camera.to(self.device) if hasattr(camera, "to") else camera)

    # ------------------------------------------------------------------ get_loss_dict (reference :614-729)
    def _rgb_loss_dict(self, outputs, batch) -> Dict[str, Tensor]:
        """SplatfactoModel.get_loss_dict [EXT nerfstudio 1.1.3]: (1-l) L1 + l (1-SSIM), optional scale reg."""
        cfg = self.config
        pred_img = outputs["rgb"]
        img = batch["image"]
        fused = ("mask" not in batch and img.shape[-1] == 3 and img.device == pred_img.device and pred_img.is_cuda
                 and self._get_downscale_factor() == 1)
        if fused and cfg.ssim_lambda > 0 and cfg.fused_ssim and pred_img.shape[0] > 10 and pred_img.shape[1] > 10:
            # (1 - l) L1 + l (1 - SSIM) in one kernel each way: pred receives a single gradient image
            main = FusedPhotometric.apply(pred_img, img, cfg.ssim_lambda)
            return {"main_loss": main, "scale_reg": self._scale_reg()}
        if fused:  # photometric L1 straight from the (uint8) image: one kernel forward, backward inside dnr_raster_bwd
            l1 = FusedL1.apply(pred_img, img, raster_holder(pred_img) if cfg.fuse_loss_backward else None)
            gt_img = None
        else:
            gt_img = self.composite_with_background(self.get_gt_img(img), outputs["background"])
            if "mask" in batch:
                mask = self._downscale_if_required(batch["mask"]).to(self.device)
                assert mask.shape[:2] == gt_img.shape[:2] == pred_img.shape[:2]
                gt_img, pred_img = gt_img * mask, pred_img * mask
            l1 = torch.abs(gt_img - pred_img).mean()
        main = (1 - cfg.ssim_lambda) * l1
        if cfg.ssim_lambda > 0:
            if cfg.fused_ssim and pred_img.is_cuda:
                # fused path: the uint8 image is read as stored (value / 255 inside the kernel)
                sim = FusedSSIM.apply(pred_img, img if gt_img is None else gt_img)
            else:
                if gt_img is None:
                    gt_img = self.get_gt_img(img)
                sim = ssim(gt_img.permute(2, 0, 1)[None], pred_img.permute(2, 0, 1)[None])
            main = main + cfg.ssim_lambda * (1 - sim)
        return {"main_loss": main, "scale_reg": self._scale_reg()}

    def _scale_reg(self) -> Tensor:
        cfg = self.config
        if cfg.use_scale_regularization and self.step % 10 == 0:
            se = torch.exp(self.scales)
            reg = torch.clamp(se.amax(dim=-1) / se.amin(dim=-1), min=cfg.max_gauss_ratio) - cfg.max_gauss_ratio
            return 0.1 * reg.mean()
        z = self.__dict__.get("_zero_scalar")
        if z is None or z.device != self.device:
            z = self.__dict__["_zero_scalar"] = torch.zeros((), device=self.device)
        return z

    def _ags_raw_ok(self, outputs, batch) -> bool:
        """Whether get_loss_dict hands the batch's maps to AGSMeshRegularization's fused kernels as stored: the ags-mesh
        strategy on a fused configuration, CUDA maps of a kernel dtype, no batch mask, no downscale, and every map the
        strategy reads present (a missing one keeps the torch code and its error)."""
        cfg = self.config
        rs = self.regularization_strategy
        if not (cfg.regularization_strategy == "ags-mesh" and rs._fusable() and "mask" not in batch
                and self._get_downscale_factor() == 1):
            return False
        u8f32 = (torch.uint8, torch.float32)
        image, conf = batch["image"], batch.get("confidence")
        if not (image.is_cuda and image.shape[-1] == 3 and image.dtype in u8f32):
            return False
        if conf is None or not conf.is_cuda or conf.dtype not in u8f32:
            return False
        if "sensor_depth" not in batch and "mono_depth" not in batch:
            return False
        if cfg.normal_supervision == "mono":
            n = batch.get("normal")
            if n is None or not n.is_cuda or n.dtype not in u8f32:
                return False
        elif cfg.normal_supervision != "depth":
            return False
        maps = (outputs["depth"], outputs["normal"], outputs["surface_normal"])
        return all(t.is_cuda and t.dtype == torch.float32 for t in maps) and not outputs["surface_normal"].requires_grad

    def get_loss_dict(self, outputs, batch, metrics_dict=None) -> Dict[str, Tensor]:
        cfg = self.config
        loss_dict = self._rgb_loss_dict(outputs, batch)
        rgb_loss, scale_reg = loss_dict["main_loss"], loss_dict["scale_reg"]
        image = batch["image"]
        # uint8 maps go to the fused regulariser as they are (scaled and clamped inside the kernels): no conversion passes
        raw_ok = (cfg.regularization_strategy == "dn-splatter" and "mask" not in batch and self._get_downscale_factor() == 1
                  and image.dtype == torch.uint8 and image.is_cuda and image.shape[-1] == 3)
        # ags-mesh on the fused kernels: the raw image, normals and confidence map go to them as stored, the rendered
        # normals in their [0,1] encoding (no 2x - 1, permute or get_gt_img passes)
        ags_raw = self._ags_raw_ok(outputs, batch)
        gt_img = image if (raw_ok or (ags_raw and image.dtype == torch.uint8)) else self.get_gt_img(image, clamp_min=10 / 255.0)  # quirk B10
        depth_out = outputs["depth"]
        sensor_depth_gt = self.get_gt_img(batch["sensor_depth"]) if "sensor_depth" in batch else None
        mono_depth_gt = self.get_gt_img(batch["mono_depth"]) if "mono_depth" in batch else None
        if "normal" in batch and not ((raw_ok or ags_raw) and batch["normal"].dtype == torch.uint8 and batch["normal"].is_cuda):
            batch["normal"] = self.get_gt_img(batch["normal"])
        if ags_raw:
            confidence = batch["confidence"]
        elif "confidence" in batch:
            confidence = 1 - self.get_gt_img(batch["confidence"]) / 255.0
        if "mask" in batch:  # quirk B11: in-place on the dicts
            mask = batch["mask"].to(self.device)
            assert mask.shape[:2] == gt_img.shape[:2] == outputs["rgb"].shape[:2]
            depth_out = depth_out * mask
            if sensor_depth_gt is not None:
                sensor_depth_gt = sensor_depth_gt * mask
            if mono_depth_gt is not None:
                mono_depth_gt = mono_depth_gt * mask
            if "normal" in batch:
                batch["normal"] = batch["normal"] * mask
            if "normal" in outputs:
                outputs["normal"] = outputs["normal"] * mask
        pred_normal = outputs["normal"]
        surface_normal = outputs["surface_normal"]
        if "normal" in batch and cfg.normal_supervision == "mono":
            gt_normal = batch["normal"]
        elif cfg.normal_supervision == "depth":
            cam = self.camera
            gt_normal = normal_from_depth_image(
                depths=depth_out.detach(), fx=float(cam.fx.flatten()[0]), fy=float(cam.fy.flatten()[0]),
                cx=float(cam.cx.flatten()[0]), cy=float(cam.cy.flatten()[0]),
                img_size=(int(cam.width.flatten()[0]), int(cam.height.flatten()[0])),
                c2w=torch.eye(4, dtype=torch.float, device=depth_out.device), device=self.device, smooth=False)
            gt_normal = (1 + torch.cat([gt_normal[..., :1], -gt_normal[..., 1:]], dim=-1)) / 2
        else:
            gt_normal = None
        depth_gt = sensor_depth_gt
        if mono_depth_gt is not None:
            depth_gt = mono_depth_gt
        if depth_gt is None and cfg.use_depth_loss:
            print("[dn_splatter_b200] use_depth_loss is True but the batch holds no depth maps")
        extra = {"scales": self.scales, "gt_img": gt_img}
        if ags_raw:
            reg = self.regularization_strategy.fused_loss(
                self.step, depth_out, depth_gt, surface_normal, gt_normal, pred_normal, confidence, gt_img, self.scales,
                confidence_raw=True)
        elif cfg.regularization_strategy == "dn-splatter":
            reg = self.regularization_strategy(pred_depth=depth_out, gt_depth=depth_gt, pred_normal=pred_normal,
                                               gt_normal=gt_normal, **extra)
        else:
            reg = self.regularization_strategy(
                step=self.step, pred_depth=depth_out, gt_depth=depth_gt, confidence_map=confidence,
                surf_normal=(2 * surface_normal - 1).permute(2, 0, 1), gt_normal=(2 * gt_normal - 1).permute(2, 0, 1),
                pred_normal=(2 * pred_normal - 1).permute(2, 0, 1), **extra)
        return {"main_loss": rgb_loss + reg, "scale_reg": scale_reg}

    # ------------------------------------------------------------------ evaluation (reference :731-926)
    def _eval_image(self, image: Tensor, outputs, keep_u8: bool) -> Tensor:
        """A batch image as the metrics compare it, on the model's device: RGBA composited with the background; uint8
        read as value / 255 (kept as stored when `keep_u8`, for the kernels to scale)."""
        image = image.to(self.device)
        if keep_u8 and image.dtype == torch.uint8 and image.shape[-1] == 3:
            return image
        background = outputs.get("background", self.background_color)
        return self.composite_with_background(u8_as_float(image), background.to(self.device))

    def _lpips(self, gt_rgb: Tensor, pred_rgb: Tensor, metrics_dict: Dict) -> None:
        if callable(self.lpips):
            metrics_dict["rgb_lpips"] = float(self.lpips(u8_as_float(gt_rgb).permute(2, 0, 1)[None],
                                                         pred_rgb.permute(2, 0, 1)[None]))

    def get_metrics_dict(self, outputs, batch) -> Dict[str, Union[float, int, Tensor]]:
        """Reference dn_model.py:731-807: rgb_mse / rgb_psnr / rgb_ssim (rgb_lpips with `self.lpips` set),
        gaussian_count, the depth_* metrics of the sensor depth when use_depth_loss, avg_min_scale.  While the training
        resolution is downscaled, the image and sensor depth are resized as torchvision's TF.resize(antialias=None)
        does (bilinear), not with the loss path's box filter."""
        d = self._get_downscale_factor()
        image, sensor_depth = batch["image"], batch.get("sensor_depth")
        if d > 1:
            image = tf_resize(image.permute(2, 0, 1), (image.shape[0] // d, image.shape[1] // d)).permute(1, 2, 0)
            if sensor_depth is not None:
                size = (sensor_depth.shape[0] // d, sensor_depth.shape[1] // d)
                sensor_depth = tf_resize(sensor_depth.permute(2, 0, 1), size).permute(1, 2, 0)
        gt_rgb = self._eval_image(image, outputs, keep_u8=True)
        pred_rgb = outputs["rgb"][0, ...] if outputs["rgb"].dim() == 4 else outputs["rgb"]
        mse, psnr, sim = rgb_metrics(pred_rgb.permute(2, 0, 1)[None], gt_rgb.permute(2, 0, 1)[None])
        metrics_dict = {"rgb_mse": float(mse), "rgb_psnr": float(psnr), "rgb_ssim": float(sim)}
        self._lpips(gt_rgb, pred_rgb, metrics_dict)
        metrics_dict["gaussian_count"] = self.num_points
        if self.config.use_depth_loss and sensor_depth is not None:
            pred_depth = outputs["depth"][0, ...] if outputs["depth"].dim() == 4 else outputs["depth"]
            values = self.depth_metrics(pred_depth.permute(2, 0, 1), sensor_depth.to(self.device).permute(2, 0, 1))
            metrics_dict.update(_depth_dict(values))
        metrics_dict["avg_min_scale"] = torch.nanmean(torch.exp(self.scales.detach()[..., -1]))
        return metrics_dict

    def get_image_metrics_and_images(self, outputs: Dict[str, Tensor], batch: Dict[str, Tensor]
                                     ) -> Tuple[Dict[str, float], Dict[str, Tensor]]:
        """Reference dn_model.py:809-926: rgb_psnr / rgb_ssim (rgb_lpips with `self.lpips` set), the depth_* metrics
        when the batch has sensor_depth, normal_mae / normal_rsme (sic) / normal_mean_err / normal_med_err when it has
        normal, and images_dict {img, depth, normal} with target and render side by side.  A batch mask multiplies
        both images and both depths per pixel (the reference's [1,3,H,W] * [H,W,1] product fails for any real image).
        The normal metrics compare the [0,1]-encoded maps as stored, as the reference does."""
        dev = self.device
        gt_rgb = self._eval_image(batch["image"], outputs, keep_u8=False)
        pred_rgb = outputs["rgb"][0, ...] if outputs["rgb"].dim() == 4 else outputs["rgb"]
        pred_depth = outputs["depth"][0, ...] if outputs["depth"].dim() == 4 else outputs["depth"]
        pred_normal = outputs["normal"][0, ...] if outputs["normal"].dim() == 4 else outputs["normal"]
        combined_rgb = torch.cat([gt_rgb, pred_rgb], dim=1)
        combined_depth, combined_normal = pred_depth, pred_normal
        mask = batch["mask"].to(dev) if "mask" in batch else None
        if mask is not None:
            gt_rgb, pred_rgb = gt_rgb * mask, pred_rgb * mask
        _, psnr, sim = rgb_metrics(pred_rgb.permute(2, 0, 1)[None], gt_rgb.permute(2, 0, 1)[None])
        metrics_dict = {"rgb_psnr": float(psnr), "rgb_ssim": float(sim)}
        self._lpips(gt_rgb, pred_rgb, metrics_dict)
        if "sensor_depth" in batch:
            gt_depth = batch["sensor_depth"].to(dev)
            if pred_depth.shape[:2] != gt_depth.shape[:2]:
                pred_depth = tf_resize(pred_depth.permute(2, 0, 1), gt_depth.shape[:2]).permute(1, 2, 0)
            gt_depth = gt_depth.to(torch.float32)
            if mask is not None:
                gt_depth, pred_depth = gt_depth * mask, pred_depth * mask
            metrics_dict.update(_depth_dict(self.depth_metrics(pred_depth.permute(2, 0, 1), gt_depth.permute(2, 0, 1))))
            combined_depth = torch.cat([gt_depth, pred_depth], dim=1)
        if "normal" in batch:
            gt_normal = u8_as_float(batch["normal"].to(dev))
            pred_normal = pred_normal.to(dev)
            if gt_normal.shape != pred_normal.shape:
                pred_normal = tf_resize(pred_normal.permute(2, 0, 1), gt_normal.shape[:2]).permute(1, 2, 0)
            mae, rmse, mean_err, med_err = self.normal_metrics(pred_normal.permute(2, 0, 1)[None],
                                                               gt_normal.permute(2, 0, 1)[None])
            metrics_dict.update({"normal_mae": float(mae), "normal_rsme": float(rmse), "normal_mean_err": float(mean_err),
                                 "normal_med_err": float(med_err)})
            combined_normal = torch.cat([gt_normal, pred_normal], dim=1)
        return metrics_dict, {"img": combined_rgb, "depth": combined_depth, "normal": combined_normal}

    def step_cb(self, step: int):
        self.step = step

    # ------------------------------------------------------------------ densification (SURVEY §8f-2; densify.py)
    def _densify_cfg(self):
        from .densify import DensifyConfig

        c = self.config
        return DensifyConfig(
            warmup_length=c.warmup_length, refine_every=c.refine_every, reset_alpha_every=c.reset_alpha_every,
            stop_split_at=c.stop_split_at, stop_screen_size_at=c.stop_screen_size_at,
            densify_grad_thresh=c.densify_grad_thresh, densify_size_thresh=c.densify_size_thresh,
            n_split_samples=c.n_split_samples, split_screen_size=c.split_screen_size, cull_alpha_thresh=c.cull_alpha_thresh,
            cull_scale_thresh=c.cull_scale_thresh, cull_screen_size=c.cull_screen_size,
            continue_cull_post_densification=c.continue_cull_post_densification)

    def after_train(self, step: int):
        """SplatfactoModel.after_train [EXT]: accumulate the view's absgrad / radii statistics."""
        from .densify import DensifyState

        assert step == self.step
        if self.__dict__.get("_densify_state") is None:
            self.__dict__["_densify_state"] = DensifyState()
        absgrad = getattr(self.xys_flat, "absgrad", None)
        if absgrad is not None:
            self._densify_state.after_train(absgrad, self.radii, self.last_size)

    def refinement_after(self, optimizers, step: int, generator=None):
        """Reference dn_model.py:271-386.  `optimizers`: {param name: torch optimizer} (densify.build_optimizers) or a
        nerfstudio `Optimizers` object exposing `.optimizers`."""
        from .densify import DensifyState, refinement_after

        assert step == self.step
        opts = getattr(optimizers, "optimizers", optimizers)
        state = self.__dict__.get("_densify_state") or DensifyState()
        self.__dict__["_densify_state"] = state
        return refinement_after(self, opts, step, state, self._densify_cfg(), self.num_train_data, generator)


def _depth_dict(values) -> Dict[str, float]:
    names = ("depth_abs_rel", "depth_sq_rel", "depth_rmse", "depth_rmse_log", "depth_a1", "depth_a2", "depth_a3")
    return {k: float(v) for k, v in zip(names, values)}
