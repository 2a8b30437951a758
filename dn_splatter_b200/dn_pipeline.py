"""DNSplatterPipeline / DNSplatterPipelineConfig with the reference's constructor contract
(/root/reference/dn_splatter/dn_pipeline.py:49-130): builds the datamanager, forwards seed points
(points3D_xyz / points3D_rgb / points3D_normals metadata) to the model, and — where the reference wraps the
model in DDP — installs the per-camera sharding + single flat all-reduce of parallel.py.
get_average_eval_image_metrics averages the image metrics of every eval view (dn_pipeline.py:133-638); its point-cloud
metrics, render dumps and MuSHRoom / FARO branches are not mirrored (SURVEY.md §2.1 #6)."""
from __future__ import annotations

from dataclasses import dataclass, field
from time import time
from typing import Any, Dict, Literal, Optional, Type

import torch
import torch.distributed as dist

from .dn_model import DNSplatterModel, DNSplatterModelConfig
from .parallel import FlatGradBucket

try:  # with nerfstudio the classes extend VanillaPipeline(Config), exactly as the reference's do (dn_pipeline.py:36-66)
    from nerfstudio.pipelines.base_pipeline import VanillaPipeline as _PipelineBase  # type: ignore
    from nerfstudio.pipelines.base_pipeline import VanillaPipelineConfig as _PipelineConfigBase  # type: ignore

    HAVE_NERFSTUDIO = True
except Exception:  # noqa: BLE001
    HAVE_NERFSTUDIO = False
    _PipelineBase = torch.nn.Module

    @dataclass
    class _PipelineConfigBase:
        pass


@dataclass
class DNSplatterPipelineConfig(_PipelineConfigBase):
    _target: Type = field(default_factory=lambda: DNSplatterPipeline)
    datamanager: Any = None  # object with .setup(device=, test_mode=, world_size=, local_rank=) or a ready datamanager
    model: DNSplatterModelConfig = field(default_factory=DNSplatterModelConfig)
    experiment_name: str = "experiment"
    skip_point_metrics: bool = True
    num_pd_points: int = 1_000_000
    save_train_images: bool = False

    def setup(self, **kwargs):
        return self._target(self, **kwargs)


class DNSplatterPipeline(_PipelineBase):
    """Datamanager contract: `next_train(step) -> (camera, batch)` with the batch keys of the reference's
    DNSplatterDataManager (image, mask, sensor_depth, mono_depth, normal, confidence; dn_datamanager.py:90-150),
    optional `train_dataparser_outputs.metadata`, `train_dataset` (len + optional scene_box/metadata)."""

    def __init__(self, config: DNSplatterPipelineConfig, device: str,
                 test_mode: Literal["test", "val", "inference"] = "val", world_size: int = 1, local_rank: int = 0,
                 grad_scaler=None):
        # like the reference (dn_pipeline.py:76): skip VanillaPipeline.__init__, which would build its own datamanager / DDP
        (super(_PipelineBase, self) if HAVE_NERFSTUDIO else super()).__init__()
        self.config, self.test_mode = config, test_mode
        dm = config.datamanager
        if hasattr(dm, "setup"):
            dm = dm.setup(device=device, test_mode=test_mode, world_size=world_size, local_rank=local_rank)
        self.datamanager = dm
        seed_pts = None
        meta = getattr(getattr(dm, "train_dataparser_outputs", None), "metadata", None) or {}
        if "points3D_xyz" in meta:
            seed_pts = (meta["points3D_xyz"], meta["points3D_rgb"])
            if "points3D_normals" in meta:
                seed_pts = seed_pts + (meta["points3D_normals"],)
        train_ds = getattr(dm, "train_dataset", None)
        assert train_ds is not None, "Missing input dataset"
        self._model = config.model.setup(num_train_data=len(train_ds), device=device, seed_points=seed_pts,
                                         metadata=getattr(train_ds, "metadata", None),
                                         scene_box=getattr(train_ds, "scene_box", None), grad_scaler=grad_scaler)
        self.world_size, self.local_rank = world_size, local_rank
        self.bucket: Optional[FlatGradBucket] = None
        if world_size > 1:  # reference :123-128 wraps in DDP + barrier
            self.bucket = FlatGradBucket(dict(self._model.gauss_params))
            if dist.is_initialized():
                dist.barrier()

    @property
    def model(self) -> DNSplatterModel:
        return self._model

    @property
    def device(self):
        return self._model.device

    def get_train_loss_dict(self, step: int):
        """VanillaPipeline.get_train_loss_dict [EXT]: one view per rank; call `reduce_gradients()` after backward."""
        camera, batch = self.datamanager.next_train(step)
        outputs = self._model(camera)
        loss_dict = self._model.get_loss_dict(outputs, batch, None)
        return outputs, loss_dict, {}

    def reduce_gradients(self):
        if self.bucket is not None:
            self.bucket.all_reduce()

    @torch.no_grad()
    def get_average_eval_image_metrics(self, step: Optional[int] = None, output_path=None, get_std: bool = False):
        """Iterates over every eval image and averages the model's get_image_metrics_and_images over them, plus
        num_rays_per_sec and fps of the render (reference dn_pipeline.py:133-638).  With `get_std`, every key also
        gets `<key>_std` (torch.std_mean: NaN for a single image).

        Datamanager contract: `datamanager.eval_dataset.cameras` is sliceable (cameras[i : i + 1] is view i) and
        `datamanager.cached_eval` is a sequence of batches in the same order.  Point-cloud metrics
        (skip_point_metrics=False; mesh_eval.point_cloud_metrics scores point clouds), render dumps (`output_path`) and
        the MuSHRoom parser's split are not supported and raise NotImplementedError."""
        if not self.config.skip_point_metrics:
            raise NotImplementedError("point-cloud metrics in the eval loop: use mesh_eval.point_cloud_metrics")
        if output_path is not None:
            raise NotImplementedError("render dumps (output_path) are not supported")
        if getattr(self.datamanager, "dataparser", None).__class__.__name__ == "MushroomDataParser":
            raise NotImplementedError("the MuSHRoom with / within split of the eval metrics is not supported")
        self.eval()
        metrics_dict_list = []
        cameras = self.datamanager.eval_dataset.cameras
        for image_idx, batch in enumerate(self.datamanager.cached_eval):
            camera = cameras[image_idx: image_idx + 1].to("cpu")
            inner_start = time()
            outputs = self.model.get_outputs_for_camera(camera=camera)
            height, width = camera.height, camera.width
            num_rays = height * width
            metrics_dict, _ = self.model.get_image_metrics_and_images(outputs, batch)
            assert "num_rays_per_sec" not in metrics_dict
            metrics_dict["num_rays_per_sec"] = (num_rays / (time() - inner_start)).item()
            assert "fps" not in metrics_dict
            metrics_dict["fps"] = (metrics_dict["num_rays_per_sec"] / (height * width)).item()
            metrics_dict_list.append(metrics_dict)
        metrics_dict = {}
        for key in metrics_dict_list[0].keys():
            values = torch.tensor([m[key] for m in metrics_dict_list])
            if get_std:
                key_std, key_mean = torch.std_mean(values)
                metrics_dict[key] = float(key_mean)
                metrics_dict[f"{key}_std"] = float(key_std)
            else:
                metrics_dict[key] = float(torch.mean(values))
        self.train()
        return metrics_dict
