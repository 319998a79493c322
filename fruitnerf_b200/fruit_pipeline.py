"""FruitPipeline -- drop-in surface of fruit_nerf.fruit_pipeline.FruitPipeline (66-260).

Differences that matter on the GPU: instead of wrapping the model in DDP (fruit_pipeline.py:117, NCCL
all-reduce of every parameter's .grad in 25 MiB buckets) the backward kernels accumulate into ONE
flat fp32 gradient buffer (ops.flat_zero_grads) and ``sync_gradients`` all-reduces that buffer in a
single NCCL collective over NVLink/NVSwitch (mean over ranks, the DDP semantics).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Literal, Optional, Type

import torch
import torch.distributed as dist
from torch import nn
from torch.nn import Parameter

from . import ops
from .compat import InstantiateConfig
from .data.fruit_datamanager import FruitDataManagerConfig
from .fruit_nerf import FruitNerfModelConfig


@dataclass
class FruitPipelineConfig(InstantiateConfig):
    """fruit_pipeline.py:54-63."""

    _target: Type = field(default_factory=lambda: FruitPipeline)
    datamanager: Any = field(default_factory=FruitDataManagerConfig)
    model: Any = field(default_factory=FruitNerfModelConfig)


def sync_gradients(flat_grad: torch.Tensor, world_size: int, group=None, async_op: bool = False):
    """Mean all-reduce of the flat gradient buffer (the reference's DDP exchange)."""
    if world_size <= 1:
        return None
    return dist.all_reduce(flat_grad, op=dist.ReduceOp.AVG if flat_grad.is_cuda else dist.ReduceOp.SUM, group=group,
                           async_op=async_op) if flat_grad.is_cuda else _cpu_mean_all_reduce(flat_grad, world_size, group)


def _cpu_mean_all_reduce(t: torch.Tensor, world_size: int, group=None):
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)  # gloo has no AVG
    t.div_(world_size)
    return None


class FruitPipeline(nn.Module):
    """fruit_pipeline.py:66-260 (constructor signature and method names kept)."""

    def __init__(self, config: FruitPipelineConfig, device: str, test_mode: Literal["test", "val", "inference", "export"] = "val",
                 world_size: int = 1, local_rank: int = 0, grad_scaler: Optional[Any] = None):
        super().__init__()
        self.config = config
        self.test_mode = test_mode
        self.datamanager = config.datamanager.setup(device=device, test_mode=test_mode, world_size=world_size, local_rank=local_rank)
        self.datamanager.to(device)
        assert self.datamanager.train_dataset is not None, "Missing input dataset"  # fruit_pipeline.py:102
        self._model = config.model.setup(
            scene_box=self.datamanager.train_dataset.scene_box,
            num_train_data=len(self.datamanager.train_dataset),
            metadata=self.datamanager.train_dataset.metadata,
            device=device,
            grad_scaler=grad_scaler,
            test_mode=test_mode,
            render_rgb_inference=True,
        )
        self._model.to(device)
        self.world_size = world_size
        self.local_rank = local_rank
        if world_size > 1:
            dist.barrier()  # fruit_pipeline.py:118

    @property
    def model(self):
        return self._model

    @property
    def device(self):
        return self._model.device

    def get_train_loss_dict(self, step: int):
        """fruit_pipeline.py:120-146."""
        ray_bundle, batch = self.datamanager.next_train(step)
        model_outputs = self._model(ray_bundle)
        metrics_dict = self.model.get_metrics_dict(model_outputs, batch)
        loss_dict = self.model.get_loss_dict(model_outputs, batch, metrics_dict)
        return model_outputs, loss_dict, metrics_dict

    @torch.no_grad()
    def get_eval_image_metrics_and_images(self, step: int):
        """fruit_pipeline.py:155-172: render one held-out image and hand it to the model's get_image_metrics_and_images
        (psnr / ssim / iou as upstream, plus ``fruit_iou``: the fruit-mask agreement of the thresholded semantic map)."""
        was_training = self.training
        self.eval()
        image_idx, camera_ray_bundle, batch = self.datamanager.next_eval_image(step)
        outputs = self.model.get_outputs_for_camera_ray_bundle(camera_ray_bundle)
        metrics, images = self.model.get_image_metrics_and_images(outputs, batch)
        assert "image_idx" not in metrics
        metrics["image_idx"] = image_idx
        assert "num_rays" not in metrics
        metrics["num_rays"] = int(camera_ray_bundle.origins.shape[0] * camera_ray_bundle.origins.shape[1])
        self.train(was_training)
        return metrics, images

    @torch.no_grad()
    def get_average_eval_image_metrics(self, step: Optional[int] = None, output_path=None) -> Dict[str, float]:
        """fruit_pipeline.py:174-227: mean of every per-image metric over the eval split (plus rays/s of the renders);
        ``output_path``: also write each image of the images dict as ``<camera>-<key>.jpg``."""
        import time

        n = len(self.datamanager.eval_dataset)
        rows = []
        for _ in range(n):
            t0 = time.time()
            metrics, images = self.get_eval_image_metrics_and_images(step or 0)
            metrics["num_rays_per_sec"] = metrics["num_rays"] / max(time.time() - t0, 1e-9)
            metrics["fps"] = metrics["num_rays_per_sec"] / metrics["num_rays"]
            if output_path is not None:
                self._save_eval_images(output_path, metrics["image_idx"], images)
            rows.append(metrics)
        return {k: float(sum(r[k] for r in rows) / n) for k in rows[0] if k not in ("image_idx", "num_rays")}

    @staticmethod
    def _save_eval_images(output_path, image_idx: int, images: Dict[str, torch.Tensor]) -> None:
        """fruit_pipeline.py:205-210: ``<camera>-<key>.jpg`` per entry of the images dict."""
        import pathlib

        import numpy as np
        from PIL import Image

        out = pathlib.Path(output_path)
        out.mkdir(parents=True, exist_ok=True)
        for key, val in images.items():
            arr = (val.detach().float().clamp(0, 1) * 255).byte().cpu().numpy()
            if arr.ndim == 3 and arr.shape[-1] == 1:
                arr = np.repeat(arr, 3, axis=-1)
            Image.fromarray(arr).save(out / f"{image_idx:06d}-{key}.jpg")

    def sync_gradients(self):
        """Call after ``loss.backward()``: one collective over the flat gradient buffer."""
        flat = ops._Render.last_flat_grad
        if flat is not None:
            sync_gradients(flat, self.world_size)

    # keys a nerfstudio-written FruitNeRF checkpoint holds that have no counterpart here: metric modules of the model
    # (fruit_nerf.py:174-177) and the datamanager's camera optimiser / ray generators
    REFERENCE_ONLY_PREFIXES = ("_model.lpips.", "_model.psnr.", "_model.ssim.", "_model.collider.", "datamanager.train_camera_optimizer.",
                               "datamanager.train_ray_generator.", "datamanager.eval_ray_generator.", "datamanager.orthographic_ray_generator.")

    def load_pipeline(self, loaded_state: Dict[str, Any], step: int, strict: bool = True) -> None:
        """fruit_pipeline.py:229-240: strip DDP's ``module.`` prefix, strict load.  ``strict=False`` is the loader for
        checkpoints the REFERENCE wrote with ``implementation='torch'``: keys of modules that only exist upstream
        (``REFERENCE_ONLY_PREFIXES``) are dropped, everything else must still match name by name and shape by shape
        (tinycudann checkpoints store packed fp16 ``params`` blobs and cannot be mapped)."""
        state = {(key[len("module."):] if key.startswith("module.") else key): value for key, value in loaded_state.items()}
        self.model.update_to_step(step)
        if not strict:
            state = {k: v for k, v in state.items() if not k.startswith(self.REFERENCE_ONLY_PREFIXES)}
            if any(k.endswith(".params") for k in state):
                raise ValueError("tinycudann checkpoint (packed fp16 `params` tensors): retrain or export with implementation='torch'")
        self.load_state_dict(state, strict=True)

    def get_training_callbacks(self, training_callback_attributes) -> List:
        """fruit_pipeline.py:242-249: datamanager callbacks followed by the model's (proposal-weight annealing)."""
        datamanager_callbacks = self.datamanager.get_training_callbacks(training_callback_attributes)
        model_callbacks = self.model.get_training_callbacks(training_callback_attributes)
        return list(datamanager_callbacks) + list(model_callbacks)

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        """fruit_pipeline.py:251-260."""
        return {**self.datamanager.get_param_groups(), **self.model.get_param_groups()}
