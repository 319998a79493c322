"""Datamanager of the plugin surface (fruit_nerf/data/fruit_datamanager.py).

Export side (SURVEY.md section 8a E1/E2): ``get_corners_of_aabb`` (42-68), ``sample_surface_points`` (71-121),
``FruitDataManager.setup_inference`` (157-172) and ``next_sample_volume`` (199-204) -- they define the export
ray grid.  Training side (section 8f rank 3): ``next_train`` / ``next_eval`` (183-215) over an in-memory data set
(images + fruit masks + cameras resident on the GPU, e.g. ``data.synthetic_scene``): uniform pixel sampling across
all training images and pinhole ray generation on the device -- no host work or H2D copy per step.  Reading
images from disk (nerfstudio's dataparser / dataloader machinery) is host I/O outside the path.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, Optional, Tuple, Type, Union

import torch
from torch import nn

from ..compat import InstantiateConfig, RayBundle
from ..components.ray_generators import OrthographicRayGenerator


def get_corners_of_aabb(aabb, device):
    """8 corners of an AABB given as (min xyz, max xyz) -- fruit_datamanager.py:42-68."""
    mn, mx = aabb[0], aabb[1]
    return torch.asarray(
        [
            [mn[0], mn[1], mn[2]],
            [mx[0], mn[1], mn[2]],
            [mn[0], mx[1], mn[2]],
            [mx[0], mx[1], mn[2]],
            [mn[0], mn[1], mx[2]],
            [mx[0], mn[1], mx[2]],
            [mn[0], mx[1], mx[2]],
            [mx[0], mx[1], mx[2]],
        ],
        dtype=torch.float32,
        device=device,
    )


def sample_surface_points(aabb, n, device, noise=False):
    """Regular grid on the z = min face of the box spanned by the 8 corners ``aabb`` and the vector
    to the opposite face (fruit_datamanager.py:71-121): int(dx/dz*n) x int(dy/dz*n) points,
    meshgrid 'ij' flattened x-major."""
    c1, c2, c3 = aabb[0], aabb[1], aabb[2]
    dxyz = torch.abs(torch.max(aabb, dim=0).values - torch.min(aabb, dim=0).values)
    const_axis = int(torch.argmax(torch.logical_and((c1 == c2), (c2 == c3)).to(int)))
    ax = torch.argmax(torch.abs(c1 - c2))
    x = torch.linspace(float(c1[ax]), float(c2[ax]), int(dxyz[0] / dxyz[const_axis] * n), dtype=torch.float32, device=device)
    ay = torch.argmax(torch.abs(c1 - c3))
    y = torch.linspace(float(c1[ay]), float(c3[ay]), int(dxyz[1] / dxyz[const_axis] * n), dtype=torch.float32, device=device)
    xx, yy = torch.meshgrid(x, y, indexing="ij")
    pts = torch.column_stack((xx.flatten(), yy.flatten(), torch.full_like(xx.flatten(), float(c3[const_axis]))))
    c4 = aabb[-1]
    plane_vector = torch.asarray(
        [[0, 0, float(torch.sign(c4[const_axis]) * torch.abs(c1[const_axis]) + torch.abs(c4[const_axis]))]],
        dtype=torch.float32, device=device)
    return pts.clone(), plane_vector


@dataclass
class FruitDataManagerConfig(InstantiateConfig):
    _target: Type = field(default_factory=lambda: FruitDataManager)
    train_num_rays_per_batch: int = 4096
    eval_num_rays_per_batch: int = 4096
    synthetic_scene: Optional[Dict] = None  # kwargs of data.synthetic_scene.make_apple_scene (no data set on disk)
    dataparser: Optional[Any] = None        # FruitNerfDataParserConfig: read transforms.json + images + fruit masks from disk
    seed: int = 0


class FruitDataManager(nn.Module):
    """Export-side subset of fruit_nerf.data.fruit_datamanager.FruitDataManager."""

    config: FruitDataManagerConfig

    def __init__(self, config: FruitDataManagerConfig, device: Union[torch.device, str] = "cpu", test_mode: str = "val",
                 world_size: int = 1, local_rank: int = 0, **kwargs):
        super().__init__()
        self.config = config
        self.device = device
        self.test_mode = test_mode
        self.world_size, self.local_rank = world_size, local_rank
        self.train_count = 0
        self.eval_count = 0
        self.train_dataset = kwargs.get("train_dataset")
        self.eval_dataset = kwargs.get("eval_dataset")
        if self.train_dataset is None and config.synthetic_scene is not None:
            from .synthetic_scene import make_apple_scene

            self.train_dataset, self.eval_dataset = make_apple_scene(**config.synthetic_scene)
        self.train_dataparser_outputs = None
        if self.train_dataset is None and config.dataparser is not None:
            # fruit_datamanager.py:137-147 (dataparser -> train / eval data sets), decoded once into memory
            from .fruitnerf_dataparser import load_fruit_datasets

            self.train_dataset, self.eval_dataset, self.train_dataparser_outputs = load_fruit_datasets(config.dataparser)
        if self.train_dataset is not None and hasattr(self.train_dataset, "to"):
            self.train_dataset = self.train_dataset.to(device)
            if self.eval_dataset is not None:
                self.eval_dataset = self.eval_dataset.to(device)
        self.orthographic_ray_generator: Optional[OrthographicRayGenerator] = None
        self._gen: Optional[torch.Generator] = None

    # ---- training / evaluation batches (fruit_datamanager.py:183-215) ------------------------------------
    def _generator(self) -> torch.Generator:
        if self._gen is None:
            self._gen = torch.Generator(device=self.device)
            self._gen.manual_seed(self.config.seed * 7919 + self.local_rank)  # each rank draws its own batch (fruit_pipeline.py:97-99)
        return self._gen

    def _pixel_batch(self, ds, num_rays: int) -> Tuple[RayBundle, Dict]:
        """nerfstudio PixelSampler.sample_method (uniform over images x rows x cols) + RayGenerator."""
        from .synthetic_scene import camera_rays

        cams = ds.cameras
        if cams.has_lens:
            return self._lens_pixel_batch(ds, num_rays)
        N, H, W = len(ds), cams.height, cams.width
        dev = ds.images.device
        if dev.type == "cuda":  # one launch (fnr_pixel_batch) after the draw, instead of ~25 indexing / elementwise kernels
            from .. import ops

            # the default generator (seeded per rank by the trainer) is the one torch can advance inside a captured graph
            r = torch.rand((num_rays, 3), device=dev)
            o, d, cam, idx, image, mask = ops.pixel_batch(r, cams.camera_to_worlds, ds.images, ds.fruit_masks, cams.fx, cams.fy, cams.cx, cams.cy)
            pa = self.__dict__.setdefault("_pixel_area_cache", {})
            if (num_rays, str(dev)) not in pa:
                pa[(num_rays, str(dev))] = torch.full((num_rays, 1), 1.0 / (cams.fx * cams.fy), device=dev)
            bundle = RayBundle(origins=o, directions=d, pixel_area=pa[(num_rays, str(dev))], camera_indices=cam[:, None])
            return bundle, {"image": image, "fruit_mask": mask, "indices": idx}
        # CUDA: the default generator (seeded per rank by the trainer) -- the one torch can advance inside a captured graph
        r = torch.rand((num_rays, 3), device=dev, generator=None if dev.type == "cuda" else self._generator())
        extent = self.__dict__.setdefault("_extent_cache", {})
        key = (N, H, W, str(dev))
        if key not in extent:
            extent[key] = torch.tensor([N, H, W], dtype=torch.float32).to(dev)
        idx = torch.floor(r * extent[key]).long()
        ci, ys, xs = idx[:, 0], idx[:, 1], idx[:, 2]
        o, d = camera_rays(cams.camera_to_worlds[ci], cams.fx, cams.fy, cams.cx, cams.cy, ys, xs)
        bundle = RayBundle(origins=o.contiguous(), directions=d.contiguous(),
                           pixel_area=torch.full((num_rays, 1), 1.0 / (cams.fx * cams.fy), device=o.device), camera_indices=ci[:, None])
        batch = {"image": ds.images[ci, ys, xs], "fruit_mask": ds.fruit_masks[ci, ys, xs], "indices": idx}
        return bundle, batch

    def _lens_pixel_batch(self, ds, num_rays: int) -> Tuple[RayBundle, Dict]:
        """``_pixel_batch`` for lens cameras (per-image intrinsics, distortion, fisheye / equirectangular): the same draws, rays
        from ``fnr_pixel_batch_lens`` on the device or from data/camera_model.py on the host.  pixel_area is 1 / (fx fy) of
        each ray's camera."""
        cams = ds.cameras
        N, H, W = len(ds), cams.height, cams.width
        dev = ds.images.device
        fx, fy, cx, cy = cams.intrinsics()  # already [N] fp32 on the device after .to(device): no copy in the step
        area = self.__dict__.setdefault("_lens_area_cache", {})
        key = (id(ds), str(dev))
        if key not in area:
            area[key] = (ds, (1.0 / (fx.double() * fy.double())).float())  # ds held so that its id stays unique
        inv_area = area[key][1]
        if dev.type == "cuda":
            from .. import ops

            r = torch.rand((num_rays, 3), device=dev)
            o, d, cam, idx, image, mask = ops.pixel_batch_lens(r, cams.camera_to_worlds, ds.images, ds.fruit_masks, fx, fy, cx, cy,
                                                               cams.distortion_params, cams.camera_type)
            bundle = RayBundle(origins=o, directions=d, pixel_area=inv_area[cam.long()][:, None], camera_indices=cam[:, None])
            return bundle, {"image": image, "fruit_mask": mask, "indices": idx}
        from .camera_model import lens_rays

        r = torch.rand((num_rays, 3), device=dev, generator=self._generator())
        idx = torch.minimum(torch.floor(r * torch.tensor([N, H, W], dtype=torch.float32)).long(), torch.tensor([N - 1, H - 1, W - 1]))
        ci, ys, xs = idx[:, 0], idx[:, 1], idx[:, 2]
        dist = cams.distortion_params
        o, d = lens_rays(cams.camera_to_worlds[ci], fx[ci], fy[ci], cx[ci], cy[ci], None if dist is None else dist[ci], cams.camera_type, ys, xs)
        bundle = RayBundle(origins=o.contiguous(), directions=d.contiguous(), pixel_area=inv_area[ci][:, None], camera_indices=ci[:, None])
        return bundle, {"image": ds.images[ci, ys, xs], "fruit_mask": ds.fruit_masks[ci, ys, xs], "indices": idx}

    def next_train(self, step: int) -> Tuple[RayBundle, Dict]:
        self.train_count += 1
        return self._pixel_batch(self.train_dataset, self.config.train_num_rays_per_batch)

    def next_eval(self, step: int) -> Tuple[RayBundle, Dict]:
        self.eval_count += 1
        return self._pixel_batch(self.eval_dataset, self.config.eval_num_rays_per_batch)

    def next_eval_image(self, step: int) -> Tuple[int, RayBundle, Dict]:
        ds = self.eval_dataset
        i = self.eval_count % len(ds)
        self.eval_count += 1
        return i, ds.cameras.generate_rays(i), {"image": ds.images[i], "fruit_mask": ds.fruit_masks[i]}

    def setup_inference(self, aabb, num_points) -> int:
        """fruit_datamanager.py:157-172: ray grid for the uniform volume; returns the ray count."""
        corners = get_corners_of_aabb(aabb=aabb, device=self.device)
        surface_points, plane_vector = sample_surface_points(corners, n=num_points, device=self.device, noise=False)
        self.orthographic_ray_generator = OrthographicRayGenerator(
            surface_points=surface_points, plane_normal=plane_vector, ray_batch_size=self.config.eval_num_rays_per_batch,
            device=self.device, aabb=aabb)
        return surface_points.shape[0]

    def next_sample_volume(self, step: int) -> Tuple[RayBundle, Optional[Dict]]:
        """fruit_datamanager.py:199-204."""
        self.train_count += 1
        return self.orthographic_ray_generator(count=self.train_count), None

    def get_param_groups(self):
        return {}

    def get_training_callbacks(self, attrs):
        return []
