"""Procedural apple-tree scene (SURVEY.md section 8f rank 3; BASELINE.json configs[1]).

The reference's Zenodo data set and fruit templates are unavailable offline, so the training / PSNR /
fruit-count configuration runs on an analytic scene: a trunk, leaf blobs, red fruit spheres, a ground
plane and a sky, ray-traced exactly (no sampling noise) into RGB images plus the binary fruit masks
Grounded-SAM would provide.  The result has the structure the reference's dataparser produces
(fruit_nerf/data/fruitnerf_dataparser.py:73-292): camera-to-world poses in the OpenGL convention scaled
into the +/-1 box, shared pinhole intrinsics, ``scene_box`` = [-1,1]^3, ``metadata["semantics"]`` with the
classes ``['apple', 'stuff']``, a 90/10 train/eval split; ``write_dataset`` emits the on-disk layout
(``transforms.json`` with ``file_path`` / ``semantic_path`` frames + PNG images and masks,
fruit_nerf/data/fruit_dataset.py:31-57 reads masks as {0,255} -> {0,1}).
"""
from __future__ import annotations

import json
import math
import pathlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple, Union

import torch
from torch import Tensor

from ..compat import RayBundle, SceneBox, Semantics


def _normalize(v: Tensor) -> Tensor:
    return v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def look_at_c2w(eye: Tensor, target: Tensor, up=(0.0, 0.0, 1.0)) -> Tensor:
    """[3,4] camera-to-world, OpenGL axes (x right, y up, camera looks along -z)."""
    back = _normalize(eye - target)
    right = _normalize(torch.linalg.cross(torch.tensor(up, dtype=eye.dtype), back))
    upv = torch.linalg.cross(back, right)
    return torch.stack([right, upv, back, eye], dim=1)


def camera_rays(c2w: Tensor, fx: float, fy: float, cx: float, cy: float, ys: Tensor, xs: Tensor) -> Tuple[Tensor, Tensor]:
    """nerfstudio Cameras.generate_rays for a pinhole: pixel centres (+0.5), directions normalised.
    c2w [...,3,4] broadcast against integer pixel rows ``ys`` / columns ``xs``."""
    x = (xs.to(torch.float32) + 0.5 - cx) / fx
    y = -(ys.to(torch.float32) + 0.5 - cy) / fy
    d_cam = torch.stack([x, y, -torch.ones_like(x)], dim=-1)
    d = (c2w[..., :3, :3] * d_cam[..., None, :]).sum(-1)
    return c2w[..., :3, 3].expand_as(d), _normalize(d)


@dataclass
class SceneGeometry:
    fruit_centers: Tensor  # [K,3]
    fruit_radius: float
    leaf_centers: Tensor  # [M,3]
    leaf_radii: Tensor  # [M]
    trunk_radius: float = 0.035
    trunk_z: Tuple[float, float] = (-0.45, 0.02)
    ground_z: float = -0.45


def make_geometry(num_fruits: int = 12, seed: int = 0) -> SceneGeometry:
    g = torch.Generator().manual_seed(seed)
    centre = torch.tensor([0.0, 0.0, 0.08])
    # leaf blobs: a lumpy canopy of radius ~0.26
    M = 14
    lc = _normalize(torch.randn(M, 3, generator=g)) * (0.10 + 0.08 * torch.rand(M, 1, generator=g)) + centre
    lr = 0.10 + 0.05 * torch.rand(M, generator=g)
    # fruits on a shell just outside the canopy, rejection-sampled for a minimum spacing (distinct clusters)
    fr = 0.04
    centers: List[Tensor] = []
    tries = 0
    while len(centers) < num_fruits and tries < 10000:
        tries += 1
        dirv = _normalize(torch.randn(3, generator=g))
        if dirv[2] < -0.55:
            continue
        c = centre + dirv * (0.27 + 0.05 * float(torch.rand(1, generator=g)))
        if all(float((c - o).norm()) > 0.14 for o in centers):
            centers.append(c)
    return SceneGeometry(fruit_centers=torch.stack(centers), fruit_radius=fr, leaf_centers=lc, leaf_radii=lr)


def trace(geom: SceneGeometry, origins: Tensor, dirs: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """Exact first-hit shading.  origins/dirs [N,3] -> rgb [N,3], fruit mask [N,1], hit distance [N]."""
    N = origins.shape[0]
    dev = origins.device
    centers = torch.cat([geom.fruit_centers, geom.leaf_centers]).to(dev)
    radii = torch.cat([torch.full((geom.fruit_centers.shape[0],), geom.fruit_radius), geom.leaf_radii]).to(dev)
    K = geom.fruit_centers.shape[0]
    inf = torch.tensor(float("inf"), device=dev)
    # spheres
    oc = origins[:, None, :] - centers[None]
    b = (oc * dirs[:, None, :]).sum(-1)
    c = (oc * oc).sum(-1) - radii[None] ** 2
    disc = b * b - c
    t_s = torch.where((disc > 0) & (-b - disc.clamp_min(0).sqrt() > 1e-4), -b - disc.clamp_min(0).sqrt(), inf)
    t_sphere, idx = t_s.min(dim=1)
    # trunk: finite z-aligned cylinder
    ox, oy, dx, dy = origins[:, 0], origins[:, 1], dirs[:, 0], dirs[:, 1]
    a2 = dx * dx + dy * dy
    b2 = ox * dx + oy * dy
    c2 = ox * ox + oy * oy - geom.trunk_radius ** 2
    disc2 = b2 * b2 - a2 * c2
    t_c = (-b2 - disc2.clamp_min(0).sqrt()) / a2.clamp_min(1e-12)
    zc = origins[:, 2] + t_c * dirs[:, 2]
    t_c = torch.where((disc2 > 0) & (t_c > 1e-4) & (zc > geom.trunk_z[0]) & (zc < geom.trunk_z[1]), t_c, inf)
    # ground plane
    t_g = (geom.ground_z - origins[:, 2]) / torch.where(dirs[:, 2].abs() < 1e-9, torch.full_like(dirs[:, 2], -1e-9), dirs[:, 2])
    t_g = torch.where((t_g > 1e-4) & (dirs[:, 2] < 0), t_g, inf)
    t_all = torch.stack([t_sphere, t_c, t_g], dim=1)
    t_hit, kind = t_all.min(dim=1)
    hit = torch.isfinite(t_hit)
    p = origins + dirs * torch.where(hit, t_hit, torch.zeros_like(t_hit))[:, None]
    light = _normalize(torch.tensor([0.4, 0.3, 0.85], device=dev))
    # normals and albedo per kind
    n_s = _normalize(p - centers[idx])
    is_fruit = (kind == 0) & (idx < K) & hit
    alb_s = torch.where((idx < K)[:, None], torch.tensor([0.85, 0.10, 0.08], device=dev),
                        torch.tensor([0.13, 0.45, 0.12], device=dev) * (0.8 + 0.4 * ((idx % 5).to(torch.float32) / 4)[:, None]))
    n_c = _normalize(torch.stack([p[:, 0], p[:, 1], torch.zeros_like(p[:, 0])], dim=-1))
    alb_c = torch.tensor([0.36, 0.23, 0.12], device=dev).expand(N, 3)
    n_g = torch.tensor([0.0, 0.0, 1.0], device=dev).expand(N, 3)
    checker = ((torch.floor(p[:, 0] * 4) + torch.floor(p[:, 1] * 4)) % 2)[:, None]
    alb_g = torch.tensor([0.42, 0.36, 0.27], device=dev) * (0.85 + 0.15 * checker)
    n = torch.where((kind == 0)[:, None], n_s, torch.where((kind == 1)[:, None], n_c, n_g))
    alb = torch.where((kind == 0)[:, None], alb_s, torch.where((kind == 1)[:, None], alb_c, alb_g))
    shade = 0.35 + 0.65 * (n * light).sum(-1).clamp_min(0.0)
    sky = torch.tensor([0.55, 0.70, 0.92], device=dev) * (0.75 + 0.25 * dirs[:, 2:3].clamp(0, 1)) + 0.08 * (1 - dirs[:, 2:3].clamp(0, 1))
    rgb = torch.where(hit[:, None], alb * shade[:, None], sky).clamp(0, 1)
    return rgb, is_fruit.to(torch.float32)[:, None], t_hit


@dataclass
class SyntheticCameras:
    """Cameras of a data set.  ``fx`` / ``fy`` / ``cx`` / ``cy`` are python floats shared by every image (the pinhole the
    synthetic scene and most captures use) or per-image [N] tensors; ``camera_type`` and ``distortion_params`` ([N,6] =
    k1 k2 k3 k4 p1 p2, or None) describe the lens (data/camera_model.py)."""

    camera_to_worlds: Tensor  # [N,3,4]
    fx: Union[float, Tensor]
    fy: Union[float, Tensor]
    cx: Union[float, Tensor]
    cy: Union[float, Tensor]
    height: int
    width: int
    camera_type: str = "perspective"
    distortion_params: Optional[Tensor] = None

    def __len__(self):
        return int(self.camera_to_worlds.shape[0])

    @property
    def has_lens(self) -> bool:
        """Anything but one shared distortion-free pinhole: these rays come from the lens kernels / camera_model."""
        return self.camera_type != "perspective" or self.distortion_params is not None or any(
            torch.is_tensor(v) for v in (self.fx, self.fy, self.cx, self.cy))

    def intrinsics(self) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """Per-image fx, fy, cx, cy [N] in fp32 on the cameras' device."""
        N, dev = len(self), self.camera_to_worlds.device
        return tuple(torch.as_tensor(v, dtype=torch.float32, device=dev).reshape(-1).expand(N).contiguous()
                     for v in (self.fx, self.fy, self.cx, self.cy))

    def subset(self, index) -> "SyntheticCameras":
        pick = lambda v: v[index] if torch.is_tensor(v) else v  # noqa: E731
        return SyntheticCameras(self.camera_to_worlds[index], pick(self.fx), pick(self.fy), pick(self.cx), pick(self.cy), self.height, self.width,
                                self.camera_type, pick(self.distortion_params))

    def to(self, device):
        if not self.has_lens:
            return SyntheticCameras(self.camera_to_worlds.to(device), self.fx, self.fy, self.cx, self.cy, self.height, self.width)
        # lens cameras keep per-image fp32 arrays on the device for the ray kernels; their values are checked here, once,
        # because the training step (captured in a CUDA graph) must not read device memory back
        from .camera_model import TYPE_TO_CAMERA_MODEL

        N = len(self)
        if self.camera_type not in TYPE_TO_CAMERA_MODEL:
            raise ValueError(f"camera_type must be one of {sorted(TYPE_TO_CAMERA_MODEL)}, got {self.camera_type!r}")
        fx, fy, cx, cy = (t.to(device) for t in self.intrinsics())
        dist = self.distortion_params
        if dist is not None:
            dist = dist.to(device=device, dtype=torch.float32).contiguous()
            if tuple(dist.shape) != (N, 6):
                raise ValueError(f"distortion_params must be [{N},6], got {tuple(dist.shape)}")
        checked = torch.stack([fx, fy, cx, cy], 1) if dist is None else torch.cat([torch.stack([fx, fy, cx, cy], 1), dist], 1)
        if not bool(torch.isfinite(checked).all()) or not bool(((fx != 0) & (fy != 0)).all()):
            raise ValueError("camera intrinsics and distortion must be finite, with non-zero focal lengths")
        return SyntheticCameras(self.camera_to_worlds.to(device), fx, fy, cx, cy, self.height, self.width, self.camera_type, dist)

    def generate_rays(self, camera_index: int) -> RayBundle:
        """Full-image bundle [H,W] for evaluation (nerfstudio Cameras.generate_rays(camera_indices=i))."""
        dev = self.camera_to_worlds.device
        H, W = self.height, self.width
        if self.has_lens:
            fx, fy, cx, cy = self.intrinsics()
            dist = self.distortion_params
            if dev.type == "cuda":
                from .. import ops

                o, d = ops.camera_rays_lens(self.camera_to_worlds, fx, fy, cx, cy, dist, self.camera_type, H, W, camera_index, 0, H * W)
            else:
                from .camera_model import lens_rays

                ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
                i = camera_index
                o, d = lens_rays(self.camera_to_worlds[i], fx[i], fy[i], cx[i], cy[i], None if dist is None else dist[i], self.camera_type,
                                 ys.reshape(-1), xs.reshape(-1))
            area = 1.0 / (float(fx[camera_index]) * float(fy[camera_index]))
        else:
            ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
            o, d = camera_rays(self.camera_to_worlds[camera_index], self.fx, self.fy, self.cx, self.cy, ys.reshape(-1), xs.reshape(-1))
            area = 1.0 / (self.fx * self.fy)
        return RayBundle(origins=o.reshape(H, W, 3).contiguous(), directions=d.reshape(H, W, 3).contiguous(),
                         pixel_area=torch.full((H, W, 1), area, device=dev),
                         camera_indices=torch.full((H, W, 1), camera_index, dtype=torch.int64, device=dev))


@dataclass
class SyntheticFruitDataset:
    """What FruitDataset (fruit_nerf/data/fruit_dataset.py:59-89) exposes to the pipeline, held in memory:
    images, ``fruit_mask`` per pixel, cameras, ``scene_box``, ``metadata['semantics']``."""

    images: Tensor  # [N,H,W,3] float32 in [0,1]
    fruit_masks: Tensor  # [N,H,W,1] float32 {0,1}
    cameras: SyntheticCameras
    scene_box: SceneBox
    metadata: Dict = field(default_factory=dict)
    geometry: Optional[SceneGeometry] = None
    dataparser_scale: float = 1.0

    def __len__(self):
        return int(self.images.shape[0])

    def to(self, device):
        return SyntheticFruitDataset(self.images.to(device), self.fruit_masks.to(device), self.cameras.to(device), self.scene_box, self.metadata,
                                     self.geometry, self.dataparser_scale)


def make_apple_scene(num_images: int = 40, height: int = 160, width: int = 160, num_fruits: int = 12, seed: int = 0, radius: float = 1.0,
                     elevations=(12.0, 30.0, 50.0), noise_std: float = 0.02, device="cpu", camera_type: str = "perspective",
                     distortion: Optional[Tensor] = None, intrinsics_jitter: float = 0.0) -> Tuple[SyntheticFruitDataset, SyntheticFruitDataset]:
    """(train, eval) data sets of the synthetic apple tree.  Cameras orbit at ``radius`` (inside the +/-1 box after the
    dataparser's auto-scaling) on three elevation rings; every 10th image goes to the eval split (train_split_fraction 0.9).

    A lens: ``camera_type`` ("perspective", "fisheye", "equirectangular"), ``distortion`` (k1 k2 k3 k4 p1 p2, shared [6]
    or per image [N,6]) and ``intrinsics_jitter`` (each image's fx / fy / cx / cy scaled by 1 + jitter * U(-1, 1), seeded)
    make lens cameras whose images are traced along the rays of data/camera_model.py.  The defaults give the shared
    pinhole and the same scene bit for bit."""
    geom = make_geometry(num_fruits, seed)
    target = torch.tensor([0.0, 0.0, 0.02])
    poses = []
    for i in range(num_images):
        az = 2 * math.pi * i / num_images + 0.37 * (i % 3)
        el = math.radians(elevations[i % len(elevations)])
        eye = target + radius * torch.tensor([math.cos(az) * math.cos(el), math.sin(az) * math.cos(el), math.sin(el)])
        poses.append(look_at_c2w(eye, target))
    c2w = torch.stack(poses).to(torch.float32)
    fx = fy = 1.1 * width
    cams = SyntheticCameras(c2w.to(device), fx, fy, width / 2.0, height / 2.0, height, width)
    if camera_type != "perspective" or distortion is not None or intrinsics_jitter:
        intr = torch.tensor([fx, fy, width / 2.0, height / 2.0], dtype=torch.float32).expand(num_images, 4)
        if intrinsics_jitter:
            gj = torch.Generator().manual_seed(seed + 777)
            intr = intr * (1.0 + intrinsics_jitter * (2.0 * torch.rand(num_images, 4, generator=gj) - 1.0))
        dist = None if distortion is None else torch.as_tensor(distortion, dtype=torch.float32).reshape(-1, 6).expand(num_images, 6).contiguous()
        cams = SyntheticCameras(c2w.to(device), *(intr[:, k].contiguous().to(device) for k in range(4)), height, width, camera_type,
                                None if dist is None else dist.to(device))
    imgs, masks = [], []
    for i in range(num_images):
        rb = cams.generate_rays(i)
        rgb, m, _ = trace(geom, rb.origins.reshape(-1, 3), rb.directions.reshape(-1, 3))
        imgs.append(rgb.reshape(height, width, 3))
        masks.append(m.reshape(height, width, 1))
    images, fruit_masks = torch.stack(imgs), torch.stack(masks)
    if noise_std > 0:
        # sensor noise: photographs never let the photometric loss reach zero; a noise-free render does, and Adam with
        # eps = 1e-15 at a constant 1e-2 learning rate then amplifies round-off-level gradients (see DESIGN.md section 7)
        gn = torch.Generator().manual_seed(seed + 12345)
        images = (images + noise_std * torch.randn(images.shape, generator=gn).to(images.device)).clamp(0.0, 1.0)
    scene_box = SceneBox(aabb=torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]], dtype=torch.float32))
    idx = torch.arange(num_images)
    eval_idx = idx[idx % 10 == 9]
    train_idx = idx[idx % 10 != 9]

    def subset(ix):
        sem = Semantics(filenames=[f"semantics/frame_{int(i):05d}.png" for i in ix], classes=["apple", "stuff"],
                        colors=torch.tensor([[255, 0, 0], [0, 0, 0]], dtype=torch.float32) / 255.0, mask_classes=["apple", "stuff"])
        cam_ix = cams.subset(ix.to(cams.camera_to_worlds.device)) if cams.has_lens else SyntheticCameras(
            cams.camera_to_worlds[ix], fx, fy, cams.cx, cams.cy, height, width)
        return SyntheticFruitDataset(images[ix], fruit_masks[ix], cam_ix, scene_box, {"semantics": sem}, geom, 1.0)

    return subset(train_idx), subset(eval_idx)


def write_dataset(ds: SyntheticFruitDataset, out_dir) -> pathlib.Path:
    """Emit the folder the reference's dataparser reads: images/, semantics/, transforms.json."""
    import numpy as np
    from PIL import Image

    out = pathlib.Path(out_dir)
    (out / "images").mkdir(parents=True, exist_ok=True)
    (out / "semantics").mkdir(parents=True, exist_ok=True)
    frames = []
    for i in range(len(ds)):
        Image.fromarray((ds.images[i].cpu().numpy() * 255 + 0.5).astype(np.uint8)).save(out / "images" / f"frame_{i:05d}.png")
        Image.fromarray((ds.fruit_masks[i, ..., 0].cpu().numpy() * 255).astype(np.uint8)).save(out / "semantics" / f"frame_{i:05d}.png")
        m = torch.eye(4)
        m[:3, :4] = ds.cameras.camera_to_worlds[i].cpu()
        frames.append({"file_path": f"images/frame_{i:05d}.png", "semantic_path": f"semantics/frame_{i:05d}.png",
                       "transform_matrix": m.tolist()})
    cams = ds.cameras
    if cams.has_lens:
        # per-frame intrinsics and distortion, and the camera model, so that the lens survives the round trip
        from .camera_model import TYPE_TO_CAMERA_MODEL

        fxs, fys, cxs, cys = (t.cpu().tolist() for t in cams.intrinsics())
        dist = None if cams.distortion_params is None else cams.distortion_params.cpu().tolist()
        for i, f in enumerate(frames):
            f.update({"fl_x": fxs[i], "fl_y": fys[i], "cx": cxs[i], "cy": cys[i]})
            if dist is not None:
                f.update(dict(zip(("k1", "k2", "k3", "k4", "p1", "p2"), dist[i])))
        meta = {"w": cams.width, "h": cams.height, "camera_model": TYPE_TO_CAMERA_MODEL[cams.camera_type], "frames": frames}
    else:
        meta = {"fl_x": cams.fx, "fl_y": cams.fy, "cx": cams.cx, "cy": cams.cy, "w": cams.width,
                "h": cams.height, "camera_model": "OPENCV", "k1": 0.0, "k2": 0.0, "p1": 0.0, "p2": 0.0, "frames": frames}
    (out / "transforms.json").write_text(json.dumps(meta, indent=1))
    return out / "transforms.json"
