"""Dataparser of the plugin surface: reads a FruitNeRF / nerfstudio data folder from disk
(fruit_nerf/data/fruitnerf_dataparser.py:44-326 + the mask reader of fruit_nerf/data/fruit_dataset.py:31-57).

``transforms.json`` (shared or per-frame intrinsics, ``file_path`` / ``semantic_path`` frames, optional
``{split}_filenames``, ``orientation_override``, ``applied_transform`` / ``applied_scale``) -> the pose pipeline of
the reference (auto-orient "up" + centre on the mean camera position + auto-scale into the +/-1 box, equally spaced
train split with the remaining frames for eval) -> an in-memory data set (images, binary fruit masks, cameras,
``scene_box``, ``metadata['semantics']``) that ``FruitDataManager`` keeps resident on the GPU.  Image decoding is host
I/O done once at start-up; nothing here is on the per-iteration path.

By default the parser keeps to ONE shared pinhole camera model (``fnr_pixel_batch``): per-frame intrinsics and non-zero
distortion coefficients are rejected with a clear error instead of being silently ignored.  With ``lens_distortion=True``
it reads what the reference passes to nerfstudio's ``Cameras`` (fruitnerf_dataparser.py:86-137, 225-246): shared or
per-frame intrinsics and distortion and the ``camera_model``, which ``fnr_pixel_batch_lens`` / ``fnr_camera_rays_lens``
model on the device (DESIGN.md section 4.3j).
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Literal, Optional, Tuple, Type

import numpy as np
import torch
from torch import Tensor

from ..compat import InstantiateConfig, SceneBox, Semantics
from .camera_model import CAMERA_MODEL_TO_TYPE, get_distortion_params
from .synthetic_scene import SyntheticCameras, SyntheticFruitDataset

MAX_AUTO_RESOLUTION = 1200  # fruitnerf_dataparser.py:39


@dataclass
class FruitNerfDataParserConfig(InstantiateConfig):
    """fruitnerf_dataparser.py:42-63 (same fields and defaults)."""

    _target: Type = field(default_factory=lambda: FruitNerf)
    data: Path = Path()
    scale_factor: float = 1.0
    downscale_factor: Optional[int] = None
    scene_scale: float = 1.0
    orientation_method: Literal["pca", "up", "vertical", "none"] = "up"
    center_method: Literal["poses", "focus", "none"] = "poses"
    auto_scale_poses: bool = True
    train_split_fraction: float = 0.9
    lens_distortion: bool = False
    """Read ``camera_model``, per-frame intrinsics and distortion coefficients (captured data sets).  Off: one shared
    distortion-free pinhole, anything else refused, ``camera_model`` ignored."""


@dataclass
class DataparserOutputs:
    """The subset of nerfstudio's DataparserOutputs the plugin uses, plus the decoded pixels."""

    image_filenames: List[Path]
    cameras: SyntheticCameras
    scene_box: SceneBox
    dataparser_scale: float
    dataparser_transform: Tensor  # [3,4]
    metadata: Dict
    images: Tensor        # [N,H,W,3] float32
    fruit_masks: Tensor   # [N,H,W,1] float32 {0,1}

    def as_dataset(self) -> SyntheticFruitDataset:
        return SyntheticFruitDataset(self.images, self.fruit_masks, self.cameras, self.scene_box, self.metadata, None, self.dataparser_scale)

    def save_dataparser_transform(self, path) -> None:
        """nerfstudio DataparserOutputs.save_dataparser_transform: what the exporter reads back as ``transform_json``
        (fruit_nerf/scripts/exporter.py:97-99)."""
        Path(path).parent.mkdir(parents=True, exist_ok=True)
        Path(path).write_text(json.dumps({"transform": self.dataparser_transform.tolist(), "scale": float(self.dataparser_scale)}, indent=4))


# ---- nerfstudio camera_utils (0.3.2), restated ----------------------------------------------------------------------
def rotation_matrix(a: Tensor, b: Tensor) -> Tensor:
    """Rotation taking direction ``a`` onto ``b`` (Rodrigues form used by camera_utils.rotation_matrix)."""
    a = a / torch.linalg.norm(a)
    b = b / torch.linalg.norm(b)
    v = torch.linalg.cross(a, b)
    c = torch.dot(a, b)
    if c < -1 + 1e-8:  # opposite vectors: perturb one of them (the reference adds random noise; a fixed nudge is reproducible)
        return rotation_matrix(a + torch.tensor([1e-3, -2e-3, 1.5e-3], dtype=a.dtype), b)
    s = torch.linalg.norm(v)
    k = torch.tensor([[0.0, -float(v[2]), float(v[1])], [float(v[2]), 0.0, -float(v[0])], [-float(v[1]), float(v[0]), 0.0]], dtype=a.dtype)
    return torch.eye(3, dtype=a.dtype) + k + k @ k * ((1 - c) / (s ** 2 + 1e-8))


def focus_of_attention(poses: Tensor, initial_focus: Tensor) -> Tensor:
    """Point closest to the optical axes of the cameras looking at it (camera_utils.focus_of_attention)."""
    active_directions = -poses[:, :3, 2:3]
    active_origins = poses[:, :3, 3:4]
    focus_pt = initial_focus
    active = torch.sum(active_directions.squeeze(-1) * (focus_pt - active_origins.squeeze(-1)), dim=-1) > 0
    done = False
    while torch.sum(active.int()) > 1 and not done:
        active_directions = active_directions[active]
        active_origins = active_origins[active]
        m = torch.eye(3) - active_directions * torch.transpose(active_directions, -2, -1)
        mt_m = torch.transpose(m, -2, -1) @ m
        focus_pt = torch.linalg.inv(mt_m.mean(0)) @ (mt_m @ active_origins).mean(0)[:, 0]
        active = torch.sum(active_directions.squeeze(-1) * (focus_pt - active_origins.squeeze(-1)), dim=-1) > 0
        done = bool(active.all())
    return focus_pt


def auto_orient_and_center_poses(poses: Tensor, method: str = "up", center_method: str = "poses") -> Tuple[Tensor, Tensor]:
    """camera_utils.auto_orient_and_center_poses: [N,4,4] c2w -> ([N,3,4] oriented poses, [3,4] transform)."""
    origins = poses[..., :3, 3]
    mean_origin = torch.mean(origins, dim=0)
    translation_diff = origins - mean_origin
    if center_method == "poses":
        translation = mean_origin
    elif center_method == "focus":
        translation = focus_of_attention(poses, mean_origin)
    elif center_method == "none":
        translation = torch.zeros_like(mean_origin)
    else:
        raise ValueError(f"Unknown value for center_method: {center_method}")
    if method == "pca":
        _, eigvec = torch.linalg.eigh(translation_diff.T @ translation_diff)
        eigvec = torch.flip(eigvec, dims=(-1,))
        if torch.linalg.det(eigvec) < 0:
            eigvec[:, 2] = -eigvec[:, 2]
        transform = torch.cat([eigvec, eigvec @ -translation[..., None]], dim=-1)
        oriented = transform @ poses
        if oriented.mean(dim=0)[2, 1] < 0:
            oriented[:, 1:3] = -1 * oriented[:, 1:3]
    elif method == "up":
        up = torch.mean(poses[:, :3, 1], dim=0)
        up = up / torch.linalg.norm(up)
        rotation = rotation_matrix(up, torch.tensor([0.0, 0.0, 1.0], dtype=poses.dtype))
        transform = torch.cat([rotation, rotation @ -translation[..., None]], dim=-1)
        oriented = transform @ poses
    elif method == "none":
        transform = torch.eye(4, dtype=poses.dtype)
        transform[:3, 3] = -translation
        transform = transform[:3, :]
        oriented = transform @ poses
    else:
        raise NotImplementedError(f"orientation_method={method!r} is not restated (the reference default is 'up')")
    return oriented, transform


# ---- pixel readers ----------------------------------------------------------------------------------------------------
def read_image(path: Path) -> Tensor:
    """nerfstudio InputDataset.get_image: uint8 -> float32 / 255; an alpha channel is dropped (alpha_color unset)."""
    from PIL import Image

    arr = np.array(Image.open(path), dtype="uint8")
    if arr.ndim == 2:
        arr = arr[:, :, None].repeat(3, axis=2)
    return torch.from_numpy(arr[:, :, :3].astype("float32") / 255.0)


def read_fruit_mask(path: Path) -> Tensor:
    """fruit_dataset.py:31-57: {0,255} masks -> {0,1}; JPEG masks are thresholded at 125 first.  Returns [H,W,1] float32."""
    from PIL import Image

    sem = torch.from_numpy(np.array(Image.open(path), dtype="int64"))
    if sem.dim() == 3:
        sem = sem[..., 0]
    sem = sem[..., None]
    if "jpg" in str(path).lower():
        sem = torch.where(sem <= 125, torch.zeros_like(sem), torch.full_like(sem, 255))
        sem = sem / 255
    elif sem.max() > 1.0:
        sem = sem / 255
    else:
        raise ValueError("Please look at mask file manually! How to normalize")  # the reference's message
    return sem.to(torch.float32)


@dataclass
class FruitNerf:
    """fruitnerf_dataparser.py:66-326."""

    config: FruitNerfDataParserConfig
    downscale_factor: Optional[int] = None

    def get_dataparser_outputs(self, split: str = "train") -> DataparserOutputs:
        return self._generate_dataparser_outputs(split)

    def _generate_dataparser_outputs(self, split: str = "train") -> DataparserOutputs:
        data = Path(self.config.data)
        assert data.exists(), f"Data directory {data} does not exist."
        if data.suffix == ".json":
            meta = json.loads(data.read_text())
            data_dir = data.parent
        else:
            meta = json.loads((data / "transforms.json").read_text())
            data_dir = data

        shared = {k: (k in meta) for k in ("fl_x", "fl_y", "cx", "cy", "h", "w")}
        image_filenames, semantic_filenames, poses, per_frame = [], [], [], []
        for frame in meta["frames"]:
            filepath = Path(frame["file_path"])
            image_filenames.append(self._get_fname(Path(filepath.as_posix().replace("\\", "/")), data_dir))
            intr = {}
            for k, present in shared.items():
                if not present:
                    assert k in frame, f"{k} not specified in frame"
                    intr[k] = float(frame[k])
            per_frame.append(intr)
            poses.append(np.array(frame["transform_matrix"]))
            if "semantic_path" in frame:
                sp = Path(Path(frame["semantic_path"]).as_posix().replace("\\", "/"))
                semantic_filenames.append(self._get_fname(sp, data_dir, downsample_folder_prefix="semantics_"))
        assert len(semantic_filenames) == 0 or len(semantic_filenames) == len(image_filenames), (
            "Different number of image and semantic filenames. "
            "You should check that mask_path is specified for every frame (or zero frames) in transforms.json.")
        lens = self.config.lens_distortion
        if not lens:
            for k in ("k1", "k2", "k3", "k4", "p1", "p2"):
                vals = [float(meta[k])] if k in meta else [float(f[k]) for f in meta["frames"] if k in f]
                if any(v != 0.0 for v in vals):
                    raise NotImplementedError(f"non-zero distortion coefficient {k}: the device ray generator is a pinhole model")

        # ---- split (fruitnerf_dataparser.py:155-187)
        has_split_files_spec = any(f"{s}_filenames" in meta for s in ("train", "val", "test"))
        if f"{split}_filenames" in meta:
            split_filenames = set(self._get_fname(Path(x), data_dir) for x in meta[f"{split}_filenames"])
            unmatched = split_filenames.difference(image_filenames)
            if unmatched:
                raise RuntimeError(f"Some filenames for split {split} were not found: {unmatched}.")
            indices = np.array([i for i, p in enumerate(image_filenames) if p in split_filenames], dtype=np.int32)
        elif has_split_files_spec:
            raise RuntimeError(f"The dataset's list of filenames for split {split} is missing.")
        else:
            num_images = len(image_filenames)
            num_train = math.ceil(num_images * self.config.train_split_fraction)
            i_all = np.arange(num_images)
            i_train = np.linspace(0, num_images - 1, num_train, dtype=int)  # equally spaced, first and last image included
            i_eval = np.setdiff1d(i_all, i_train)
            assert len(i_eval) == num_images - num_train
            if split == "train":
                indices = i_train
            elif split in ("val", "test"):
                indices = i_eval
            else:
                raise ValueError(f"Unknown dataparser split {split}")

        # ---- poses: orient, centre, scale BEFORE the split is applied (fruitnerf_dataparser.py:189-213)
        orientation = meta.get("orientation_override", self.config.orientation_method)
        poses_t = torch.from_numpy(np.array(poses).astype(np.float32))
        poses_t, transform = auto_orient_and_center_poses(poses_t, method=orientation, center_method=self.config.center_method)
        scale = 1.0
        if self.config.auto_scale_poses:
            scale /= float(torch.max(torch.abs(poses_t[:, :3, 3])))
        scale *= self.config.scale_factor
        poses_t[:, :3, 3] *= scale
        idx = torch.tensor(indices, dtype=torch.long)
        poses_t = poses_t[idx]
        image_filenames = [image_filenames[i] for i in indices]
        semantic_filenames = [semantic_filenames[i] for i in indices] if semantic_filenames else []

        s = self.config.scene_scale
        scene_box = SceneBox(aabb=torch.tensor([[-s, -s, -s], [s, s, s]], dtype=torch.float32))

        def intrinsic(k):
            if shared[k]:
                return float(meta[k])
            vals = {per_frame[i][k] for i in indices}
            if len(vals) != 1:
                if k in ("h", "w") and lens:
                    raise NotImplementedError(f"per-frame image sizes ({k} differs between frames): the pixel sampler draws from one [N,H,W] image stack")
                raise NotImplementedError(f"per-frame intrinsics ({k} differs between frames): the device ray generator takes one shared pinhole camera")
            return vals.pop()

        assert self.downscale_factor is not None
        r = 1.0 / self.downscale_factor  # Cameras.rescale_output_resolution
        height, width = int(intrinsic("h") * r), int(intrinsic("w") * r)
        if lens:
            # fruitnerf_dataparser.py:225-246: shared values as python floats, per-frame ones as fp32 tensors of the split
            idx_np = np.asarray(indices, dtype=np.int64)
            fx, fy, cx, cy = (float(meta[k]) * r if shared[k] else torch.tensor([f[k] for f in per_frame], dtype=torch.float32)[idx_np] * r
                              for k in ("fl_x", "fl_y", "cx", "cy"))
            camera_type, distortion = _lens_model(meta, idx_np)
        else:
            fx, fy, cx, cy = (intrinsic(k) * r for k in ("fl_x", "fl_y", "cx", "cy"))
            camera_type, distortion = "perspective", None

        metadata = {}
        if semantic_filenames:
            classes = ["apple", "stuff"]  # fruitnerf_dataparser.py:254-261
            colors = torch.zeros(len(classes))
            colors[1] = 255
            colors /= 255.0
            metadata["semantics"] = Semantics(filenames=semantic_filenames, classes=classes, colors=colors, mask_classes=classes)

        if "applied_transform" in meta:
            applied = torch.tensor(meta["applied_transform"], dtype=transform.dtype)
            transform = transform @ torch.cat([applied, torch.tensor([[0, 0, 0, 1]], dtype=transform.dtype)], 0)
        if "applied_scale" in meta:
            scale *= float(meta["applied_scale"])

        images = torch.stack([read_image(p) for p in image_filenames]) if image_filenames else torch.zeros(0, height, width, 3)
        if images.shape[1:3] != (height, width):
            raise ValueError(f"image size {tuple(images.shape[1:3])} does not match the camera model ({height}, {width})")
        if semantic_filenames:
            masks = torch.stack([read_fruit_mask(p) for p in semantic_filenames])
        else:
            masks = torch.zeros(images.shape[0], height, width, 1)
        cams = SyntheticCameras(poses_t[:, :3, :4].contiguous(), fx, fy, cx, cy, height, width, camera_type, distortion)
        return DataparserOutputs(image_filenames=image_filenames, cameras=cams, scene_box=scene_box, dataparser_scale=scale,
                                 dataparser_transform=transform, metadata=metadata, images=images, fruit_masks=masks)

    def _get_fname(self, filepath: Path, data_dir: Path, downsample_folder_prefix: str = "images_") -> Path:
        """fruitnerf_dataparser.py:294-326: resolve the (optionally pre-downscaled) file of a frame."""
        filepath = Path(filepath)
        if self.downscale_factor is None:
            if self.config.downscale_factor is None:
                from PIL import Image

                test_img = Image.open(data_dir / filepath)
                h, w = test_img.size
                max_res = max(h, w)
                df = 0
                while True:
                    if (max_res / 2 ** df) < MAX_AUTO_RESOLUTION:
                        break
                    if not (data_dir / f"{downsample_folder_prefix}{2 ** (df + 1)}" / filepath.name).exists():
                        break
                    df += 1
                self.downscale_factor = 2 ** df
            else:
                self.downscale_factor = self.config.downscale_factor
        if self.downscale_factor > 1:
            return data_dir / f"{downsample_folder_prefix}{self.downscale_factor}" / filepath.name
        return data_dir / filepath


def _lens_model(meta: Dict, indices: np.ndarray) -> Tuple[str, Optional[Tensor]]:
    """camera_type and the [N,6] distortion of the split ``indices`` (None when every coefficient is zero: the undistortion
    is then the identity).  fruitnerf_dataparser.py:92-137, 236-246, including its test for shared coefficients: only
    k1, k2, k3, p1, p2 at the top level make them shared (k4 alone does not), and then all six are read from the top."""
    model = meta.get("camera_model", "OPENCV")
    if model not in CAMERA_MODEL_TO_TYPE:
        if model.startswith(("OMNIDIRECTIONALSTEREO", "VR180")):
            raise NotImplementedError(f"camera_model {model!r}: stereo cameras are not supported")
        raise ValueError(f"unknown camera_model {model!r} (known: {sorted(CAMERA_MODEL_TO_TYPE)})")
    camera_type = CAMERA_MODEL_TO_TYPE[model]
    keys = ("k1", "k2", "k3", "k4", "p1", "p2")
    if any(k in meta for k in ("k1", "k2", "k3", "p1", "p2")):
        dist = get_distortion_params(**{k: float(meta[k]) if k in meta else 0.0 for k in keys}).expand(len(indices), 6).contiguous()
    else:
        dist = torch.stack([get_distortion_params(**{k: float(f[k]) if k in f else 0.0 for k in keys}) for f in meta["frames"]])[indices]
    if len(indices) == 0 or not bool((dist != 0).any()):
        return camera_type, None
    if not bool(torch.isfinite(dist).all()):
        raise ValueError("distortion coefficients must be finite")
    return camera_type, dist


def load_fruit_datasets(config: FruitNerfDataParserConfig) -> Tuple[SyntheticFruitDataset, SyntheticFruitDataset, DataparserOutputs]:
    """(train, eval) in-memory data sets of a data folder + the train-split outputs (transform / scale for the exporter)."""
    parser = config.setup() if hasattr(config, "setup") else FruitNerf(config)
    train = parser.get_dataparser_outputs("train")
    ev = parser.get_dataparser_outputs("val")
    if "semantics" not in train.metadata:
        raise AssertionError("No semantic instance could be found! Is a semantic folder included in the input folder and transform.json file?")
    return train.as_dataset(), ev.as_dataset(), train
