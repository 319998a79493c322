"""``ns-export-semantics semantic-pointcloud`` (fruit_nerf/scripts/exporter.py:54-144).

Same dataclass fields and defaults as the reference.  ``main`` either takes an already-built pipeline or builds one
from ``load_config`` with ``eval_setup`` below -- the counterpart of nerfstudio's ``eval_setup`` for the run folders
``fruitnerf_b200.trainer.Trainer`` writes (``config.yml`` + ``nerfstudio_models/step-*.ckpt`` +
``dataparser_transforms.json``).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from dataclasses import dataclass
from pathlib import Path
from typing import Optional, Tuple

import torch

from ..export.exporter_utils import (export_poisson_mesh, export_textured_meshes, export_tsdf_mesh, generate_point_cloud, sample_volume,
                                     write_ply)


def eval_setup(config_path, eval_num_rays_per_chunk: Optional[int] = None, test_mode: str = "test", device: Optional[str] = None):
    """nerfstudio.utils.eval_utils.eval_setup for this package's run folders: load ``config.yml`` (the pickled-by-yaml
    TrainerSpec, as nerfstudio does with its TrainerConfig), build the pipeline in ``test_mode``, load the newest
    ``step-*.ckpt`` under ``<run>/nerfstudio_models`` and put the pipeline in eval mode.
    Returns (config, pipeline, checkpoint_path, step); ``config.load_dir`` is set like upstream (exporter.py:111)."""
    import yaml

    config_path = Path(config_path)
    config = yaml.load(config_path.read_text(), Loader=yaml.Loader)
    if eval_num_rays_per_chunk:
        config.pipeline.model.eval_num_rays_per_chunk = eval_num_rays_per_chunk
    config.load_dir = config_path.parent / "nerfstudio_models"
    dev = torch.device(device or ("cuda:0" if torch.cuda.is_available() else "cpu"))
    if dev.type == "cuda":
        torch.cuda.set_device(dev)
    pipeline = config.pipeline.setup(device=dev, test_mode=test_mode)
    pipeline.eval()
    ckpts = sorted(config.load_dir.glob("step-*.ckpt"))
    if not ckpts:
        raise FileNotFoundError(f"no step-*.ckpt under {config.load_dir}")
    path = ckpts[-1]
    state = torch.load(path, map_location=dev, weights_only=False)
    step = int(state["step"])
    pipeline.load_pipeline(state["pipeline"], step)
    return config, pipeline, path, step


@dataclass
class Exporter:
    load_config: Optional[Path]
    output_dir: Path


@dataclass
class ExportSemanticPointCloud(Exporter):
    """exporter.py:64-77 (+ ``stratified_jitter``, see ``FruitModel.get_export_outputs``)."""

    use_bounding_box: bool = True
    bounding_box_min: Tuple[float, float, float] = (-1, -1, -1)
    bounding_box_max: Tuple[float, float, float] = (1, 1, 1)
    num_rays_per_batch: int = 32768
    num_points_per_side: int = 1000
    stratified_jitter: bool = True
    """True = the reference's behaviour: its export sampler is created after ``eval_setup`` and therefore still in
    training mode, so every sample is jittered inside its bin.  False = the deterministic regular grid."""

    def main(self, pipeline=None, config=None, transform_json: Optional[dict] = None) -> dict:
        """exporter.py:80-121; ``pipeline`` may be supplied by the caller (test_mode='export')."""
        if pipeline is None:
            if self.load_config is None:
                raise ValueError("pass load_config (a run folder's config.yml) or an already built pipeline")
            config, pipeline, _, _ = eval_setup(self.load_config, test_mode="export")
        self.output_dir = Path(self.output_dir)
        self.output_dir.mkdir(parents=True, exist_ok=True)
        pipeline.datamanager.config.eval_num_rays_per_batch = self.num_rays_per_batch
        pipeline.model.setup_inference(render_rgb=True, num_inference_samples=self.num_points_per_side)
        pipeline.model.proposal_sampler.train(self.stratified_jitter)
        num_points = pipeline.datamanager.setup_inference(num_points=self.num_points_per_side,
                                                          aabb=(self.bounding_box_min, self.bounding_box_max))
        if transform_json is None and self.load_config is not None:
            with open(Path(self.load_config).parent / "dataparser_transforms.json", "r") as fp:
                transform_json = json.load(fp)
        pcds = sample_volume(pipeline=pipeline, num_points=num_points, output_dir=self.output_dir, config=config,
                             transform_json=transform_json, world_size=getattr(pipeline, "world_size", 1),
                             rank=getattr(pipeline, "local_rank", 0))
        for name, pcd in pcds.items():
            path = pcd["path"] or str(self.output_dir / f"{name}.ply")
            os.makedirs(os.path.dirname(path), exist_ok=True)
            write_ply(path, pcd["points"], pcd["colors"])
            pcd["path"] = path
        return pcds


@dataclass
class ExportPointCloud(Exporter):
    """nerfstudio 0.3.2 ExportPointCloud (the reference CLI's ``pointcloud`` subcommand, exporter.py:124-129): the RGB
    surface cloud of the scene from rendered training rays, with normals.  Single GPU."""

    num_points: int = 1000000
    remove_outliers: bool = True
    reorient_normals: bool = True
    normal_method: str = "model_output"
    """"open3d": estimate normals from the cloud; "model_output": take them from the model, which FruitModel cannot."""
    normal_output_name: str = "normals"
    depth_output_name: str = "depth"
    rgb_output_name: str = "rgb"
    use_bounding_box: bool = True
    bounding_box_min: Tuple[float, float, float] = (-1, -1, -1)
    bounding_box_max: Tuple[float, float, float] = (1, 1, 1)
    num_rays_per_batch: int = 32768
    std_ratio: float = 10.0

    def main(self, pipeline=None) -> dict:
        """Writes ``output_dir/point_cloud.ply`` (points in the dataparser frame) and returns generate_point_cloud's dict
        with its 'path'.  Exits with status 1 for ``normal_method="model_output"`` when the model renders no
        ``normal_output_name``, as nerfstudio's validate_pipeline does."""
        if self.normal_method not in ("open3d", "model_output"):
            raise ValueError(f"normal_method must be 'open3d' or 'model_output', got {self.normal_method!r}")
        self.output_dir = Path(self.output_dir)
        self.output_dir.mkdir(parents=True, exist_ok=True)
        if pipeline is None:
            if self.load_config is None:
                raise ValueError("pass load_config (a run folder's config.yml) or an already built pipeline")
            _, pipeline, _, _ = eval_setup(self.load_config)
        if self.normal_method == "model_output":
            _require_normal_output(pipeline, self.normal_output_name)
        pipeline.datamanager.config.train_num_rays_per_batch = self.num_rays_per_batch
        estimate = self.normal_method == "open3d"
        pcd = generate_point_cloud(pipeline, num_points=self.num_points, remove_outliers=self.remove_outliers,
                                   reorient_normals=self.reorient_normals, estimate_normals=estimate, rgb_output_name=self.rgb_output_name,
                                   depth_output_name=self.depth_output_name,
                                   normal_output_name=None if estimate else self.normal_output_name,
                                   use_bounding_box=self.use_bounding_box, bounding_box_min=self.bounding_box_min,
                                   bounding_box_max=self.bounding_box_max, std_ratio=self.std_ratio)
        pcd["path"] = str(self.output_dir / "point_cloud.ply")
        write_ply(pcd["path"], pcd["points"], pcd["colors"], normals=pcd["normals"])
        return pcd


@dataclass
class ExportTSDFMesh(Exporter):
    """nerfstudio 0.3.2 ExportTSDFMesh: a surface mesh of the scene by TSDF fusion of rendered depth maps, plus the mesh of
    the fruit surfaces (faces whose vertices have a fused fruit probability >= 0.5).  Single GPU.  The PLYs carry vertex
    colours.  ``texture_method="nerf"`` with ``unwrap_method="custom"`` also writes both meshes as OBJs textured by the
    NeRF, ``px_per_uv_triangle`` texels per face (DESIGN section 4.3p); with ``unwrap_method="charts"`` the texture is one
    square atlas of ``num_pixels_per_side`` texels a side whose texel density follows surface area (DESIGN section 4.3r);
    the xatlas unwrap is not available.
    ``target_num_faces`` decimates each textured mesh on the GPU first (DESIGN section 4.3q); unlike nerfstudio's 50 000
    its default is None, the full mesh."""

    downscale_factor: int = 2
    depth_output_name: str = "depth"
    rgb_output_name: str = "rgb"
    resolution: Tuple[int, ...] = (128,)
    batch_size: int = 10
    use_bounding_box: bool = True
    bounding_box_min: Tuple[float, float, float] = (-1, -1, -1)
    bounding_box_max: Tuple[float, float, float] = (1, 1, 1)
    texture_method: str = "tsdf"
    refine_mesh_using_initial_aabb_estimate: bool = False
    refinement_epsilon: float = 1e-2
    unwrap_method: str = "xatlas"
    px_per_uv_triangle: int = 4
    target_num_faces: Optional[int] = None
    num_pixels_per_side: int = 1024

    def validate(self) -> None:
        """Refuse what cannot run, before anything is loaded."""
        _validate_target_num_faces(self.texture_method, self.target_num_faces)
        if self.texture_method not in ("tsdf", "nerf"):
            raise ValueError(f"texture_method must be 'tsdf' or 'nerf', got {self.texture_method!r}")
        _validate_nerf_texture(self.texture_method, self.unwrap_method, self.px_per_uv_triangle, self.num_pixels_per_side, "tsdf")
        res = tuple(self.resolution) if isinstance(self.resolution, (list, tuple)) else (self.resolution,)
        if len(res) not in (1, 3) or min(int(r) for r in res) < 2:
            raise ValueError(f"resolution must be one or three integers >= 2, got {list(res)}")
        if self.downscale_factor < 1:
            raise ValueError(f"downscale_factor must be >= 1, got {self.downscale_factor}")
        if self.batch_size < 1:
            raise ValueError(f"batch_size must be >= 1, got {self.batch_size}")
        if self.use_bounding_box and not all(lo < hi for lo, hi in zip(self.bounding_box_min, self.bounding_box_max)):
            raise ValueError("Bounding box min must be smaller than max")

    def main(self, pipeline=None) -> dict:
        """Writes ``output_dir/tsdf_mesh.ply`` and ``output_dir/fruit_mesh.ply``, and with NeRF texturing then
        ``mesh.obj`` / ``material_0.{mtl,png}`` and ``fruit_mesh.obj`` / ``fruit_material_0.{mtl,png}`` (no fruit OBJ for an
        empty fruit mesh); returns export_tsdf_mesh's dict, the OBJ, MTL and PNG paths added to its 'paths'.  An atlas
        over texture.MAX_SIDE a side raises texture.AtlasTooLargeError after the PLYs are written, before any OBJ."""
        self.validate()
        if pipeline is None:
            if self.load_config is None:
                raise ValueError("pass load_config (a run folder's config.yml) or an already built pipeline")
            _, pipeline, _, _ = eval_setup(self.load_config)
        res = list(self.resolution) if isinstance(self.resolution, (list, tuple)) else [self.resolution]
        out = export_tsdf_mesh(pipeline, Path(self.output_dir), downscale_factor=self.downscale_factor, depth_output_name=self.depth_output_name,
                               rgb_output_name=self.rgb_output_name, resolution=res, batch_size=self.batch_size,
                               use_bounding_box=self.use_bounding_box, bounding_box_min=self.bounding_box_min,
                               bounding_box_max=self.bounding_box_max,
                               refine_mesh_using_initial_aabb_estimate=self.refine_mesh_using_initial_aabb_estimate,
                               refinement_epsilon=self.refinement_epsilon)
        if self.texture_method == "nerf":
            out["paths"].update(export_textured_meshes(pipeline, out, Path(self.output_dir), self.px_per_uv_triangle,
                                                         self.target_num_faces, self.unwrap_method, self.num_pixels_per_side))
        return out


@dataclass
class ExportPoissonMesh(Exporter):
    """nerfstudio 0.3.2 ExportPoissonMesh: a watertight mesh of the scene by screened Poisson reconstruction of the surface
    cloud, trimmed at the 0.1 quantile of vertex density, plus the mesh of the fruit surfaces (faces whose vertices have a
    fruit probability >= 0.5).  Single GPU.  The PLYs carry vertex colours.  ``texture_method="nerf"`` with
    ``unwrap_method="custom"`` also writes both meshes as OBJs textured by the NeRF, ``px_per_uv_triangle`` texels per
    face (DESIGN section 4.3p), or with ``unwrap_method="charts"`` in one ``num_pixels_per_side``-square chart atlas (DESIGN
    section 4.3r); the xatlas unwrap is not available.  ``target_num_faces`` decimates each textured mesh on
    the GPU first (DESIGN section 4.3q); unlike nerfstudio's 50 000 its default is None, the full mesh.  ``depth`` (open3d's octree depth, here the dense grid's 2^depth cells per axis) is
    the one option upstream does not have."""

    num_points: int = 1000000
    remove_outliers: bool = True
    reorient_normals: bool = True
    depth_output_name: str = "depth"
    rgb_output_name: str = "rgb"
    normal_method: str = "model_output"
    """"open3d": estimate normals from the cloud; "model_output": take them from the model, which FruitModel cannot."""
    normal_output_name: str = "normals"
    save_point_cloud: bool = False
    use_bounding_box: bool = True
    bounding_box_min: Tuple[float, float, float] = (-1, -1, -1)
    bounding_box_max: Tuple[float, float, float] = (1, 1, 1)
    num_rays_per_batch: int = 32768
    texture_method: str = "point_cloud"
    std_ratio: float = 10.0
    depth: int = 9
    unwrap_method: str = "xatlas"
    px_per_uv_triangle: int = 4
    target_num_faces: Optional[int] = None
    num_pixels_per_side: int = 1024

    def validate(self) -> None:
        """Refuse what cannot run, before anything is loaded."""
        from .. import poisson

        _validate_target_num_faces(self.texture_method, self.target_num_faces)
        if self.texture_method not in ("point_cloud", "nerf"):
            raise ValueError(f"texture_method must be 'point_cloud' or 'nerf', got {self.texture_method!r}")
        _validate_nerf_texture(self.texture_method, self.unwrap_method, self.px_per_uv_triangle, self.num_pixels_per_side, "point_cloud")
        if self.normal_method not in ("open3d", "model_output"):
            raise ValueError(f"normal_method must be 'open3d' or 'model_output', got {self.normal_method!r}")
        poisson.check_depth(self.depth)
        if self.num_points < 1:
            raise ValueError(f"num_points must be >= 1, got {self.num_points}")
        if self.use_bounding_box and not all(lo < hi for lo, hi in zip(self.bounding_box_min, self.bounding_box_max)):
            raise ValueError("Bounding box min must be smaller than max")

    def main(self, pipeline=None) -> dict:
        """Writes ``output_dir/poisson_mesh.ply`` and ``output_dir/fruit_poisson_mesh.ply``, and with NeRF texturing the
        OBJs as ExportTSDFMesh.main does; returns export_poisson_mesh's dict.  Exits with status 1 for
        ``normal_method="model_output"`` when the model renders no ``normal_output_name``."""
        self.validate()
        if pipeline is None:
            if self.load_config is None:
                raise ValueError("pass load_config (a run folder's config.yml) or an already built pipeline")
            _, pipeline, _, _ = eval_setup(self.load_config)
        if self.normal_method == "model_output":
            _require_normal_output(pipeline, self.normal_output_name)
        pipeline.datamanager.config.train_num_rays_per_batch = self.num_rays_per_batch
        out = export_poisson_mesh(pipeline, Path(self.output_dir), num_points=self.num_points, remove_outliers=self.remove_outliers,
                                  reorient_normals=self.reorient_normals, depth_output_name=self.depth_output_name,
                                  rgb_output_name=self.rgb_output_name, save_point_cloud=self.save_point_cloud,
                                  use_bounding_box=self.use_bounding_box, bounding_box_min=self.bounding_box_min,
                                  bounding_box_max=self.bounding_box_max, std_ratio=self.std_ratio, depth=self.depth)
        if self.texture_method == "nerf":
            out["paths"].update(export_textured_meshes(pipeline, out, Path(self.output_dir), self.px_per_uv_triangle,
                                                         self.target_num_faces, self.unwrap_method, self.num_pixels_per_side))
        return out


def _validate_nerf_texture(texture_method: str, unwrap_method: str, px_per_uv_triangle: int, num_pixels_per_side: int,
                           vertex_colours: str) -> None:
    """The options of NeRF texturing: the per-face ("custom") unwrap at >= 2 texels per triangle, or the chart ("charts")
    unwrap into a square atlas of num_pixels_per_side texels a side; xatlas is not available."""
    from ..texture import check_num_pixels_per_side, check_px_per_uv_triangle

    if unwrap_method not in ("xatlas", "custom", "charts"):
        raise ValueError(f"unwrap_method must be 'xatlas', 'custom' or 'charts', got {unwrap_method!r}")
    if texture_method == "nerf" and unwrap_method == "xatlas":
        raise ValueError(f"texture_method 'nerf' with the xatlas UV unwrap needs the xatlas package, which is not available; use "
                         f"--unwrap-method custom (one atlas triangle per face), --unwrap-method charts (area-proportional charts in "
                         f"one square atlas) or texture_method '{vertex_colours}' (vertex colours)")
    check_px_per_uv_triangle(px_per_uv_triangle)
    if unwrap_method == "charts":
        check_num_pixels_per_side(num_pixels_per_side)


def _validate_target_num_faces(texture_method: str, target_num_faces: Optional[int]) -> None:
    """Decimation only feeds NeRF texturing: without it the option would do nothing."""
    if target_num_faces is None:
        return
    if int(target_num_faces) < 1:
        raise ValueError(f"target_num_faces must be >= 1, got {target_num_faces}")
    if texture_method != "nerf":
        raise ValueError("--target-num-faces decimates the mesh before NeRF texturing and needs --texture-method nerf; the PLYs "
                         "are never decimated")


def _require_normal_output(pipeline, normal_output_name: str) -> None:
    """nerfstudio validate_pipeline: render one ray and exit(1) if ``normal_output_name`` is not among the outputs."""
    from ..compat import RayBundle

    dev = next(pipeline.model.parameters()).device
    origins = torch.zeros((1, 3), device=dev)
    bundle = RayBundle(origins=origins, directions=torch.ones_like(origins), pixel_area=torch.ones_like(origins[..., :1]),
                       camera_indices=torch.zeros((1, 1), dtype=torch.long, device=dev))
    with torch.no_grad():
        outputs = pipeline.model(bundle)
    if normal_output_name not in outputs:
        print(f"Warning: Normal output '{normal_output_name}' not found in pipeline outputs.")
        print(f"Available outputs: {list(outputs.keys())}")
        print("Warning: Please train a model with normals (e.g., nerfacto with predicted normals turned on).")
        print("Warning: Or change --normal-method")
        print("Exiting early.")
        sys.exit(1)


def _flag(s: str) -> bool:
    return s.lower() in ("1", "true", "yes")


def add_pointcloud_parser(sub) -> argparse.ArgumentParser:
    """The ``pointcloud`` subcommand: ExportPointCloud's fields as nerfstudio's option names, same defaults."""
    d = ExportPointCloud(load_config=None, output_dir=Path("."))
    p = sub.add_parser("pointcloud", help="RGB surface point cloud with normals from rendered training rays")
    p.add_argument("--load-config", type=Path, required=True)
    p.add_argument("--output-dir", type=Path, required=True)
    p.add_argument("--num-points", type=int, default=d.num_points)
    p.add_argument("--remove-outliers", type=_flag, default=d.remove_outliers)
    p.add_argument("--reorient-normals", type=_flag, default=d.reorient_normals)
    p.add_argument("--normal-method", choices=("open3d", "model_output"), default=d.normal_method)
    p.add_argument("--normal-output-name", default=d.normal_output_name)
    p.add_argument("--depth-output-name", default=d.depth_output_name)
    p.add_argument("--rgb-output-name", default=d.rgb_output_name)
    p.add_argument("--use-bounding-box", type=_flag, default=d.use_bounding_box)
    p.add_argument("--bounding-box-min", type=float, nargs=3, default=d.bounding_box_min)
    p.add_argument("--bounding-box-max", type=float, nargs=3, default=d.bounding_box_max)
    p.add_argument("--num-rays-per-batch", type=int, default=d.num_rays_per_batch)
    p.add_argument("--std-ratio", type=float, default=d.std_ratio)
    return p


def add_tsdf_parser(sub) -> argparse.ArgumentParser:
    """The ``tsdf`` subcommand: ExportTSDFMesh's fields as nerfstudio's option names, same defaults except the texture
    method, which stays ``tsdf``: nerfstudio's default, ``nerf`` with the xatlas unwrap, is not available."""
    d = ExportTSDFMesh(load_config=None, output_dir=Path("."))
    p = sub.add_parser("tsdf", help="surface meshes of the scene and of the fruit by TSDF fusion of rendered depth")
    p.add_argument("--load-config", type=Path, required=True)
    p.add_argument("--output-dir", type=Path, required=True)
    p.add_argument("--downscale-factor", type=int, default=d.downscale_factor)
    p.add_argument("--depth-output-name", default=d.depth_output_name)
    p.add_argument("--rgb-output-name", default=d.rgb_output_name)
    p.add_argument("--resolution", type=int, nargs="+", default=list(d.resolution))
    p.add_argument("--batch-size", type=int, default=d.batch_size)
    p.add_argument("--use-bounding-box", type=_flag, default=d.use_bounding_box)
    p.add_argument("--bounding-box-min", type=float, nargs=3, default=d.bounding_box_min)
    p.add_argument("--bounding-box-max", type=float, nargs=3, default=d.bounding_box_max)
    p.add_argument("--texture-method", choices=("tsdf", "nerf"), default=d.texture_method)
    p.add_argument("--refine-mesh-using-initial-aabb-estimate", type=_flag, default=d.refine_mesh_using_initial_aabb_estimate)
    p.add_argument("--refinement-epsilon", type=float, default=d.refinement_epsilon)
    p.add_argument("--unwrap-method", choices=("xatlas", "custom", "charts"), default=d.unwrap_method)
    p.add_argument("--px-per-uv-triangle", type=int, default=d.px_per_uv_triangle)
    p.add_argument("--num-pixels-per-side", type=int, default=d.num_pixels_per_side,
                   help="side of the square texture atlas of --unwrap-method charts, in texels")
    p.add_argument("--target-num-faces", type=int, default=None,
                   help="decimate each textured mesh to this many faces on the GPU first (with --texture-method nerf); "
                        "default: no decimation, unlike nerfstudio's 50000, so the full mesh is textured")
    return p


def add_poisson_parser(sub) -> argparse.ArgumentParser:
    """The ``poisson`` subcommand: ExportPoissonMesh's fields as nerfstudio's option names, same defaults, plus ``--depth``."""
    d = ExportPoissonMesh(load_config=None, output_dir=Path("."))
    p = sub.add_parser("poisson", help="watertight meshes of the scene and of the fruit by screened Poisson reconstruction")
    p.add_argument("--load-config", type=Path, required=True)
    p.add_argument("--output-dir", type=Path, required=True)
    p.add_argument("--num-points", type=int, default=d.num_points)
    p.add_argument("--remove-outliers", type=_flag, default=d.remove_outliers)
    p.add_argument("--reorient-normals", type=_flag, default=d.reorient_normals)
    p.add_argument("--depth-output-name", default=d.depth_output_name)
    p.add_argument("--rgb-output-name", default=d.rgb_output_name)
    p.add_argument("--normal-method", choices=("open3d", "model_output"), default=d.normal_method)
    p.add_argument("--normal-output-name", default=d.normal_output_name)
    p.add_argument("--save-point-cloud", type=_flag, default=d.save_point_cloud)
    p.add_argument("--use-bounding-box", type=_flag, default=d.use_bounding_box)
    p.add_argument("--bounding-box-min", type=float, nargs=3, default=d.bounding_box_min)
    p.add_argument("--bounding-box-max", type=float, nargs=3, default=d.bounding_box_max)
    p.add_argument("--num-rays-per-batch", type=int, default=d.num_rays_per_batch)
    p.add_argument("--texture-method", choices=("point_cloud", "nerf"), default=d.texture_method)
    p.add_argument("--std-ratio", type=float, default=d.std_ratio)
    p.add_argument("--depth", type=int, default=d.depth)
    p.add_argument("--unwrap-method", choices=("xatlas", "custom", "charts"), default=d.unwrap_method)
    p.add_argument("--px-per-uv-triangle", type=int, default=d.px_per_uv_triangle)
    p.add_argument("--num-pixels-per-side", type=int, default=d.num_pixels_per_side,
                   help="side of the square texture atlas of --unwrap-method charts, in texels")
    p.add_argument("--target-num-faces", type=int, default=None,
                   help="decimate each textured mesh to this many faces on the GPU first (with --texture-method nerf); "
                        "default: no decimation, unlike nerfstudio's 50000, so the full mesh is textured")
    return p


def poisson_exporter_from_args(a) -> ExportPoissonMesh:
    return ExportPoissonMesh(load_config=a.load_config, output_dir=a.output_dir, num_points=a.num_points, remove_outliers=a.remove_outliers,
                             reorient_normals=a.reorient_normals, depth_output_name=a.depth_output_name, rgb_output_name=a.rgb_output_name,
                             normal_method=a.normal_method, normal_output_name=a.normal_output_name, save_point_cloud=a.save_point_cloud,
                             use_bounding_box=a.use_bounding_box, bounding_box_min=tuple(a.bounding_box_min),
                             bounding_box_max=tuple(a.bounding_box_max), num_rays_per_batch=a.num_rays_per_batch,
                             texture_method=a.texture_method, std_ratio=a.std_ratio, depth=a.depth, unwrap_method=a.unwrap_method,
                             px_per_uv_triangle=a.px_per_uv_triangle, target_num_faces=a.target_num_faces,
                             num_pixels_per_side=a.num_pixels_per_side)


def _run_mesh_export(exp, parser):
    """validate (argparse error, status 2), run, exit 1 on an empty mesh or an atlas that is too large, print the two
    meshes (and their textured OBJs)."""
    from ..texture import AtlasTooLargeError

    try:
        exp.validate()
    except ValueError as e:
        parser.error(str(e))
    try:
        res = exp.main()
    except RuntimeError as e:
        if "empty mesh" not in str(e) and not isinstance(e, AtlasTooLargeError):
            raise
        print(f"error: {e}", file=sys.stderr)
        sys.exit(1)
    for key in ("mesh", "fruit_mesh"):
        m = res[key]
        print(f"{key}: {m['vertices'].shape[0]} vertices, {m['faces'].shape[0]} faces -> {res['paths'][key]}")
        if f"{key}_obj" in res["paths"]:
            print(f"{key}: textured -> {res['paths'][f'{key}_obj']} ({res['paths'][f'{key}_png']})")
    return res


def tsdf_exporter_from_args(a) -> ExportTSDFMesh:
    return ExportTSDFMesh(load_config=a.load_config, output_dir=a.output_dir, downscale_factor=a.downscale_factor,
                          depth_output_name=a.depth_output_name, rgb_output_name=a.rgb_output_name, resolution=tuple(a.resolution),
                          batch_size=a.batch_size, use_bounding_box=a.use_bounding_box, bounding_box_min=tuple(a.bounding_box_min),
                          bounding_box_max=tuple(a.bounding_box_max), texture_method=a.texture_method,
                          refine_mesh_using_initial_aabb_estimate=a.refine_mesh_using_initial_aabb_estimate,
                          refinement_epsilon=a.refinement_epsilon, unwrap_method=a.unwrap_method,
                          px_per_uv_triangle=a.px_per_uv_triangle, target_num_faces=a.target_num_faces,
                          num_pixels_per_side=a.num_pixels_per_side)


def entrypoint(argv=None):
    """``ns-export-semantics semantic-pointcloud --load-config RUN/config.yml --output-dir OUT [...]`` (exporter.py:124-144;
    upstream parses the same dataclass with tyro, which is not available offline -- argparse with the same option names)
    , ``ns-export-semantics pointcloud ...`` (nerfstudio ExportPointCloud), ``ns-export-semantics tsdf ...`` (nerfstudio
    ExportTSDFMesh) and ``ns-export-semantics poisson ...`` (nerfstudio ExportPoissonMesh)."""
    ap = argparse.ArgumentParser(prog="ns-export-semantics")
    sub = ap.add_subparsers(dest="command", required=True)
    add_pointcloud_parser(sub)
    tsdf_parser = add_tsdf_parser(sub)
    poisson_parser = add_poisson_parser(sub)
    p = sub.add_parser("semantic-pointcloud", help="uniform-volume export of the fruit point clouds")
    p.add_argument("--load-config", type=Path, required=True)
    p.add_argument("--output-dir", type=Path, required=True)
    p.add_argument("--use-bounding-box", type=lambda s: s.lower() in ("1", "true", "yes"), default=True)
    p.add_argument("--bounding-box-min", type=float, nargs=3, default=(-1, -1, -1))
    p.add_argument("--bounding-box-max", type=float, nargs=3, default=(1, 1, 1))
    p.add_argument("--num-rays-per-batch", type=int, default=32768)
    p.add_argument("--num-points-per-side", type=int, default=1000)
    p.add_argument("--stratified-jitter", type=lambda s: s.lower() in ("1", "true", "yes"), default=True)
    a = ap.parse_args(argv)
    if a.command == "poisson":
        return _run_mesh_export(poisson_exporter_from_args(a), poisson_parser)
    if a.command == "tsdf":
        return _run_mesh_export(tsdf_exporter_from_args(a), tsdf_parser)
    if a.command == "pointcloud":
        exp = ExportPointCloud(load_config=a.load_config, output_dir=a.output_dir, num_points=a.num_points, remove_outliers=a.remove_outliers,
                               reorient_normals=a.reorient_normals, normal_method=a.normal_method, normal_output_name=a.normal_output_name,
                               depth_output_name=a.depth_output_name, rgb_output_name=a.rgb_output_name, use_bounding_box=a.use_bounding_box,
                               bounding_box_min=tuple(a.bounding_box_min), bounding_box_max=tuple(a.bounding_box_max),
                               num_rays_per_batch=a.num_rays_per_batch, std_ratio=a.std_ratio)
        pcd = exp.main()
        print(f"point_cloud: {pcd['points'].shape[0]} points -> {pcd['path']}")
        return pcd
    exp = ExportSemanticPointCloud(load_config=a.load_config, output_dir=a.output_dir, use_bounding_box=a.use_bounding_box,
                                   bounding_box_min=tuple(a.bounding_box_min), bounding_box_max=tuple(a.bounding_box_max),
                                   num_rays_per_batch=a.num_rays_per_batch, num_points_per_side=a.num_points_per_side,
                                   stratified_jitter=a.stratified_jitter)
    pcds = exp.main()
    for name, pcd in pcds.items():
        print(f"{name}: {pcd['points'].shape[0]} points -> {pcd['path']}")
    return pcds


if __name__ == "__main__":
    entrypoint()
