"""FruitModel -- drop-in for fruit_nerf.fruit_nerf.FruitModel (fruit_nerf/fruit_nerf.py:62-458).

Same config fields, output-dict keys, param-group names and test_mode dispatch as the reference;
the per-ray work (field + weights + renderers) is ONE native call (fruitnerf_b200.ops.render), the
volume-export branch is the fused export kernel (ops.export_batch).
"""
from __future__ import annotations

from collections import defaultdict
from dataclasses import dataclass, field
from typing import Any, Dict, List, Literal, Optional, Tuple, Type, Union

import numpy as np
import torch
from torch import Tensor, nn
from torch.nn import Parameter

from . import _lib as L
from . import ops
from .compat import FieldHeadNames, InstantiateConfig, RayBundle, RaySamples, SceneBox, Semantics
from .components.ray_samplers import UniformLinDispPiecewiseSampler, UniformSamplerWithNoise
from .components.proposal_sampler import ProposalNetworkSampler
from .density_field import HashMLPDensityField
from .fruit_field import FruitField, SceneContraction


@dataclass
class FruitNerfModelConfig(InstantiateConfig):
    """FruitNerfModelConfig(NerfactoModelConfig) (fruit_nerf.py:50-59) with the nerfstudio-0.3.2
    NerfactoModelConfig defaults the hot path reads (SURVEY.md section 2.3)."""

    _target: Type = field(default_factory=lambda: FruitModel)
    # FruitNeRF additions
    semantic_loss_weight: float = 1.0
    pass_semantic_gradients: bool = False
    num_layers_semantic: int = 2
    hidden_dim_semantics: int = 64
    geo_feat_dim: int = 15
    # NerfactoModelConfig
    near_plane: float = 0.05
    far_plane: float = 1000.0
    background_color: Literal["random", "last_sample", "black", "white"] = "last_sample"
    hidden_dim: int = 64
    hidden_dim_color: int = 64
    hidden_dim_transient: int = 64
    num_levels: int = 16
    max_res: int = 2048
    log2_hashmap_size: int = 19
    num_proposal_samples_per_ray: Tuple[int, ...] = (256, 96)
    num_nerf_samples_per_ray: int = 48
    proposal_update_every: int = 5
    proposal_warmup: int = 5000
    num_proposal_iterations: int = 2
    use_same_proposal_network: bool = False
    proposal_net_args_list: List[Dict] = field(
        default_factory=lambda: [
            {"hidden_dim": 16, "log2_hashmap_size": 17, "num_levels": 5, "max_res": 128, "use_linear": False},
            {"hidden_dim": 16, "log2_hashmap_size": 17, "num_levels": 5, "max_res": 256, "use_linear": False},
        ]
    )
    proposal_initial_sampler: Literal["piecewise", "uniform"] = "piecewise"
    interlevel_loss_mult: float = 1.0
    distortion_loss_mult: float = 0.002
    use_proposal_weight_anneal: bool = True
    use_average_appearance_embedding: bool = True
    proposal_weights_anneal_slope: float = 10.0
    proposal_weights_anneal_max_num_iters: int = 1000
    use_single_jitter: bool = True
    disable_scene_contraction: bool = False
    use_gradient_scaling: bool = False
    appearance_embed_dim: int = 32
    eval_num_rays_per_chunk: int = 4096
    implementation: Literal["tcnn", "torch", "b200"] = "b200"


def _sdist(ray_samples: RaySamples) -> Tensor:
    """nerfstudio ray_samples_to_sdist: [R, S+1] spacing bins."""
    return torch.cat([ray_samples.spacing_starts[..., 0], ray_samples.spacing_ends[..., -1:, 0]], dim=-1)


def _median_depth(weights: Tensor, ray_samples: RaySamples) -> Tensor:
    """nerfstudio DepthRenderer(method="median") for the proposal levels (visualisation outputs)."""
    if weights.is_cuda:
        return ops.median_depth(weights[..., 0], ray_samples.frustums.starts[..., 0], ray_samples.frustums.ends[..., 0])
    with torch.no_grad():
        steps = (ray_samples.frustums.starts + ray_samples.frustums.ends) / 2
        cum = torch.cumsum(weights[..., 0], dim=-1)
        split = torch.ones((*weights.shape[:-2], 1), device=weights.device) * 0.5
        idx = torch.clamp(torch.searchsorted(cum, split, side="left"), 0, steps.shape[-2] - 1)
        return torch.gather(steps[..., 0], dim=-1, index=idx)


class FruitModel(nn.Module):
    """FruitModel based on the Nerfacto model (fruit_nerf.py:62-458)."""

    config: FruitNerfModelConfig

    def __init__(self, config: FruitNerfModelConfig, metadata: Dict, scene_box: SceneBox = None, num_train_data: int = 1,
                 **kwargs) -> None:
        assert "semantics" in metadata.keys() and isinstance(metadata["semantics"], Semantics)  # fruit_nerf.py:72
        super().__init__()
        self.semantics = metadata["semantics"]
        self.test_mode = kwargs["test_mode"]  # fruit_nerf.py:74 (KeyError if absent, as upstream)
        self.config = config
        self.scene_box = scene_box
        self.num_train_data = num_train_data
        self.kwargs = kwargs
        self.render_rgb = kwargs.get("render_rgb_inference", True)
        self.device_indicator_param = nn.Parameter(torch.empty(0))
        self.populate_modules()
        self.colormap = self.semantics.colors.clone().detach()

    @property
    def device(self):
        return self.device_indicator_param.device

    def populate_modules(self):
        """fruit_nerf.py:78-177."""
        cfg = self.config
        if cfg.use_gradient_scaling:
            # nerfacto's scale_gradients_by_distance_squared hook between the field and the renderers: the fused kernel has
            # no such stage, and silently training without it would not be the configuration that was asked for
            raise NotImplementedError("use_gradient_scaling=True is not implemented by the fused render kernels (reference default: False)")
        scene_contraction = None if cfg.disable_scene_contraction else SceneContraction(order=float("inf"))
        self.field = FruitField(
            self.scene_box.aabb,
            num_levels=cfg.num_levels,
            max_res=cfg.max_res,
            num_layers_semantic=cfg.num_layers_semantic,
            hidden_dim_semantics=cfg.hidden_dim_semantics,
            log2_hashmap_size=cfg.log2_hashmap_size,
            spatial_distortion=scene_contraction,
            num_images=self.num_train_data,
            geo_feat_dim=cfg.geo_feat_dim,
            use_average_appearance_embedding=cfg.use_average_appearance_embedding,
            use_semantics=True,
            test_mode=self.test_mode,
            num_semantic_classes=1,
            pass_semantic_gradients=cfg.pass_semantic_gradients,
        )
        # Proposal networks + sampler (fruit_nerf.py:104-158)
        self.density_fns = []
        num_prop_nets = cfg.num_proposal_iterations
        self.proposal_networks = nn.ModuleList()
        if cfg.use_same_proposal_network:
            assert len(cfg.proposal_net_args_list) == 1, "Only one proposal network is allowed."
            prop_net_args = {k: v for k, v in cfg.proposal_net_args_list[0].items()}
            network = HashMLPDensityField(self.scene_box.aabb, spatial_distortion=scene_contraction, **prop_net_args)
            self.proposal_networks.append(network)
            self.density_fns.extend([network.density_fn for _ in range(num_prop_nets)])
        else:
            for i in range(num_prop_nets):
                prop_net_args = cfg.proposal_net_args_list[min(i, len(cfg.proposal_net_args_list) - 1)]
                network = HashMLPDensityField(self.scene_box.aabb, spatial_distortion=scene_contraction, **prop_net_args)
                self.proposal_networks.append(network)
            self.density_fns.extend([network.density_fn for network in self.proposal_networks])

        def update_schedule(step):
            return np.clip(np.interp(step, [0, cfg.proposal_warmup], [0, cfg.proposal_update_every]), 1, cfg.proposal_update_every)

        if cfg.proposal_initial_sampler == "uniform":
            # upstream leaves self.proposal_sampler unset on this branch (fruit_nerf.py:145-149): reject instead of crashing later
            raise NotImplementedError('proposal_initial_sampler="uniform" builds no sampler in the reference either')
        if num_prop_nets >= 1:
            self.proposal_sampler = ProposalNetworkSampler(
                num_nerf_samples_per_ray=cfg.num_nerf_samples_per_ray,
                num_proposal_samples_per_ray=cfg.num_proposal_samples_per_ray,
                num_proposal_network_iterations=cfg.num_proposal_iterations,
                single_jitter=cfg.use_single_jitter,
                update_sched=update_schedule,
                initial_sampler=None,
            )
        else:  # nerfstudio with zero proposal iterations: the initial sampler draws the final bins
            self.proposal_sampler = UniformLinDispPiecewiseSampler(num_samples=cfg.num_nerf_samples_per_ray, single_jitter=cfg.use_single_jitter)
        self.near_plane, self.far_plane = cfg.near_plane, cfg.far_plane
        self.rgb_loss = nn.MSELoss()
        self.binary_cross_entropy_loss = nn.BCEWithLogitsLoss(reduction="mean")
        self.step = 0

    def setup_inference(self, render_rgb, num_inference_samples):
        """fruit_nerf.py:179-183."""
        self.render_rgb = render_rgb
        self.num_inference_samples = num_inference_samples
        self.proposal_sampler = UniformSamplerWithNoise(num_samples=self.num_inference_samples, single_jitter=False)
        self.field.spatial_distortion = None

    def get_param_groups(self) -> Dict[str, List[Parameter]]:
        """fruit_nerf.py:185-189 (names must match the optimizer keys of fruit_nerf_config.py)."""
        return {"proposal_networks": list(self.proposal_networks.parameters()), "fields": list(self.field.parameters())}

    def update_to_step(self, step: int) -> None:
        self.step = step

    # ---- collider (nerfstudio NearFarCollider: only fills missing nears / fars) ------------------
    def collider(self, ray_bundle: RayBundle) -> RayBundle:
        if ray_bundle.nears is not None and ray_bundle.fars is not None:
            return ray_bundle
        ones = torch.ones_like(ray_bundle.origins[..., 0:1])
        # NearFarCollider.set_nears_and_fars: `near_plane = self.near_plane if self.training else 0` -- evaluation and
        # inference renders start sampling at the camera centre
        near_plane = self.near_plane if self.training else 0.0
        ray_bundle.nears = ones * near_plane
        ray_bundle.fars = ones * self.far_plane
        return ray_bundle

    # ---- hot path ---------------------------------------------------------------------------------
    def _render(self, ray_samples: RaySamples) -> Dict[str, Tensor]:
        f = self.field
        shape, o, d, s, e, cam = FruitField.ray_tensors(ray_samples)
        mode = f.appearance_mode()
        if mode == L.FNR_APP_PER_CAMERA and cam is None:
            raise AttributeError("Camera indices are not provided.")
        return ops.render(f.kernel_shape(), f.kernel_params(), o, d, s, e, cam, f.position_mode(), mode,
                          clamp_rgb=not self.training, impl=f.kernel_impl)

    def get_outputs(self, ray_bundle: RayBundle):
        """fruit_nerf.py:316-357 (and 272-314 for test_mode == 'inference')."""
        if isinstance(self.proposal_sampler, ProposalNetworkSampler):
            ray_samples, weights_list, ray_samples_list = self.proposal_sampler(ray_bundle, density_fns=self.density_fns)
        else:
            ray_samples, weights_list, ray_samples_list = self.proposal_sampler(ray_bundle), [], []
        out = self._render(ray_samples)
        R = out["rgb"].shape[0]
        weights = out["weights"].unsqueeze(-1)
        weights_list.append(weights)
        ray_samples_list.append(ray_samples)
        outputs = {
            "rgb": out["rgb"],
            "accumulation": out["accumulation"].view(R, 1),
            "depth": out["depth"].view(R, 1),
            "weights_list": weights_list,
            "ray_samples_list": ray_samples_list,
        }
        for i in range(len(weights_list) - 1):  # prop_depth_i: median depth of each proposal level (fruit_nerf.py:339-340)
            outputs[f"prop_depth_{i}"] = _median_depth(weights_list[i], ray_samples_list[i])
        outputs["semantics"] = out["semantics"].view(R, 1)
        semantic_labels = torch.sigmoid(outputs["semantics"].detach())
        threshold = 0.9
        semantic_labels = torch.heaviside(semantic_labels - threshold, torch.zeros((), device=semantic_labels.device)).to(torch.long)
        if self.colormap.device != semantic_labels.device:  # moved once, not per call (and never inside a graph capture)
            self.colormap = self.colormap.to(semantic_labels.device)
        cmap = self.colormap[semantic_labels]
        outputs["semantics_colormap"] = cmap.repeat(1, 3) if self.test_mode == "inference" else cmap  # fruit_nerf.py:312 / 355
        return outputs

    get_inference_outputs = get_outputs

    def get_rgba_image(self, outputs: Dict[str, Tensor], output_name: str = "rgb") -> Tensor:
        """nerfstudio Model.get_rgba_image for the "last_sample" background FruitModel renders with: the colour and the
        accumulation of each ray side by side, [..., 4]."""
        accumulation_name = output_name.replace("rgb", "accumulation")
        if output_name not in outputs or accumulation_name not in outputs:
            raise NotImplementedError(f"get_rgba_image needs '{output_name}' and '{accumulation_name}' among the outputs")
        rgb, acc = outputs[output_name], outputs[accumulation_name]
        if acc.dim() < rgb.dim():
            acc = acc.unsqueeze(-1)
        return torch.cat((rgb, acc), dim=-1)

    def get_export_outputs(self, ray_bundle: RayBundle, buffers: Optional[ops.ExportBuffers] = None, point_base: int = 0,
                           dense: bool = True):
        """fruit_nerf.py:251-269: uniform bins -> field (aabb-normalised, mean appearance) ->
        rgb / point_location / semantics / density / semantics_colormap, one fused kernel.  When
        ``buffers`` is given the kernel also performs sample_volume's threshold + compaction."""
        S = self.num_inference_samples
        dev = ray_bundle.origins.device
        sampler = self.proposal_sampler
        if isinstance(sampler, UniformSamplerWithNoise) and sampler.train_stratified and sampler.training:
            # The reference exporter calls setup_inference() AFTER eval_setup() put the pipeline in eval mode, so its
            # freshly built sampler module is still in training mode and jitters every sample inside its bin
            # (components/ray_samplers.py:78-87, single_jitter=False): per-ray bins [B, S+1].  `sampler.eval()` (or
            # ExportSemanticPointCloud(stratified_jitter=False)) selects the deterministic regular grid instead.
            bins = sampler.spacing_bins(ray_bundle.origins.shape[0], S, dev).contiguous()
        else:
            bins = torch.linspace(0.0, 1.0, S + 1).to(dev)  # host linspace, as components/ray_samplers.py:75
        normal = [float(v) for v in ray_bundle.directions[0].tolist()]
        near = float(ray_bundle.nears[0]) if ray_bundle.nears is not None else self.near_plane
        far = float(ray_bundle.fars[0]) if ray_bundle.fars is not None else self.far_plane
        if buffers is None:
            buffers = ops.ExportBuffers(capacity=1, device=dev)
        res = ops.export_batch(self.field.kernel_shape(), self.field.kernel_params(), ray_bundle.origins, normal, bins, near, far,
                               buffers, point_base=point_base, dense_out=dense)
        return res if res is not None else {}

    def forward(self, ray_bundle: RayBundle, **kw) -> Dict[str, Union[torch.Tensor, List]]:
        """fruit_nerf.py:374-394."""
        ray_bundle = self.collider(ray_bundle)
        if self.test_mode == "export":
            return self.get_export_outputs(ray_bundle, **kw)
        return self.get_outputs(ray_bundle)

    def get_loss_dict(self, outputs, batch, metrics_dict=None):
        """fruit_nerf.py:359-372."""
        loss_dict = {}
        loss_dict["rgb_loss"], loss_dict["semantics_loss"], _ = self._fused_losses(outputs, batch)
        if self.training:
            loss_dict["interlevel_loss"] = ops.interlevel_loss(
                [w[..., 0] for w in outputs["weights_list"]], [_sdist(rs) for rs in outputs["ray_samples_list"]], self.config.interlevel_loss_mult
            )
        return loss_dict

    def get_metrics_dict(self, outputs, batch):
        """fruit_nerf.py:396-401: PSNR (data_range 1)."""
        metrics = {"psnr": self._fused_losses(outputs, batch)[2]}
        # nerfstudio distortion_loss on the final level: a logged metric only (fruit_nerf.py:400)
        metrics["distortion"] = ops.distortion_metric(outputs["weights_list"][-1][..., 0], _sdist(outputs["ray_samples_list"][-1]))
        return metrics

    def get_image_metrics_and_images(self, outputs: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor]):
        """fruit_nerf.py:403-458: metrics (psnr, ssim, iou; lpips needs downloaded weights and is omitted; ``fruit_iou`` added) and
        the images a logger / viewer shows, for ONE full image rendered by get_outputs_for_camera_ray_bundle.  Computed on the
        device the rendered outputs live on (the chunked renderer returns CPU tensors, as upstream)."""
        from .image_metrics import image_metrics_and_images

        return image_metrics_and_images(outputs, batch, self.config.num_proposal_iterations, outputs["rgb"].device)

    def _fused_losses(self, outputs, batch):
        """(MSELoss, semantic_loss_weight * BCEWithLogitsLoss, PSNR) from ONE launch, shared by get_metrics_dict and
        get_loss_dict (the reference evaluates the MSE twice, fruit_nerf.py:361 and :398)."""
        cached = outputs.get("_losses")
        if cached is None:
            cached = ops.render_losses(outputs["rgb"], outputs["semantics"], batch["image"].to(self.device), batch["fruit_mask"].to(self.device),
                                       self.config.semantic_loss_weight)
            outputs["_losses"] = cached
        return cached

    def get_training_callbacks(self, training_callback_attributes=None) -> List[Dict]:
        """fruit_nerf.py:191-223: anneal the proposal weights before each iteration, count steps after."""
        callbacks = []
        if self.config.use_proposal_weight_anneal and isinstance(self.proposal_sampler, ProposalNetworkSampler):
            N = self.config.proposal_weights_anneal_max_num_iters

            def set_anneal(step):
                train_frac = np.clip(step / N, 0, 1)
                b = self.config.proposal_weights_anneal_slope
                self.proposal_sampler.set_anneal(b * train_frac / ((b - 1) * train_frac + 1))

            callbacks.append({"where_to_run": "BEFORE_TRAIN_ITERATION", "update_every_num_iters": 1, "func": set_anneal})
            callbacks.append({"where_to_run": "AFTER_TRAIN_ITERATION", "update_every_num_iters": 1, "func": self.proposal_sampler.step_cb})
        return callbacks

    @torch.no_grad()
    def get_outputs_for_camera_ray_bundle(self, camera_ray_bundle: RayBundle) -> Dict[str, torch.Tensor]:
        """fruit_nerf.py:225-249: chunked full-image evaluation."""
        num_rays_per_chunk = self.config.eval_num_rays_per_chunk
        image_height, image_width = camera_ray_bundle.origins.shape[:2]
        num_rays = image_height * image_width
        outputs_lists = defaultdict(list)
        for i in range(0, num_rays, num_rays_per_chunk):
            ray_bundle = camera_ray_bundle.get_row_major_sliced_ray_bundle(i, i + num_rays_per_chunk)
            outputs = self.forward(ray_bundle=ray_bundle)
            for output_name, output in outputs.items():
                if not torch.is_tensor(output):
                    continue
                outputs_lists[output_name].append(output.cpu())
        return {k: torch.cat(v).view(image_height, image_width, -1) for k, v in outputs_lists.items()}


FruitNerfModel = FruitModel  # name used by BASELINE.json / north_star
