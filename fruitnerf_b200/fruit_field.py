"""FruitField -- the reference's field (fruit_nerf/fruit_field.py:43-301) as a parameter holder
whose forward runs in the native sm_90a kernels.

Constructor signature, attribute names and state-dict keys follow the reference under
nerfstudio's torch path, so ``load_state_dict(strict=True)`` round-trips
(fruit_nerf/fruit_pipeline.py:229-240):

    mlp_base_grid.hash_table, mlp_base_mlp.layers.{i}.{weight,bias}, mlp_base.{0,1}.* (aliases of
    the Sequential, fruit_field.py:141), mlp_semantics.layers.*, field_head_semantics.net.*,
    mlp_head.layers.*, embedding_appearance.embedding.weight, buffers aabb / max_res / num_levels /
    log2_hashmap_size (fruit_field.py:98-103).

The holder modules below own parameters only; they have no Python forward (no PyTorch fallback).
"""
from __future__ import annotations

from typing import Dict, Literal, Optional, Tuple

import numpy as np
import torch
from torch import Tensor, nn

from . import _lib as L
from . import ops
from .compat import FieldHeadNames, RaySamples


class SceneContraction(nn.Module):
    """Marker for nerfstudio's SceneContraction; only order=inf (fruit_nerf.py:85) is implemented
    (inside the kernels: fnr_common.cuh field_position)."""

    def __init__(self, order=float("inf")) -> None:
        super().__init__()
        if order != float("inf"):
            raise NotImplementedError("only the L-inf scene contraction used by FruitNeRF is implemented")
        self.order = order


class _Holder(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(
            f"{type(self).__name__} is a parameter holder: its arithmetic runs inside the fused native kernels "
            "(fruitnerf_b200.ops); there is no PyTorch fallback"
        )


class HashEncoding(_Holder):
    """nerfstudio HashEncoding parameters (reference ctor call fruit_field.py:124-131)."""

    def __init__(self, num_levels=16, min_res=16, max_res=1024, log2_hashmap_size=19, features_per_level=2,
                 hash_init_scale=0.001) -> None:
        super().__init__()
        self.num_levels = num_levels
        self.min_res = min_res
        self.features_per_level = features_per_level
        self.log2_hashmap_size = log2_hashmap_size
        self.hash_table_size = 2**log2_hashmap_size
        levels = torch.arange(num_levels)
        # same expression as nerfstudio (float32 pow through Tensor.__rpow__): the kernels take
        # this array as is and never recompute it (SURVEY.md section 7, "float-fragile")
        growth_factor = np.exp((np.log(max_res) - np.log(min_res)) / (num_levels - 1)) if num_levels > 1 else 1
        self.scalings = torch.floor(min_res * growth_factor**levels)
        self.hash_offset = levels * self.hash_table_size
        table = torch.rand(size=(self.hash_table_size * num_levels, features_per_level)) * 2 - 1
        table *= hash_init_scale
        self.hash_table = nn.Parameter(table)

    def get_out_dim(self) -> int:
        return self.num_levels * self.features_per_level


class MLP(_Holder):
    """nerfstudio MLP (torch path) parameters: ``num_layers`` nn.Linear layers in ``layers``."""

    def __init__(self, in_dim: int, num_layers: int, layer_width: int, out_dim: Optional[int] = None) -> None:
        super().__init__()
        self.in_dim = in_dim
        self.out_dim = out_dim if out_dim is not None else layer_width
        self.num_layers = num_layers
        self.layer_width = layer_width
        layers = []
        if num_layers == 1:
            layers.append(nn.Linear(in_dim, self.out_dim))
        else:
            for i in range(num_layers - 1):
                layers.append(nn.Linear(in_dim if i == 0 else layer_width, layer_width))
            layers.append(nn.Linear(layer_width, self.out_dim))
        self.layers = nn.ModuleList(layers)

    def get_out_dim(self) -> int:
        return self.out_dim

    def dims(self):
        return [self.layers[0].in_features] + [l.out_features for l in self.layers]


class Embedding(_Holder):
    """nerfstudio Embedding: wraps torch.nn.Embedding as ``.embedding`` (fruit_field.py:108)."""

    def __init__(self, in_dim: int, out_dim: int) -> None:
        super().__init__()
        self.in_dim, self.out_dim = in_dim, out_dim
        self.embedding = nn.Embedding(in_dim, out_dim)

    def mean(self, dim=0):
        return self.embedding.weight.mean(dim)


class SemanticFieldHead(_Holder):
    """fruit_nerf/components/field_heads.py:29-40: nerfstudio FieldHead = ``net = Linear(in, classes)``."""

    def __init__(self, num_classes: int, in_dim: Optional[int] = None, activation=None) -> None:
        super().__init__()
        self.in_dim, self.out_dim = in_dim, num_classes
        self.field_head_name = FieldHeadNames.SEMANTICS
        self.activation = activation
        self.net = nn.Linear(in_dim, num_classes)


class FruitField(nn.Module):
    """Drop-in for fruit_nerf.fruit_field.FruitField (same constructor, fruit_field.py:70-95)."""

    aabb: Tensor

    def __init__(
        self,
        aabb: Tensor,
        num_images: int,
        num_layers: int = 2,
        hidden_dim: int = 64,
        geo_feat_dim: int = 15,
        num_levels: int = 16,
        base_res: int = 16,
        max_res: int = 2048,
        log2_hashmap_size: int = 19,
        num_layers_color: int = 3,
        num_layers_semantic: int = 2,
        features_per_level: int = 2,
        hidden_dim_color: int = 64,
        hidden_dim_semantics: int = 64,
        hidden_dim_transient: int = 64,
        appearance_embedding_dim: int = 32,
        use_semantics: bool = False,
        test_mode: str = None,
        num_semantic_classes: int = 100,
        pass_semantic_gradients: bool = False,
        use_average_appearance_embedding: bool = False,
        spatial_distortion: Optional[nn.Module] = None,
        implementation: Literal["tcnn", "torch", "b200"] = "b200",
    ) -> None:
        super().__init__()
        self.register_buffer("aabb", torch.as_tensor(aabb, dtype=torch.float32))
        self.geo_feat_dim = geo_feat_dim
        self.register_buffer("max_res", torch.tensor(max_res))
        self.register_buffer("num_levels", torch.tensor(num_levels))
        self.register_buffer("log2_hashmap_size", torch.tensor(log2_hashmap_size))

        self.spatial_distortion = spatial_distortion
        self.num_images = num_images
        self.appearance_embedding_dim = appearance_embedding_dim
        self.embedding_appearance = Embedding(self.num_images, self.appearance_embedding_dim)
        self.use_average_appearance_embedding = use_average_appearance_embedding
        self.use_semantics = use_semantics
        self.test_mode = test_mode
        self.pass_semantic_gradients = pass_semantic_gradients
        self.base_res = base_res
        self.implementation = implementation
        self.kernel_impl = L.FNR_IMPL_AUTO

        self.mlp_base_grid = HashEncoding(
            num_levels=num_levels,
            min_res=base_res,
            max_res=max_res,
            log2_hashmap_size=log2_hashmap_size,
            features_per_level=features_per_level,
        )
        self.mlp_base_mlp = MLP(
            in_dim=self.mlp_base_grid.get_out_dim(), num_layers=num_layers, layer_width=hidden_dim, out_dim=1 + self.geo_feat_dim
        )
        self.mlp_base = torch.nn.Sequential(self.mlp_base_grid, self.mlp_base_mlp)

        if not self.use_semantics:
            raise NotImplementedError("FruitNeRF always builds the field with use_semantics=True (fruit_nerf.py:99)")
        if num_semantic_classes != 1:
            raise NotImplementedError("FruitNeRF uses a single fruit logit (num_semantic_classes=1, fruit_nerf.py:101)")
        self.mlp_semantics = MLP(
            in_dim=self.geo_feat_dim, num_layers=num_layers_semantic, layer_width=hidden_dim_semantics, out_dim=hidden_dim_transient
        )
        self.field_head_semantics = SemanticFieldHead(in_dim=self.mlp_semantics.get_out_dim(), num_classes=num_semantic_classes)
        self.mlp_head = MLP(
            in_dim=16 + self.geo_feat_dim + self.appearance_embedding_dim, num_layers=num_layers_color, layer_width=hidden_dim_color, out_dim=3
        )

    # -- native plumbing ---------------------------------------------------------------------
    def kernel_shape(self) -> ops.FieldShape:
        """Static kernel description; cached (building it reads the aabb buffer, a device sync)."""
        key = (self.pass_semantic_gradients, self.num_images, self.aabb._version, self.aabb.data_ptr())
        cached = getattr(self, "_kernel_shape_cache", None)
        if cached is not None and cached[0] == key:
            return cached[1]
        shape = self._build_kernel_shape()
        object.__setattr__(self, "_kernel_shape_cache", (key, shape))
        return shape

    def _build_kernel_shape(self) -> ops.FieldShape:
        g = self.mlp_base_grid
        return ops.FieldShape(
            num_levels=g.num_levels,
            features_per_level=g.features_per_level,
            log2_hashmap_size=g.log2_hashmap_size,
            scalings=[float(v) for v in g.scalings],
            geo_feat_dim=self.geo_feat_dim,
            appearance_dim=self.appearance_embedding_dim,
            num_images=self.num_images,
            base_dims=self.mlp_base_mlp.dims(),
            semantic_dims=self.mlp_semantics.dims(),
            color_dims=self.mlp_head.dims(),
            aabb=[float(v) for v in self.aabb.reshape(-1)],
            pass_semantic_gradients=self.pass_semantic_gradients,
        )

    def kernel_params(self):
        ps = [self.mlp_base_grid.hash_table]
        for m in (self.mlp_base_mlp, self.mlp_semantics):
            for l in m.layers:
                ps += [l.weight, l.bias]
        ps += [self.field_head_semantics.net.weight, self.field_head_semantics.net.bias]
        for l in self.mlp_head.layers:
            ps += [l.weight, l.bias]
        ps.append(self.embedding_appearance.embedding.weight)
        return ps

    def position_mode(self) -> int:
        return L.FNR_POS_CONTRACT if self.spatial_distortion is not None else L.FNR_POS_AABB

    def appearance_mode(self) -> int:
        if self.test_mode in ("inference", "export"):
            return L.FNR_APP_MEAN  # get_inference_outputs, fruit_field.py:217-219
        if self.training:
            return L.FNR_APP_PER_CAMERA  # fruit_field.py:250-251
        return L.FNR_APP_MEAN if self.use_average_appearance_embedding else L.FNR_APP_ZEROS

    @staticmethod
    def ray_tensors(ray_samples: RaySamples):
        fr = ray_samples.frustums
        shape = tuple(fr.starts.shape[:-1])
        S = shape[-1] if len(shape) > 1 else 1
        R = int(np.prod(shape)) // S
        origins = fr.origins.reshape(R, S, 3)[:, 0, :]
        directions = fr.directions.reshape(R, S, 3)[:, 0, :]
        starts = fr.starts.reshape(R, S)
        ends = fr.ends.reshape(R, S)
        cam = None
        if ray_samples.camera_indices is not None:
            cam = ray_samples.camera_indices.reshape(R, S)[:, 0]
        return shape, origins, directions, starts, ends, cam

    # -- reference API -----------------------------------------------------------------------
    def forward(self, ray_samples: RaySamples) -> Dict[FieldHeadNames, Tensor]:
        """fruit_field.py:283-301.  Returns DENSITY [...,1], RGB [...,3], SEMANTICS [...,1]."""
        shape, o, d, s, e, cam = self.ray_tensors(ray_samples)
        mode = self.appearance_mode()
        if mode == L.FNR_APP_PER_CAMERA and cam is None:
            raise AttributeError("Camera indices are not provided.")  # fruit_field.py:240-241
        sd, srgb, ssem = ops.field(self.kernel_shape(), self.kernel_params(), o, d, s, e, cam, self.position_mode(), mode,
                                   impl=self.kernel_impl)
        return {
            FieldHeadNames.RGB: srgb.view(*shape, 3),
            FieldHeadNames.SEMANTICS: ssem.view(*shape, 1),
            FieldHeadNames.DENSITY: sd.view(*shape, 1),
        }

    def get_density(self, ray_samples: RaySamples) -> Tuple[Tensor, Optional[Tensor]]:
        """fruit_field.py:168-193.  The fused kernels never materialise the geo features in HBM,
        so the second element (density embedding) is None; use ``forward`` for the field heads."""
        return self.forward(ray_samples)[FieldHeadNames.DENSITY], None

    def get_outputs(self, ray_samples: RaySamples, density_embedding: Optional[Tensor] = None) -> Dict[FieldHeadNames, Tensor]:
        """fruit_field.py:234-281 (RGB + SEMANTICS); evaluated by the same fused kernel."""
        out = self.forward(ray_samples)
        return {k: v for k, v in out.items() if k != FieldHeadNames.DENSITY}

    def get_inference_outputs(self, ray_samples: RaySamples, density_embedding: Optional[Tensor] = None, render_rgb: bool = False):
        """fruit_field.py:195-232: mean appearance embedding regardless of train/eval."""
        shape, o, d, s, e, cam = self.ray_tensors(ray_samples)
        sd, srgb, ssem = ops.field(self.kernel_shape(), self.kernel_params(), o, d, s, e, None, self.position_mode(),
                                   L.FNR_APP_MEAN, impl=self.kernel_impl)
        return {FieldHeadNames.SEMANTICS: ssem.view(*shape, 1), FieldHeadNames.RGB: srgb.view(*shape, 3)}
