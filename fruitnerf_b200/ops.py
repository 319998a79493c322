"""PyTorch-facing ops of the native hot path: thin autograd wrappers over the C ABI.

PyTorch is plumbing here (device memory, streams, autograd bookkeeping); all arithmetic happens in
libfruitnerf_b200.so.  Every op requires CUDA tensors and raises otherwise -- there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib as L


@dataclass
class FieldShape:
    """Static shape of a FruitField as the kernels see it (fruit_nerf/fruit_field.py:70-166)."""

    num_levels: int
    features_per_level: int
    log2_hashmap_size: int
    scalings: Sequence[float]
    geo_feat_dim: int
    appearance_dim: int
    num_images: int
    base_dims: Sequence[int]
    semantic_dims: Sequence[int]
    color_dims: Sequence[int]
    aabb: Sequence[float]  # 6 floats: min xyz, max xyz
    pass_semantic_gradients: bool = False

    def desc(self, position_mode: int, appearance_mode: int, impl: int = L.FNR_IMPL_AUTO) -> L.FieldDesc:
        cache = self.__dict__.setdefault("_desc_cache", {})
        key = (position_mode, appearance_mode, impl)
        if key not in cache:
            cache[key] = self._make_desc(position_mode, appearance_mode, impl)
        return cache[key]

    def _make_desc(self, position_mode: int, appearance_mode: int, impl: int) -> L.FieldDesc:
        d = L.FieldDesc()
        d.num_levels = self.num_levels
        d.features_per_level = self.features_per_level
        d.log2_hashmap_size = self.log2_hashmap_size
        for i, s in enumerate(self.scalings):
            d.scalings[i] = float(s)
        d.geo_feat_dim = self.geo_feat_dim
        d.appearance_dim = self.appearance_dim
        d.num_images = self.num_images
        for m, dims in ((d.base, self.base_dims), (d.semantic, self.semantic_dims), (d.color, self.color_dims)):
            m.n_layers = len(dims) - 1
            for i, v in enumerate(dims):
                m.dims[i] = int(v)
        for i, v in enumerate(self.aabb):
            d.aabb[i] = float(v)
        d.position_mode = position_mode
        d.appearance_mode = appearance_mode
        d.pass_semantic_gradients = int(self.pass_semantic_gradients)
        d.impl = impl
        return d

    def param_layout(self) -> List[str]:
        """Fixed order of the parameter tensors passed to the ops."""
        names = ["hash_table"]
        for pre, dims in (("base", self.base_dims), ("sem", self.semantic_dims)):
            for i in range(len(dims) - 1):
                names += [f"{pre}_w{i}", f"{pre}_b{i}"]
        names += ["head_w", "head_b"]
        for i in range(len(self.color_dims) - 1):
            names += [f"col_w{i}", f"col_b{i}"]
        names.append("app_embedding")
        return names


def _ptr(t: Optional[Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _require_cuda(*ts: Optional[Tensor]) -> torch.device:
    dev = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise L.FruitNerfNativeError(
                "fruitnerf_b200 ops need CUDA tensors: the hot path is hand-written sm_90a CUDA with no CPU fallback"
            )
        dev = t.device
    return dev


def _f32c(t: Tensor) -> Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _params_struct(shape: FieldShape, tensors: Sequence[Tensor]) -> L.FieldParams:
    names = shape.param_layout()
    assert len(names) == len(tensors), (len(names), len(tensors))
    p = L.FieldParams()
    for name, t in zip(names, tensors):
        assert t.dtype == torch.float32 and t.is_contiguous(), name
        if name in ("hash_table", "head_w", "head_b", "app_embedding"):
            setattr(p, name, t.data_ptr())
        else:
            kind, idx = name[:-1], int(name[-1])  # e.g. base_w / 0
            getattr(p, kind)[idx] = t.data_ptr()
    return p


def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def flat_grad_numel(tensors: Sequence[Tensor]) -> int:
    """Elements of the flat gradient buffer of these parameters (every view 16-byte aligned)."""
    return sum((t.numel() + 3) // 4 * 4 for t in tensors)


def flat_zero_grads(tensors: Sequence[Tensor], out: Optional[Tensor] = None) -> Tuple[Tensor, List[Tensor]]:
    """One flat, zero-filled fp32 buffer with a 16-byte aligned view per parameter.  The backward
    kernels accumulate straight into it; the multi-GPU path all-reduces it in one collective.  ``out``: a persistent
    buffer of the caller (e.g. the symmetric allocation of the NVLS gradient exchange) that is re-zeroed instead of
    allocating a new one every step."""
    offs, total = [], 0
    for t in tensors:
        offs.append(total)
        total += (t.numel() + 3) // 4 * 4
    if out is not None:
        if out.dtype != torch.float32 or out.numel() < total or out.device != tensors[0].device or not out.is_contiguous():
            raise ValueError(f"flat gradient buffer must be contiguous fp32 with >= {total} elements on {tensors[0].device}")
        flat = out
        flat.zero_()
    else:
        flat = torch.zeros(total, dtype=torch.float32, device=tensors[0].device)
    views = [flat[o : o + t.numel()].view_as(t) for o, t in zip(offs, tensors)]
    return flat, views


class _Render(torch.autograd.Function):
    """Field forward (+ optional compositing) and its backward through the C ABI."""

    @staticmethod
    def forward(ctx, shape: FieldShape, mode: Dict, origins, directions, starts, ends, camera_indices, *params):
        dev = _require_cuda(origins, directions, starts, ends, *params)
        lib = L.load()
        ctx.set_materialize_grads(False)
        R, S = starts.shape[0], starts.shape[1]
        origins, directions, starts, ends = map(_f32c, (origins, directions, starts, ends))
        cam = None
        if camera_indices is not None:
            cam = camera_indices.reshape(-1)
            if cam.dtype != torch.int32:
                cam = cam.to(torch.int32)
            cam = cam.contiguous()
        params = [p.detach() for p in params]
        need_grad = any(ctx.needs_input_grad[7:])
        composite = mode["composite"]
        desc = shape.desc(mode["position_mode"], mode["appearance_mode"], mode["impl"])
        pstruct = _params_struct(shape, params)
        rays = L.RayBatch(R, S, _ptr(origins), _ptr(directions), _ptr(starts), _ptr(ends), _ptr(cam))

        f32 = dict(dtype=torch.float32, device=dev)
        sd = torch.empty((R, S), **f32)
        srgb = torch.empty((R, S, 3), **f32)
        ssem = torch.empty((R, S), **f32)
        stash = torch.empty((R, S, shape.num_levels * shape.features_per_level), **f32) if need_grad else None
        if composite:
            rgb = torch.empty((R, 3), **f32)
            acc = torch.empty((R,), **f32)
            depth = torch.empty((R,), **f32)
            didx = torch.empty((R,), dtype=torch.int32, device=dev)
            sem = torch.empty((R,), **f32)
            w = torch.empty((R, S), **f32)
        else:
            rgb = acc = depth = didx = sem = w = None
        out = L.RenderOut(_ptr(rgb), _ptr(acc), _ptr(depth), _ptr(didx), _ptr(sem), _ptr(w), _ptr(sd), _ptr(srgb),
                          _ptr(ssem), _ptr(stash), int(mode.get("clamp_rgb", False)))
        L.check(lib.fnr_render_forward(C.byref(desc), C.byref(pstruct), C.byref(rays), C.byref(out), _stream(dev)))

        ctx.shape, ctx.mode = shape, mode
        ctx.rs = (R, S)
        ctx.saved = (origins, directions, starts, ends, cam, params, sd, srgb, ssem, stash, w, acc)
        if composite:
            ctx.mark_non_differentiable(depth, didx)
            return rgb, acc, depth, didx, sem, w, sd, srgb, ssem
        return sd, srgb, ssem

    @staticmethod
    def backward(ctx, *g):
        lib = L.load()
        shape, mode = ctx.shape, ctx.mode
        origins, directions, starts, ends, cam, params, sd, srgb, ssem, stash, w, acc = ctx.saved
        dev = sd.device
        R, S = ctx.rs
        if mode["composite"]:
            g_rgb, g_acc, _, _, g_sem, g_w, g_sd, g_srgb, g_ssem = g
        else:
            g_sd, g_srgb, g_ssem = g
            g_rgb = g_acc = g_sem = g_w = None
        gs = [None if t is None else _f32c(t) for t in (g_rgb, g_acc, g_sem, g_w, g_sd, g_srgb, g_ssem)]
        desc = shape.desc(mode["position_mode"], mode["appearance_mode"], mode["impl"])
        pstruct = _params_struct(shape, params)
        flat, views = flat_zero_grads(params, out=mode.get("flat_grad"))
        gstruct = _params_struct(shape, views)
        rays = L.RayBatch(R, S, _ptr(origins), _ptr(directions), _ptr(starts), _ptr(ends), _ptr(cam))
        saved = L.RenderSaved(_ptr(w), _ptr(sd), _ptr(srgb), _ptr(ssem), _ptr(stash), _ptr(acc))
        up = L.RenderGrads(*[_ptr(t) for t in gs])
        nbytes = C.c_size_t(0)
        L.check(lib.fnr_render_backward_scratch_bytes(C.byref(desc), R, S, C.byref(nbytes)))
        scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        L.check(
            lib.fnr_render_backward(C.byref(desc), C.byref(pstruct), C.byref(rays), C.byref(saved), C.byref(up),
                                    C.byref(gstruct), scratch.data_ptr(), nbytes.value, _stream(dev))
        )
        _Render.last_flat_grad = flat
        return (None, None, None, None, None, None, None, *views)

    last_flat_grad: Optional[Tensor] = None


def render(shape: FieldShape, params: Sequence[Tensor], origins: Tensor, directions: Tensor, starts: Tensor, ends: Tensor,
           camera_indices: Optional[Tensor], position_mode: int, appearance_mode: int, clamp_rgb: bool = False,
           impl: int = L.FNR_IMPL_AUTO, flat_grad: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """Fused FruitField.forward + get_weights + renderers (fruit_nerf/fruit_nerf.py:320-348).

    origins/directions [R,3]; starts/ends [R,S]; camera_indices [R] or None.  ``flat_grad``: persistent flat gradient
    buffer the backward accumulates into (``flat_zero_grads``).
    """
    mode = dict(composite=True, position_mode=position_mode, appearance_mode=appearance_mode, clamp_rgb=clamp_rgb, impl=impl,
                flat_grad=flat_grad)
    rgb, acc, depth, didx, sem, w, sd, srgb, ssem = _Render.apply(shape, mode, origins, directions, starts, ends, camera_indices, *params)
    return {
        "rgb": rgb,
        "accumulation": acc,
        "depth": depth,
        "depth_index": didx,
        "semantics": sem,
        "weights": w,
        "sample_density": sd,
        "sample_rgb": srgb,
        "sample_semantics": ssem,
    }


def field(shape: FieldShape, params: Sequence[Tensor], origins: Tensor, directions: Tensor, starts: Tensor, ends: Tensor,
          camera_indices: Optional[Tensor], position_mode: int, appearance_mode: int, impl: int = L.FNR_IMPL_AUTO):
    """FruitField.forward (fruit_nerf/fruit_field.py:283-301): per-sample density, rgb, semantic logit."""
    mode = dict(composite=False, position_mode=position_mode, appearance_mode=appearance_mode, impl=impl)
    return _Render.apply(shape, mode, origins, directions, starts, ends, camera_indices, *params)


def hash_indices(shape: FieldShape, origins, directions, starts, ends, position_mode: int):
    """Hash-table rows [R,S,L,8] (nerfstudio corner order) and masked positions [R,S,3]."""
    dev = _require_cuda(origins, directions, starts, ends)
    lib = L.load()
    R, S = starts.shape
    origins, directions, starts, ends = map(_f32c, (origins, directions, starts, ends))
    rows = torch.empty((R, S, shape.num_levels, 8), dtype=torch.int32, device=dev)
    pos = torch.empty((R, S, 3), dtype=torch.float32, device=dev)
    desc = shape.desc(position_mode, L.FNR_APP_ZEROS)
    rays = L.RayBatch(R, S, _ptr(origins), _ptr(directions), _ptr(starts), _ptr(ends), None)
    L.check(lib.fnr_hash_indices(C.byref(desc), C.byref(rays), rows.data_ptr(), pos.data_ptr(), _stream(dev)))
    return rows, pos


class ExportBuffers:
    """Device-side compaction buffers of the volume export (three point sets, see include/)."""

    def __init__(self, capacity: int, device, dense: bool = False):
        self.capacity = capacity
        self.rows = [torch.empty((capacity, 7), dtype=torch.float32, device=device) for _ in range(3)]
        self.keys = [torch.empty((capacity,), dtype=torch.int64, device=device) for _ in range(3)]
        self.counts = torch.zeros(3, dtype=torch.int32, device=device)
        self.dense = dense


def export_batch(shape: FieldShape, params: Sequence[Tensor], origins: Tensor, normal: Sequence[float], bins: Tensor,
                 near: float, far: float, buffers: ExportBuffers, point_base: int = 0, dense_out: bool = False,
                 thresholds=(3.0, 70.0, 0.9), impl: int = L.FNR_IMPL_AUTO) -> Optional[Dict[str, Tensor]]:
    """One batch of FruitModel.get_export_outputs + the selection of sample_volume
    (fruit_nerf/fruit_nerf.py:251-269; fruit_nerf/export/exporter_utils.py:100-153)."""
    dev = _require_cuda(origins, bins, *params)
    lib = L.load()
    origins = _f32c(origins)
    bins = _f32c(bins)
    B = origins.shape[0]
    if bins.dim() == 2 and bins.shape[0] != 1:  # per-ray bins [B, S+1]: the sampler's stratified jitter (training-mode module)
        if bins.shape[0] != B:
            raise ValueError(f"per-ray bins need one row per ray: {tuple(bins.shape)} for {B} rays")
        S, stride = bins.shape[1] - 1, bins.shape[1]
    else:
        S, stride = bins.numel() - 1, 0
    params = [p.detach() for p in params]
    desc = shape.desc(L.FNR_POS_AABB, L.FNR_APP_MEAN, impl)
    pstruct = _params_struct(shape, params)
    xp = L.ExportParams(float(thresholds[0]), float(thresholds[1]), float(thresholds[2]), buffers.capacity, stride)
    out = L.ExportOut()
    for k in range(3):
        out.rows[k] = buffers.rows[k].data_ptr()
        out.keys[k] = buffers.keys[k].data_ptr()
    out.counts = buffers.counts.data_ptr()
    dense = None
    if dense_out:
        dense = {
            "rgb": torch.empty((B, S, 3), dtype=torch.float32, device=dev),
            "point_location": torch.empty((B, S, 3), dtype=torch.float32, device=dev),
            "semantics": torch.empty((B, S), dtype=torch.float32, device=dev),
            "density": torch.empty((B, S), dtype=torch.float32, device=dev),
            "semantics_colormap": torch.empty((B, S), dtype=torch.int64, device=dev),
        }
        out.sample_rgb = dense["rgb"].data_ptr()
        out.point_location = dense["point_location"].data_ptr()
        out.sample_semantics = dense["semantics"].data_ptr()
        out.sample_density = dense["density"].data_ptr()
        out.semantics_colormap = dense["semantics_colormap"].data_ptr()
    n3 = (C.c_float * 3)(*[float(v) for v in normal])
    L.check(
        lib.fnr_export_forward(C.byref(desc), C.byref(pstruct), origins.data_ptr(), n3, bins.data_ptr(), float(near),
                               float(far), B, S, int(point_base), C.byref(xp), C.byref(out), _stream(dev))
    )
    return dense


# ======================================================================================================
# Proposal-sampling stage (fruit_nerf/fruit_nerf.py:104-158, 318)
# ======================================================================================================
@dataclass
class DensityShape:
    """Static shape of a nerfstudio HashMLPDensityField as the kernels see it."""

    num_levels: int
    log2_hashmap_size: int
    hidden_dim: int
    scalings: Sequence[float]
    aabb: Sequence[float]

    def desc(self, position_mode: int) -> L.DensityDesc:
        cache = self.__dict__.setdefault("_desc_cache", {})
        if position_mode not in cache:
            d = L.DensityDesc()
            d.num_levels, d.log2_hashmap_size, d.hidden_dim = self.num_levels, self.log2_hashmap_size, self.hidden_dim
            for i, v in enumerate(self.scalings):
                d.scalings[i] = float(v)
            for i, v in enumerate(self.aabb):
                d.aabb[i] = float(v)
            d.position_mode = position_mode
            cache[position_mode] = d
        return cache[position_mode]


def _density_params(tensors: Sequence[Tensor]) -> L.DensityParams:
    p = L.DensityParams()
    p.hash_table, p.w0, p.b0, p.w1, p.b1 = [t.data_ptr() for t in tensors]
    return p


class _ProposalWeights(torch.autograd.Function):
    """HashMLPDensityField.density_fn(frustum midpoints) + RaySamples.get_weights, fused."""

    @staticmethod
    def forward(ctx, shape: DensityShape, position_mode: int, origins, directions, starts, ends, *params):
        dev = _require_cuda(origins, directions, starts, ends, *params)
        lib = L.load()
        R, S = starts.shape
        origins, directions, starts, ends = map(_f32c, (origins, directions, starts, ends))
        params = [p.detach() for p in params]
        density = torch.empty((R, S), dtype=torch.float32, device=dev)
        weights = torch.empty((R, S), dtype=torch.float32, device=dev)
        rays = L.RayBatch(R, S, _ptr(origins), _ptr(directions), _ptr(starts), _ptr(ends), None)
        desc = shape.desc(position_mode)
        L.check(lib.fnr_proposal_weights_forward(C.byref(desc), C.byref(_density_params(params)), C.byref(rays), density.data_ptr(),
                                                 weights.data_ptr(), _stream(dev)))
        ctx.shape, ctx.position_mode = shape, position_mode
        ctx.saved = (origins, directions, starts, ends, params, density, weights)
        return weights

    @staticmethod
    def backward(ctx, g_w):
        lib = L.load()
        origins, directions, starts, ends, params, density, weights = ctx.saved
        dev = density.device
        R, S = starts.shape
        flat, views = flat_zero_grads(params)
        rays = L.RayBatch(R, S, _ptr(origins), _ptr(directions), _ptr(starts), _ptr(ends), None)
        desc = ctx.shape.desc(ctx.position_mode)
        L.check(lib.fnr_proposal_weights_backward(C.byref(desc), C.byref(_density_params(params)), C.byref(rays), density.data_ptr(),
                                                  weights.data_ptr(), _f32c(g_w).data_ptr(), C.byref(_density_params(views)), _stream(dev)))
        return (None, None, None, None, None, None, *views)


def proposal_weights(shape: DensityShape, params: Sequence[Tensor], origins, directions, starts, ends, position_mode: int) -> Tensor:
    """weights [R,S] of one proposal level."""
    return _ProposalWeights.apply(shape, position_mode, origins, directions, starts, ends, *params)


_LINSPACE_CACHE: Dict = {}


def _linspace_cached(lo: float, hi: float, steps: int, dev) -> Tensor:
    key = (lo, hi, steps, str(dev))
    if key not in _LINSPACE_CACHE:
        _LINSPACE_CACHE[key] = torch.linspace(lo, hi, steps=steps, device=dev)
    return _LINSPACE_CACHE[key]


def pdf_sample(weights: Tensor, existing_bins: Tensor, num_samples: int, u_rand: Optional[Tensor], anneal: float, nears: Tensor, fars: Tensor,
               histogram_padding: float = 0.01):
    """PDFSampler + spacing->euclidean map.  Returns (new spacing bins [R,n+1], starts [R,n], ends [R,n]); no gradient
    flows through the sampler (the reference detaches the bins)."""
    dev = _require_cuda(weights, existing_bins, nears, fars)
    lib = L.load()
    R, S = weights.shape
    weights, existing_bins = _f32c(weights.detach()), _f32c(existing_bins.detach())
    nears, fars = _f32c(nears.reshape(-1)), _f32c(fars.reshape(-1))
    nb = num_samples + 1
    # as the reference: torch.linspace on the device the cdf lives on
    u_base = _linspace_cached(0.0, 1.0 - (1.0 / nb), nb, dev)
    stride = 0
    if u_rand is not None:
        u_rand = _f32c(u_rand)
        stride = 1 if u_rand.numel() == R else nb
    bins = torch.empty((R, nb), dtype=torch.float32, device=dev)
    starts = torch.empty((R, num_samples), dtype=torch.float32, device=dev)
    ends = torch.empty((R, num_samples), dtype=torch.float32, device=dev)
    anneal_dev = None
    if torch.is_tensor(anneal):  # device scalar: the schedule advances between CUDA-graph replays
        anneal_dev, anneal = _f32c(anneal), 1.0
    L.check(lib.fnr_pdf_sample(weights.data_ptr(), existing_bins.data_ptr(), R, S, num_samples, u_base.data_ptr(), _ptr(u_rand), stride,
                               float(anneal), _ptr(anneal_dev), float(histogram_padding), nears.data_ptr(), fars.data_ptr(), bins.data_ptr(),
                               starts.data_ptr(), ends.data_ptr(), _stream(dev)))
    return bins, starts, ends


class _InterlevelLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, c, w, cp, wp, mult: float):
        dev = _require_cuda(c, w, cp, wp)
        lib = L.load()
        R, Sc = w.shape
        Sp = wp.shape[1]
        c, w, cp, wpc = map(_f32c, (c.detach(), w.detach(), cp.detach(), wp.detach()))
        loss = torch.zeros((), dtype=torch.float32, device=dev)
        d_wp = torch.empty((R, Sp), dtype=torch.float32, device=dev) if ctx.needs_input_grad[3] else None
        L.check(lib.fnr_interlevel_loss(c.data_ptr(), w.data_ptr(), cp.data_ptr(), wpc.data_ptr(), R, Sc, Sp, float(mult), loss.data_ptr(),
                                        _ptr(d_wp), _stream(dev)))
        ctx.d_wp = d_wp
        return loss

    @staticmethod
    def backward(ctx, g):
        return None, None, None, (ctx.d_wp * g if ctx.d_wp is not None else None), None


def interlevel_loss(weights_list: Sequence[Tensor], sdist_list: Sequence[Tensor], mult: float = 1.0) -> Tensor:
    """nerfstudio losses.interlevel_loss: weights_list[i] [R,S_i], sdist_list[i] [R,S_i+1]; the last entry is the final level."""
    c, w = sdist_list[-1], weights_list[-1]
    total = None
    for sdist, wp in zip(sdist_list[:-1], weights_list[:-1]):
        term = _InterlevelLoss.apply(c, w, sdist, wp, mult)
        total = term if total is None else total + term
    if total is None:
        total = torch.zeros((), dtype=torch.float32, device=w.device)
    return total


# ======================================================================================================
# Per-ray glue of a training iteration (fnr_glue.cu): one launch each instead of dozens of torch kernels
# ======================================================================================================
def pixel_batch(rand: Tensor, c2w: Tensor, images: Tensor, masks: Tensor, fx: float, fy: float, cx: float, cy: float):
    """PixelSampler.sample + RayGenerator (fruit_datamanager.py:183-192).  Returns origins, directions [R,3], camera_indices
    [R] int32, indices [R,3] int64, image [R,3], fruit_mask [R,1]."""
    dev = _require_cuda(rand, c2w, images, masks)
    R = rand.shape[0]
    N, H, W = images.shape[0], images.shape[1], images.shape[2]
    rand, c2w, images, masks = _f32c(rand), _f32c(c2w), _f32c(images), _f32c(masks)
    f32 = dict(dtype=torch.float32, device=dev)
    o, d, img, m = torch.empty((R, 3), **f32), torch.empty((R, 3), **f32), torch.empty((R, 3), **f32), torch.empty((R, 1), **f32)
    cam = torch.empty((R,), dtype=torch.int32, device=dev)
    idx = torch.empty((R, 3), dtype=torch.int64, device=dev)
    L.check(L.load().fnr_pixel_batch(rand.data_ptr(), c2w.data_ptr(), images.data_ptr(), masks.data_ptr(), N, H, W, float(fx), float(fy),
                                     float(cx), float(cy), R, o.data_ptr(), d.data_ptr(), cam.data_ptr(), idx.data_ptr(), img.data_ptr(),
                                     m.data_ptr(), _stream(dev)))
    return o, d, cam, idx, img, m


def spaced_bins(base_bins: Tensor, t_rand: Optional[Tensor], nears: Tensor, fars: Tensor, num_samples: int, mode: int):
    """SpacedSampler bins (spacing space) + euclidean starts / ends.  base_bins [S+1] (host-made linspace, already on the device)."""
    dev = _require_cuda(base_bins, nears, fars)
    R = nears.reshape(-1).shape[0]
    nears, fars = _f32c(nears.reshape(-1)), _f32c(fars.reshape(-1))
    stride = 0
    if t_rand is not None:
        t_rand = _f32c(t_rand)
        stride = 1 if t_rand.numel() == R else num_samples + 1
    f32 = dict(dtype=torch.float32, device=dev)
    bins, starts, ends = torch.empty((R, num_samples + 1), **f32), torch.empty((R, num_samples), **f32), torch.empty((R, num_samples), **f32)
    L.check(L.load().fnr_spaced_bins(_f32c(base_bins.reshape(-1)).data_ptr(), _ptr(t_rand), stride, nears.data_ptr(), fars.data_ptr(), R, num_samples,
                                     mode, bins.data_ptr(), starts.data_ptr(), ends.data_ptr(), _stream(dev)))
    return bins, starts, ends


class _RenderLosses(torch.autograd.Function):
    """(MSE(image, rgb), weight * BCEWithLogits(semantics, mask), PSNR) with the gradients produced by the same launch."""

    @staticmethod
    def forward(ctx, rgb, semantics, image, fruit_mask, weight: float):
        dev = _require_cuda(rgb, semantics, image, fruit_mask)
        R = rgb.shape[0]
        rgb_c, sem_c = _f32c(rgb.detach()), _f32c(semantics.detach().reshape(-1))
        out = torch.empty(4, dtype=torch.float32, device=dev)
        need = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        d_rgb = torch.empty_like(rgb_c) if need else None
        d_sem = torch.empty_like(sem_c) if need else None
        L.check(L.load().fnr_render_losses(rgb_c.data_ptr(), sem_c.data_ptr(), _f32c(image).data_ptr(), _f32c(fruit_mask.reshape(-1)).data_ptr(), R,
                                           float(weight), out.data_ptr(), _ptr(d_rgb), _ptr(d_sem), _stream(dev)))
        ctx.saved = (d_rgb, d_sem, semantics.shape)
        ctx.mark_non_differentiable(out)
        return out[0], out[1], out
    # out[0] / out[1] are views of `out`: returned as separate 0-d tensors that carry the graph

    @staticmethod
    def backward(ctx, g_mse, g_bce, _g_out):
        d_rgb, d_sem, sem_shape = ctx.saved
        gr = d_rgb * g_mse if (g_mse is not None and ctx.needs_input_grad[0]) else None
        gs = (d_sem * g_bce).view(sem_shape) if (g_bce is not None and ctx.needs_input_grad[1]) else None
        return gr, gs, None, None, None


def render_losses(rgb: Tensor, semantics: Tensor, image: Tensor, fruit_mask: Tensor, semantic_weight: float = 1.0):
    """Returns (rgb_loss, semantics_loss, psnr): nn.MSELoss, semantic_weight * nn.BCEWithLogitsLoss(mean), -10 log10(mse)."""
    mse, bce, out = _RenderLosses.apply(rgb, semantics, image, fruit_mask, semantic_weight)
    return mse, bce, out[2]


def distortion_metric(weights: Tensor, sdist: Tensor) -> Tensor:
    """nerfstudio distortion_loss([weights], [ray_samples]) for one level, mean over rays (no gradient: a logged metric)."""
    dev = _require_cuda(weights, sdist)
    R, S = weights.shape
    out = torch.zeros((), dtype=torch.float32, device=dev)
    L.check(L.load().fnr_ray_metrics(_f32c(weights.detach()).data_ptr(), _f32c(sdist.detach()).data_ptr(), None, None, R, S, out.data_ptr(), None,
                                     _stream(dev)))
    return out


def median_depth(weights: Tensor, starts: Tensor, ends: Tensor) -> Tensor:
    """DepthRenderer(method="median") of one level: [R,1]."""
    dev = _require_cuda(weights, starts, ends)
    R, S = weights.shape
    depth = torch.empty((R, 1), dtype=torch.float32, device=dev)
    L.check(L.load().fnr_ray_metrics(_f32c(weights.detach()).data_ptr(), None, _f32c(starts.detach()).data_ptr(), _f32c(ends.detach()).data_ptr(), R, S,
                                     None, depth.data_ptr(), _stream(dev)))
    return depth


# ======================================================================================================
# Fruit counting on the exported cloud (fnr_cluster.cu; clustering/clustering_base.py:138-143, 183-259)
# ======================================================================================================
def cluster_points(points: Tensor) -> Tensor:
    """[n,3] fp64 contiguous copy/view of a CUDA point tensor (float32 is upcast).  Non-finite coordinates raise ValueError."""
    _require_cuda(points)
    pts = points.detach().reshape(-1, 3)
    if pts.dtype != torch.float64:
        pts = pts.double()
    pts = pts.contiguous()
    if pts.shape[0] and not bool(torch.isfinite(pts).all()):
        raise ValueError("point cloud has non-finite coordinates")
    return pts


def _bounds(pts: Tensor):
    """Per-axis minimum and maximum as host double[3] arrays: the grid origin and extent of fnr_cluster.cu."""
    if pts.shape[0] == 0:
        return None, None
    lo, hi = torch.aminmax(pts, dim=0)
    b = torch.stack([lo, hi]).cpu().tolist()
    return (C.c_double * 3)(*b[0]), (C.c_double * 3)(*b[1])


def _cluster_scratch(n: int, dev) -> Tensor:
    nbytes = C.c_size_t(0)
    L.check(L.load().fnr_cluster_scratch_bytes(n, C.byref(nbytes)))
    return torch.empty(nbytes.value, dtype=torch.uint8, device=dev)


def radius_count(points: Tensor, radius: float, cap: int) -> Tensor:
    """int32 [n]: min(cap, number of points within ``radius`` of each point, itself included) -- the
    NearestNeighbors(radius).radius_neighbors list lengths, saturated."""
    pts = cluster_points(points)
    n, dev = pts.shape[0], pts.device
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    lo, hi = _bounds(pts)
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_radius_count(_ptr(pts), n, lo, hi, float(radius), int(cap), _ptr(counts), _ptr(scratch), scratch.numel(),
                                      _stream(dev)))
    return counts


def voxel_down_sample(points: Tensor, voxel: float) -> Tensor:
    """[m,3] fp64: clustering.voxel_down_sample bit for bit (one mean per occupied voxel, lexicographic voxel order)."""
    pts = cluster_points(points)
    n, dev = pts.shape[0], pts.device
    if n == 0 or voxel <= 0:
        return pts
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    num = torch.zeros(1, dtype=torch.int32, device=dev)
    lo, hi = _bounds(pts)
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_voxel_down_sample(_ptr(pts), n, lo, hi, float(voxel), _ptr(out), _ptr(num), _ptr(scratch), scratch.numel(),
                                           _stream(dev)))
    return out[: int(num.item())]


def dbscan(points: Tensor, eps: float, min_samples: int) -> Tuple[Tensor, int]:
    """(labels int32 [n], number of clusters): sklearn.cluster.DBSCAN(eps, min_samples).labels_, noise = -1."""
    pts = cluster_points(points)
    n, dev = pts.shape[0], pts.device
    labels = torch.empty(n, dtype=torch.int32, device=dev)
    num = torch.zeros(1, dtype=torch.int32, device=dev)
    lo, hi = _bounds(pts)
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_dbscan(_ptr(pts), n, lo, hi, float(eps), int(min_samples), _ptr(labels), _ptr(num), _ptr(scratch),
                                scratch.numel(), _stream(dev)))
    return labels, int(num.item())


def cluster_sums(points: Tensor, labels: Tensor, num_clusters: int) -> Tuple[Tensor, Tensor]:
    """(fp64 coordinate sums [K,3], int32 point counts [K]) of the labels 0..K-1 (deterministic)."""
    pts = cluster_points(points)
    _require_cuda(labels)
    n, dev = pts.shape[0], pts.device
    labels = labels.reshape(-1).to(torch.int32).contiguous()
    if labels.shape[0] != n:
        raise ValueError(f"{labels.shape[0]} labels for {n} points")
    sums = torch.zeros((num_clusters, 3), dtype=torch.float64, device=dev)
    counts = torch.zeros(num_clusters, dtype=torch.int32, device=dev)
    if num_clusters == 0:
        return sums, counts
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_cluster_sums(_ptr(pts), _ptr(labels), n, int(num_clusters), _ptr(sums), _ptr(counts), _ptr(scratch),
                                      scratch.numel(), _stream(dev)))
    return sums, counts


# ======================================================================================================
# The `pointcloud` export (fnr_cluster.cu; nerfstudio ExportPointCloud / generate_point_cloud)
# ======================================================================================================
def knn_mean_distance(points: Tensor, k: int) -> Tensor:
    """fp64 [n]: mean Euclidean distance to the min(k, n) nearest neighbours, the point itself included, summed in
    ascending order (open3d remove_statistical_outlier's per-point statistic)."""
    pts = cluster_points(points)
    n, dev = pts.shape[0], pts.device
    out = torch.empty(n, dtype=torch.float64, device=dev)
    lo, hi = _bounds(pts)
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_knn_mean_distance(_ptr(pts), n, lo, hi, int(k), _ptr(out), _ptr(scratch), scratch.numel(), _stream(dev)))
    return out


def estimate_normals(points: Tensor, k: int, view_dirs: Optional[Tensor] = None) -> Tensor:
    """fp64 [n,3] unit normals from the min(k, n) nearest neighbours (open3d estimate_normals with KNN(k)); with
    ``view_dirs`` [n,3], normals facing along their view direction (fp32 dot product > 0) are flipped."""
    pts = cluster_points(points)
    n, dev = pts.shape[0], pts.device
    if view_dirs is not None:
        _require_cuda(view_dirs)
        view_dirs = _f32c(view_dirs.detach().reshape(-1, 3))
        if view_dirs.shape[0] != n:
            raise ValueError(f"{view_dirs.shape[0]} view directions for {n} points")
    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    lo, hi = _bounds(pts)
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_estimate_normals(_ptr(pts), n, lo, hi, int(k), _ptr(view_dirs), _ptr(out), _ptr(scratch), scratch.numel(),
                                          _stream(dev)))
    return out


class PointBuffers:
    """Device rows a point-cloud export appends to: xyz, rgb and view direction ([capacity,3] fp32 each) and the
    running row count (a device int32)."""

    def __init__(self, capacity: int, device):
        f32 = dict(dtype=torch.float32, device=device)
        self.capacity = capacity
        self.points = torch.empty((capacity, 3), **f32)
        self.colors = torch.empty((capacity, 3), **f32)
        self.view_dirs = torch.empty((capacity, 3), **f32)
        self.count = torch.zeros(1, dtype=torch.int32, device=device)


def backproject_select(origins: Tensor, directions: Tensor, depth: Tensor, rgb: Tensor, accumulation: Tensor, buffers: PointBuffers,
                       bounding_box=None) -> None:
    """Appends the rays of one rendered batch with accumulation > 0.5 (and, with ``bounding_box`` = (min xyz, max xyz),
    their point strictly inside it) to ``buffers`` in ray order: point = origin + direction * depth in fp32."""
    dev = _require_cuda(origins, directions, depth, rgb, accumulation)
    R = origins.reshape(-1, 3).shape[0]
    o, d, c = (_f32c(t.detach().reshape(-1, 3)) for t in (origins, directions, rgb))
    t, a = (_f32c(x.detach().reshape(-1)) for x in (depth, accumulation))
    if not (d.shape[0] == c.shape[0] == t.shape[0] == a.shape[0] == R):
        raise ValueError("origins, directions, depth, rgb and accumulation must describe the same rays")
    bmin = bmax = None
    if bounding_box is not None:
        bmin = (C.c_float * 3)(*[float(v) for v in bounding_box[0]])
        bmax = (C.c_float * 3)(*[float(v) for v in bounding_box[1]])
    L.check(L.load().fnr_backproject_select(_ptr(o), _ptr(d), _ptr(t), _ptr(c), _ptr(a), R, int(bounding_box is not None), bmin, bmax,
                                            buffers.capacity, _ptr(buffers.points), _ptr(buffers.colors), _ptr(buffers.view_dirs),
                                            _ptr(buffers.count), _stream(dev)))


# ======================================================================================================
# Stage 3 of the fruit count (fnr_fruit_split.cu; clustering/clustering_base.py:261-429)
# ======================================================================================================
def _segments(bounds, num: int, what: str) -> Tuple[np.ndarray, int]:
    """Host int64 segment bounds checked against ``num`` rows, and the largest segment."""
    b = np.asarray(bounds.cpu() if isinstance(bounds, Tensor) else bounds, dtype=np.int64)
    lo, hi = (b[:-1], b[1:]) if b.ndim == 1 else (b[:, 0], b[:, 1])
    if b.ndim not in (1, 2) or (b.ndim == 2 and b.shape[1] != 2) or bool((lo < 0).any()) or bool((hi > num).any()) or bool((hi < lo).any()):
        raise ValueError(f"{what}: segment bounds must be ascending offsets or (begin, end) rows within {num} rows")
    return b, int((hi - lo).max(initial=0))


def icp_scaled(source: Tensor, targets: Tensor, target_offsets, init_translation: Tensor, max_distance: float = 0.01,
               max_iteration: int = 2000, relative_fitness: float = 1e-6, relative_rmse: float = 1e-6):
    """Scaled point-to-point ICP of one ``source`` cloud [m,3] onto each target segment (rows target_offsets[b] ..
    target_offsets[b+1] of ``targets``), starting from a translation ``init_translation`` [B,3]: clustering.icp_scaled
    batched.  ``target_offsets``: host sequence of B+1 ascending ints.  Returns (transforms [B,4,4] fp64, fitness [B],
    rmse [B], iterations [B] int32)."""
    src, tgt, init = cluster_points(source), cluster_points(targets), cluster_points(init_translation)
    dev = tgt.device
    offs, max_n = _segments(target_offsets, tgt.shape[0], "icp_scaled")
    B = offs.shape[0] - 1
    if init.shape[0] != B:
        raise ValueError(f"{init.shape[0]} initial translations for {B} problems")
    if B and (offs[1:] == offs[:-1]).any():
        raise ValueError("icp_scaled: every target segment needs at least one point")
    T = torch.empty((B, 4, 4), dtype=torch.float64, device=dev)
    fitness, rmse = torch.empty(B, dtype=torch.float64, device=dev), torch.empty(B, dtype=torch.float64, device=dev)
    iters = torch.empty(B, dtype=torch.int32, device=dev)
    offs_d = torch.from_numpy(offs).to(dev)
    L.check(L.load().fnr_icp_scaled(_ptr(src), src.shape[0], _ptr(tgt), _ptr(offs_d), B, max(max_n, 1), _ptr(init), float(max_distance),
                                    int(max_iteration), float(relative_fitness), float(relative_rmse), _ptr(T), _ptr(fitness), _ptr(rmse),
                                    _ptr(iters), _stream(dev)))
    return T, fitness, rmse, iters


def ward_cut(points: Tensor, offsets) -> Tensor:
    """clustering.ward_cut_centres for each segment (rows offsets[b] .. offsets[b+1] of ``points``; at most 4096 rows,
    more raise the library's unsupported error): [B,20,3] fp64.  ``offsets``: host sequence of B+1 ascending ints."""
    pts = cluster_points(points)
    dev = pts.device
    offs, max_n = _segments(offsets, pts.shape[0], "ward_cut")
    B = offs.shape[0] - 1
    out = torch.empty((B, 20, 3), dtype=torch.float64, device=dev)
    offs_d = torch.from_numpy(offs).to(dev)
    L.check(L.load().fnr_ward_cut(_ptr(pts), _ptr(offs_d), B, max(max_n, 1), _ptr(out), _stream(dev)))
    return out


def hausdorff(a: Tensor, a_ranges, b: Tensor, b_ranges) -> Tensor:
    """Symmetric Hausdorff distances [P] fp64 of the pairs (rows a_ranges[p] of ``a``, rows b_ranges[p] of ``b``):
    clustering.hausdorff batched, bit for bit.  Ranges: host [P,2] (begin, end) ints; empty sets raise ValueError."""
    pa, pb = cluster_points(a), cluster_points(b)
    dev = pa.device
    ra, _ = _segments(a_ranges, pa.shape[0], "hausdorff")
    rb, _ = _segments(b_ranges, pb.shape[0], "hausdorff")
    if ra.ndim != 2 or rb.ndim != 2 or ra.shape[0] != rb.shape[0]:
        raise ValueError("hausdorff: a_ranges and b_ranges must both be [P,2]")
    if (ra[:, 1] == ra[:, 0]).any() or (rb[:, 1] == rb[:, 0]).any():
        raise ValueError("hausdorff: every set needs at least one point")
    P = ra.shape[0]
    out = torch.empty(P, dtype=torch.float64, device=dev)
    ra_d, rb_d = torch.from_numpy(np.ascontiguousarray(ra)).to(dev), torch.from_numpy(np.ascontiguousarray(rb)).to(dev)
    L.check(L.load().fnr_hausdorff(_ptr(pa), _ptr(ra_d), _ptr(pb), _ptr(rb_d), P, _ptr(out), _stream(dev)))
    return out


# ======================================================================================================
# Novel-view rendering (fnr_render.cu; nerfstudio ns-render, the reference's debug/render.py)
# ======================================================================================================
CAMERA_TYPES = {"perspective": L.FNR_CAMERA_PERSPECTIVE, "fisheye": L.FNR_CAMERA_FISHEYE, "equirectangular": L.FNR_CAMERA_EQUIRECTANGULAR}


def camera_rays(c2w: Tensor, fx: Tensor, fy: Tensor, cx: Tensor, cy: Tensor, camera_type: str, height: int, width: int, frame: int,
                pixel_start: int, num_pixels: int, out: Optional[Tuple[Tensor, Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """Origins and unit directions [n,3] of pixels [pixel_start, pixel_start + n) (row-major) of frame ``frame`` of a camera
    set: c2w [F,3,4] (CUDA, fp32), per-frame fx / fy / cx / cy [F] (CUDA, taken as fp64).  ``out``: preallocated (origins, directions) with at
    least n rows, of which the first n are written and returned."""
    dev = _require_cuda(c2w, fx, fy, cx, cy)
    if camera_type not in CAMERA_TYPES:
        raise ValueError(f"camera_type must be one of {sorted(CAMERA_TYPES)}, got {camera_type!r}")
    c2w = _f32c(c2w)
    fx, fy, cx, cy = (t.to(torch.float64).contiguous() for t in (fx, fy, cx, cy))
    F = c2w.shape[0]
    if c2w.shape[1:] != (3, 4) or not (fx.numel() == fy.numel() == cx.numel() == cy.numel() == F):
        raise ValueError(f"c2w must be [F,3,4] with F intrinsics each, got {tuple(c2w.shape)} and {fx.numel()} fx")
    if out is None:
        o = torch.empty((num_pixels, 3), dtype=torch.float32, device=dev)
        d = torch.empty((num_pixels, 3), dtype=torch.float32, device=dev)
    else:
        _require_cuda(*out)
        o, d = out[0][:num_pixels], out[1][:num_pixels]
        if o.shape != (num_pixels, 3) or d.shape != (num_pixels, 3) or not (o.is_contiguous() and d.is_contiguous()):
            raise ValueError("out buffers must be contiguous fp32 [>= n, 3]")
    L.check(L.load().fnr_camera_rays(_ptr(c2w), _ptr(fx), _ptr(fy), _ptr(cx), _ptr(cy), F, CAMERA_TYPES[camera_type], int(height), int(width),
                                     int(frame), int(pixel_start), int(num_pixels), _ptr(o), _ptr(d), _stream(dev)))
    return o, d


@dataclass
class FrameImage:
    """One requested output of a frame for ``compose_frame``: ``image`` [H*W, 3] (kind "color") or [H*W] / [H*W,1]
    ("turbo", "depth"); depth ``near`` / ``far`` of None take the frame's own min / max."""

    image: Tensor
    kind: str
    near: Optional[float] = None
    far: Optional[float] = None


_FRAME_KINDS = {"color": L.FNR_FRAME_COLOR, "turbo": L.FNR_FRAME_TURBO, "depth": L.FNR_FRAME_DEPTH}


def compose_frame(images: Sequence[FrameImage], accumulation: Optional[Tensor], height: int, width: int, turbo: Tensor,
                  scratch: Optional[Tensor] = None, out: Optional[Tensor] = None) -> Tensor:
    """uint8 [H, W*k, 3] on the device: every image colour-mapped (nerfstudio apply_colormap / apply_depth_colormap),
    side by side, quantised as uint8(clip(x, 0, 1) * 255 + 0.5).  ``turbo``: [256,3] CUDA fp32 table."""
    k = len(images)
    if not 1 <= k <= L.FNR_MAX_FRAME_OUTPUTS:
        raise ValueError(f"compose_frame takes 1..{L.FNR_MAX_FRAME_OUTPUTS} images, got {k}")
    dev = _require_cuda(turbo, accumulation, *[im.image for im in images])
    P = height * width
    arr = (L.FrameOutput * k)()
    keep = []
    any_auto = False
    for j, im in enumerate(images):
        if im.kind not in _FRAME_KINDS:
            raise ValueError(f"unknown frame image kind {im.kind!r}")
        t = _f32c(im.image)
        want = 3 * P if im.kind == "color" else P
        if t.numel() != want:
            raise ValueError(f"{im.kind} image {j} has {t.numel()} values, expected {want} for {width}x{height}")
        keep.append(t)
        auto = (L.FNR_RANGE_AUTO_NEAR if im.near is None else 0) | (L.FNR_RANGE_AUTO_FAR if im.far is None else 0) if im.kind == "depth" else 0
        any_auto |= auto != 0
        arr[j] = L.FrameOutput(t.data_ptr(), _FRAME_KINDS[im.kind], auto, float(im.near or 0.0), float(im.far or 0.0))
    acc = None if accumulation is None else _f32c(accumulation)
    if acc is not None and acc.numel() != P:
        raise ValueError(f"accumulation has {acc.numel()} values for {width}x{height}")
    turbo = _f32c(turbo)
    if turbo.numel() != 768:
        raise ValueError("turbo table must be [256,3]")
    if any_auto and scratch is None:
        scratch = torch.empty(L.FNR_COMPOSE_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
    if out is None:
        out = torch.empty((height, width * k, 3), dtype=torch.uint8, device=dev)
    elif out.dtype != torch.uint8 or out.shape != (height, width * k, 3) or not out.is_contiguous():
        raise ValueError(f"out must be contiguous uint8 [{height}, {width * k}, 3]")
    L.check(L.load().fnr_compose_frame(arr, k, _ptr(acc), int(height), int(width), _ptr(turbo), _ptr(scratch), _ptr(out), _stream(dev)))
    return out
