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


def pixel_batch_lens(rand: Tensor, c2w: Tensor, images: Tensor, masks: Tensor, fx: Tensor, fy: Tensor, cx: Tensor, cy: Tensor,
                     distortion: Optional[Tensor], camera_type: str):
    """``pixel_batch`` for lens cameras (DESIGN.md section 4.3j): per-image fx / fy / cx / cy [N] and distortion [N,6] (k1 k2 k3 k4
    p1 p2, or None), all fp32 on the device, and a camera type of ``CAMERA_TYPES``.  Same outputs as ``pixel_batch``.  Nothing
    here reads device memory, so the call can be captured in a CUDA graph: the values are checked when the data set is
    moved to the device (``SyntheticCameras.to``)."""
    dev = _require_cuda(rand, c2w, images, masks, fx, fy, cx, cy, distortion)
    if camera_type not in CAMERA_TYPES:
        raise ValueError(f"camera_type must be one of {sorted(CAMERA_TYPES)}, got {camera_type!r}")
    R = rand.shape[0]
    N, H, W = images.shape[0], images.shape[1], images.shape[2]
    fx, fy, cx, cy = (_f32c(t.reshape(-1)) for t in (fx, fy, cx, cy))
    if not (fx.numel() == fy.numel() == cx.numel() == cy.numel() == N) or (distortion is not None and tuple(distortion.shape) != (N, 6)):
        raise ValueError(f"lens cameras need [N] intrinsics and [N,6] distortion for N = {N} images")
    distortion = None if distortion is None else _f32c(distortion)
    rand, c2w, images, masks = _f32c(rand), _f32c(c2w), _f32c(images), _f32c(masks)
    f32 = dict(dtype=torch.float32, device=dev)
    o, d, img, m = torch.empty((R, 3), **f32), torch.empty((R, 3), **f32), torch.empty((R, 3), **f32), torch.empty((R, 1), **f32)
    cam = torch.empty((R,), dtype=torch.int32, device=dev)
    idx = torch.empty((R, 3), dtype=torch.int64, device=dev)
    L.check(L.load().fnr_pixel_batch_lens(rand.data_ptr(), c2w.data_ptr(), images.data_ptr(), masks.data_ptr(), N, H, W, fx.data_ptr(),
                                          fy.data_ptr(), cx.data_ptr(), cy.data_ptr(), _ptr(distortion), CAMERA_TYPES[camera_type], R,
                                          o.data_ptr(), d.data_ptr(), cam.data_ptr(), idx.data_ptr(), img.data_ptr(), m.data_ptr(), _stream(dev)))
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


def _host_radii(radii, caps, what: str):
    """(double[R], int32[R], R) host arrays of the multi-radius calls; the library checks the values."""
    r, c = [float(v) for v in radii], [int(v) for v in caps]
    if len(r) != len(c):
        raise ValueError(f"{what}: {len(r)} radii for {len(c)} caps")
    return (C.c_double * max(len(r), 1))(*r), (C.c_int32 * max(len(c), 1))(*c), len(r)


def radius_count_multi(points: Tensor, radii: Sequence[float], caps: Sequence[int]) -> Tensor:
    """int32 [R,n]: row k is ``radius_count(points, radii[k], caps[k])``, bit for bit, from one grid walk (1 <= R <= 16,
    max(radii) <= 4 min(radii))."""
    pts = cluster_points(points)
    n, dev = pts.shape[0], pts.device
    r, c, R = _host_radii(radii, caps, "radius_count_multi")
    counts = torch.empty((R, n), dtype=torch.int32, device=dev)
    lo, hi = _bounds(pts)
    scratch = _cluster_scratch(n, dev)
    L.check(L.load().fnr_radius_count_multi(_ptr(pts), n, lo, hi, r, c, R, _ptr(counts), _ptr(scratch), scratch.numel(), _stream(dev)))
    return counts


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


def camera_rays_lens(c2w: Tensor, fx: Tensor, fy: Tensor, cx: Tensor, cy: Tensor, distortion: Optional[Tensor], camera_type: str, height: int,
                     width: int, frame: int, pixel_start: int, num_pixels: int) -> Tuple[Tensor, Tensor]:
    """``camera_rays`` for lens cameras: fp32 fx / fy / cx / cy [F] and distortion [F,6] or None on the device.  The ray of pixel
    (frame, y, x) is bit-identical to the one ``pixel_batch_lens`` draws for it."""
    dev = _require_cuda(c2w, fx, fy, cx, cy, distortion)
    if camera_type not in CAMERA_TYPES:
        raise ValueError(f"camera_type must be one of {sorted(CAMERA_TYPES)}, got {camera_type!r}")
    c2w = _f32c(c2w)
    F = c2w.shape[0]
    fx, fy, cx, cy = (_f32c(t.reshape(-1)) for t in (fx, fy, cx, cy))
    if c2w.shape[1:] != (3, 4) or not (fx.numel() == fy.numel() == cx.numel() == cy.numel() == F) or (
            distortion is not None and tuple(distortion.shape) != (F, 6)):
        raise ValueError(f"c2w must be [F,3,4] with F intrinsics each and [F,6] distortion, got {tuple(c2w.shape)} and {fx.numel()} fx")
    distortion = None if distortion is None else _f32c(distortion)
    o = torch.empty((num_pixels, 3), dtype=torch.float32, device=dev)
    d = torch.empty((num_pixels, 3), dtype=torch.float32, device=dev)
    L.check(L.load().fnr_camera_rays_lens(_ptr(c2w), _ptr(fx), _ptr(fy), _ptr(cx), _ptr(cy), _ptr(distortion), F, CAMERA_TYPES[camera_type],
                                          int(height), int(width), int(frame), int(pixel_start), int(num_pixels), _ptr(o), _ptr(d), _stream(dev)))
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


# ======================================================================================================
# Surface meshes (fnr_mesh.cu; nerfstudio ns-export tsdf)
# ======================================================================================================
def _host3(v, what: str):
    """HOST float[3] of a per-axis value (a scalar, three values or a tensor)."""
    a = [float(x) for x in (v.detach().cpu().reshape(-1).tolist() if torch.is_tensor(v) else np.asarray(v, dtype=np.float64).reshape(-1))]
    if len(a) == 1:
        a = a * 3
    if len(a) != 3:
        raise ValueError(f"{what} must be one or three values, got {len(a)}")
    return (C.c_float * 3)(*a)


def _grid_dims(values: Tensor) -> Tuple[int, int, int]:
    if values.dim() != 3 or values.dtype != torch.float32 or not values.is_contiguous():
        raise ValueError(f"grid values must be a contiguous fp32 [X,Y,Z] tensor, got {values.dtype} {tuple(values.shape)}")
    return tuple(int(d) for d in values.shape)


def tsdf_integrate(values: Tensor, weights: Tensor, colors: Tensor, fruit_state: Optional[Tensor], origin, voxel_size, truncation: float,
                   c2w: Tensor, fx, fy, cx, cy, depth: Tensor, rgb: Tensor, fruit: Optional[Tensor] = None) -> None:
    """Fuse B frames into a TSDF grid in place (fnr_tsdf_integrate): state ``values`` / ``weights`` / ``fruit_state`` [X,Y,Z]
    and ``colors`` [X,Y,Z,3], contiguous fp32 CUDA tensors; frames c2w [B,3,4], fx / fy / cx / cy [B] (or scalars),
    depth [B,H,W] (ray distance), rgb [B,H,W,3], fruit [B,H,W] or None."""
    dev = _require_cuda(values, weights, colors, fruit_state, c2w, depth, rgb, fruit)
    X, Y, Z = _grid_dims(values)
    for name, t, shape in (("weights", weights, (X, Y, Z)), ("colors", colors, (X, Y, Z, 3)), ("fruit_state", fruit_state, (X, Y, Z))):
        if t is not None and (tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous fp32 {list(shape)} tensor")
    if fruit is not None and fruit_state is None:
        raise ValueError("frame fruit probabilities need a fruit_state grid")
    B = int(c2w.shape[0])
    c2w = _f32c(c2w.detach().reshape(B, 3, 4))
    depth = _f32c(depth.detach())
    H, W = int(depth.shape[1]), int(depth.shape[2])
    depth = depth.reshape(B, H, W)
    rgb = _f32c(rgb.detach().reshape(B, H, W, 3))
    fruit = None if fruit is None else _f32c(fruit.detach().reshape(B, H, W))
    fx, fy, cx, cy = (_f32c(torch.as_tensor(t, dtype=torch.float32, device=dev).reshape(-1).expand(B)) for t in (fx, fy, cx, cy))
    L.check(L.load().fnr_tsdf_integrate(_ptr(values), _ptr(weights), _ptr(colors), _ptr(fruit_state) if fruit is not None else None, X, Y, Z,
                                        _host3(origin, "origin"), _host3(voxel_size, "voxel_size"), float(truncation), _ptr(c2w), _ptr(fx),
                                        _ptr(fy), _ptr(cx), _ptr(cy), _ptr(depth), _ptr(rgb), _ptr(fruit), B, H, W, _stream(dev)))


def marching_cubes(values: Tensor, origin, voxel_size, colors: Optional[Tensor] = None, fruit: Optional[Tensor] = None) -> dict:
    """Level-0 isosurface of a CUDA fp32 grid [X,Y,Z] (fnr_marching_cubes_count / _emit): {'vertices' [V,3], 'normals' [V,3],
    'colors' [V,3] or None, 'fruit' [V] or None (fp32), 'faces' [F,3] int64}, all on the device.  One host read (the
    vertex and face counts) between the passes."""
    dev = _require_cuda(values, colors, fruit)
    values = _f32c(values.detach())
    X, Y, Z = _grid_dims(values)
    colors = None if colors is None else _f32c(colors.detach().reshape(X, Y, Z, 3))
    fruit = None if fruit is None else _f32c(fruit.detach().reshape(X, Y, Z))
    lib = L.load()
    nbytes = C.c_size_t(0)
    L.check(lib.fnr_marching_cubes_scratch_bytes(X, Y, Z, C.byref(nbytes)))
    scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    totals = torch.zeros(2, dtype=torch.int64, device=dev)
    L.check(lib.fnr_marching_cubes_count(_ptr(values), X, Y, Z, _ptr(scratch), nbytes.value, _ptr(totals), _stream(dev)))
    V, F = (int(v) for v in totals.cpu().tolist())
    if V > 0x7FFFFFFF:  # the library refuses it before touching any output
        L.check(lib.fnr_marching_cubes_emit(_ptr(values), None, None, X, Y, Z, _host3(origin, "origin"), _host3(voxel_size, "voxel_size"),
                                            _ptr(scratch), nbytes.value, V, F, None, None, None, None, None, _stream(dev)))
    f32 = dict(dtype=torch.float32, device=dev)
    out = {"vertices": torch.empty((V, 3), **f32), "normals": torch.empty((V, 3), **f32),
           "colors": None if colors is None else torch.empty((V, 3), **f32), "fruit": None if fruit is None else torch.empty(V, **f32),
           "faces": torch.empty((F, 3), dtype=torch.int64, device=dev)}
    L.check(lib.fnr_marching_cubes_emit(_ptr(values), _ptr(colors), _ptr(fruit), X, Y, Z, _host3(origin, "origin"), _host3(voxel_size, "voxel_size"),
                                        _ptr(scratch), nbytes.value, V, F, _ptr(out["vertices"]), _ptr(out["normals"]), _ptr(out["colors"]),
                                        _ptr(out["fruit"]), _ptr(out["faces"]), _stream(dev)))
    return out


# ======================================================================================================
# Screened Poisson reconstruction (fnr_poisson.cu; nerfstudio ns-export poisson)
# ======================================================================================================
def _poisson_inputs(points: Tensor, normals: Tensor, colors: Optional[Tensor], fruit: Optional[Tensor]):
    dev = _require_cuda(points, normals, colors, fruit)
    pts = points.detach().to(torch.float64).reshape(-1, 3).contiguous()
    n = int(pts.shape[0])
    if n < 1:
        raise ValueError("the Poisson reconstruction needs at least one point")
    nrm = _f32c(normals.detach().reshape(n, 3))
    col = None if colors is None else _f32c(colors.detach().reshape(n, 3))
    fr = None if fruit is None else _f32c(fruit.detach().reshape(n))
    return dev, pts, n, nrm, col, fr


def _cube(origin, side: float):
    o = (C.c_double * 3)(*[float(v) for v in np.asarray(origin, np.float64).reshape(3)])
    return o, float(side)


def _poisson_scratch(n: int, depth: int, dev) -> Tuple[Tensor, int]:
    nbytes = C.c_size_t(0)
    L.check(L.load().fnr_poisson_scratch_bytes(n, int(depth), C.byref(nbytes)))
    return torch.empty(nbytes.value, dtype=torch.uint8, device=dev), nbytes.value


def poisson_splat(points: Tensor, normals: Tensor, depth: int, origin, side: float, colors: Optional[Tensor] = None,
                  fruit: Optional[Tensor] = None, scratch: Optional[Tuple[Tensor, int]] = None) -> dict:
    """The node sums and right-hand side of the screened Poisson system (fnr_poisson_splat) on the cube ``origin`` / ``side``
    at ``depth``: {'density' [M], 'normal_field' [M,3], 'colors' [M,3] or None, 'fruit' [M] or None, 'rhs' [M]} fp32 with
    M = (2^depth + 1)^3 in C order, and 'scratch' (the sorted points, which ``poisson_apply`` reads)."""
    dev, pts, n, nrm, col, fr = _poisson_inputs(points, normals, colors, fruit)
    M = (2 ** int(depth) + 1) ** 3
    buf, nbytes = scratch if scratch is not None else _poisson_scratch(n, depth, dev)
    f32 = dict(dtype=torch.float32, device=dev)
    out = {"density": torch.empty(M, **f32), "normal_field": torch.empty((M, 3), **f32),
           "colors": None if col is None else torch.empty((M, 3), **f32), "fruit": None if fr is None else torch.empty(M, **f32),
           "rhs": torch.empty(M, **f32)}
    o, s = _cube(origin, side)
    L.check(L.load().fnr_poisson_splat(_ptr(pts), _ptr(nrm), _ptr(col), _ptr(fr), n, int(depth), o, s, _ptr(buf), nbytes, _ptr(out["density"]),
                                       _ptr(out["normal_field"]), _ptr(out["colors"]), _ptr(out["fruit"]), _ptr(out["rhs"]), _stream(dev)))
    out["scratch"] = (buf, nbytes)
    return out


def poisson_apply(x: Tensor, num_points: int, depth: int, scratch: Tuple[Tensor, int], alpha: float = 2.0) -> Tensor:
    """y = (K + alpha a S^T S) x (fnr_poisson_apply) for the points ``poisson_splat`` left in ``scratch``."""
    dev = _require_cuda(x)
    M = (2 ** int(depth) + 1) ** 3
    x = _f32c(x.detach().reshape(-1))
    if x.numel() != M:
        raise ValueError(f"x must have (2^depth + 1)^3 = {M} entries, got {x.numel()}")
    y = torch.empty_like(x)
    buf, nbytes = scratch
    L.check(L.load().fnr_poisson_apply(int(num_points), int(depth), float(alpha), _ptr(buf), nbytes, _ptr(x), _ptr(y), _stream(dev)))
    return y


def poisson_solve(points: Tensor, normals: Tensor, depth: int, origin, side: float, colors: Optional[Tensor] = None,
                  fruit: Optional[Tensor] = None, alpha: float = 2.0, max_iters: int = 2000, tolerance: float = 1e-5) -> dict:
    """Coarse-to-fine solve of the screened Poisson system (fnr_poisson_solve): {'chi' [M], 'density' [M], 'colors' [M,3]
    or None, 'fruit' [M] or None, 'iterations' (finest level), 'total_iterations', 'residual' (|r| / |b|)}."""
    dev, pts, n, nrm, col, fr = _poisson_inputs(points, normals, colors, fruit)
    M = (2 ** int(depth) + 1) ** 3
    buf, nbytes = _poisson_scratch(n, depth, dev)
    f32 = dict(dtype=torch.float32, device=dev)
    out = {"chi": torch.empty(M, **f32), "density": torch.empty(M, **f32), "colors": None if col is None else torch.empty((M, 3), **f32),
           "fruit": None if fr is None else torch.empty(M, **f32)}
    iters = (C.c_int64 * 2)()
    res = C.c_double(0.0)
    o, s = _cube(origin, side)
    L.check(L.load().fnr_poisson_solve(_ptr(pts), _ptr(nrm), _ptr(col), _ptr(fr), n, int(depth), o, s, float(alpha), int(max_iters),
                                       float(tolerance), _ptr(buf), nbytes, _ptr(out["chi"]), _ptr(out["density"]), _ptr(out["colors"]),
                                       _ptr(out["fruit"]), iters, C.byref(res), _stream(dev)))
    out.update(iterations=int(iters[0]), total_iterations=int(iters[1]), residual=float(res.value))
    return out


def poisson_sample(points: Tensor, grid: Tensor, depth: int, origin, side: float) -> Tensor:
    """Trilinear samples [n] fp32 of a node grid [M] at the points (fnr_poisson_sample)."""
    dev = _require_cuda(points, grid)
    pts = points.detach().to(torch.float64).reshape(-1, 3).contiguous()
    grid = _f32c(grid.detach().reshape(-1))
    if grid.numel() != (2 ** int(depth) + 1) ** 3:
        raise ValueError("grid must have (2^depth + 1)^3 entries")
    out = torch.empty(pts.shape[0], dtype=torch.float32, device=dev)
    o, s = _cube(origin, side)
    L.check(L.load().fnr_poisson_sample(_ptr(pts), int(pts.shape[0]), int(depth), o, s, _ptr(grid), _ptr(out), _stream(dev)))
    return out


# ======================================================================================================
# Per-fruit measurement of triangle meshes (fnr_measure.cu)
# ======================================================================================================
def _mesh_inputs(vertices: Optional[Tensor], faces: Tensor):
    """(device, vertices [V,3] fp64 or None, faces [F,3] int64), contiguous."""
    dev = _require_cuda(vertices, faces)
    v = None if vertices is None else vertices.detach().to(torch.float64).reshape(-1, 3).contiguous()
    f = faces.detach().to(torch.int64).reshape(-1, 3).contiguous()
    return dev, v, f


def _measure_scratch(num_vertices: int, num_faces: int, dev) -> Tuple[Tensor, int]:
    nbytes = C.c_size_t(0)
    L.check(L.load().fnr_mesh_measure_scratch_bytes(int(num_vertices), int(num_faces), C.byref(nbytes)))
    return torch.empty(nbytes.value, dtype=torch.uint8, device=dev), nbytes.value


def mesh_components(faces: Tensor, num_vertices: int) -> Tuple[Tensor, int]:
    """(int32 [F] labels, number of groups): the connected components of the faces through shared vertex indices
    (fnr_mesh_components), numbered in the order of their smallest vertex index."""
    dev, _, f = _mesh_inputs(None, faces)
    F = int(f.shape[0])
    labels = torch.empty(F, dtype=torch.int32, device=dev)
    buf, nbytes = _measure_scratch(num_vertices, F, dev)
    num = C.c_int64(0)
    L.check(L.load().fnr_mesh_components(_ptr(f), F, int(num_vertices), _ptr(buf), nbytes, _ptr(labels), C.byref(num), _stream(dev)))
    return labels, int(num.value)


def mesh_assign_centers(vertices: Tensor, faces: Tensor, centers: Tensor, max_distance: float = float("inf")) -> Tensor:
    """int32 [F]: the index of the centre [K,3] nearest each face centroid, -1 beyond ``max_distance``
    (fnr_mesh_assign_centers)."""
    dev, v, f = _mesh_inputs(vertices, faces)
    _require_cuda(centers)
    c = centers.detach().to(torch.float64).reshape(-1, 3).contiguous()
    F = int(f.shape[0])
    labels = torch.empty(F, dtype=torch.int32, device=dev)
    flag = torch.empty(L.FNR_MESH_ASSIGN_SCRATCH_BYTES, dtype=torch.uint8, device=dev)
    L.check(L.load().fnr_mesh_assign_centers(_ptr(v), _ptr(f), F, int(v.shape[0]), _ptr(c), int(c.shape[0]), float(max_distance), _ptr(flag),
                                             flag.numel(), _ptr(labels), _stream(dev)))
    return labels


def mesh_measure_groups(vertices: Tensor, faces: Tensor, face_group: Tensor, num_groups: int) -> Dict[str, Tensor]:
    """Per-group measurements of the labels 0..G-1 (fnr_mesh_measure_groups), device tensors: 'faces', 'boundary_edges',
    'nonmanifold_edges' [G] int64, 'area' [G], 'centroid' [G,3], 'sphere' [G,5] (centre, radius, rms), 'volume' [G],
    'coverage' [G] fp64, 'fit_ok' [G] int32, and 'unassigned_faces' / 'unassigned_area' [1] for the label -1 faces."""
    dev, v, f = _mesh_inputs(vertices, faces)
    _require_cuda(face_group)
    g = face_group.detach().to(torch.int32).reshape(-1).contiguous()
    V, F, G = int(v.shape[0]), int(f.shape[0]), int(num_groups)
    if g.shape[0] != F:
        raise ValueError(f"{g.shape[0]} face labels for {F} faces")
    buf, nbytes = _measure_scratch(V, F, dev)
    i64 = dict(dtype=torch.int64, device=dev)
    f64 = dict(dtype=torch.float64, device=dev)
    G0 = max(G, 0)
    out = {"faces": torch.empty(G0, **i64), "boundary_edges": torch.empty(G0, **i64), "nonmanifold_edges": torch.empty(G0, **i64),
           "area": torch.empty(G0, **f64), "centroid": torch.empty((G0, 3), **f64), "sphere": torch.empty((G0, 5), **f64),
           "volume": torch.empty(G0, **f64), "coverage": torch.empty(G0, **f64), "fit_ok": torch.empty(G0, dtype=torch.int32, device=dev),
           "unassigned_faces": torch.empty(1, **i64), "unassigned_area": torch.empty(1, **f64)}
    p = lambda k: _ptr(out[k]) if G0 else None  # noqa: E731
    L.check(L.load().fnr_mesh_measure_groups(_ptr(v), _ptr(f), F, V, _ptr(g), G, _ptr(buf), nbytes, p("faces"), p("boundary_edges"),
                                             p("nonmanifold_edges"), p("area"), p("centroid"), p("sphere"), p("volume"), p("coverage"),
                                             p("fit_ok"), _ptr(out["unassigned_faces"]), _ptr(out["unassigned_area"]), _stream(dev)))
    return out


# ======================================================================================================
# Held-out evaluation scores of one rendered view (fnr_metrics.cu; the `eval` command)
# ======================================================================================================
def image_metrics_scratch(height: int, width: int, dev) -> Tensor:
    """The uint8 device scratch ``image_stats`` and ``image_ssim`` share for images of this size."""
    nbytes = C.c_size_t(0)
    L.check(L.load().fnr_image_metrics_scratch_bytes(int(height), int(width), C.byref(nbytes)))
    return torch.empty(nbytes.value, dtype=torch.uint8, device=dev)


def _metric_input(t: Tensor, numel: int, what: str) -> Tensor:
    if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != numel:
        raise ValueError(f"{what} must be a contiguous fp32 tensor of {numel} values, got {t.dtype} {tuple(t.shape)}"
                         f"{'' if t.is_contiguous() else ' (not contiguous)'}")
    return t


def _metric_record(record: Optional[Tensor], dev) -> Tensor:
    if record is None:
        return torch.zeros(L.FNR_IMAGE_RECORD_DOUBLES, dtype=torch.float64, device=dev)
    _require_cuda(record)
    if record.dtype != torch.float64 or not record.is_contiguous() or record.numel() != L.FNR_IMAGE_RECORD_DOUBLES:
        raise ValueError(f"record must be a contiguous fp64 tensor of {L.FNR_IMAGE_RECORD_DOUBLES} values, got {record.dtype} {tuple(record.shape)}")
    return record


def _image_size(image: Tensor) -> Tuple[int, int]:
    if image.dim() != 3 or image.shape[2] != 3:
        raise ValueError(f"image must be [H,W,3], got {tuple(image.shape)}")
    return int(image.shape[0]), int(image.shape[1])


def image_stats(rgb: Tensor, semantics: Tensor, accumulation: Tensor, image: Tensor, fruit_mask: Tensor, record: Optional[Tensor] = None,
                scratch: Optional[Tensor] = None) -> Tensor:
    """One pass over a rendered view (fnr_image_stats): ``rgb`` [H*W,3] as rendered, ``semantics`` logits and
    ``accumulation`` [H*W] or [H*W,1], against ``image`` [H,W,3] and ``fruit_mask`` [H,W,1] or [H,W]; all CUDA fp32 and
    contiguous.  Fills and returns ``record`` (fp64 [12], slots ``_lib.IMAGE_RECORD_FIELDS``; e.g. one row of an [N,12]
    tensor): squared error of the clamped rgb, both value ranges, accumulation sum and fruit confusion counts."""
    dev = _require_cuda(rgb, semantics, accumulation, image, fruit_mask, scratch)
    H, W = _image_size(image)
    P = H * W
    _metric_input(image, 3 * P, "image")
    _metric_input(rgb, 3 * P, "rgb")
    _metric_input(semantics, P, "semantics")
    _metric_input(accumulation, P, "accumulation")
    _metric_input(fruit_mask, P, "fruit_mask")
    record = _metric_record(record, dev)
    if scratch is None:
        scratch = image_metrics_scratch(H, W, dev)
    L.check(L.load().fnr_image_stats(_ptr(rgb), _ptr(semantics), _ptr(accumulation), _ptr(image), _ptr(fruit_mask), H, W, _ptr(scratch),
                                     scratch.numel() * scratch.element_size(), _ptr(record), _stream(dev)))
    return record


def image_ssim(rgb: Tensor, image: Tensor, record: Tensor, scratch: Optional[Tensor] = None) -> Tensor:
    """torchmetrics' SSIM of the clamped ``rgb`` [H*W,3] against ``image`` [H,W,3] (fnr_ssim) into ``record``, which
    ``image_stats`` of the same pair has filled on this stream (the data range comes from its min / max slots).  Images
    with H or W < 11 are refused."""
    dev = _require_cuda(rgb, image, record, scratch)
    H, W = _image_size(image)
    _metric_input(image, 3 * H * W, "image")
    _metric_input(rgb, 3 * H * W, "rgb")
    record = _metric_record(record, dev)
    if scratch is None:
        scratch = image_metrics_scratch(H, W, dev)
    L.check(L.load().fnr_ssim(_ptr(rgb), _ptr(image), H, W, _ptr(scratch), scratch.numel() * scratch.element_size(), _ptr(record), _stream(dev)))
    return record
