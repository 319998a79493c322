"""Restatement of the nerfstudio-0.3.2 *torch-fallback* components FruitNeRF's hot path calls.

TEST INFRASTRUCTURE (see oracle/__init__.py).  PARITY UNPINNED: nerfstudio is absent from this
image and from /root/reference; each function names the reference call site whose behaviour it
restates and the [NS] class it stands in for.  All arithmetic is fp32 on the CPU, written as
separate elementwise torch ops (no fused multiply-add), which is what the CUDA path's
index-defining arithmetic reproduces bit-for-bit.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

HASH_PRIMES = (1, 2654435761, 805459861)  # [NS] HashEncoding.hash_fn multipliers


# --------------------------------------------------------------------------------------
# Hash-grid encoding            (reference ctor call: fruit_nerf/fruit_field.py:124-131)
# --------------------------------------------------------------------------------------
def hash_scalings(num_levels: int, min_res: int, max_res: int) -> Tensor:
    """[NS] HashEncoding.__init__: ``floor(min_res * growth**levels)``.

    ``growth`` is a numpy float64, ``levels`` an int64 tensor: ``np.float64 ** Tensor`` defers to
    ``Tensor.__rpow__`` and evaluates in float32 -- the top level of max_res=2048 is 2047, not
    2048 (SURVEY.md section 7 "float-fragile").  Restated with the very same expression so the
    values are whatever torch produces; the CUDA path receives this array and never recomputes it.
    """
    levels = torch.arange(num_levels)
    growth = np.exp((np.log(max_res) - np.log(min_res)) / (num_levels - 1)) if num_levels > 1 else 1
    return torch.floor(min_res * growth**levels).to(torch.float32)


def hash_fn(coords: Tensor, log2_hashmap_size: int, num_levels: int) -> Tensor:
    """[NS] HashEncoding.hash_fn.  coords: int32 [..., L, 3] -> int64 table row [..., L].

    int32 * int64 promotes to int64; xor and ``% 2**T`` only look at the low T bits, so this is
    identical to uint32 wrap-around arithmetic (what the kernel does) for T <= 32.
    """
    t = coords * torch.tensor(HASH_PRIMES, dtype=torch.int64)
    x = torch.bitwise_xor(t[..., 0], t[..., 1])
    x = torch.bitwise_xor(x, t[..., 2])
    x = x % (2**log2_hashmap_size)
    x = x + torch.arange(num_levels, dtype=torch.int64) * (2**log2_hashmap_size)
    return x


def hash_corner_indices(p: Tensor, scalings: Tensor, log2_hashmap_size: int) -> Tuple[Tensor, Tensor]:
    """Corner rows and trilinear offsets of [NS] HashEncoding.pytorch_fwd.

    p: [N,3] in [0,1].  Returns (idx [N,L,8] int64 in the [NS] corner order 0..7, offset [N,L,3]).
    Corner order (c = ceil, f = floor): 0 ccc, 1 cfc, 2 ffc, 3 fcc, 4 ccf, 5 cff, 6 fff, 7 fcf.
    """
    L = scalings.numel()
    scaled = p[..., None, :] * scalings.view(-1, 1)  # [N, L, 3]
    c = torch.ceil(scaled).type(torch.int32)
    f = torch.floor(scaled).type(torch.int32)
    offset = scaled - f

    def pick(sel: str) -> Tensor:
        parts = [(c if s == "c" else f)[..., i : i + 1] for i, s in enumerate(sel)]
        return hash_fn(torch.cat(parts, dim=-1), log2_hashmap_size, L)

    order = ("ccc", "cfc", "ffc", "fcc", "ccf", "cff", "fff", "fcf")
    idx = torch.stack([pick(s) for s in order], dim=-1)  # [N, L, 8]
    return idx, offset


def hash_encode(p: Tensor, table: Tensor, scalings: Tensor, log2_hashmap_size: int) -> Tensor:
    """[NS] HashEncoding.pytorch_fwd: [N,3] -> [N, L*F], level-major."""
    idx, offset = hash_corner_indices(p, scalings, log2_hashmap_size)
    f = [table[idx[..., k]] for k in range(8)]  # each [N, L, F]
    ox, oy, oz = offset[..., 0:1], offset[..., 1:2], offset[..., 2:3]
    f_03 = f[0] * ox + f[3] * (1 - ox)
    f_12 = f[1] * ox + f[2] * (1 - ox)
    f_56 = f[5] * ox + f[6] * (1 - ox)
    f_47 = f[4] * ox + f[7] * (1 - ox)
    f0312 = f_03 * oy + f_12 * (1 - oy)
    f4756 = f_47 * oy + f_56 * (1 - oy)
    enc = f0312 * oz + f4756 * (1 - oz)
    return torch.flatten(enc, start_dim=-2, end_dim=-1)


# --------------------------------------------------------------------------------------
# MLP / heads / activations     (fruit_field.py:132-166; components/field_heads.py:29-40)
# --------------------------------------------------------------------------------------
def mlp_forward(x: Tensor, weights: Sequence[Tensor], biases: Sequence[Tensor], out_activation: Optional[str] = None,
                preacts: Optional[List[Tensor]] = None) -> Tensor:
    """[NS] MLP.pytorch_fwd without skip connections: Linear(+bias) layers, ReLU between.
    ``preacts`` (test hook) collects the detached ReLU inputs of the hidden layers."""
    n = len(weights)
    for i, (w, b) in enumerate(zip(weights, biases)):
        x = torch.nn.functional.linear(x, w, b)
        if i < n - 1:
            if preacts is not None:
                preacts.append(x.detach())
            x = torch.relu(x)
    if out_activation == "sigmoid":
        x = torch.sigmoid(x)
    elif out_activation is not None:
        raise ValueError(out_activation)
    return x


class _TruncExp(torch.autograd.Function):
    """[NS] field_components.activations.trunc_exp (fruit_field.py:191): exp forward,
    ``g * exp(clamp(x, -15, 15))`` backward."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(-15, 15))


trunc_exp = _TruncExp.apply


def sh_degree4(d: Tensor) -> Tensor:
    """[NS] SHEncoding(levels=4).pytorch_fwd = components_from_spherical_harmonics(4, d).

    FruitField passes ``shift_directions_for_tcnn(d) = (d+1)/2`` (fruit_field.py:208,243) and the
    torch fallback evaluates the basis on that shifted vector as given -- restated literally.
    """
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    xx, yy, zz = x**2, y**2, z**2
    c = torch.zeros((*d.shape[:-1], 16), dtype=d.dtype)
    c[..., 0] = 0.28209479177387814
    c[..., 1] = 0.4886025119029199 * y
    c[..., 2] = 0.4886025119029199 * z
    c[..., 3] = 0.4886025119029199 * x
    c[..., 4] = 1.0925484305920792 * x * y
    c[..., 5] = 1.0925484305920792 * y * z
    c[..., 6] = 0.9461746957575601 * zz - 0.31539156525251999
    c[..., 7] = 1.0925484305920792 * x * z
    c[..., 8] = 0.5462742152960396 * (xx - yy)
    c[..., 9] = 0.5900435899266435 * y * (3 * xx - yy)
    c[..., 10] = 2.890611442640554 * x * y * z
    c[..., 11] = 0.4570457994644658 * y * (5 * zz - 1)
    c[..., 12] = 0.3731763325901154 * z * (5 * zz - 3)
    c[..., 13] = 0.4570457994644658 * x * (5 * zz - 1)
    c[..., 14] = 1.445305721320277 * z * (xx - yy)
    c[..., 15] = 0.5900435899266435 * x * (xx - 3 * yy)
    return c


# --------------------------------------------------------------------------------------
# Positions                     (fruit_field.py:170-179)
# --------------------------------------------------------------------------------------
def frustum_positions(origins: Tensor, directions: Tensor, starts: Tensor, ends: Tensor) -> Tensor:
    """[NS] Frustums.get_positions: ``o + d * (start + end) / 2`` in that op order."""
    return origins + directions * (starts + ends) / 2


def scene_contraction_inf(x: Tensor) -> Tensor:
    """[NS] SceneContraction(order=inf) (fruit_nerf.py:85): x if |x|inf < 1 else (2 - 1/m) * (x/m)."""
    mag = torch.linalg.norm(x, ord=float("inf"), dim=-1)[..., None]
    return torch.where(mag < 1, x, (2 - (1 / mag)) * (x / mag))


def normalized_positions(x: Tensor, aabb: Tensor) -> Tensor:
    """[NS] SceneBox.get_normalized_positions (fruit_field.py:175): (x - aabb[0]) / (aabb[1]-aabb[0])."""
    lengths = aabb[1] - aabb[0]
    return (x - aabb[0]) / lengths


# --------------------------------------------------------------------------------------
# Compositing                   (fruit_nerf.py:325-348)
# --------------------------------------------------------------------------------------
def get_weights(deltas: Tensor, densities: Tensor) -> Tensor:
    """[NS] RaySamples.get_weights (fruit_nerf.py:325).  deltas, densities: [R,S,1]."""
    delta_density = deltas * densities
    alphas = 1 - torch.exp(-delta_density)
    transmittance = torch.cumsum(delta_density[..., :-1, :], dim=-2)
    transmittance = torch.cat([torch.zeros((*transmittance.shape[:1], 1, 1)), transmittance], dim=-2)
    transmittance = torch.exp(-transmittance)
    weights = alphas * transmittance
    return torch.nan_to_num(weights)


def render_rgb_last_sample(rgb: Tensor, weights: Tensor, training: bool) -> Tensor:
    """[NS] RGBRenderer(background_color="last_sample") (fruit_nerf.py:164,329)."""
    if not training:
        rgb = torch.nan_to_num(rgb)
    comp = torch.sum(weights * rgb, dim=-2)
    acc = torch.sum(weights, dim=-2)
    background = rgb[..., -1, :]
    comp = comp + background * (1.0 - acc)
    if not training:
        comp = torch.clamp(comp, min=0.0, max=1.0)
    return comp


def render_accumulation(weights: Tensor) -> Tensor:
    """[NS] AccumulationRenderer (fruit_nerf.py:331)."""
    return torch.sum(weights, dim=-2)


def render_depth_median(weights: Tensor, starts: Tensor, ends: Tensor) -> Tuple[Tensor, Tensor]:
    """[NS] DepthRenderer(method="median") (fruit_nerf.py:330).  Returns (depth [R,1], index [R,1])."""
    steps = (starts + ends) / 2
    cumulative = torch.cumsum(weights[..., 0], dim=-1)
    split = torch.ones((*weights.shape[:-2], 1)) * 0.5
    idx = torch.searchsorted(cumulative, split, side="left")
    idx = torch.clamp(idx, 0, steps.shape[-2] - 1)
    return torch.gather(steps[..., 0], dim=-1, index=idx), idx


def render_semantics(semantics: Tensor, weights: Tensor) -> Tensor:
    """[NS] SemanticRenderer (fruit_nerf.py:346-348): sum(w * logits)."""
    return torch.sum(weights * semantics, dim=-2)


# --------------------------------------------------------------------------------------
# Export sampling               (components/ray_samplers.py:54-104, ray_generators.py:46-66,
#                                data/fruit_datamanager.py:42-121)
# --------------------------------------------------------------------------------------
def uniform_bins(nears: Tensor, fars: Tensor, num_samples: int, t_rand: Tensor = None) -> Tuple[Tensor, Tensor]:
    """UniformSamplerWithNoise.generate_ray_samples (components/ray_samplers.py:54-104).  nears/fars [B,1] ->
    (starts [B,S,1], ends [B,S,1]).  ``t_rand`` = None: module in eval mode, the regular grid.  ``t_rand`` [B,S+1] (or
    [B,1], single_jitter): the stratified jitter of a module in TRAINING mode (ray_samplers.py:78-87) -- the state the
    reference exporter actually runs it in, because setup_inference() creates the sampler after eval_setup() called
    pipeline.eval() (scripts/exporter.py:87-95)."""
    bins = torch.linspace(0.0, 1.0, num_samples + 1)[None, ...]
    if t_rand is not None:
        bin_centers = (bins[..., 1:] + bins[..., :-1]) / 2.0
        bin_upper = torch.cat([bin_centers, bins[..., -1:]], -1)
        bin_lower = torch.cat([bins[..., :1], bin_centers], -1)
        bins = bin_lower + (bin_upper - bin_lower) * t_rand
    euclid = bins * fars + (1 - bins) * nears  # spacing_fn = identity
    return euclid[..., :-1, None], euclid[..., 1:, None]


def aabb_corners(aabb) -> Tensor:
    """get_corners_of_aabb (fruit_datamanager.py:42-68)."""
    mn, mx = aabb[0], aabb[1]
    return torch.tensor(
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
    )


def surface_points(aabb, n: int) -> Tuple[Tensor, Tensor]:
    """sample_surface_points (fruit_datamanager.py:71-121) on the 8 corners of ``aabb``.

    Returns (points [nx*ny, 3] x-major, plane_vector [1,3])."""
    corners = aabb_corners(aabb)
    c1, c2, c3 = corners[0], corners[1], corners[2]
    dxyz = torch.abs(torch.max(corners, dim=0).values - torch.min(corners, dim=0).values)
    const_axis = int(torch.argmax(torch.logical_and(c1 == c2, c2 == c3).to(int)))
    ax = torch.argmax(torch.abs(c1 - c2))
    x = torch.linspace(float(c1[ax]), float(c2[ax]), int(dxyz[0] / dxyz[const_axis] * n), dtype=torch.float32)
    ay = torch.argmax(torch.abs(c1 - c3))
    y = torch.linspace(float(c1[ay]), float(c3[ay]), int(dxyz[1] / dxyz[const_axis] * n), dtype=torch.float32)
    xx, yy = torch.meshgrid(x, y, indexing="ij")
    pts = torch.column_stack((xx.flatten(), yy.flatten(), torch.full_like(xx.flatten(), float(c3[const_axis]))))
    c4 = corners[-1]
    plane = torch.tensor(
        [[0, 0, float(torch.sign(c4[const_axis]) * torch.abs(c1[const_axis]) + torch.abs(c4[const_axis]))]],
        dtype=torch.float32,
    )
    return pts, plane


def orthographic_rays(points: Tensor, plane_vector: Tensor, batch: int, count: int):
    """OrthographicRayGenerator.forward (ray_generators.py:46-66); ``count`` is 1-based."""
    start, end = batch * (count - 1), batch * count
    if batch * count >= points.shape[0]:
        end = points.shape[0]
    normal = torch.nn.functional.normalize(plane_vector)
    norm = torch.linalg.norm(plane_vector)
    o = points[start:end]
    n = o.shape[0]
    return o, normal.repeat(n, 1), torch.zeros(n, 1), torch.ones(n, 1) * norm


# --------------------------------------------------------------------------------------
# Losses                        (fruit_nerf.py:359-372)
# --------------------------------------------------------------------------------------
def rgb_mse(image: Tensor, rgb: Tensor) -> Tensor:
    return torch.nn.functional.mse_loss(image, rgb)


def semantic_bce(logits: Tensor, mask: Tensor) -> Tensor:
    return torch.nn.functional.binary_cross_entropy_with_logits(logits, mask, reduction="mean")


# --------------------------------------------------------------------------------------
# Proposal stage                (fruit_nerf.py:104-158, 318; SURVEY.md section 8a row A13)
# --------------------------------------------------------------------------------------
def lindisp_piecewise_fn(x: Tensor) -> Tensor:
    """[NS] UniformLinDispPiecewiseSampler spacing_fn: x/2 below 1, 1 - 1/(2x) above."""
    return torch.where(x < 1, x / 2, 1 - 1 / (2 * x))


def lindisp_piecewise_inv(x: Tensor) -> Tensor:
    """[NS] UniformLinDispPiecewiseSampler spacing_fn_inv."""
    return torch.where(x < 0.5, 2 * x, 1 / (2 - 2 * x))


def spaced_bins(num_rays: int, num_samples: int, t_rand: Optional[Tensor]) -> Tensor:
    """[NS] SpacedSampler.generate_ray_samples bins in spacing space.  ``t_rand`` [R,1] (single
    jitter) or [R,S+1], or None for the deterministic (eval) bins."""
    bins = torch.linspace(0.0, 1.0, num_samples + 1)[None, ...]
    if t_rand is not None:
        centers = (bins[..., 1:] + bins[..., :-1]) / 2.0
        upper = torch.cat([centers, bins[..., -1:]], -1)
        lower = torch.cat([bins[..., :1], centers], -1)
        bins = lower + (upper - lower) * t_rand
    return bins.expand(num_rays, num_samples + 1)


def spacing_to_euclidean(bins: Tensor, nears: Tensor, fars: Tensor) -> Tensor:
    """x -> spacing_fn_inv(x * s_far + (1 - x) * s_near) for the piecewise sampler."""
    s_near, s_far = lindisp_piecewise_fn(nears), lindisp_piecewise_fn(fars)
    return lindisp_piecewise_inv(bins * s_far + (1 - bins) * s_near)


def select_density(density: Tensor, selector: Tensor) -> Tensor:
    """``density * selector`` of HashMLPDensityField.get_density: samples outside the selector have density 0 and pass no
    gradient to the network."""
    return density * selector[..., None]


def proposal_density(positions: Tensor, table: Tensor, scalings: Tensor, log2_hashmap_size: int, w0: Tensor, b0: Tensor, w1: Tensor,
                     b1: Tensor, aabb: Tensor, contraction: bool = True, hook: Optional[Dict] = None) -> Tensor:
    """[NS] HashMLPDensityField.get_density (through Field.density_fn): contraction -> (x+2)/4 ->
    selector mask -> hash grid -> Linear/ReLU/Linear -> trunc_exp * selector.  positions [...,3] -> [...,1].
    ``hook`` (test hook) receives the detached hidden pre-activations [..., hidden] and the selector [...]."""
    pos = positions
    if contraction:
        pos = (scene_contraction_inf(pos) + 2.0) / 4.0
    else:
        pos = normalized_positions(pos, aabb)
    selector = ((pos > 0.0) & (pos < 1.0)).all(dim=-1)
    pos = pos * selector[..., None]
    flat = pos.reshape(-1, 3)
    out, pre = [], []
    for a in range(0, flat.shape[0], 65536):
        enc = hash_encode(flat[a : a + 65536], table, scalings, log2_hashmap_size)
        out.append(mlp_forward(enc, [w0, w1], [b0, b1], preacts=pre))
    dba = torch.cat(out).view(*pos.shape[:-1], 1)
    if hook is not None:
        hook["preacts"] = torch.cat(pre).view(*pos.shape[:-1], -1)
        hook["selector"] = selector
    return select_density(trunc_exp(dba), selector)


def pdf_sample(weights: Tensor, existing_bins: Tensor, num_samples: int, u_rand: Optional[Tensor], histogram_padding: float = 0.01,
               eps: float = 1e-5) -> Tensor:
    """[NS] PDFSampler.generate_ray_samples (include_original=False) in spacing space.

    weights [R,S] (already annealed), existing_bins [R,S+1] -> new spacing bins [R,num_samples+1]
    (detached).  ``u_rand``: the torch.rand draw of the reference ([R,1] single jitter or
    [R,num_samples+1]) or None for the eval-mode midpoints."""
    num_bins = num_samples + 1
    weights = weights + histogram_padding
    weights_sum = torch.sum(weights, dim=-1, keepdim=True)
    padding = torch.relu(eps - weights_sum)
    weights = weights + padding / weights.shape[-1]
    weights_sum = weights_sum + padding
    pdf = weights / weights_sum
    cdf = torch.min(torch.ones_like(pdf), torch.cumsum(pdf, dim=-1))
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    u = torch.linspace(0.0, 1.0 - (1.0 / num_bins), steps=num_bins)
    if u_rand is not None:
        u = u.expand(*cdf.shape[:-1], num_bins) + u_rand / num_bins
    else:
        u = (u + 1.0 / (2 * num_bins)).expand(*cdf.shape[:-1], num_bins)
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, side="right")
    below = torch.clamp(inds - 1, 0, existing_bins.shape[-1] - 1)
    above = torch.clamp(inds, 0, existing_bins.shape[-1] - 1)
    cdf_g0 = torch.gather(cdf, -1, below)
    bins_g0 = torch.gather(existing_bins, -1, below)
    cdf_g1 = torch.gather(cdf, -1, above)
    bins_g1 = torch.gather(existing_bins, -1, above)
    t = torch.clip(torch.nan_to_num((u - cdf_g0) / (cdf_g1 - cdf_g0), 0), 0, 1)
    bins = bins_g0 + t * (bins_g1 - bins_g0)
    return bins.detach()


def _outer(t0_starts, t0_ends, t1_starts, t1_ends, y1):
    cy1 = torch.cat([torch.zeros_like(y1[..., :1]), torch.cumsum(y1, dim=-1)], dim=-1)
    idx_lo = torch.searchsorted(t1_starts.contiguous(), t0_starts.contiguous(), side="right") - 1
    idx_lo = torch.clamp(idx_lo, min=0, max=y1.shape[-1] - 1)
    idx_hi = torch.searchsorted(t1_ends.contiguous(), t0_ends.contiguous(), side="right")
    idx_hi = torch.clamp(idx_hi, min=0, max=y1.shape[-1] - 1)
    cy1_lo = torch.take_along_dim(cy1[..., :-1], idx_lo, dim=-1)
    cy1_hi = torch.take_along_dim(cy1[..., 1:], idx_hi, dim=-1)
    return cy1_hi - cy1_lo


def lossfun_outer(t, w, t_env, w_env):
    """[NS] losses.lossfun_outer (EPS = 1e-7)."""
    w_outer = _outer(t[..., :-1], t[..., 1:], t_env[..., :-1], t_env[..., 1:], w_env)
    return torch.clip(w - w_outer, min=0) ** 2 / (w + 1.0e-7)


def interlevel_loss(weights_list: Sequence[Tensor], sdist_list: Sequence[Tensor]) -> Tensor:
    """[NS] losses.interlevel_loss (fruit_nerf.py:368-370).  weights_list[i] [R,S_i];
    sdist_list[i] [R,S_i+1] = cat(spacing_starts, spacing_ends[-1]); last entries = final level (detached)."""
    c = sdist_list[-1].detach()
    w = weights_list[-1].detach()
    loss = 0.0
    for sdist, weights in zip(sdist_list[:-1], weights_list[:-1]):
        loss = loss + torch.mean(lossfun_outer(c, w, sdist, weights))
    return loss


def distortion_loss(weights: Tensor, sdist: Tensor) -> Tensor:
    """[NS] losses.distortion_loss on the final level (a metric in FruitNeRF, fruit_nerf.py:400)."""
    t, w = sdist, weights
    ut = (t[..., 1:] + t[..., :-1]) / 2
    dut = torch.abs(ut[..., :, None] - ut[..., None, :])
    loss_inter = torch.sum(w * torch.sum(w[..., None, :] * dut, dim=-1), dim=-1)
    loss_intra = torch.sum(w**2 * (t[..., 1:] - t[..., :-1]), dim=-1) / 3
    return torch.mean(loss_inter + loss_intra)
