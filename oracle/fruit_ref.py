"""Oracle restatement of FruitField / FruitModel / export on plain tensors.

TEST INFRASTRUCTURE, PARITY UNPINNED (see oracle/__init__.py).  Parameters come in as a dict with
the reference's state-dict names (``FruitField`` under nerfstudio's torch path):

    mlp_base_grid.hash_table                 [L * 2**T, F]
    mlp_base_mlp.layers.{0,1}.{weight,bias}
    mlp_semantics.layers.{i}.{weight,bias}
    field_head_semantics.net.{weight,bias}
    mlp_head.layers.{0,1,2}.{weight,bias}
    embedding_appearance.embedding.weight    [num_images, 32]
    aabb                                     [2, 3]
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch
from torch import Tensor

from . import ns_torch as ns


@dataclass
class FieldSpec:
    """Hyper-parameters of FruitField.__init__ (fruit_nerf/fruit_field.py:70-95)."""

    num_levels: int = 16
    base_res: int = 16
    max_res: int = 2048
    log2_hashmap_size: int = 19
    features_per_level: int = 2
    geo_feat_dim: int = 15
    appearance_embedding_dim: int = 32
    pass_semantic_gradients: bool = False

    def scalings(self) -> Tensor:
        return ns.hash_scalings(self.num_levels, self.base_res, self.max_res)


def _layers(params: Dict[str, Tensor], prefix: str):
    ws, bs = [], []
    i = 0
    while f"{prefix}.layers.{i}.weight" in params:
        ws.append(params[f"{prefix}.layers.{i}.weight"])
        bs.append(params[f"{prefix}.layers.{i}.bias"])
        i += 1
    return ws, bs


def sample_positions(origins, directions, starts, ends, aabb, contraction: bool):
    """fruit_field.py:170-179 -> (positions in [0,1]^3 after masking, selector)."""
    pos = ns.frustum_positions(origins, directions, starts, ends)
    if contraction:
        pos = ns.scene_contraction_inf(pos)
        pos = (pos + 2.0) / 4.0
    else:
        pos = ns.normalized_positions(pos, aabb)
    selector = ((pos > 0.0) & (pos < 1.0)).all(dim=-1)
    pos = pos * selector[..., None]
    return pos, selector


def field_forward(
    params: Dict[str, Tensor],
    spec: FieldSpec,
    origins: Tensor,  # [R,S,3] (or broadcastable [R,1,3])
    directions: Tensor,  # [R,S,3]
    starts: Tensor,  # [R,S,1]
    ends: Tensor,  # [R,S,1]
    camera_indices: Optional[Tensor],  # [R] or [R,S] int64, needed for appearance="train"
    contraction: bool = True,
    appearance: str = "train",  # "train" | "mean" | "zeros"
    chunk: int = 32768,
) -> Dict[str, Tensor]:
    """FruitField.forward (fruit_field.py:283-301): get_density (168-193) then get_outputs
    (234-281; appearance "train"/"zeros"/"mean") or get_inference_outputs (195-232; "mean")."""
    R, S = starts.shape[0], starts.shape[1]
    origins = origins.expand(R, S, 3)
    directions = directions.expand(R, S, 3)
    pos, selector = sample_positions(origins, directions, starts, ends, params["aabb"], contraction)
    table = params["mlp_base_grid.hash_table"]
    scal = spec.scalings()
    bw, bb = _layers(params, "mlp_base_mlp")
    sw, sb = _layers(params, "mlp_semantics")
    cw, cb = _layers(params, "mlp_head")
    emb = params["embedding_appearance.embedding.weight"]
    G = spec.geo_feat_dim

    pos_flat = pos.reshape(-1, 3)
    dirs_flat = ((directions + 1.0) / 2.0).reshape(-1, 3)  # shift_directions_for_tcnn
    if appearance == "train":
        cam = camera_indices
        if cam.dim() == 1:
            cam = cam[:, None].expand(R, S)
        cam_flat = cam.reshape(-1)
    dens, rgbs, sems, geos, encs, margins = [], [], [], [], [], []
    N = pos_flat.shape[0]
    for a in range(0, N, chunk):
        b = min(N, a + chunk)
        enc = ns.hash_encode(pos_flat[a:b], table, scal, spec.log2_hashmap_size)
        pre: list = []
        h = ns.mlp_forward(enc, bw, bb, preacts=pre)
        d_before, geo = torch.split(h, [1, G], dim=-1)
        dens.append(ns.trunc_exp(d_before))
        sem_in = geo if spec.pass_semantic_gradients else geo.detach()
        x = ns.mlp_forward(sem_in, sw, sb, preacts=pre)
        sems.append(torch.nn.functional.linear(x, params["field_head_semantics.net.weight"], params["field_head_semantics.net.bias"]))
        sh = ns.sh_degree4(dirs_flat[a:b])
        if appearance == "train":
            app = emb[cam_flat[a:b]]
        elif appearance == "mean":
            app = torch.ones((b - a, spec.appearance_embedding_dim)) * emb.mean(dim=0)
        elif appearance == "zeros":
            app = torch.zeros((b - a, spec.appearance_embedding_dim))
        else:
            raise ValueError(appearance)
        rgbs.append(ns.mlp_forward(torch.cat([sh, geo, app], dim=-1), cw, cb, out_activation="sigmoid", preacts=pre))
        # ReLU margin of each point: min |pre-activation| / rms(layer), over every hidden unit (test hook: the
        # gradient of a sample is only well-defined up to the mask of units this close to zero)
        margins.append(torch.stack([(t.abs() / t.pow(2).mean().sqrt().clamp_min(1e-20)).amin(dim=-1) for t in pre], dim=-1).amin(dim=-1))
        geos.append(geo)
        encs.append(enc)
    density = torch.cat(dens).view(R, S, 1) * selector[..., None]
    return {
        "density": density,
        "rgb": torch.cat(rgbs).view(R, S, 3),
        "semantics": torch.cat(sems).view(R, S, 1),
        "geo": torch.cat(geos).view(R, S, G),
        "encoding": torch.cat(encs).view(R, S, -1),
        "positions": pos,
        "selector": selector,
        "relu_margin": torch.cat(margins).view(R, S),
    }


def render(field_out: Dict[str, Tensor], starts: Tensor, ends: Tensor, training: bool = True,
           pass_semantic_gradients: bool = False) -> Dict[str, Tensor]:
    """FruitModel.get_outputs after the field call (fruit_nerf.py:325-355), without the proposal
    entries.  ``semantics`` uses detached weights unless ``pass_semantic_gradients`` (301-305, 343-345)."""
    deltas = ends - starts
    weights = ns.get_weights(deltas, field_out["density"])
    rgb = ns.render_rgb_last_sample(field_out["rgb"], weights, training)
    depth, depth_idx = ns.render_depth_median(weights, starts, ends)
    acc = ns.render_accumulation(weights)
    sem = ns.render_semantics(field_out["semantics"], weights if pass_semantic_gradients else weights.detach())
    labels = torch.heaviside(torch.sigmoid(sem.detach()) - 0.9, torch.tensor(0.0, dtype=sem.dtype)).to(torch.long)
    return {
        "rgb": rgb,
        "accumulation": acc,
        "depth": depth,
        "depth_index": depth_idx,
        "semantics": sem,
        "semantic_labels": labels,
        "weights": weights,
    }


def loss_dict(outputs: Dict[str, Tensor], image: Tensor, fruit_mask: Tensor, semantic_loss_weight: float = 1.0):
    """FruitModel.get_loss_dict (fruit_nerf.py:359-366) without the interlevel term."""
    return {
        "rgb_loss": ns.rgb_mse(image, outputs["rgb"]),
        "semantics_loss": semantic_loss_weight * ns.semantic_bce(outputs["semantics"], fruit_mask),
    }


def export_outputs(params, spec, origins, directions, nears, fars, num_samples: int, chunk: int = 32768, t_rand=None):
    """FruitModel.get_export_outputs (fruit_nerf.py:251-269) after setup_inference (179-183):
    uniform bins (jittered by ``t_rand`` when the sampler module is in training mode, see ns.uniform_bins), field with
    spatial_distortion=None (aabb normalisation), mean appearance."""
    starts, ends = ns.uniform_bins(nears, fars, num_samples, t_rand)
    B = origins.shape[0]
    o = origins[:, None, :].expand(B, num_samples, 3)
    d = directions[:, None, :].expand(B, num_samples, 3)
    f = field_forward(params, spec, o, d, starts, ends, None, contraction=False, appearance="mean", chunk=chunk)
    sem = f["semantics"][..., 0]
    labels = torch.heaviside(torch.sigmoid(sem) - 0.9, torch.tensor(0.0, dtype=sem.dtype)).to(torch.long)
    return {
        "rgb": f["rgb"],
        "point_location": ns.frustum_positions(o, d, starts, ends),
        "semantics": sem,
        "density": f["density"][..., 0],
        "semantics_colormap": labels,
    }


def export_select(out: Dict[str, Tensor]) -> Dict[str, Dict[str, Tensor]]:
    """Threshold + selection of sample_volume (export/exporter_utils.py:100-153) for one batch.

    Three clouds: 'semantic_colormap' = (label >= 0.999) & (density >= 70); 'semantic' =
    (logit >= 3) & (density >= 70); 'density' = (density >= 70).  Colours are rgb plus a 4th
    column sigmoid(logit) (sigmoid(density) for the density cloud)."""
    pts = out["point_location"].reshape(-1, 3)
    sem = out["semantics"].reshape(-1)
    lab = out["semantics_colormap"].reshape(-1)
    den = out["density"].reshape(-1)
    rgb = out["rgb"].reshape(-1, 3)
    m_sem, m_den, m_lab = sem >= 3, den >= 70, lab >= 0.999
    res = {}
    for name, m, fourth in (
        ("semantic_colormap", m_lab & m_den, sem),
        ("semantic", m_sem & m_den, sem),
        ("density", m_den, den),
    ):
        res[name] = {"points": pts[m], "colors": torch.hstack([rgb[m], torch.sigmoid(fourth[m]).unsqueeze(-1)])}
    return res


# --------------------------------------------------------------------------------------------------
# Proposal stage (fruit_nerf.py:104-158, 318): nerfstudio ProposalNetworkSampler on plain tensors
# --------------------------------------------------------------------------------------------------
@dataclass
class DensitySpec:
    """proposal_net_args_list entry (fruit_nerf.py:121-127) of a HashMLPDensityField."""

    num_levels: int = 5
    max_res: int = 128
    log2_hashmap_size: int = 17
    base_res: int = 16
    hidden_dim: int = 16

    def scalings(self) -> Tensor:
        return ns.hash_scalings(self.num_levels, self.base_res, self.max_res)


def proposal_weights(pp: Dict[str, Tensor], spec: DensitySpec, origins, directions, starts, ends, aabb, contraction: bool = True,
                     relu_margin: bool = False):
    """density_fn(frustum midpoints) -> get_weights for one level.  starts/ends [R,S] -> weights [R,S].

    ``relu_margin`` (test hook, as field_forward's): also return [R,S] min |hidden pre-activation| / rms of the hidden layer
    over the batch, +inf for samples outside the selector (their density is 0 and they pass no gradient)."""
    pos = ns.frustum_positions(origins[:, None, :], directions[:, None, :], starts[..., None], ends[..., None])
    hook = {} if relu_margin else None
    dens = ns.proposal_density(pos, pp["encoding.hash_table"], spec.scalings(), spec.log2_hashmap_size, pp["mlp_base.1.layers.0.weight"],
                               pp["mlp_base.1.layers.0.bias"], pp["mlp_base.1.layers.1.weight"], pp["mlp_base.1.layers.1.bias"], aabb, contraction,
                               hook=hook)
    weights = ns.get_weights((ends - starts)[..., None], dens)[..., 0]
    if not relu_margin:
        return weights
    pre = hook["preacts"]
    margin = (pre.abs() / pre.pow(2).mean().sqrt().clamp_min(1e-20)).amin(dim=-1)
    return weights, margin.masked_fill(~hook["selector"], float("inf"))


def proposal_sampler(prop_params, prop_specs, origins, directions, nears, fars, num_prop_samples, num_nerf_samples, aabb, t_rand0=None,
                     u_rands=None, anneal: float = 1.0):
    """ProposalNetworkSampler.generate_ray_samples.  ``t_rand0``: jitter of the initial sampler (None = eval);
    ``u_rands``: list of PDF draws per PDF level (None = eval).  Returns (starts, ends, final_bins, weights_list, sdist_list)
    where the lists cover the proposal levels only."""
    R = origins.shape[0]
    n = len(prop_params)
    weights_list, sdist_list = [], []
    bins = ns.spaced_bins(R, num_prop_samples[0], t_rand0)
    weights = None
    for lvl in range(n + 1):
        is_prop = lvl < n
        if lvl > 0:
            ns_ = num_prop_samples[lvl] if is_prop else num_nerf_samples
            u = None if u_rands is None else u_rands[lvl - 1]
            bins = ns.pdf_sample(torch.pow(weights, anneal), bins, ns_, u)
        e = ns.spacing_to_euclidean(bins, nears, fars)
        starts, ends = e[:, :-1], e[:, 1:]
        if is_prop:
            weights = proposal_weights(prop_params[lvl], prop_specs[lvl], origins, directions, starts, ends, aabb)
            weights_list.append(weights)
            sdist_list.append(bins)
    return starts, ends, bins, weights_list, sdist_list
