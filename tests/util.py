"""Shared helpers of the test-suite (oracle-side glue + tolerances)."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch

from fruitnerf_b200 import synthetic as syn
from fruitnerf_b200.fruit_field import FruitField, SceneContraction
from oracle import fruit_ref as fr
from oracle import ns_torch as ns

REL = 1e-3  # north_star tolerance: 1e-3 relative on RGB / density / semantics
FLOOR = 0.01  # elements below 1% of the tensor's max magnitude are compared absolutely (against rel * 1% * max)


def assert_rel(actual, expected, rel=REL, floor=FLOOR, what=""):
    """|a-b| <= rel * max(|b|, floor * max|b|) element-wise."""
    a = actual.detach().double().cpu().reshape(-1)
    b = expected.detach().double().cpu().reshape(-1)
    assert a.shape == b.shape, (what, actual.shape, expected.shape)
    assert torch.isfinite(a).all(), f"{what}: non-finite values"
    scale = float(b.abs().max()) if b.numel() else 0.0
    tol = rel * torch.maximum(b.abs(), torch.full_like(b, floor * scale)) + 1e-30
    err = (a - b).abs()
    bad = err > tol
    if bad.any():
        i = int(torch.argmax(err / tol))
        raise AssertionError(
            f"{what}: {int(bad.sum())}/{a.numel()} elements off; worst idx {i}: got {a[i]:.8g} want {b[i]:.8g} "
            f"(err {err[i]:.3g}, tol {tol[i]:.3g}, scale {scale:.3g})"
        )


def variant(name: str):
    """Field hyper-parameters of "small" (fruit_nerf), "big" (fruit_nerf_big) or "huge" (fruit_nerf_huge: the big network
    on a max_res 8192 grid)."""
    if name == "huge":
        return dict(syn.BIG, max_res=8192)
    return dict(syn.SMALL if name == "small" else syn.BIG)


def make_state(name: str, table_scale=0.5, weight_gain=1.5, num_images=7, log2T=None):
    v = variant(name)
    T = log2T or v["log2_hashmap_size"]
    sd = syn.field_state(geo=v["geo"], sem_dims=v["sem_dims"], log2_hashmap_size=T, num_images=num_images,
                         table_scale=table_scale, weight_gain=weight_gain)
    spec = fr.FieldSpec(max_res=v["max_res"], log2_hashmap_size=T, geo_feat_dim=v["geo"])
    return sd, spec


HASH_KEY = "mlp_base_grid.hash_table"
# Gradient bar against the float64 oracle, both implementations.  On one H100 the worst normalized errors of
# tests/test_gpu_backward_configs.py are 4.4e-5 (simt) and 3.8e-4 (wgmma: bf16 hi/lo operands, ~2^-17 per product, summed
# over a tile and accumulated with fp32 atomics); the fp32 oracle sits at 1e-5.  tests/test_backward_bars_host.py pins the
# bar from both sides on the CPU.
GRAD_REL = 1e-3
GRAD_FLOOR = 0.05  # elements below 5% of their group's scale are compared against rel * 5% * scale
RELU_MARGIN = 1e-4  # samples with a hidden pre-activation within 1e-4 (relative to the layer rms) of zero


def _grad_scales(want: torch.Tensor, key: str, num_levels: int, own_rows=None, hash_key: str = HASH_KEY) -> torch.Tensor:
    """Per-element scale of a gradient tensor: its max |value|; for the hash table (``hash_key``: the field's, or a proposal
    network's PROP_HASH_KEY) the max of each of its ``num_levels`` levels, and ``own_rows`` (flat table rows) each scaled by
    themselves, outside their level's scale."""
    b = want.abs()
    if key != hash_key:
        return b.amax().expand_as(b)
    lv = b.reshape(num_levels, -1, b.shape[-1])
    own = torch.zeros(lv.shape[:2], dtype=torch.bool)
    if own_rows is not None:
        own.view(-1)[torch.as_tensor(own_rows).reshape(-1)] = True
    level_scale = lv.masked_fill(own[..., None], 0.0).amax(dim=(1, 2), keepdim=True).expand_as(lv)
    row_scale = lv.amax(dim=2, keepdim=True).expand_as(lv)
    return torch.where(own[..., None], row_scale, level_scale).reshape(b.shape)


def grad_errors(got: dict, want: dict, num_levels: int = 16, floor: float = GRAD_FLOOR, own_rows=None, hash_key: str = HASH_KEY) -> dict:
    """Worst normalized error per tensor: max |a - b| / max(|b|, floor * scale), scales from ``_grad_scales``.  A tensor
    whose reference is exactly zero gets an infinite error for any nonzero element (and 0 when it is zero too)."""
    res = {}
    for key, b in want.items():
        a = got[key].detach().double().cpu()
        b = b.detach().double().cpu()
        assert a.shape == b.shape, (key, a.shape, b.shape)
        assert bool(torch.isfinite(a).all()), f"grad {key}: non-finite values"
        den = torch.maximum(b.abs(), floor * _grad_scales(b, key, num_levels, own_rows, hash_key))
        err = (a - b).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / den)  # den == 0 and err > 0 -> inf
        res[key] = float(ratio.max()) if ratio.numel() else 0.0
    return res


def assert_grads(got: dict, want: dict, rel: float = GRAD_REL, what: str = "", **kw) -> float:
    """Every gradient tensor within ``rel`` (normalized, see grad_errors) of the reference; returns the worst error."""
    errs = grad_errors(got, want, **kw)
    bad = {k: f"{v:.3g}" for k, v in errs.items() if not v <= rel}
    assert not bad, f"{what}: gradients off the {rel:g} bar: {bad}"
    worst = max(errs.values())
    print(f"{what}: worst normalized gradient error {worst:.3g} ({max(errs, key=errs.get)}), bar {rel:g}")
    return worst


def safe_ray_weights(f, min_rays: int = 8) -> torch.Tensor:
    """[R] 1 for rays whose samples all keep a ReLU margin, else 0.  d relu(x)/dx at x ~ 0 depends on the last bits of x:
    the tensor-core path computes pre-activations to ~2^-16 (bf16 hi/lo operands), so masks may legitimately differ there and
    the sample's gradient changes discretely.  Such rays get zero loss weight on both sides."""
    ok = (f["relu_margin"] > RELU_MARGIN).all(dim=1).double()
    assert ok.sum() >= min_rays, f"only {int(ok.sum())} of {ok.numel()} rays keep a ReLU margin; enlarge the batch"
    return ok


UPSTREAM_KEYS = ("rgb", "accumulation", "semantics", "weights", "sample_density", "sample_rgb", "sample_semantics")


def oracle_outputs(f, starts, ends, training=True, pass_semantic_gradients=False) -> dict:
    """fr.render of a field_forward result, in the shapes ops.render returns ([R,3], [R], [R], [R,S], [R,S], [R,S,3], [R,S])."""
    r = fr.render(f, starts[..., None], ends[..., None], training=training, pass_semantic_gradients=pass_semantic_gradients)
    return {"rgb": r["rgb"], "accumulation": r["accumulation"][..., 0], "semantics": r["semantics"][..., 0],
            "weights": r["weights"][..., 0], "sample_density": f["density"][..., 0], "sample_rgb": f["rgb"],
            "sample_semantics": f["semantics"][..., 0]}


def upstream_coefficients(R: int, S: int, salt: int = 0) -> dict:
    """Fixed U(-1,1) coefficients of a linear loss on every differentiable output of ops.render (density's scaled by 0.1)."""
    shapes = {"rgb": (R, 3), "accumulation": (R,), "semantics": (R,), "weights": (R, S), "sample_density": (R, S),
              "sample_rgb": (R, S, 3), "sample_semantics": (R, S)}
    coefs = {}
    for i, (k, shp) in enumerate(shapes.items()):
        n = 1
        for v in shp:
            n *= v
        c = syn.hash_uniform(n, 700 + 10 * salt + i, "cpu").view(shp)
        coefs[k] = c * 0.1 if k == "sample_density" else c
    return coefs


def coefficient_loss(coefs: dict, keys=UPSTREAM_KEYS):
    """loss(out, w) = sum over ``keys`` of sum(w_ray * c * out[key])."""
    def loss(out, w):
        total = 0.0
        for k in keys:
            c = coefs[k].to(out[k].device, out[k].dtype)
            total = total + (w.to(c).view(-1, *[1] * (c.dim() - 1)) * c * out[k]).sum()
        return total
    return loss


def mse_bce_loss(image, mask, batch_rays=None):
    """FruitModel's rgb MSE + semantic BCE (fruit_nerf.py:359-366), each ray weighted by w.  The means are over
    ``batch_rays`` rays (default: the rays given), so that the rays of a part of a batch get the whole batch's loss terms."""
    def loss(out, w):
        w = w.to(out["rgb"])
        R = w.shape[0] if batch_rays is None else batch_rays
        bce = torch.nn.functional.binary_cross_entropy_with_logits(out["semantics"], mask.to(out["rgb"]).reshape(-1), reduction="none")
        return (w[:, None] * (image.to(out["rgb"]) - out["rgb"]) ** 2).sum() / (3 * R) + (w * bce).sum() / R
    return loss


def ray_loss(kind: str, R: int, S: int, keys=UPSTREAM_KEYS):
    """loss_of(rays=slice(None)) -> loss(out, w) of the rays ``rays`` (a slice or index tensor) of an R x S batch:
    "mse_bce" (mse_bce_loss of syn.targets(R)) or the linear loss of upstream_coefficients(R, S) on ``keys``.  Both are sums
    over rays, so the losses of disjoint sets of rays add up to the whole batch's."""
    if kind == "mse_bce":
        img, mask = syn.targets(R)
        return lambda rays=slice(None): mse_bce_loss(img[rays], mask[rays], batch_rays=R)
    coefs = upstream_coefficients(R, S)
    return lambda rays=slice(None): coefficient_loss({k: c[rays] for k, c in coefs.items()}, keys)


@dataclass
class OracleRun:
    grads: dict
    field: dict
    out: dict
    ray_weights: torch.Tensor
    loss: torch.Tensor


def oracle_params(sd, dtype=torch.float64) -> dict:
    """The parameters of a state dict as ``dtype`` leaves that require grad (the aabb and integer buffers as they are)."""
    return {k: v.detach().to(dtype, copy=True).requires_grad_(True) if v.is_floating_point() and k != "aabb" else v
            for k, v in sd.items()}


def oracle_backward(sd, spec, rays, loss_fn, contraction=True, appearance="train", training=True, pass_semantic_gradients=False,
                    dtype=torch.float64, ray_weights=None, mutate=None, min_rays=8, params=None) -> OracleRun:
    """Autograd through the oracle with the parameters in ``dtype``.  Rays stay float32, so sample positions (and hash rows
    and trilinear offsets) are bit-equal to the kernels' (test_gpu_parity.py::test_hash_rows_bit_exact).  ``ray_weights``:
    per-ray loss weights (default: this run's ReLU margins); ``mutate(out) -> out`` edits the outputs before the loss.
    ``params``: oracle_params(sd, dtype) to add this run's gradients to (default: fresh ones)."""
    o, d, s, e, cam = rays
    if params is None:
        params = oracle_params(sd, dtype)
    sp = replace(spec, pass_semantic_gradients=pass_semantic_gradients)
    f = fr.field_forward(params, sp, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, contraction=contraction,
                         appearance=appearance)
    out = oracle_outputs(f, s, e, training, pass_semantic_gradients)
    if ray_weights is None:
        ray_weights = safe_ray_weights(f, min_rays)
    if mutate is not None:
        out = mutate(out)
    loss = loss_fn(out, ray_weights)
    loss.backward()
    grads = {k: (p.grad if p.grad is not None else torch.zeros_like(p)).detach() for k, p in params.items() if p.requires_grad}
    return OracleRun(grads, f, out, ray_weights, loss.detach())


def chunked_oracle_backward(sd, spec, rays, loss_of, chunk=512, contraction=True, appearance="train", training=True,
                            pass_semantic_gradients=False, dtype=torch.float64, ray_weights=None, min_rays=8) -> OracleRun:
    """oracle_backward of the loss ``loss_of()`` (see ray_loss) over chunks of ``chunk`` rays, the gradients of the chunks'
    losses ``loss_of(chunk)`` summed: exact, since the loss is a sum over rays, and it bounds the autograd graph (at 4096 x 48
    samples one graph in float64 takes several GB).  The default ray weights are the unchunked run's: safe_ray_weights of one
    forward over the whole batch, whose ReLU margins are relative to the layer rms over field_forward's own sample chunks.
    ``field`` and ``out`` hold the chunks' tensors concatenated, detached."""
    R = rays[2].shape[0]
    params = oracle_params(sd, dtype)
    if ray_weights is None:
        o, d, s, e, cam = rays
        with torch.no_grad():
            f = fr.field_forward(params, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, contraction=contraction,
                                 appearance=appearance)
        ray_weights = safe_ray_weights(f, min_rays)
        del f
    fields, outs, loss = [], [], 0.0
    for a in range(0, R, chunk):
        part = slice(a, min(R, a + chunk))
        run = oracle_backward(sd, spec, tuple(t[part] for t in rays), loss_of(part), contraction=contraction, appearance=appearance,
                              training=training, pass_semantic_gradients=pass_semantic_gradients, dtype=dtype,
                              ray_weights=ray_weights[part], params=params)
        fields.append({k: v.detach() for k, v in run.field.items()})
        outs.append({k: v.detach() for k, v in run.out.items()})
        loss = loss + run.loss
    grads = {k: (p.grad if p.grad is not None else torch.zeros_like(p)).detach() for k, p in params.items() if p.requires_grad}
    return OracleRun(grads, {k: torch.cat([f[k] for f in fields]) for k in fields[0]},
                     {k: torch.cat([o[k] for o in outs]) for k in outs[0]}, ray_weights, loss)


# ---- the field backward's tile schedule ---------------------------------------------------------------------------------------
TILE_POINTS = 128  # points of one warpgroup tile of the field kernels
RESIDENT_GROUPS = 2  # warpgroups per CTA of the small family's tensor-core backward


def resident_backward_rounds(N: int, sms: int):
    """([tiles] round of each tile, CTA count) of the small family's tensor-core backward over N points on a GPU of ``sms``
    SMs (fnr_simt.cu: launch_field, simt_field_backward_kernel): min(ceil(N / 256), sms) CTAs of two warpgroups;
    warpgroup g of CTA b takes tile 2b + g, then every (2 * CTAs)-th tile after it, so tile t runs in round
    t // (2 * CTAs).  A CTA keeps its weight gradients on chip over all its rounds and flushes them after the last."""
    tiles = -(-N // TILE_POINTS)
    grid = min(-(-N // (RESIDENT_GROUPS * TILE_POINTS)), sms)
    return torch.arange(tiles) // (RESIDENT_GROUPS * grid), grid


def live_rays_per_round(rounds: torch.Tensor, ray_weights: torch.Tensor, S: int) -> list:
    """Per round, the number of rays of nonzero weight with a sample in one of the round's tiles."""
    R = ray_weights.shape[0]
    point_round = rounds.repeat_interleave(TILE_POINTS)[:R * S].view(R, S)
    live = ray_weights > 0
    return [int((live & (point_round == k).any(dim=1)).sum()) for k in range(int(rounds.max()) + 1)]


def make_field(name: str, sd, spec, device, contraction=True, test_mode=None, **kw) -> FruitField:
    v = variant(name)
    f = FruitField(
        aabb=sd["aabb"], num_images=sd["embedding_appearance.embedding.weight"].shape[0], geo_feat_dim=v["geo"],
        max_res=v["max_res"], log2_hashmap_size=spec.log2_hashmap_size, num_layers_semantic=len(v["sem_dims"]) - 1,
        hidden_dim_semantics=v["sem_dims"][1], use_semantics=True, num_semantic_classes=1, test_mode=test_mode,
        spatial_distortion=SceneContraction(order=float("inf")) if contraction else None, **kw,
    )
    missing, unexpected = f.load_state_dict({k: v_ for k, v_ in sd.items()}, strict=False)
    # only the Sequential aliases and registered scalar buffers may be absent from the synthetic dict
    assert not unexpected, unexpected
    assert all(k.startswith("mlp_base.") or k in ("max_res", "num_levels", "log2_hashmap_size") for k in missing), missing
    return f.to(device)


# ---- proposal stage ------------------------------------------------------------------------------------------------------------
PROP_HASH_KEY = "encoding.hash_table"
PROP_KEYS = (PROP_HASH_KEY, "mlp_base.1.layers.0.weight", "mlp_base.1.layers.0.bias", "mlp_base.1.layers.1.weight",
             "mlp_base.1.layers.1.bias")


def proposal_rays(R: int, S: int, salt: int = 0, far: float = 30.0):
    """(origins, directions, starts, ends) float32: syn.ray_batch rays with nears 0.05 and fars ``far``, S bins spaced by the
    piecewise linear-in-disparity map of the initial sampler (one jitter per ray)."""
    o, d, _, _, _ = syn.ray_batch(R, 4, salt=salt)
    nears, fars = torch.full((R, 1), 0.05), torch.full((R, 1), far)
    bins = ns.spaced_bins(R, S, (syn.hash_uniform(R, 77 + salt).view(R, 1) + 1) * 0.5)
    e = ns.spacing_to_euclidean(bins, nears, fars)
    return o, d, e[:, :-1].contiguous(), e[:, 1:].contiguous()


def weight_coefficients(R: int, S: int, salt: int = 0) -> torch.Tensor:
    """[R,S] U(-1,1) coefficients of a linear loss on the proposal weights.  Signed: with one-signed coefficients the gradient
    of the output bias (a sum of d loss / d log-density over every sample) cancels ~3000-fold, and fp32 arithmetic alone
    (the float32 oracle's) leaves it 2e-3 off the float64 value."""
    return syn.hash_uniform(R * S, 91 + salt).view(R, S)


@dataclass
class ProposalRun:
    grads: dict
    weights: torch.Tensor
    ray_weights: torch.Tensor


def proposal_oracle_backward(sd, spec, rays, coef, contraction=True, dtype=torch.float64, ray_weights=None, chunk=1024,
                             min_rays=8) -> ProposalRun:
    """Gradients of sum(ray_w * coef * w) by autograd through fr.proposal_weights with the parameters in ``dtype``, formed
    over chunks of ``chunk`` rays (the loss is a sum over rays).  Rays stay float32, so sample positions, hash rows and
    trilinear offsets are the kernels'.  ``ray_weights`` default: 1 for the rays whose samples all keep RELU_MARGIN."""
    o, d, s, e = rays
    params = {k: v.detach().to(dtype, copy=True).requires_grad_(True) for k, v in sd.items() if k != "aabb"}
    aabb = sd["aabb"]
    R = s.shape[0]
    ws, rws = [], []
    for a in range(0, R, chunk):
        b = min(R, a + chunk)
        w, margin = fr.proposal_weights(params, spec, o[a:b], d[a:b], s[a:b], e[a:b], aabb, contraction, relu_margin=True)
        rw = (margin > RELU_MARGIN).all(dim=1).to(dtype) if ray_weights is None else ray_weights[a:b].to(dtype)
        (rw[:, None] * coef[a:b].to(dtype) * w).sum().backward()
        ws.append(w.detach())
        rws.append(rw)
    rw = torch.cat(rws)
    assert rw.sum() >= min_rays, f"only {int(rw.sum())} of {R} rays keep a ReLU margin"
    grads = {k: (p.grad if p.grad is not None else torch.zeros_like(p)).detach() for k, p in params.items()}
    return ProposalRun(grads, torch.cat(ws), rw)


def proposal_net(sd, spec, contraction=True, device="cuda"):
    """HashMLPDensityField of ``spec`` holding the parameters of a syn.density_state dict."""
    from fruitnerf_b200.density_field import HashMLPDensityField

    net = HashMLPDensityField(sd["aabb"], hidden_dim=spec.hidden_dim, log2_hashmap_size=spec.log2_hashmap_size, num_levels=spec.num_levels,
                              max_res=spec.max_res, spatial_distortion=SceneContraction() if contraction else None)
    missing, unexpected = net.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("mlp_base.0") or k in ("max_res", "num_levels", "log2_hashmap_size") for k in missing)
    return net.to(device)


def proposal_edge_case(spec, R: int = 509, S: int = 96, salt: int = 3):
    """AABB-mode batch (positions normalized by the box, no contraction) of R ordinary rays out to t = 30, most of which leave
    the box, and three edge rays appended:
      R     every sample outside the box (selector 0 everywhere: density 0, no gradient);
      R + 1 every other bin of zero width;
      R + 2 S bins of 1e-8 around t = 1e-3, all in the same grid cells, whose table rows are set so that the density's
            pre-activation h is 17: past trunc_exp's backward clamp at 15, with sigma * delta ~ 0.25 per bin.
    Returns (state, (origins, directions, starts, ends)) with R + 3 rays."""
    sd = syn.density_state(num_levels=spec.num_levels, log2_hashmap_size=spec.log2_hashmap_size, salt=7000 + salt)
    o, d, s, e = proposal_rays(R, S, salt=salt)
    out_o, out_d = torch.tensor([[3.0, 3.0, 3.0]]), torch.tensor([[0.6, 0.0, 0.8]])
    zw_s, zw_e = s[:1].clone(), e[:1].clone()
    zw_e[:, 1::2] = zw_s[:, 1::2]
    cl_o, cl_d = torch.tensor([[0.3, -0.2, 0.1]]), torch.tensor([[0.0, 0.6, 0.8]])
    cl_s = (1e-3 + 1e-8 * torch.arange(S, dtype=torch.float32))[None]
    cl_e = (1e-3 + 1e-8 * torch.arange(1, S + 1, dtype=torch.float32))[None]
    o = torch.cat([o, out_o, o[:1], cl_o]).contiguous()
    d = torch.cat([d, out_d, d[:1], cl_d]).contiguous()
    s = torch.cat([s, s[:1], zw_s, cl_s]).contiguous()
    e = torch.cat([e, e[:1], zw_e, cl_e]).contiguous()
    # the clamp ray: every corner row of its cells, every level, holds (a, a); h(a) = 17 solved by bisection on the side of a
    # along which h grows without bound
    p = ns.normalized_positions(ns.frustum_positions(cl_o[:, None], cl_d[:, None], cl_s[..., None], cl_e[..., None]), sd["aabb"])
    rows = ns.hash_corner_indices(p.reshape(-1, 3), spec.scalings(), spec.log2_hashmap_size)[0].unique()
    w0, b0 = sd["mlp_base.1.layers.0.weight"].double(), sd["mlp_base.1.layers.0.bias"].double()
    w1, b1 = sd["mlp_base.1.layers.1.weight"].double()[0], float(sd["mlp_base.1.layers.1.bias"])
    rs = w0.sum(dim=1)

    def h(a):
        return b1 + float((w1 * torch.relu(a * rs + b0)).sum())

    sign = 1.0 if h(1e4) > h(-1e4) else -1.0
    lo, hi = 0.0, sign * 1e4
    assert h(hi) > 17.0 > h(lo), "the density MLP does not reach the clamp along (a, a)"
    for _ in range(100):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if h(mid) < 17.0 else (lo, mid)
    sd["encoding.hash_table"][rows] = float(hi)
    return sd, (o, d, s, e)


def interlevel_inputs(R: int, prop_samples, Sc: int, salt: int = 0):
    """Final-level bins c [R,Sc+1] and weights w [R,Sc] and, per proposal level, bins cp [R,Sp+1] and weights wp [R,Sp]:
    sorted U(0,1) interior bin edges and softmax weights (sums 0.9 and 0.8)."""
    def edges(n, s):
        return torch.sort(torch.cat([torch.zeros(R, 1), (syn.hash_uniform(R * (n - 1), s).view(R, n - 1) + 1) * 0.5, torch.ones(R, 1)], 1), 1).values

    c = edges(Sc, 1 + 100 * salt)
    w = torch.softmax(syn.hash_uniform(R * Sc, 2 + 100 * salt).view(R, Sc) * 3, -1) * 0.9
    props = [(edges(Sp, 10 + k + 100 * salt), torch.softmax(syn.hash_uniform(R * Sp, 20 + k + 100 * salt).view(R, Sp) * 2, -1) * 0.8)
             for k, Sp in enumerate(prop_samples)]
    return c, w, props


def interlevel_reference(c, w, props, ray_weights=None, mult: float = 1.0, dtype=torch.float64):
    """nerfstudio interlevel_loss (ns.interlevel_loss) with per-ray weights: sum over levels of sum(ray_w * lossfun_outer) / (R*Sc),
    and its gradient with respect to each level's weights.  Returns (loss, [d loss / d wp])."""
    R, Sc = w.shape
    rw = torch.ones(R, dtype=dtype) if ray_weights is None else ray_weights.to(dtype)
    wps = [wp.detach().to(dtype).requires_grad_(True) for _, wp in props]
    loss = 0.0
    for (cp, _), wp in zip(props, wps):
        loss = loss + (rw[:, None] * ns.lossfun_outer(c, w.to(dtype), cp, wp)).sum() / (R * Sc) * mult
    loss.backward()
    return loss.detach(), [wp.grad for wp in wps]


def proposal_configs():
    """{"<method>/L<k>": (DensitySpec, samples per ray, rays per batch)} for each proposal level of the fruit_nerf, fruit_nerf_big
    and fruit_nerf_huge methods, read from their configs; and {"<method>": (proposal samples, nerf samples)}."""
    from fruitnerf_b200.fruit_nerf_config import METHODS

    levels, interlevel = {}, {}
    for name in ("fruit_nerf", "fruit_nerf_big", "fruit_nerf_huge"):
        m = METHODS[name].pipeline.model
        R = METHODS[name].pipeline.datamanager.train_num_rays_per_batch
        for k, S in enumerate(m.num_proposal_samples_per_ray):
            a = m.proposal_net_args_list[min(k, len(m.proposal_net_args_list) - 1)]
            spec = fr.DensitySpec(num_levels=a["num_levels"], max_res=a["max_res"], log2_hashmap_size=a["log2_hashmap_size"],
                                  hidden_dim=a["hidden_dim"])
            levels[f"{name}/L{k}"] = (spec, S, R)
        interlevel[name] = (tuple(m.num_proposal_samples_per_ray), m.num_nerf_samples_per_ray)
    return levels, interlevel


def interlevel_bar(f32_grads, ref_grads) -> float:
    """Bar of the interlevel gradient: GRAD_REL, or twice the float32 oracle's distance from the float64 one if that is larger.
    The gradient -2 (w - w_outer) / w of each final interval divides the rounding of w_outer, a difference of two entries of
    the proposal weights' cumulative sum (~2^-24 absolute), by the final weight w: at Sc = 128 final samples the smallest
    w are ~1e-4 and fp32 arithmetic alone leaves the gradient ~1.1e-3 off the float64 value."""
    errs = grad_errors({k: g for k, g in enumerate(f32_grads)}, {k: g for k, g in enumerate(ref_grads)})
    bar = max(GRAD_REL, 2.0 * max(errs.values()))
    assert bar <= INTERLEVEL_BAR_CAP, f"the float32 interlevel gradient is {max(errs.values()):.3g} off: more than rounding explains"
    return bar


INTERLEVEL_BAR_CAP = 2.5e-3  # fp32 rounding reaches 1.1e-3 at the training shapes; a bar past 2.5e-3 means the reference drifted
