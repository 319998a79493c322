"""Shared helpers of the test-suite (oracle-side glue + tolerances)."""
from __future__ import annotations

from dataclasses import dataclass, replace

import torch

from fruitnerf_b200 import synthetic as syn
from fruitnerf_b200.fruit_field import FruitField, SceneContraction
from oracle import fruit_ref as fr

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


def _grad_scales(want: torch.Tensor, key: str, num_levels: int, own_rows=None) -> torch.Tensor:
    """Per-element scale of a gradient tensor: its max |value|; for the hash table the max of each level, and ``own_rows``
    (flat table rows) each scaled by themselves, outside their level's scale."""
    b = want.abs()
    if key != HASH_KEY:
        return b.amax().expand_as(b)
    lv = b.reshape(num_levels, -1, b.shape[-1])
    own = torch.zeros(lv.shape[:2], dtype=torch.bool)
    if own_rows is not None:
        own.view(-1)[torch.as_tensor(own_rows).reshape(-1)] = True
    level_scale = lv.masked_fill(own[..., None], 0.0).amax(dim=(1, 2), keepdim=True).expand_as(lv)
    row_scale = lv.amax(dim=2, keepdim=True).expand_as(lv)
    return torch.where(own[..., None], row_scale, level_scale).reshape(b.shape)


def grad_errors(got: dict, want: dict, num_levels: int = 16, floor: float = GRAD_FLOOR, own_rows=None) -> dict:
    """Worst normalized error per tensor: max |a - b| / max(|b|, floor * scale), scales from ``_grad_scales``.  A tensor
    whose reference is exactly zero gets an infinite error for any nonzero element (and 0 when it is zero too)."""
    res = {}
    for key, b in want.items():
        a = got[key].detach().double().cpu()
        b = b.detach().double().cpu()
        assert a.shape == b.shape, (key, a.shape, b.shape)
        assert bool(torch.isfinite(a).all()), f"grad {key}: non-finite values"
        den = torch.maximum(b.abs(), floor * _grad_scales(b, key, num_levels, own_rows))
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


def mse_bce_loss(image, mask):
    """FruitModel's rgb MSE + semantic BCE (fruit_nerf.py:359-366), each ray weighted by w."""
    def loss(out, w):
        w = w.to(out["rgb"])
        R = w.shape[0]
        bce = torch.nn.functional.binary_cross_entropy_with_logits(out["semantics"], mask.to(out["rgb"]).reshape(-1), reduction="none")
        return (w[:, None] * (image.to(out["rgb"]) - out["rgb"]) ** 2).sum() / (3 * R) + (w * bce).sum() / R
    return loss


@dataclass
class OracleRun:
    grads: dict
    field: dict
    out: dict
    ray_weights: torch.Tensor
    loss: torch.Tensor


def oracle_backward(sd, spec, rays, loss_fn, contraction=True, appearance="train", training=True, pass_semantic_gradients=False,
                    dtype=torch.float64, ray_weights=None, mutate=None, min_rays=8) -> OracleRun:
    """Autograd through the oracle with the parameters in ``dtype``.  Rays stay float32, so sample positions (and hash rows
    and trilinear offsets) are bit-equal to the kernels' (test_gpu_parity.py::test_hash_rows_bit_exact).  ``ray_weights``:
    per-ray loss weights (default: this run's ReLU margins); ``mutate(out) -> out`` edits the outputs before the loss."""
    o, d, s, e, cam = rays
    params = {k: v.detach().to(dtype, copy=True).requires_grad_(True) if v.is_floating_point() and k != "aabb" else v
              for k, v in sd.items()}
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
