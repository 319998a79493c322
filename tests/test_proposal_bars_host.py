"""CPU pins of the gradient bar the proposal-stage GPU tests use (tests/test_gpu_proposal_configs.py: tests/util.py grad_errors at
GRAD_REL, the proposal hash table level by level).

On reduced-R versions of those tests' inputs the float32 oracle must pass against the float64 oracle with at least a 2x margin
(the bar is not tighter than fp32 arithmetic allows), and the bar must reject gradients that are wrong in the ways the proposal
kernels could go subtly wrong (it is not looser than it has to be): a ray left out, 1% on the finest hash level, trunc_exp's
backward clamp dropped, the transmittance gradient of the second 32-sample chunk summed from the wrong later chunks, the
selector ignored in the backward, and the two proposal levels' interlevel gradients exchanged.

Measured: the float32 oracle sits at 6.6e-5 (huge_L1) and 5.4e-5 (edge_aabb) of the 1e-3 bar; the mutations land at 3.7 (ray
removed), 1.0e-2 (level x 0.99), 0.94 (wrong chunk), 5.7 (no clamp) and 1.2e3 (selector ignored).  The float32 interlevel
gradient sits at 3.0e-4, 1.1e-3 and 6.4e-4 of the float64 one at the fruit_nerf, big and huge shapes (tests/util.py:interlevel_bar).
"""
import pytest
import torch

from fruitnerf_b200 import synthetic as syn
from oracle import ns_torch as ns

from .util import (GRAD_REL, PROP_HASH_KEY, grad_errors, interlevel_bar, interlevel_inputs, interlevel_reference, proposal_configs, proposal_edge_case,
                   proposal_oracle_backward, proposal_rays, weight_coefficients)

R = 512
_GET_WEIGHTS = ns.get_weights


def _weights_case(kind):
    levels, _ = proposal_configs()
    if kind == "huge_L1":  # 7 levels up to 2048, 512 samples out to t = 1000
        spec, S, _ = levels["fruit_nerf_huge/L1"]
        sd = syn.density_state(num_levels=spec.num_levels, log2_hashmap_size=spec.log2_hashmap_size)
        return sd, spec, proposal_rays(R, S, salt=2, far=1000.0), True
    spec, _, _ = levels["fruit_nerf/L1"]
    sd, rays = proposal_edge_case(spec, R=R - 3)
    return sd, spec, rays, False


@pytest.fixture(scope="module", params=["huge_L1", "edge_aabb"])
def wruns(request):
    sd, spec, rays, contraction = _weights_case(request.param)
    coef = weight_coefficients(*rays[2].shape)
    ref = proposal_oracle_backward(sd, spec, rays, coef, contraction)
    f32 = proposal_oracle_backward(sd, spec, rays, coef, contraction, dtype=torch.float32, ray_weights=ref.ray_weights)
    return dict(kind=request.param, sd=sd, spec=spec, rays=rays, coef=coef, contraction=contraction, ref=ref, f32=f32)


def _errors(got, ref, spec):
    return grad_errors(got, ref.grads, num_levels=spec.num_levels, hash_key=PROP_HASH_KEY)


def test_fp32_oracle_passes_with_margin(wruns):
    errs = _errors(wruns["f32"].grads, wruns["ref"], wruns["spec"])
    worst = max(errs.values())
    print(f"{wruns['kind']}: fp32 oracle vs fp64: worst normalized error {worst:.3g} ({max(errs, key=errs.get)}), bar {GRAD_REL:g}")
    assert worst <= GRAD_REL / 2, errs


def _f32(runs, ray_weights=None):
    return proposal_oracle_backward(runs["sd"], runs["spec"], runs["rays"], runs["coef"], runs["contraction"], dtype=torch.float32,
                                    ray_weights=runs["ref"].ray_weights if ray_weights is None else ray_weights).grads


def _drop_ray(runs, monkeypatch):
    w = runs["ref"].ray_weights.clone()
    w[int(torch.nonzero(w)[0])] = 0.0
    return _f32(runs, w)


def _scale_level(runs, monkeypatch):
    g = dict(runs["f32"].grads)
    L = runs["spec"].num_levels
    t = g[PROP_HASH_KEY].clone()
    t.view(L, -1, 2)[L - 1] *= 0.99
    g[PROP_HASH_KEY] = t
    return g


def _no_clamp(runs, monkeypatch):
    monkeypatch.setattr(ns, "trunc_exp", torch.exp)
    return _f32(runs)


def _no_selector(runs, monkeypatch):
    monkeypatch.setattr(ns, "select_density", lambda dens, sel: dens - (dens * (~sel)[..., None]).detach())
    return _f32(runs)


class _WrongChunkSuffix(torch.autograd.Function):
    """get_weights with the backward the kernels use, dL/dx_j = G_j T_{j+1} - sum_{i>j} G_i w_i, except that samples 32..63
    take the later-chunk part of their suffix sum from chunk 2's lane (chunks after 2) instead of chunk 1's (chunks after 1)."""

    @staticmethod
    def forward(ctx, deltas, densities):
        w = _GET_WEIGHTS(deltas, densities)
        ctx.save_for_backward(deltas, densities, w)
        return w

    @staticmethod
    def backward(ctx, g):
        deltas, densities, w = ctx.saved_tensors
        x, G, w = (deltas * densities)[..., 0], g[..., 0], w[..., 0]
        gw = G * w
        suffix = gw.flip(-1).cumsum(-1).flip(-1) - gw
        suffix[:, 32:64] -= gw[:, 64:96].sum(-1, keepdim=True)
        dx = G * torch.exp(-torch.cumsum(x, -1)) - suffix
        return None, (dx * deltas[..., 0])[..., None]


def _wrong_chunk(runs, monkeypatch):
    assert runs["rays"][2].shape[1] >= 96
    monkeypatch.setattr(ns, "get_weights", _WrongChunkSuffix.apply)
    return _f32(runs)


MUTATIONS = {"one ray removed": ("huge_L1", _drop_ray), "hash level L-1 x 0.99": ("huge_L1", _scale_level),
             "trunc_exp clamp removed": ("edge_aabb", _no_clamp), "suffix of chunk 1 from chunk 2": ("huge_L1", _wrong_chunk),
             "selector ignored in the backward": ("edge_aabb", _no_selector)}


@pytest.mark.parametrize("wruns,mutation", [(kind, m) for m, (kind, _) in MUTATIONS.items()], indirect=["wruns"])
def test_bar_rejects_mutation(wruns, mutation, monkeypatch):
    _, fn = MUTATIONS[mutation]
    errs = _errors(fn(wruns, monkeypatch), wruns["ref"], wruns["spec"])
    worst = max(errs.values())
    print(f"{mutation}: worst normalized error {worst:.3g} ({max(errs, key=errs.get)}), bar {GRAD_REL:g}")
    assert worst > GRAD_REL, f"{mutation} passes the bar: {errs}"


def test_wrong_chunk_mutation_is_exact_elsewhere():
    """The wrong-chunk backward agrees with autograd through get_weights outside samples 32..63: that chunk is all it changes."""
    x = torch.rand(3, 100, 1, dtype=torch.float64) * 0.1
    d = torch.rand(3, 100, 1, dtype=torch.float64).requires_grad_(True)
    g = torch.rand(3, 100, 1, dtype=torch.float64)
    (a,) = torch.autograd.grad(_GET_WEIGHTS(x, d), d, g)
    (b,) = torch.autograd.grad(_WrongChunkSuffix.apply(x, d), d, g)
    assert not torch.allclose(a[:, 32:64], b[:, 32:64]) and torch.allclose(a[:, :32], b[:, :32]) and torch.allclose(a[:, 64:], b[:, 64:])


# ---- interlevel loss ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["fruit_nerf", "fruit_nerf_big", "fruit_nerf_huge"])
def iruns(request):
    _, inter = proposal_configs()
    props_n, Sc = inter[request.param]
    c, w, props = interlevel_inputs(R, props_n, Sc)
    _, ref = interlevel_reference(c.double(), w, [(cp.double(), wp) for cp, wp in props])
    _, f32 = interlevel_reference(c, w, props, dtype=torch.float32)
    return dict(name=request.param, c=c, w=w, props=props, ref=ref, f32=f32)


def _ilevels(gs):
    return {f"level {k}": g for k, g in enumerate(gs)}


def test_interlevel_fp32_passes_with_margin(iruns):
    """The bar is GRAD_REL or twice the float32 oracle's distance, whichever is larger (interlevel_bar refuses a bar past
    INTERLEVEL_BAR_CAP); on the fruit_nerf shape at these 512 rays it is GRAD_REL."""
    errs = grad_errors(_ilevels(iruns["f32"]), _ilevels(iruns["ref"]))
    worst = max(errs.values())
    bar = interlevel_bar(iruns["f32"], iruns["ref"])
    print(f"{iruns['name']}: fp32 interlevel gradient vs fp64: worst normalized error {worst:.3g}, bar {bar:.3g}")
    assert worst <= bar / 2, errs
    if iruns["name"] == "fruit_nerf":
        assert bar == GRAD_REL


def test_interlevel_bar_rejects_dropped_ray(iruns):
    rw = torch.ones(R)
    rw[7] = 0.0
    _, got = interlevel_reference(iruns["c"], iruns["w"], iruns["props"], ray_weights=rw, dtype=torch.float32)
    errs = grad_errors(_ilevels(got), _ilevels(iruns["ref"]))
    assert max(errs.values()) > interlevel_bar(iruns["f32"], iruns["ref"]), errs


@pytest.mark.parametrize("iruns", ["fruit_nerf_huge"], indirect=True)
def test_interlevel_bar_rejects_swapped_levels(iruns):
    """At (512, 512) + 64 both levels' gradients have one shape, so a kernel could write each into the other's."""
    errs = grad_errors(_ilevels(iruns["f32"][::-1]), _ilevels(iruns["ref"]))
    print(f"swapped levels: worst normalized error {max(errs.values()):.3g}")
    assert max(errs.values()) > interlevel_bar(iruns["f32"], iruns["ref"]), errs
