"""CPU pins of the gradient bar the GPU backward tests use (tests/util.py: assert_grads, GRAD_REL, GRAD_FLOOR).

On the inputs of tests/test_gpu_backward_configs.py the float32 oracle must pass against the float64 oracle with at least a
2x margin (the bar is not tighter than fp32 arithmetic allows), and the bar must reject gradients that are wrong in the ways a
backward kernel goes subtly wrong (it is not looser than it has to be).
"""
import pytest
import torch

from fruitnerf_b200 import synthetic as syn

from .util import (GRAD_REL, HASH_KEY, coefficient_loss, grad_errors, make_state, mse_bce_loss, oracle_backward,
                   upstream_coefficients)

R, S = 128, 48  # the ray batch of the GPU tests


def _case(name, loss_kind):
    sd, spec = make_state(name, log2T=15)
    rays = syn.ray_batch(R, S, salt=5, far=3.0, num_images=7)
    if loss_kind == "mse_bce":
        img, mask = syn.targets(R)
        loss = mse_bce_loss(img, mask)
    else:
        loss = coefficient_loss(upstream_coefficients(R, S))
    return sd, spec, rays, loss


@pytest.fixture(scope="module", params=[("small", "mse_bce"), ("big", "mse_bce"), ("small", "all7")],
                ids=["small-mse_bce", "big-mse_bce", "small-all7"])
def runs(request):
    name, loss_kind = request.param
    sd, spec, rays, loss = _case(name, loss_kind)
    ref = oracle_backward(sd, spec, rays, loss, pass_semantic_gradients=True)
    f32 = oracle_backward(sd, spec, rays, loss, pass_semantic_gradients=True, dtype=torch.float32, ray_weights=ref.ray_weights)
    return dict(sd=sd, spec=spec, rays=rays, loss=loss, ref=ref, f32=f32)


def test_fp32_oracle_passes_with_margin(runs):
    errs = grad_errors(runs["f32"].grads, runs["ref"].grads)
    worst = max(errs.values())
    print(f"fp32 oracle vs fp64: worst normalized error {worst:.3g} ({max(errs, key=errs.get)}), bar {GRAD_REL:g}")
    assert worst <= GRAD_REL / 2, errs


def _drop_ray(runs):
    w = runs["ref"].ray_weights.clone()
    w[int(torch.nonzero(w)[0])] = 0.0
    return oracle_backward(runs["sd"], runs["spec"], runs["rays"], runs["loss"], pass_semantic_gradients=True, dtype=torch.float32,
                           ray_weights=w).grads


def _scale_level(runs, level=15):
    g = dict(runs["f32"].grads)
    t = g[HASH_KEY].clone()
    t.view(16, -1, 2)[level] *= 0.99
    g[HASH_KEY] = t
    return g


def _no_semantic_pass(runs):
    return oracle_backward(runs["sd"], runs["spec"], runs["rays"], runs["loss"], pass_semantic_gradients=False, dtype=torch.float32,
                           ray_weights=runs["ref"].ray_weights).grads


def _no_background(runs):
    def mutate(out):
        term = out["sample_rgb"][:, -1, :] * (1.0 - out["accumulation"][:, None])
        return dict(out, rgb=out["rgb"] - term + term.detach())  # same values, no gradient through the background term
    return oracle_backward(runs["sd"], runs["spec"], runs["rays"], runs["loss"], pass_semantic_gradients=True, dtype=torch.float32,
                           ray_weights=runs["ref"].ray_weights, mutate=mutate).grads


def _wrong_camera_row(runs):
    g = dict(runs["f32"].grads)
    key = "embedding_appearance.embedding.weight"
    t = g[key].clone()
    c = int(t.norm(dim=1).argmax())
    t[(c + 1) % t.shape[0]] += t[c]
    t[c] = 0.0
    g[key] = t
    return g


MUTATIONS = {"one ray removed": _drop_ray, "hash level 15 x 0.99": _scale_level, "pass_semantic_gradients ignored": _no_semantic_pass,
             "background term omitted": _no_background, "appearance to the wrong camera row": _wrong_camera_row}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_bar_rejects_mutation(runs, mutation):
    errs = grad_errors(MUTATIONS[mutation](runs), runs["ref"].grads)
    worst = max(errs.values())
    print(f"{mutation}: worst normalized error {worst:.3g} ({max(errs, key=errs.get)}), bar {GRAD_REL:g}")
    assert worst > GRAD_REL, f"{mutation} passes the bar: {errs}"
