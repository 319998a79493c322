"""CPU pins of the gradient bar tests/test_gpu_backward_training_shapes.py holds the field backward to at fruit_nerf's
training batch (4096 rays x 48 samples: 1536 tiles, six rounds of the small family's resident backward on the 132 SMs of an
H100 SXM), as tests/test_backward_bars_host.py pins it at R = 128.

The float32 oracle must pass against the float64 oracle with at least a 2x margin, and the bar must reject float64
gradients changed the way a bug confined to a warpgroup's later tiles would change them: a live ray of the last round left
out, the same ray counted twice (one tile flushed twice), every ray of one CTA's tiles after its first round left out (a
warpgroup that stops after one tile), and one ray's semantic-branch gradient missing under pass_semantic_gradients.  The
losses are sums over rays, so each mutation is the float64 run plus or minus the float64 gradients of the rays it changes.

Measured: the float32 oracle sits at 2.1e-5 (small, all7), 1.1e-5 (small, MSE + BCE with pass_semantic_gradients) and
8.5e-6 (big, all7) of the 1e-3 bar.  The mutations land at 2.4 to 8.2, on the hash table; on the other tensors alone at 1.5
(last-round ray removed or doubled), 5.1 (CTA stops after one round) and 5.6e-2 (semantic branch missing), and for the big
family at 0.98 and 1.3.

The chunked oracle these shapes need (tests/util.py:chunked_oracle_backward) is checked against one unchunked run.
"""
import pytest
import torch

from fruitnerf_b200 import synthetic as syn

from .util import (GRAD_REL, HASH_KEY, RESIDENT_GROUPS, TILE_POINTS, chunked_oracle_backward, grad_errors, live_rays_per_round,
                   make_state, oracle_backward, ray_loss, resident_backward_rounds)

R, S = 4096, 48
H100_SXM_SMS = 132
# name -> (family, loss, pass_semantic_gradients): the inputs of the GPU test's cases of the same names
CASES = {"small-all7": ("small", "all7", False), "small-pass_sem": ("small", "mse_bce", True), "big-all7": ("big", "all7", False)}


@pytest.fixture(scope="module", params=list(CASES))
def runs(request):
    name, loss, pass_sem = CASES[request.param]
    sd, spec = make_state(name, num_images=7)  # the family's own table (T = 19 / 21)
    rays = syn.ray_batch(R, S, salt=5, far=3.0, num_images=7)
    loss_of = ray_loss(loss, R, S)
    ref = chunked_oracle_backward(sd, spec, rays, loss_of, pass_semantic_gradients=pass_sem)
    f32 = chunked_oracle_backward(sd, spec, rays, loss_of, pass_semantic_gradients=pass_sem, dtype=torch.float32,
                                  ray_weights=ref.ray_weights)
    rounds, grid = resident_backward_rounds(R * S, H100_SXM_SMS)
    return dict(case=request.param, sd=sd, spec=spec, rays=rays, loss_of=loss_of, pass_sem=pass_sem, ref=ref, f32=f32, rounds=rounds,
                grid=grid)


def test_schedule_reaches_every_round(runs):
    """Six rounds, warpgroups with five tiles and with six, and live rays in every round."""
    rounds, grid = runs["rounds"], runs["grid"]
    per_group = torch.bincount(torch.arange(rounds.numel()) % (RESIDENT_GROUPS * grid))
    live = live_rays_per_round(rounds, runs["ref"].ray_weights, S)
    print(f"{runs['case']}: {rounds.numel()} tiles, {grid} CTAs, tiles per warpgroup {int(per_group.min())}..{int(per_group.max())}, "
          f"live rays per round {live}")
    assert int(rounds.max()) + 1 >= 4 and int(per_group.min()) < int(per_group.max())
    assert min(live) > 0


def test_fp32_oracle_passes_with_margin(runs):
    errs = grad_errors(runs["f32"].grads, runs["ref"].grads)
    worst = max(errs.values())
    print(f"{runs['case']}: fp32 oracle vs fp64: worst normalized error {worst:.3g} ({max(errs, key=errs.get)}), "
          f"{GRAD_REL / worst:.3g}x inside the bar {GRAD_REL:g}")
    assert worst <= GRAD_REL / 2, errs


def _ray_grads(runs, rays, pass_sem=None):
    """float64 gradients of the loss terms of the rays ``rays`` (indices) alone."""
    idx = torch.as_tensor(rays).reshape(-1)
    return oracle_backward(runs["sd"], runs["spec"], tuple(t[idx] for t in runs["rays"]), runs["loss_of"](idx),
                           pass_semantic_gradients=runs["pass_sem"] if pass_sem is None else pass_sem,
                           ray_weights=torch.ones(idx.numel(), dtype=torch.float64)).grads


def _combine(ref, *terms):
    """ref + sum of c * g over the (c, g) in ``terms``, tensor by tensor."""
    return {k: v + sum(c * g[k] for c, g in terms) for k, v in ref.items()}


def _last_round_ray(runs):
    """The last live ray; all its samples lie in the last round."""
    r = int(torch.nonzero(runs["ref"].ray_weights)[-1])
    point_round = runs["rounds"].repeat_interleave(TILE_POINTS)[:R * S].view(R, S)
    assert bool((point_round[r] == runs["rounds"].max()).all())
    return r


def _drop_last_round_ray(runs):
    return _combine(runs["ref"].grads, (-1.0, _ray_grads(runs, [_last_round_ray(runs)])))


def _double_last_round_ray(runs):
    return _combine(runs["ref"].grads, (1.0, _ray_grads(runs, [_last_round_ray(runs)])))


def _cta_stops_after_first_round(runs):
    """CTA 0's tiles of rounds 1 and later left out: every live ray with a sample in them."""
    rounds, grid = runs["rounds"], runs["grid"]
    t = torch.arange(rounds.numel())
    tiles = t[(t % (RESIDENT_GROUPS * grid) < RESIDENT_GROUPS) & (rounds >= 1)]
    points = (tiles[:, None] * TILE_POINTS + torch.arange(TILE_POINTS)).reshape(-1)
    rays = torch.unique(points[points < R * S] // S)
    rays = rays[runs["ref"].ray_weights[rays] > 0]
    assert rays.numel() > 0
    return _combine(runs["ref"].grads, (-1.0, _ray_grads(runs, rays)))


def _no_semantic_pass_on_one_ray(runs):
    assert runs["pass_sem"]
    r = [_last_round_ray(runs)]
    return _combine(runs["ref"].grads, (-1.0, _ray_grads(runs, r)), (1.0, _ray_grads(runs, r, pass_sem=False)))


MUTATIONS = {"last-round ray removed": ("small-all7", _drop_last_round_ray),
             "last-round ray counted twice": ("small-all7", _double_last_round_ray),
             "CTA 0 stops after its first round": ("small-all7", _cta_stops_after_first_round),
             "one ray without its semantic-branch gradient": ("small-pass_sem", _no_semantic_pass_on_one_ray),
             "big: last-round ray removed": ("big-all7", _drop_last_round_ray),
             "big: CTA 0 stops after its first round": ("big-all7", _cta_stops_after_first_round)}


@pytest.mark.parametrize("runs,mutation", [(case, m) for m, (case, _) in MUTATIONS.items()], indirect=["runs"])
def test_bar_rejects_mutation(runs, mutation):
    errs = grad_errors(MUTATIONS[mutation][1](runs), runs["ref"].grads)
    worst = max(errs.values())
    mlp = max((v, k) for k, v in errs.items() if k != HASH_KEY)
    print(f"{mutation}: worst normalized error {worst:.3g} ({max(errs, key=errs.get)}), {worst / GRAD_REL:.3g}x the bar {GRAD_REL:g}; "
          f"outside the table {mlp[0]:.3g} ({mlp[1]})")
    assert worst > GRAD_REL, f"{mutation} passes the bar: {errs}"


@pytest.mark.parametrize("loss", ["mse_bce", "all7"])
def test_chunked_oracle_is_the_unchunked_one(loss):
    """Over 1024 x 48 samples (two of field_forward's sample chunks) in chunks of 100 rays: the same safe rays, and gradients
    equal to float64 rounding."""
    R_, S_ = 1024, 48
    sd, spec = make_state("small", log2T=15)
    rays = syn.ray_batch(R_, S_, salt=5, far=3.0, num_images=7)
    loss_of = ray_loss(loss, R_, S_)
    whole = oracle_backward(sd, spec, rays, loss_of(), pass_semantic_gradients=True)
    chunked = chunked_oracle_backward(sd, spec, rays, loss_of, chunk=100, pass_semantic_gradients=True)
    assert torch.equal(whole.ray_weights, chunked.ray_weights)
    assert 0 < int(whole.ray_weights.sum()) < R_
    assert abs(float(whole.loss - chunked.loss)) <= 1e-12 * abs(float(whole.loss))
    errs = grad_errors(chunked.grads, whole.grads)
    assert max(errs.values()) <= 1e-9, errs
    for k, v in whole.out.items():
        assert torch.allclose(chunked.out[k], v.detach(), rtol=1e-12, atol=0.0), k
