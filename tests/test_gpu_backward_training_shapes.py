"""The render backward at the batch training launches, in every configuration, against autograd through the float64 oracle.

At R = 128, S = 48 (tests/test_gpu_backward_configs.py) the field backward has 48 tiles for the 264 warpgroups of an H100,
so no warpgroup takes a second tile.  At fruit_nerf's training batch, 4096 x 48 (1536 tiles), the small family's resident
tensor-core backward runs six rounds of tiles per CTA on an H100: its on-chip weight gradients accumulate over all of them
and are flushed once at the CTA's end, and its recompute of enc, h1 and the branches' ReLU masks runs on every later tile.
Each case first asserts, from the SM count of the GPU it runs on, that the shape gives at least four rounds, warpgroups
with unequal tile counts, and rays of nonzero loss weight in every round, the last ragged one included.  The big family's
staged kernel (one warpgroup per CTA, several CTAs per SM) gets at least 4 x (2 x SMs) tiles.

Every gradient tensor of both implementations is held to tests/util.py:assert_grads at GRAD_REL; the worst errors are
printed.  Measured on one H100 80GB HBM3 (700 W power limit), the worst per case lies between 1.5e-4 and 2.6e-4 on the
tensor cores (pass_semantic_gradients highest: 2.6e-4 small, 2.5e-4 big) and between 1.1e-5 and 1.4e-4 on simt (AABB mode
highest), as at R = 128.  tests/test_backward_training_shapes_host.py shows on the same inputs that the float32 oracle passes that bar with
a wide margin and that it rejects a live ray of the last round left out or counted twice, a CTA that stops after its first
round, and one ray's missing semantic-branch gradient.  The float64 oracle runs over ray chunks
(util.chunked_oracle_backward), once per case.  Rays whose samples come within RELU_MARGIN of a ReLU kink get zero loss
weight on both sides (util.safe_ray_weights).

The tensor-core forward at 4096 x 48 in AABB mode (training, with the encoding stash) and in inference mode (no_grad,
mean appearance, no stash) is compared with the same oracle runs at assert_rel's 1e-3.
"""
from functools import lru_cache

import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn
from oracle import ns_torch as ns

from .test_gpu_backward_configs import FIELD_ONLY_KEYS, IMPL_IDS, IMPLS, _backward_through_abi, _gpu_backward
from .util import (HASH_KEY, RESIDENT_GROUPS, TILE_POINTS, UPSTREAM_KEYS, assert_grads, assert_rel, chunked_oracle_backward,
                   live_rays_per_round, make_field, make_state, ray_loss, resident_backward_rounds, upstream_coefficients)

pytestmark = pytest.mark.gpu

# name -> (family, R, S, loss, upstream keys, contraction, appearance, pass_semantic_gradients, num_images).  The small family
# at fruit_nerf's batch (and a ragged one), the big family at the same batch, and the huge method's scalings (the big network
# on a max_res 8192 grid) at 4096 x 36: 1152 tiles, the fewest samples per ray that give the staged kernel 4 x 264 tiles.
CASES = {
    "small-mse_bce": ("small", 4096, 48, "mse_bce", UPSTREAM_KEYS, True, "train", False, 7),
    "small-all7": ("small", 4096, 48, "all7", UPSTREAM_KEYS, True, "train", False, 7),
    "small-pass_sem": ("small", 4096, 48, "mse_bce", UPSTREAM_KEYS, True, "train", True, 7),
    "small-aabb": ("small", 4096, 48, "all7", UPSTREAM_KEYS, False, "train", False, 7),
    "small-field_only_mean": ("small", 4096, 48, "all7", FIELD_ONLY_KEYS, True, "mean", False, 40),
    "small-field_only_zeros": ("small", 4096, 48, "all7", FIELD_ONLY_KEYS, True, "zeros", False, 40),
    "small-ragged_4093x47": ("small", 4093, 47, "all7", UPSTREAM_KEYS, True, "train", False, 7),
    "big-mse_bce": ("big", 4096, 48, "mse_bce", UPSTREAM_KEYS, True, "train", False, 7),
    "big-all7": ("big", 4096, 48, "all7", UPSTREAM_KEYS, True, "train", False, 7),
    "big-pass_sem": ("big", 4096, 48, "mse_bce", UPSTREAM_KEYS, True, "train", True, 7),
    "big-aabb": ("big", 4096, 48, "all7", UPSTREAM_KEYS, False, "train", False, 7),
    "huge-all7": ("huge", 4096, 36, "all7", UPSTREAM_KEYS, True, "train", False, 7),
}


@lru_cache(maxsize=2)  # the tests of one case run one after another; a case of the big family holds ~2 GB
def _case(case):
    """(state, spec, rays, loss_of, float64 oracle run) of one case, shared by both implementations."""
    name, R, S, loss, keys, contraction, appearance, pass_sem, num_images = CASES[case]
    sd, spec = make_state(name, num_images=num_images)  # the family's own table: T = 19 (small) / 21 (big, huge)
    rays = syn.ray_batch(R, S, salt=5, far=3.0, num_images=num_images)
    loss_of = ray_loss(loss, R, S, keys)
    ref = chunked_oracle_backward(sd, spec, rays, loss_of, contraction=contraction, appearance=appearance,
                                  training=appearance == "train", pass_semantic_gradients=pass_sem)
    return sd, spec, rays, loss_of, ref


def _assert_every_round_covered(case, ray_weights):
    """The schedule of this shape on this GPU reaches several rounds, and live rays reach each of them."""
    name, R, S = CASES[case][:3]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if name == "small":
        rounds, grid = resident_backward_rounds(R * S, sms)
        per_group = torch.bincount(torch.arange(rounds.numel()) % (RESIDENT_GROUPS * grid))
        assert int(rounds.max()) + 1 >= 4, f"{case}: only {int(rounds.max()) + 1} rounds on {sms} SMs"
        assert int(per_group.min()) < int(per_group.max()), f"{case}: every warpgroup takes {int(per_group.max())} tiles"
    else:  # the staged kernel: up to per_sm CTAs of one warpgroup per SM; rounds of 2 x SMs tiles stand for it
        rounds = torch.arange(-(-R * S // TILE_POINTS)) // (2 * sms)
        assert rounds.numel() >= 4 * 2 * sms, f"{case}: {rounds.numel()} tiles for {sms} SMs"
    live = live_rays_per_round(rounds, ray_weights, S)
    print(f"{case}: {rounds.numel()} tiles in {len(live)} rounds on {sms} SMs, live rays per round {live}")
    assert min(live) > 0, f"{case}: a round without live rays: {live}"


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("case", list(CASES))
def test_gradients_at_training_shape(native_lib, cuda_device, case, impl):
    name, R, S, loss, keys, contraction, appearance, pass_sem, num_images = CASES[case]
    sd, spec, rays, loss_of, ref = _case(case)
    _assert_every_round_covered(case, ref.ray_weights)
    what = f"{case}/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}"
    got, _, _ = _gpu_backward(name, sd, spec, rays, loss_of(), ref.ray_weights, impl, contraction=contraction, appearance=appearance,
                              pass_sem=pass_sem, composite=appearance == "train")
    emb = "embedding_appearance.embedding.weight"
    if appearance == "zeros":
        assert int(torch.count_nonzero(got[emb])) == 0
    elif appearance == "mean":
        assert float(ref.grads[emb].abs().min()) > 0.0
    if contraction:
        assert_grads(got, ref.grads, what=what)
        return
    # AABB positions: samples outside the box have density 0 but keep their colour and semantic gradients, which all scatter
    # into the table rows of the masked position 0; those rows are compared on their own scale
    sel, live = ref.field["selector"], ref.ray_weights.bool()
    masked = ~sel & live[:, None]
    assert float(masked.float().sum() / (live.sum() * S)) > 0.3, "too few samples outside the box"
    assert bool((upstream_coefficients(R, S)["sample_rgb"][masked].abs().sum(-1) > 0).all())
    rows0, _ = ns.hash_corner_indices(torch.zeros(1, 3), spec.scalings(), spec.log2_hashmap_size)
    own = rows0[0, :, 0]  # corner 0 carries the whole trilinear weight at the origin
    g0 = ref.grads[HASH_KEY][own]
    assert float(g0.abs().min()) > 0.0
    assert_grads(got, ref.grads, own_rows=own, what=what)
    assert_grads({HASH_KEY: got[HASH_KEY].cpu()[own]}, {HASH_KEY: g0}, num_levels=16, what=f"{what} position-0 rows")


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
def test_recompute_encoding_at_training_shape(native_lib, cuda_device, impl):
    """A NULL stash_encoding makes the field backward hash-encode the points again, on every tile of every round: the
    stashed and the recomputing backward both match the oracle."""
    case = "small-all7"
    sd, spec, rays, loss_of, ref = _case(case)
    field = make_field("small", sd, spec, "cuda").train()
    o, d, s, e, cam = (t.cuda() for t in rays)
    out = ops.render(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam, field.position_mode(), field.appearance_mode(), impl=impl)
    upstream = torch.autograd.grad(loss_of()(out, ref.ray_weights.cuda()), [out[k] for k in UPSTREAM_KEYS], retain_graph=True)
    tag = f"{case}/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}"
    stashed = _backward_through_abi(field, out, upstream, impl, stash=True)
    assert_grads(stashed, ref.grads, what=f"{tag} stashed")
    recomputed = _backward_through_abi(field, out, upstream, impl, stash=False)
    assert_grads(recomputed, ref.grads, what=f"{tag} recomputed")


FORWARD_KEYS = ("sample_density", "sample_rgb", "sample_semantics", "weights", "rgb", "accumulation", "semantics")


def test_tensor_core_forward_aabb_mode(native_lib, cuda_device):
    """Every sample and ray of the AABB-mode training forward (per-camera appearance, encoding stash)."""
    sd, spec, rays, _, ref = _case("small-aabb")
    field = make_field("small", sd, spec, "cuda", contraction=False).train()
    o, d, s, e, cam = (t.cuda() for t in rays)
    out = ops.render(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam, field.position_mode(), field.appearance_mode(),
                     impl=L.FNR_IMPL_TCGEN05)
    assert out["rgb"].grad_fn.saved[9] is not None  # the encoding stash was written
    for k in FORWARD_KEYS:
        assert_rel(out[k], ref.out[k], what=f"aabb forward {k}")


def test_tensor_core_forward_inference_mode(native_lib, cuda_device):
    """Every sample and ray of the inference forward: no_grad (no encoding stash), mean appearance over 40 images, clamped
    rgb."""
    sd, spec, rays, _, ref = _case("small-field_only_mean")
    field = make_field("small", sd, spec, "cuda", test_mode="inference").eval()
    assert field.appearance_mode() == L.FNR_APP_MEAN
    o, d, s, e, cam = (t.cuda() for t in rays)
    with torch.no_grad():
        out = ops.render(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam, field.position_mode(), field.appearance_mode(),
                         clamp_rgb=True, impl=L.FNR_IMPL_TCGEN05)
    for k in FORWARD_KEYS:
        assert_rel(out[k], ref.out[k], what=f"inference forward {k}")
