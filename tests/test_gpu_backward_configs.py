"""The render backward (fnr_render_backward: compositing backward + field backward, simt and wgmma instantiations) in the
configurations training can reach, against autograd through the float64 oracle.

Every gradient tensor is held to tests/util.py:assert_grads (GRAD_REL of max(|g|, 5% of the tensor's scale), the hash table
level by level); tests/test_backward_bars_host.py shows on the same inputs that the bar passes the float32 oracle with a wide
margin and rejects a dropped ray, a 1% error on one hash level, an ignored pass_semantic_gradients, a missing background
term and an appearance gradient on the wrong camera row.  Rays whose samples come within RELU_MARGIN of a ReLU kink get zero
loss weight on both sides (util.safe_ray_weights).
"""
import ctypes as C
from functools import lru_cache

import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn
from oracle import ns_torch as ns

from .util import (GRAD_REL, HASH_KEY, UPSTREAM_KEYS, assert_grads, coefficient_loss, grad_errors, make_field, make_state,
                   mse_bce_loss, oracle_backward, upstream_coefficients)

pytestmark = pytest.mark.gpu

IMPLS = [L.FNR_IMPL_SIMT, L.FNR_IMPL_TCGEN05]
IMPL_IDS = ["simt", "tcgen05"]
FIELD_ONLY_KEYS = ("sample_density", "sample_rgb", "sample_semantics")


def _loss(kind, R, S, keys=UPSTREAM_KEYS):
    if kind == "mse_bce":
        img, mask = syn.targets(R)
        return mse_bce_loss(img, mask)
    return coefficient_loss(upstream_coefficients(R, S), keys)


@lru_cache(maxsize=None)
def _case(name="small", R=128, S=48, loss="mse_bce", keys=UPSTREAM_KEYS, contraction=True, appearance="train", pass_sem=False,
          num_images=7, min_rays=8, masked=True):
    """(state, spec, rays, loss_fn, float64 oracle run) of one configuration, shared by both implementations."""
    sd, spec = make_state(name, log2T=15, num_images=num_images)
    rays = syn.ray_batch(R, S, salt=5, far=3.0, num_images=num_images)
    loss_fn = _loss(loss, R, S, keys)
    ref = oracle_backward(sd, spec, rays, loss_fn, contraction=contraction, appearance=appearance, training=appearance == "train",
                          pass_semantic_gradients=pass_sem, min_rays=min_rays, ray_weights=None if masked else torch.ones(R, dtype=torch.float64))
    return sd, spec, rays, loss_fn, ref


def _gpu_backward(name, sd, spec, rays, loss_fn, ray_w, impl, contraction=True, appearance="train", pass_sem=False, composite=True):
    """Gradients of loss_fn(ops outputs) w.r.t. a FruitField's parameters, by the native backward."""
    field = make_field(name, sd, spec, "cuda", contraction=contraction, pass_semantic_gradients=pass_sem,
                       use_average_appearance_embedding=appearance == "mean").train(appearance == "train")
    field.kernel_impl = impl
    o, d, s, e, cam = (t.cuda() for t in rays)
    if composite:
        out = ops.render(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam, field.position_mode(), field.appearance_mode(),
                         impl=impl)
    else:
        sdn, srgb, ssem = ops.field(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam if appearance == "train" else None,
                                    field.position_mode(), field.appearance_mode(), impl=impl)
        out = {"sample_density": sdn, "sample_rgb": srgb, "sample_semantics": ssem}
    loss_fn(out, ray_w.cuda()).backward()
    return {k: p.grad for k, p in field.named_parameters()}, out, field


# ---- pass_semantic_gradients=True ------------------------------------------------------------------------------------------
DENSITY_PATH = ("mlp_base_mlp.layers.0.weight", "mlp_base_mlp.layers.0.bias", "mlp_base_mlp.layers.1.weight",
                "mlp_base_mlp.layers.1.bias", HASH_KEY)


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("name", ["small", "big"])
def test_pass_semantic_gradients(native_lib, cuda_device, name, impl):
    """The semantic loss reaches the weights (compositing backward: G += gsem * s_i) and the geometry features (field
    backward: the semantic MLP's input gradient, a 15- / 30-wide wgmma GEMM)."""
    sd, spec, rays, loss_fn, ref = _case(name, pass_sem=True)
    got, _, _ = _gpu_backward(name, sd, spec, rays, loss_fn, ref.ray_weights, impl, pass_sem=True)
    assert_grads(got, ref.grads, what=f"pass_semantic_gradients {name}/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}")
    off, _, _ = _gpu_backward(name, sd, spec, rays, loss_fn, ref.ray_weights, impl, pass_sem=False)
    diff = grad_errors({k: off[k] for k in DENSITY_PATH}, {k: got[k] for k in DENSITY_PATH})
    assert all(v > 25 * GRAD_REL for v in diff.values()), f"the flag barely changes the density path: {diff}"


# ---- AABB positions (disable_scene_contraction=True) --------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
def test_aabb_mode_masked_samples(native_lib, cuda_device, impl):
    """Samples outside the box have density 0 (no d_sigma) but keep their colour and semantic gradients, which all scatter
    into the table rows of the masked position 0; those rows are compared on their own scale."""
    sd, spec, rays, loss_fn, ref = _case("small", loss="all7", contraction=False)
    sel = ref.field["selector"]
    live = ref.ray_weights.bool()
    masked = ~sel & live[:, None]
    assert float(masked.float().sum() / (live.sum() * sel.shape[1])) > 0.3, "too few samples outside the box"
    # colour upstream of the masked samples: the sample_rgb term of the loss (and the background term on the last sample)
    assert bool((upstream_coefficients(*sel.shape)["sample_rgb"][masked].abs().sum(-1) > 0).all())
    rows0, _ = ns.hash_corner_indices(torch.zeros(1, 3), spec.scalings(), spec.log2_hashmap_size)
    own = rows0[0, :, 0]  # corner 0 carries the whole trilinear weight at the origin
    g0 = ref.grads[HASH_KEY][own]
    assert float(g0.abs().min()) > 0.0
    got, _, _ = _gpu_backward("small", sd, spec, rays, loss_fn, ref.ray_weights, impl, contraction=False)
    assert_grads(got, ref.grads, own_rows=own, what=f"aabb/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}")
    assert_grads({HASH_KEY: got[HASH_KEY][own]}, {HASH_KEY: g0}, num_levels=16, what="position-0 rows")


# ---- upstream gradients of every differentiable output ------------------------------------------------------------------------
@pytest.mark.parametrize("key", UPSTREAM_KEYS)
def test_single_upstream_gradient(native_lib, cuda_device, key):
    sd, spec, rays, loss_fn, ref = _case("small", loss="all7", keys=(key,))
    got, _, _ = _gpu_backward("small", sd, spec, rays, loss_fn, ref.ray_weights, L.FNR_IMPL_SIMT)
    assert_grads(got, ref.grads, what=f"upstream {key}/simt")


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("name", ["small", "big"])
def test_all_upstream_gradients(native_lib, cuda_device, name, impl):
    sd, spec, rays, loss_fn, ref = _case(name, loss="all7")
    got, _, _ = _gpu_backward(name, sd, spec, rays, loss_fn, ref.ray_weights, impl)
    assert_grads(got, ref.grads, what=f"all upstream {name}/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}")


# ---- appearance modes of the eval-mode field backward ---------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("mode", ["mean", "zeros"])
def test_field_only_appearance_modes(native_lib, cuda_device, mode, impl):
    """MEAN spreads 1/num_images of the embedding gradient over every row (40 rows: more than one per lane); ZEROS has none."""
    sd, spec, rays, loss_fn, ref = _case("small", loss="all7", keys=FIELD_ONLY_KEYS, appearance=mode, num_images=40)
    got, _, _ = _gpu_backward("small", sd, spec, rays, loss_fn, ref.ray_weights, impl, appearance=mode, composite=False)
    emb = "embedding_appearance.embedding.weight"
    if mode == "zeros":
        assert int(torch.count_nonzero(got[emb])) == 0
    else:
        assert float(ref.grads[emb].abs().min()) > 0.0
    assert_grads(got, ref.grads, what=f"appearance {mode}/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}")


# ---- ray shapes ------------------------------------------------------------------------------------------------------------------
# Gradients that reach their parameter through no hidden ReLU: exact under any ReLU-mask difference, so the 1100-sample rays
# (no ray of which keeps a ReLU margin on every sample) are compared on these with every ray weighted.
FLIP_FREE = ("mlp_head.layers.2.weight", "mlp_head.layers.2.bias", "field_head_semantics.net.weight", "field_head_semantics.net.bias",
             "mlp_semantics.layers.1.weight", "mlp_semantics.layers.1.bias")


def _flip_free(g):
    res = {k: g[k] for k in FLIP_FREE}
    res["density row of mlp_base_mlp.layers.1.weight"] = g["mlp_base_mlp.layers.1.weight"][0]  # d_sigma * exp(h0) * h1
    res["density row of mlp_base_mlp.layers.1.bias"] = g["mlp_base_mlp.layers.1.bias"][:1]
    return res


SHAPES = {"S1xR300": dict(R=300, S=1), "S1100xR6": dict(R=6, S=1100, masked=False), "R7xS11": dict(R=7, S=11, min_rays=3),
          "R111xS50": dict(R=111, S=50)}


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_ray_shapes(native_lib, cuda_device, shape, impl):
    """S = 1 (the only sample is the background sample; per-ray cameras differ across every warp); S > 1024 (the suffix sums
    of the compositing backward switch to total - prefix); 77 points (less than one 128-point tile); a ragged last tile."""
    kw = SHAPES[shape]
    sd, spec, rays, loss_fn, ref = _case("small", loss="all7", **kw)
    if kw["S"] == 1:
        cam = rays[4]
        assert all(cam[i:i + 32].unique().numel() > 1 for i in range(0, 288, 32)), "need per-lane camera rows"
    got, _, _ = _gpu_backward("small", sd, spec, rays, loss_fn, ref.ray_weights, impl)
    what = f"{shape}/{IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]}"
    if kw.get("masked", True):
        assert_grads(got, ref.grads, what=what)
    else:
        assert_grads(_flip_free(got), _flip_free(ref.grads), what=what)


# ---- the recompute path (no encoding stash) ----------------------------------------------------------------------------------------
def _backward_through_abi(field, out, upstream, impl, stash):
    """fnr_render_backward on the tensors ops.render saved, with or without the encoding stash -> {name: grad}."""
    node = out["rgb"].grad_fn  # the _Render context
    origins, directions, starts, ends, cam, params, sd, srgb, ssem, stash_t, w, acc = node.saved
    lib = L.load()
    shape = field.kernel_shape()
    R, S = starts.shape
    desc = shape.desc(field.position_mode(), field.appearance_mode(), impl)
    pstruct = ops._params_struct(shape, params)
    _, views = ops.flat_zero_grads(params)
    gstruct = ops._params_struct(shape, views)
    p = ops._ptr
    rays = L.RayBatch(R, S, p(origins), p(directions), p(starts), p(ends), p(cam))
    saved = L.RenderSaved(p(w), p(sd), p(srgb), p(ssem), p(stash_t) if stash else None, p(acc))
    ups = [g.float().contiguous() for g in upstream]
    up = L.RenderGrads(*[p(g) for g in ups])
    nbytes = C.c_size_t(0)
    L.check(lib.fnr_render_backward_scratch_bytes(C.byref(desc), R, S, C.byref(nbytes)))
    scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=sd.device)
    L.check(lib.fnr_render_backward(C.byref(desc), C.byref(pstruct), C.byref(rays), C.byref(saved), C.byref(up), C.byref(gstruct),
                                    scratch.data_ptr(), nbytes.value, ops._stream(sd.device)))
    torch.cuda.synchronize()
    names = {t.data_ptr(): k for k, t in field.named_parameters()}
    return {names[t.data_ptr()]: v for t, v in zip(params, views)}


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
def test_recompute_encoding_backward(native_lib, cuda_device, impl):
    """A NULL stash_encoding makes the field backward hash-encode the points again: same gradients as the stashed run."""
    sd, spec, rays, loss_fn, ref = _case("small", loss="all7")
    field = make_field("small", sd, spec, "cuda").train()
    o, d, s, e, cam = (t.cuda() for t in rays)
    out = ops.render(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam, field.position_mode(), field.appearance_mode(), impl=impl)
    loss = loss_fn(out, ref.ray_weights.cuda())
    upstream = torch.autograd.grad(loss, [out[k] for k in UPSTREAM_KEYS], retain_graph=True)
    stashed = _backward_through_abi(field, out, upstream, impl, stash=True)
    recomputed = _backward_through_abi(field, out, upstream, impl, stash=False)
    assert not torch.equal(stashed[HASH_KEY], torch.zeros_like(stashed[HASH_KEY]))
    tag = IMPL_IDS[impl == L.FNR_IMPL_TCGEN05]
    assert_grads(recomputed, stashed, what=f"recompute vs stash/{tag}")
    assert_grads(recomputed, ref.grads, what=f"recompute vs oracle/{tag}")
    loss.backward()  # and the autograd path itself agrees with the direct call
    assert_grads({k: t.grad for k, t in field.named_parameters()}, ref.grads, what=f"stashed autograd/{tag}")
