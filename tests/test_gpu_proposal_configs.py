"""The proposal stage (fnr_proposal.cu) at the shapes training runs it, against float64 references.

(a) proposal_weights forward and backward for every proposal level of the fruit_nerf, fruit_nerf_big and fruit_nerf_huge
    methods (nets and samples per ray read from fruit_nerf_config.py, log2_hashmap_size 17) at 4096 rays, and the huge
    method's finest net at its 16384-ray batch (96 samples): several rays per warp and many warps per CTA gradient
    accumulator.  Also 9000 rays of 37 samples (a ragged chunk, more rays than the forward grid has warps) and rays of one
    sample, and an AABB-mode batch with a ray wholly outside the box, a ray with zero-width bins and a ray past
    trunc_exp's backward clamp.  Weights are held to assert_rel, every parameter gradient to tests/util.py:assert_grads at
    GRAD_REL, the hash table level by level.  Rays with a sample within RELU_MARGIN of a hidden ReLU kink get zero loss
    weight on both sides.
(b) pdf_sample at the training shapes (512 -> 256 and 256 -> 96 new samples, 9000 rays: each warp's shared CDF serves
    several rays) against ns.pdf_sample.
(c) interlevel_loss at the three methods' level shapes, 4096 rays: the value, and the gradient of each proposal level held
    to tests/util.py:interlevel_bar (GRAD_REL, or twice the float32 oracle's own distance where fp32 arithmetic cannot
    reach GRAD_REL: at (512, 256) + 128 it is 1.1e-3 off; never past 2.5e-3).
(d) one FruitModel training step, end to end: the rgb MSE + semantic BCE + interlevel loss of get_loss_dict, ray by ray,
    through interlevel backward, proposal-weights backward and the field backward, against train_step_reference rebuilt in
    float64 from the GPU's own sample bins.  Every gradient of both proposal networks and of the field at GRAD_REL, each hash
    table level by level; the model of test_gpu_proposal.py's train-step test, and the same with the big method's
    proposal settings.

tests/test_proposal_bars_host.py pins the bars of (a) and (c) on the CPU from both sides.

Worst normalized gradient errors on one H100 (80 GB): (a) fruit_nerf L0 3.0e-5, L1 2.0e-5; fruit_nerf_big L0 1.2e-4, L1
2.7e-5; fruit_nerf_huge L0 1.0e-4, L1 4.2e-5, L1 at 16384 rays 4.8e-5; 9000 x 37 1.2e-5; S = 1 1.8e-6; edge rays 1.1e-5,
the clamp ray alone 2.5e-6.  (c) fruit_nerf 5.5e-4 (bar 1.03e-3), fruit_nerf_big 1.5e-3 (bar 2.2e-3), fruit_nerf_huge 1.1e-3
(bar 2.1e-3).  (d) base: field 4.2e-4, proposal nets 1.2e-4 and 1.8e-4; big proposals: field 3.3e-4, proposal nets 6.2e-4 and
3.2e-4 (the float32 oracle: 1.3e-4 and 2.5e-4).  The whole file takes ~50 s there, most of it the float64 oracles on the CPU.
"""
from functools import lru_cache

import pytest
import torch

from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn
from fruitnerf_b200.compat import RayBundle, SceneBox, Semantics
from fruitnerf_b200.fruit_nerf import FruitModel, FruitNerfModelConfig, _sdist
from oracle import fruit_ref as fr
from oracle import ns_torch as ns

from .util import (PROP_HASH_KEY, PROP_KEYS, RELU_MARGIN, assert_grads, mse_bce_loss, assert_rel, interlevel_bar, interlevel_inputs,
                   interlevel_reference, proposal_configs, proposal_edge_case, proposal_net, proposal_oracle_backward,
                   proposal_rays, weight_coefficients)

pytestmark = pytest.mark.gpu

LEVELS, INTERLEVEL = proposal_configs()


def _weight_cases():
    cases = {}
    for key, (spec, S, R) in LEVELS.items():
        # 4096 rays (the fruit_nerf batch); level 0 out to t = 1000, level 1 to t = 30
        cases[f"{key}-S{S}"] = (key, S, 4096, 1000.0 if key.endswith("L0") else 30.0)
    # the huge method's batch on its finest net: ~8 rays per backward warp.  96 samples per ray keep its float64 oracle short.
    cases["fruit_nerf_huge/L1-S96-R16384"] = ("fruit_nerf_huge/L1", 96, LEVELS["fruit_nerf_huge/L1"][2], 30.0)
    cases["fruit_nerf/L0-S37-R9000"] = ("fruit_nerf/L0", 37, 9000, 1000.0)
    cases["fruit_nerf/L1-S1"] = ("fruit_nerf/L1", 1, 4096, 30.0)
    return cases


WEIGHT_CASES = _weight_cases()


@lru_cache(maxsize=None)
def _weights_ref(case):
    key, S, R, far = WEIGHT_CASES[case]
    spec = LEVELS[key][0]
    sd = syn.density_state(num_levels=spec.num_levels, log2_hashmap_size=spec.log2_hashmap_size)
    rays = proposal_rays(R, S, salt=2, far=far)
    coef = weight_coefficients(R, S)
    return spec, sd, rays, coef, proposal_oracle_backward(sd, spec, rays, coef)


def _gpu_weights(sd, spec, rays, coef, ray_weights, contraction=True):
    net = proposal_net(sd, spec, contraction)
    w = net.weights(*[t.cuda() for t in rays])
    (w * (ray_weights[:, None] * coef).float().cuda()).sum().backward()
    named = dict(net.named_parameters())
    return w, {k: named[k].grad for k in PROP_KEYS}


@pytest.mark.parametrize("case", list(WEIGHT_CASES))
def test_proposal_weights_configs(native_lib, cuda_device, case):
    spec, sd, rays, coef, ref = _weights_ref(case)
    R = rays[2].shape[0]
    assert ref.ray_weights.sum() >= R // 2, f"{int(ref.ray_weights.sum())} of {R} rays keep a ReLU margin"
    w, got = _gpu_weights(sd, spec, rays, coef, ref.ray_weights)
    assert_rel(w, ref.weights, what=f"{case} weights")
    assert_grads(got, ref.grads, num_levels=spec.num_levels, hash_key=PROP_HASH_KEY, what=case)


def test_proposal_weights_edge_rays(native_lib, cuda_device):
    spec = LEVELS["fruit_nerf/L1"][0]
    sd, rays = proposal_edge_case(spec)
    R, S = rays[2].shape
    coef = weight_coefficients(R, S, salt=1)
    ref = proposal_oracle_backward(sd, spec, rays, coef, contraction=False)
    assert bool(ref.ray_weights[-3:].all()), "the edge rays must carry loss weight"
    w, got = _gpu_weights(sd, spec, rays, coef, ref.ray_weights, contraction=False)
    assert int(torch.count_nonzero(w[-3])) == 0, "a ray outside the box has zero weights"
    assert int(torch.count_nonzero(w[-2, 1::2])) == 0, "zero-width bins have zero weight"
    assert_rel(w, ref.weights, what="edge weights")
    assert_rel(w[-1], ref.weights[-1], what="clamp ray weights")
    assert_grads(got, ref.grads, num_levels=spec.num_levels, hash_key=PROP_HASH_KEY, what="edge rays")
    # the clamp ray alone: its gradient is the clamped one (trunc_exp's backward at h = 17 uses exp(15))
    only = torch.zeros(R, dtype=torch.float64)
    only[-1] = 1.0
    ref1 = proposal_oracle_backward(sd, spec, rays, coef, contraction=False, ray_weights=only, min_rays=1)
    _, got1 = _gpu_weights(sd, spec, rays, coef, only, contraction=False)
    assert float(ref1.grads["mlp_base.1.layers.1.bias"].abs()) > 0
    assert_grads(got1, ref1.grads, num_levels=spec.num_levels, hash_key=PROP_HASH_KEY, what="clamp ray")


# ---- (b) pdf_sample -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["eval", "single_jitter", "per_bin"])
@pytest.mark.parametrize("S,n,anneal", [(512, 256, 1.0), (512, 256, 0.37), (256, 96, 1.0), (256, 96, 0.37)])
def test_pdf_sample_training_shapes(native_lib, cuda_device, mode, S, n, anneal):
    R = 9000
    w = (syn.hash_uniform(R * S, 5).view(R, S) + 1.0).pow(6) * 0.01
    w[3] = 0.0  # zero-weight ray: the reference's eps padding path
    w[4, : S // 2] = 0.0
    existing = ns.spaced_bins(R, S, (syn.hash_uniform(R, 6).view(R, 1) + 1) * 0.5).contiguous()
    nears, fars = torch.full((R, 1), 0.05), torch.full((R, 1), 1000.0)
    u = None
    if mode == "single_jitter":
        u = (syn.hash_uniform(R, 8).view(R, 1) + 1) * 0.5
    elif mode == "per_bin":
        u = (syn.hash_uniform(R * (n + 1), 9).view(R, n + 1) + 1) * 0.5
    ref_bins = ns.pdf_sample(torch.pow(w, anneal), existing, n, u)
    bins, starts, ends = ops.pdf_sample(w.cuda(), existing.cuda(), n, None if u is None else u.cuda(), anneal, nears.cuda(), fars.cuda())
    # positions are continuous in u, so searchsorted ties only move a bin by rounding noise
    assert torch.allclose(bins.cpu(), ref_bins, atol=2e-6, rtol=1e-5), float((bins.cpu() - ref_bins).abs().max())
    # the spacing -> euclidean map of the kernel's own bins: 1 / (2 - 2x) near fars = 1000 turns the bins' rounding noise
    # (2e-6) into 2e-3 relative, so the map is checked on the bins it was given (test_gpu_proposal.py::
    # test_pdf_sample_matches_oracle still maps the reference's bins, at 64 rays)
    e_ref = ns.spacing_to_euclidean(bins.cpu(), nears, fars)
    assert torch.allclose(starts.cpu(), e_ref[:, :-1], rtol=2e-4, atol=1e-6) and torch.allclose(ends.cpu(), e_ref[:, 1:], rtol=2e-4, atol=1e-6)
    assert bool((bins[:, 1:] >= bins[:, :-1]).all()), "bins must be sorted"


# ---- (c) interlevel loss --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", list(INTERLEVEL))
def test_interlevel_loss_training_shapes(native_lib, cuda_device, method):
    props_n, Sc = INTERLEVEL[method]
    R = 4096
    c, w, props = interlevel_inputs(R, props_n, Sc)
    loss_ref, ref = interlevel_reference(c.double(), w, [(cp.double(), wp) for cp, wp in props])
    _, f32 = interlevel_reference(c, w, props, dtype=torch.float32)
    bar = interlevel_bar(f32, ref)
    gw = [wp.cuda().requires_grad_(True) for _, wp in props]
    out = ops.interlevel_loss(gw + [w.cuda()], [cp.cuda() for cp, _ in props] + [c.cuda()], 1.0)
    out.backward()
    assert_rel(out.detach(), loss_ref, what="interlevel loss")
    assert_grads({f"level {k}": g.grad for k, g in enumerate(gw)}, {f"level {k}": g for k, g in enumerate(ref)}, rel=bar,
                 what=f"interlevel {method}")


# ---- (d) one training step's proposal and field gradients, end to end ------------------------------------------------------------
def _train_model_config(kind):
    """FruitNerfModelConfig of the model test_gpu_proposal.py::test_model_train_step_produces_all_gradients trains ("base"), or the
    same model with the big method's proposal settings (nets, samples per level, final samples; hidden_dim 16)."""
    from fruitnerf_b200.fruit_nerf_config import METHODS

    if kind == "base":
        nets = [{"hidden_dim": 16, "log2_hashmap_size": 14, "num_levels": 5, "max_res": 128, "use_linear": False},
                {"hidden_dim": 16, "log2_hashmap_size": 14, "num_levels": 5, "max_res": 256, "use_linear": False}]
        return FruitNerfModelConfig(log2_hashmap_size=15, proposal_net_args_list=nets)
    big = METHODS["fruit_nerf_big"].pipeline.model
    return FruitNerfModelConfig(log2_hashmap_size=15, proposal_net_args_list=[dict(a) for a in big.proposal_net_args_list],
                                num_proposal_samples_per_ray=tuple(big.num_proposal_samples_per_ray),
                                num_nerf_samples_per_ray=big.num_nerf_samples_per_ray)


def train_step_reference(fsd, fspec, psds, pspecs, rays, cam, levels, image, mask, mult, dtype=torch.float64, ray_weights=None):
    """FruitModel's training loss on fixed sample bins, by autograd with the parameters in ``dtype``: each proposal level's
    weights (fr.proposal_weights), the field on the final bins and its render, rgb MSE + semantic BCE + interlevel loss
    (nerfstudio's, final level detached), each ray weighted.  ``levels``: per level (starts [R,S], ends [R,S], spacing bins
    [R,S+1]) float32, the last the final level.  ``ray_weights`` default: the rays whose samples keep RELU_MARGIN in both
    proposal nets and the field.  Returns (field grads, [proposal grads], ray weights)."""
    o, d = rays
    R = o.shape[0]
    fp = {k: v.detach().to(dtype, copy=True).requires_grad_(True) if v.is_floating_point() and k != "aabb" else v for k, v in fsd.items()}
    pps = [{k: v.detach().to(dtype, copy=True).requires_grad_(True) for k, v in sd.items() if k != "aabb"} for sd in psds]
    wps, keep = [], torch.ones(R, dtype=torch.bool)
    for pp, spec, (s, e, _) in zip(pps, pspecs, levels[:-1]):
        w, margin = fr.proposal_weights(pp, spec, o, d, s, e, psds[0]["aabb"], True, relu_margin=True)
        wps.append(w)
        keep &= (margin > RELU_MARGIN).all(dim=1)
    s, e, c = levels[-1]
    f = fr.field_forward(fp, fspec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, True, "train")
    keep &= (f["relu_margin"] > RELU_MARGIN).all(dim=1)
    rw = keep.to(dtype) if ray_weights is None else ray_weights.to(dtype)
    r = fr.render(f, s[..., None], e[..., None], training=True)
    loss = mse_bce_loss(image, mask)({"rgb": r["rgb"], "semantics": r["semantics"][..., 0]}, rw)
    w_final = r["weights"][..., 0].detach()
    for wp, (_, _, cp) in zip(wps, levels[:-1]):
        loss = loss + (rw[:, None] * ns.lossfun_outer(c, w_final, cp, wp)).sum() / w_final.numel() * mult
    loss.backward()
    grad = lambda p: (p.grad if p.grad is not None else torch.zeros_like(p)).detach()  # noqa: E731
    return ({k: grad(p) for k, p in fp.items() if torch.is_tensor(p) and p.requires_grad},
            [{k: grad(p) for k, p in pp.items()} for pp in pps], rw)


@pytest.mark.parametrize("kind", ["base", "big_proposals"])
def test_train_step_gradients_end_to_end(native_lib, cuda_device, kind):
    """One FruitModel training step: its proposal networks' and field's gradients against train_step_reference rebuilt from
    the GPU's own ray_samples_list bins (sampling positions carry no gradient, and pdf-sampling ties cannot split the sides)."""
    cfg = _train_model_config(kind)
    sem = Semantics(filenames=[], classes=["fruit"], colors=torch.tensor([[0.0, 0, 0], [1.0, 0, 0]]))
    model = FruitModel(cfg, metadata={"semantics": sem}, scene_box=SceneBox(torch.tensor([[-1.0, -1, -1], [1, 1, 1]])),
                       num_train_data=7, test_mode="val")
    fsd = syn.field_state(log2_hashmap_size=15, num_images=7, table_scale=0.5, weight_gain=1.5)
    model.field.load_state_dict(fsd, strict=False)
    fspec = fr.FieldSpec(log2_hashmap_size=15)
    psds, pspecs = [], []
    for i, (net, a) in enumerate(zip(model.proposal_networks, cfg.proposal_net_args_list)):
        sd = syn.density_state(num_levels=a["num_levels"], log2_hashmap_size=a["log2_hashmap_size"], salt=6000 + 100 * i, table_scale=1.0,
                               weight_gain=2.0)
        net.load_state_dict(sd, strict=False)
        psds.append(sd)
        pspecs.append(fr.DensitySpec(num_levels=a["num_levels"], max_res=a["max_res"], log2_hashmap_size=a["log2_hashmap_size"]))
    model = model.to(cuda_device).train()
    for cb in model.get_training_callbacks():
        if cb["where_to_run"] == "BEFORE_TRAIN_ITERATION":
            cb["func"](1000)
    R = 2048  # 512 samples of two nets and 128 of the field: ~5% of the rays keep every ReLU margin
    o, d, _, _, _ = syn.ray_batch(R, 4, salt=6)
    cam = ((syn.hash_uniform(R, 41) + 1.0) * 3.5).to(torch.int64).clamp_(0, 6)
    img, mask = syn.targets(R)
    rb = RayBundle(origins=o.cuda(), directions=d.cuda(), camera_indices=cam[:, None].cuda(), nears=torch.full((R, 1), 0.05, device=cuda_device),
                   fars=torch.full((R, 1), 1000.0, device=cuda_device))
    out = model(rb)
    rsl = out["ray_samples_list"]
    levels = [(rs.frustums.starts[..., 0].cpu(), rs.frustums.ends[..., 0].cpu(), _sdist(rs).cpu()) for rs in rsl]
    mult = cfg.interlevel_loss_mult
    fgrads, pgrads, rw = train_step_reference(fsd, fspec, psds, pspecs, (o, d), cam, levels, img, mask, mult)
    assert rw.sum() >= 64, f"only {int(rw.sum())} of {R} rays keep a ReLU margin"

    # the loss of get_loss_dict, ray by ray: MSE + BCE on the rendered outputs, the interlevel loss over the kept rays
    keep = rw.bool().cuda()
    loss = mse_bce_loss(img, mask)({"rgb": out["rgb"], "semantics": out["semantics"][:, 0]}, rw.cuda())
    inter = ops.interlevel_loss([w[keep][..., 0] for w in out["weights_list"]], [_sdist(rs)[keep] for rs in rsl], mult)
    (loss + inter * (float(keep.sum()) / R)).backward()

    named = dict(model.field.named_parameters(remove_duplicate=False))
    worst = assert_grads({k: named[k].grad for k in fgrads}, fgrads, what=f"{kind} field")
    for i, net in enumerate(model.proposal_networks):
        pn = dict(net.named_parameters())
        assert float(pgrads[i][PROP_HASH_KEY].abs().max()) > 0, f"proposal net {i} receives no gradient"
        worst = max(worst, assert_grads({k: pn[k].grad for k in PROP_KEYS}, pgrads[i], num_levels=pspecs[i].num_levels, hash_key=PROP_HASH_KEY,
                                        what=f"{kind} proposal net {i}"))
    print(f"{kind}: worst normalized gradient error of the step {worst:.3g}")
