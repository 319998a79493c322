"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Bars (north_star): bit-exact hash rows / sample indices; 1e-3 relative on RGB, density and
semantics (tests/util.py:assert_rel).  The oracle restates nerfstudio's torch-fallback semantics
and is itself unpinned by the reference (no upstream tests) -- see oracle/__init__.py.
"""
import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn
from fruitnerf_b200.compat import FieldHeadNames, Frustums, RaySamples
from oracle import fruit_ref as fr
from oracle import ns_torch as ns

from .util import assert_grads, assert_rel, make_field, make_state, mse_bce_loss, oracle_backward

pytestmark = pytest.mark.gpu

IMPLS = [L.FNR_IMPL_SIMT, L.FNR_IMPL_TCGEN05]
IMPL_IDS = ["simt", "tcgen05"]


def _rays(R, S, salt=0, far=2.0, num_images=7):
    return syn.ray_batch(R, S, salt=salt, far=far, num_images=num_images)


def _edge_rays(S=16):
    """Rays that hit the corner cases: outside the unit cube (contraction shell / masked in aabb
    mode), exactly on cell boundaries, zero-length bins."""
    o = torch.tensor([[0.0, 0.0, 0.0], [-1.0, -1.0, -1.0], [0.5, 0.25, -0.75], [3.0, 0.0, 0.0], [0.0, 0.0, -2.0]])
    d = torch.tensor([[1.0, 0.0, 0.0], [1.0, 1.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    d = d / d.norm(dim=-1, keepdim=True)
    t = torch.linspace(0.0, 4.0, S + 1)[None, :].repeat(o.shape[0], 1)
    starts, ends = t[:, :-1].contiguous(), t[:, 1:].contiguous()
    ends[:, 3] = starts[:, 3]  # zero-width bin
    cam = torch.arange(o.shape[0]) % 7
    return o, d, starts, ends, cam


def _oracle_field(sd, spec, o, d, s, e, cam, contraction, appearance):
    return fr.field_forward(sd, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam,
                            contraction=contraction, appearance=appearance)


@pytest.mark.parametrize("name", ["small", "big"])
@pytest.mark.parametrize("contraction", [True, False])
def test_hash_rows_bit_exact(native_lib, cuda_device, name, contraction):
    sd, spec = make_state(name)
    field = make_field(name, sd, spec, "cpu", contraction=contraction)
    shape = field.kernel_shape()
    for o, d, s, e, _ in (_rays(257, 48, far=6.0), _edge_rays()):
        rows, pos = ops.hash_indices(shape, o.cuda(), d.cuda(), s.cuda(), e.cuda(), field.position_mode())
        R, S = s.shape
        p_ref, _ = fr.sample_positions(o[:, None, :].expand(R, S, 3), d[:, None, :].expand(R, S, 3), s[..., None], e[..., None],
                                       sd["aabb"], contraction)
        idx_ref, _ = ns.hash_corner_indices(p_ref.reshape(-1, 3), spec.scalings(), spec.log2_hashmap_size)
        assert torch.equal(pos.cpu().reshape(-1, 3).abs(), p_ref.reshape(-1, 3).abs()), "positions differ bitwise"
        assert torch.equal(rows.cpu().reshape(-1, 16, 8).long(), idx_ref), "hash rows differ"


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("name", ["small", "big"])
@pytest.mark.parametrize("mode", ["train", "mean", "zeros"])
def test_field_forward_matches_oracle(native_lib, cuda_device, name, mode, impl):
    sd, spec = make_state(name)
    field = make_field(name, sd, spec, cuda_device, contraction=True, use_average_appearance_embedding=(mode == "mean"))
    field.kernel_impl = impl
    field.train(mode == "train")
    for o, d, s, e, cam in (_rays(129, 48, far=4.0), _edge_rays()):
        R, S = s.shape
        rs = RaySamples(
            frustums=Frustums(origins=o[:, None, :].expand(R, S, 3).cuda(), directions=d[:, None, :].expand(R, S, 3).cuda(),
                              starts=s[..., None].cuda(), ends=e[..., None].cuda()),
            camera_indices=cam[:, None, None].expand(R, S, 1).cuda(),
        )
        with torch.no_grad():
            out = field(rs)
        ref = _oracle_field(sd, spec, o, d, s, e, cam, True, mode)
        assert_rel(out[FieldHeadNames.DENSITY], ref["density"], what="density")
        assert_rel(out[FieldHeadNames.RGB], ref["rgb"], what="rgb")
        assert_rel(out[FieldHeadNames.SEMANTICS], ref["semantics"], what="semantics")


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
def test_huge_variant_forward_matches_oracle(native_lib, cuda_device, impl):
    """fruit_nerf_huge: the big network on a max_res 8192 grid (fruit_nerf_config.py:113-153), 64 samples per ray."""
    v = dict(syn.BIG, max_res=8192)
    sd = syn.field_state(geo=v["geo"], sem_dims=v["sem_dims"], log2_hashmap_size=21, num_images=5, table_scale=0.5, weight_gain=1.5)
    spec = fr.FieldSpec(max_res=8192, log2_hashmap_size=21, geo_feat_dim=30)
    from fruitnerf_b200.fruit_field import FruitField, SceneContraction

    field = FruitField(aabb=sd["aabb"], num_images=5, geo_feat_dim=30, max_res=8192, log2_hashmap_size=21, num_layers_semantic=3,
                       hidden_dim_semantics=128, use_semantics=True, num_semantic_classes=1, test_mode=None,
                       spatial_distortion=SceneContraction(order=float("inf")))
    field.load_state_dict(sd, strict=False)
    field = field.to(cuda_device).train()
    o, d, s, e, cam = _rays(100, 64, salt=8, far=3.0, num_images=5)
    with torch.no_grad():
        out = _render_gpu(field, o, d, s, e, cam, impl)
    f = _oracle_field(sd, spec, o, d, s, e, cam, True, "train")
    ref = fr.render(f, s[..., None], e[..., None], training=True)
    assert_rel(out["sample_density"], f["density"][..., 0], what="density")
    assert_rel(out["rgb"], ref["rgb"], what="rgb")
    assert_rel(out["semantics"], ref["semantics"][..., 0], what="semantics")
    _check_depth_index(out["depth_index"], ref, ref["weights"])


def test_missing_camera_indices_raises(native_lib, cuda_device):
    sd, spec = make_state("small")
    field = make_field("small", sd, spec, cuda_device).train()
    o, d, s, e, _ = _rays(4, 8)
    rs = RaySamples(frustums=Frustums(o[:, None, :].expand(4, 8, 3).cuda(), d[:, None, :].expand(4, 8, 3).cuda(),
                                      s[..., None].cuda(), e[..., None].cuda()))
    with pytest.raises(AttributeError):  # fruit_field.py:240-241
        field(rs)


def _render_gpu(field, o, d, s, e, cam, impl, clamp=False):
    return ops.render(field.kernel_shape(), field.kernel_params(), o.cuda(), d.cuda(), s.cuda(), e.cuda(),
                      None if cam is None else cam.cuda(), field.position_mode(), field.appearance_mode(), clamp_rgb=clamp, impl=impl)


def _check_depth_index(gpu_idx, ref_out, weights_ref):
    """Median index: exact, or off by one only where the cumulative weight ties 0.5 within 1e-6."""
    gi = gpu_idx.cpu().long().reshape(-1)
    ri = ref_out["depth_index"].reshape(-1)
    cum = torch.cumsum(weights_ref[..., 0], dim=-1)
    for r in torch.nonzero(gi != ri).reshape(-1).tolist():
        lo, hi = sorted((int(gi[r]), int(ri[r])))
        assert hi - lo == 1 and abs(float(cum[r, lo]) - 0.5) < 1e-5, f"median index mismatch on ray {r}: {gi[r]} vs {ri[r]}"


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("name,S", [("small", 48), ("small", 192), ("big", 128), ("small", 37)])
def test_render_forward_matches_oracle(native_lib, cuda_device, name, S, impl):
    sd, spec = make_state(name)
    field = make_field(name, sd, spec, cuda_device).train()
    o, d, s, e, cam = _rays(96, S, salt=3, far=3.0)
    with torch.no_grad():
        out = _render_gpu(field, o, d, s, e, cam, impl)
    f = _oracle_field(sd, spec, o, d, s, e, cam, True, "train")
    ref = fr.render(f, s[..., None], e[..., None], training=True)
    assert_rel(out["rgb"], ref["rgb"], what="rgb")
    assert_rel(out["accumulation"], ref["accumulation"], what="accumulation")
    assert_rel(out["semantics"], ref["semantics"], what="semantics")
    assert_rel(out["weights"], ref["weights"], what="weights")
    assert_rel(out["sample_density"], f["density"], what="sample density")
    _check_depth_index(out["depth_index"], ref, ref["weights"])
    same = out["depth_index"].cpu().long().reshape(-1) == ref["depth_index"].reshape(-1)
    assert_rel(out["depth"].cpu()[same], ref["depth"].reshape(-1)[same], what="depth")


def test_render_eval_clamp_and_composite_edge_cases(native_lib, cuda_device):
    """sigma = 0, huge sigma (saturating weights), eval-mode clamp (nerfstudio RGBRenderer)."""
    sd, spec = make_state("small", table_scale=4.0, weight_gain=3.0)
    field = make_field("small", sd, spec, cuda_device).eval()
    o, d, s, e, cam = _edge_rays(S=32)
    with torch.no_grad():
        out = _render_gpu(field, o, d, s, e, None, L.FNR_IMPL_SIMT, clamp=True)
    f = _oracle_field(sd, spec, o, d, s, e, None, True, "zeros")
    ref = fr.render(f, s[..., None], e[..., None], training=False)
    assert_rel(out["rgb"], ref["rgb"], what="rgb(eval)")
    assert_rel(out["weights"], ref["weights"], what="weights")
    assert float(out["rgb"].min()) >= 0.0 and float(out["rgb"].max()) <= 1.0


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
def test_infinite_density_keeps_the_first_sample(native_lib, cuda_device, impl):
    """trunc_exp overflow (h0 > 88.7 -> sigma = +inf): torch's get_weights gives weight 1 to the first such sample (T = 1 in
    front of it, alpha = 1) and 0 behind it -- not NaN -> 0 everywhere, which would silence the whole ray."""
    sd, spec = make_state("small")
    sd = dict(sd)
    sd["mlp_base_mlp.layers.1.bias"] = sd["mlp_base_mlp.layers.1.bias"].clone()
    sd["mlp_base_mlp.layers.1.bias"][0] = 120.0
    field = make_field("small", sd, spec, cuda_device).eval()
    o, d, s, e, cam = _rays(32, 48, salt=9, far=2.0)
    with torch.no_grad():
        out = _render_gpu(field, o, d, s, e, None, impl, clamp=True)
    f = _oracle_field(sd, spec, o, d, s, e, None, True, "zeros")
    ref = fr.render(f, s[..., None], e[..., None], training=False)
    assert bool(torch.isinf(f["density"]).any())
    w = out["weights"].cpu()
    assert torch.equal(w, ref["weights"][..., 0]) or torch.allclose(w, ref["weights"][..., 0], atol=1e-6)
    inside = torch.isinf(f["density"][:, 0, 0])  # rays whose first sample is inside the box (selector = 1)
    assert bool(inside.any()) and bool((w[inside, 0] == 1.0).all()) and bool((w[inside, 1:] == 0.0).all())
    assert_rel(out["rgb"], ref["rgb"], what="rgb")
    assert_rel(out["accumulation"], ref["accumulation"][..., 0], what="accumulation")


RELU_MARGIN = 1e-4  # samples with a hidden pre-activation within 1e-4 (relative to the layer rms) of zero


def _safe_ray_weights(f, R):
    """1 for rays whose samples all keep a ReLU margin, else 0.  d relu(x)/dx at x ~ 0 depends on the
    last bits of x: the tensor-core path computes pre-activations to ~2^-16 (bf16 hi/lo operands), the
    oracle to ~2^-24, so masks may legitimately differ there and the sample's gradient changes
    discretely.  Such rays get zero loss weight (on both sides), everything else is compared exactly."""
    ok = (f["relu_margin"] > RELU_MARGIN).all(dim=1).float()
    assert ok.sum() >= 8, f"only {int(ok.sum())} of {R} rays keep a ReLU margin; enlarge the batch"
    return ok


@pytest.mark.parametrize("impl", [L.FNR_IMPL_SIMT, L.FNR_IMPL_TCGEN05, L.FNR_IMPL_AUTO], ids=["simt", "tcgen05", "auto"])
@pytest.mark.parametrize("name,R,S", [("small", 128, 48), ("big", 128, 48), ("small", 111, 50), ("big", 77, 37)])
def test_backward_matches_oracle_autograd(native_lib, cuda_device, name, R, S, impl):
    """tcgen05 and auto both run the wgmma forward and backward kernels, simt the fp32 ones; 111 x 50 = 5550 points
    exercises a ragged last tile and warps that span rays."""
    sd, spec = make_state(name, log2T=15)  # small table keeps the oracle's dense grad comparison cheap
    field = make_field(name, sd, spec, cuda_device).train()
    o, d, s, e, cam = _rays(R, S, salt=5, far=3.0)
    img, mask = syn.targets(R)
    loss_of = mse_bce_loss(img, mask)
    ref = oracle_backward(sd, spec, (o, d, s, e, cam), loss_of)  # float64 autograd, ReLU-margin ray weights

    out = _render_gpu(field, o, d, s, e, cam, impl)
    loss = loss_of(out, ref.ray_weights.cuda())
    loss.backward()
    assert_rel(loss.detach(), ref.loss, what="loss")
    # every tensor within GRAD_REL of max(|g|, 5% of its scale), the hash table level by level (tests/test_backward_bars_host.py)
    assert_grads({k: t.grad for k, t in field.named_parameters()}, ref.grads, what=f"{name} {R}x{S}")


@pytest.mark.parametrize("impl", [L.FNR_IMPL_SIMT, L.FNR_IMPL_TCGEN05, L.FNR_IMPL_AUTO], ids=["simt", "tcgen05", "auto"])
def test_field_only_backward(native_lib, cuda_device, impl):
    """FruitField.forward users: gradients w.r.t. per-sample outputs flow to the parameters."""
    sd, spec = make_state("small", log2T=15)
    field = make_field("small", sd, spec, cuda_device).train()
    field.kernel_impl = impl
    R, S = 32, 16
    o, d, s, e, cam = _rays(R, S, salt=9, far=2.0)
    rs = RaySamples(frustums=Frustums(o[:, None, :].expand(R, S, 3).cuda(), d[:, None, :].expand(R, S, 3).cuda(),
                                      s[..., None].cuda(), e[..., None].cuda()),
                    camera_indices=cam[:, None, None].expand(R, S, 1).cuda())
    sd_ref = {k: v.clone().requires_grad_(v.is_floating_point() and k != "aabb") for k, v in sd.items()}
    f = _oracle_field(sd_ref, spec, o, d, s, e, cam, True, "train")
    w = (f["relu_margin"] > RELU_MARGIN).float()[..., None]  # per-sample weights (see _safe_ray_weights)
    (w * f["rgb"]).sum().add(0.1 * (w * f["density"]).sum()).add((w * f["semantics"].pow(2)).sum()).backward()
    out = field(rs)
    wg = w.cuda()
    ((wg * out[FieldHeadNames.RGB]).sum() + 0.1 * (wg * out[FieldHeadNames.DENSITY]).sum()
     + (wg * out[FieldHeadNames.SEMANTICS].pow(2)).sum()).backward()
    named = dict(field.named_parameters())
    for key in ("mlp_base_grid.hash_table", "mlp_base_mlp.layers.0.weight", "mlp_semantics.layers.1.weight",
                "field_head_semantics.net.bias", "mlp_head.layers.0.weight", "embedding_appearance.embedding.weight"):
        assert_rel(named[key].grad, sd_ref[key].grad, rel=2e-3, floor=0.25, what=f"grad {key}")


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("name,n", [("small", 12), ("big", 12), ("small", 37)])
def test_export_matches_oracle(native_lib, cuda_device, name, n, impl):
    """get_export_outputs + sample_volume selection on a small grid, thresholds lowered so that
    all three sets are populated (the reference constants 3 / 70 / 0.9 are covered below)."""
    sd, spec = make_state(name, table_scale=2.0, weight_gain=2.5)
    field = make_field(name, sd, spec, cuda_device, contraction=False, test_mode="export").eval()
    pts, plane = ns.surface_points(((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), n)
    o, dirs, nears, fars = ns.orthographic_rays(pts, plane, batch=10_000, count=1)
    bins = torch.linspace(0.0, 1.0, n + 1)
    ref = fr.export_outputs(sd, spec, o, dirs, nears, fars, n)
    dens = ref["density"].reshape(-1)
    sem = ref["semantics"].reshape(-1)
    for thr in ((float(sem.median()), float(dens.median()), 0.5), (3.0, 70.0, 0.9)):
        buf = ops.ExportBuffers(capacity=o.shape[0] * n, device=cuda_device)
        dense = ops.export_batch(field.kernel_shape(), field.kernel_params(), o.cuda(), [float(v) for v in dirs[0]], bins.cuda(),
                                 float(nears[0]), float(fars[0]), buf, dense_out=True, thresholds=thr, impl=impl)
        assert_rel(dense["density"], ref["density"], what="density")
        assert_rel(dense["semantics"], ref["semantics"], what="logit")
        assert_rel(dense["rgb"], ref["rgb"], what="rgb")
        assert torch.equal(dense["point_location"].cpu(), ref["point_location"]), "sample positions differ bitwise"
        # selection parity: same point sets unless a value sits within tolerance of its threshold
        lab = torch.heaviside(torch.sigmoid(sem) - thr[2], torch.tensor(0.0))
        masks = {0: (lab >= 0.999) & (dens >= thr[1]), 1: (sem >= thr[0]) & (dens >= thr[1]), 2: dens >= thr[1]}
        near_thr = ((sem - thr[0]).abs() < 1e-3 * (1 + abs(thr[0]))) | ((dens - thr[1]).abs() < 1e-3 * (1 + abs(thr[1]))) | (
            (torch.sigmoid(sem) - thr[2]).abs() < 1e-4)
        counts = buf.counts.cpu()
        for k in range(3):
            got = set(buf.keys[k][: int(counts[k])].cpu().tolist())
            want = set(torch.nonzero(masks[k]).reshape(-1).tolist())
            diff = got ^ want
            assert all(bool(near_thr[i]) for i in diff), f"set {k}: {len(diff)} selection mismatches away from the thresholds"
            rows = buf.rows[k][: int(counts[k])].cpu()
            keys = buf.keys[k][: int(counts[k])].cpu()
            if len(keys):
                assert torch.equal(rows[:, :3], ref["point_location"].reshape(-1, 3)[keys])
                fourth = torch.sigmoid(dens[keys]) if k == 2 else torch.sigmoid(sem[keys])
                assert_rel(rows[:, 6], fourth, what=f"set {k} 4th column")
                assert_rel(rows[:, 3:6], ref["rgb"].reshape(-1, 3)[keys], what=f"set {k} rgb")


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
@pytest.mark.parametrize("name", ["small", "big"])
def test_export_with_stratified_jitter_matches_oracle(native_lib, cuda_device, name, impl):
    """The reference exporter's sampler is a module in TRAINING mode (created after eval_setup): every sample is jittered inside
    its bin (components/ray_samplers.py:78-87).  Same t_rand on both sides -> per-ray bins [B, S+1] through the kernel."""
    from fruitnerf_b200.components.ray_samplers import UniformSamplerWithNoise

    n = 21
    sd, spec = make_state(name, table_scale=2.0, weight_gain=2.5)
    field = make_field(name, sd, spec, cuda_device, contraction=False, test_mode="export").eval()
    pts, plane = ns.surface_points(((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), n)
    o, dirs, nears, fars = ns.orthographic_rays(pts, plane, batch=10_000, count=1)
    B = o.shape[0]
    t_rand = torch.rand((B, n + 1), generator=torch.Generator().manual_seed(5))
    ref = fr.export_outputs(sd, spec, o, dirs, nears, fars, n, t_rand=t_rand)
    # the host-side sampler produces the same spacing bins from the same draws (training-mode module)
    sampler = UniformSamplerWithNoise(num_samples=n, single_jitter=False)
    assert sampler.training
    base = torch.linspace(0.0, 1.0, n + 2 - 1)[None]
    centers = (base[..., 1:] + base[..., :-1]) / 2.0
    bins = torch.cat([base[..., :1], centers], -1) + (torch.cat([centers, base[..., -1:]], -1) - torch.cat([base[..., :1], centers], -1)) * t_rand
    buf = ops.ExportBuffers(capacity=B * n, device=cuda_device)
    dense = ops.export_batch(field.kernel_shape(), field.kernel_params(), o.cuda(), [float(v) for v in dirs[0]], bins.cuda().contiguous(),
                             float(nears[0]), float(fars[0]), buf, dense_out=True, thresholds=(float(ref["semantics"].median()), float(ref["density"].median()), 0.5),
                             impl=impl)
    assert torch.equal(dense["point_location"].cpu(), ref["point_location"]), "jittered sample positions differ bitwise"
    assert not torch.equal(ref["point_location"], fr.export_outputs(sd, spec, o, dirs, nears, fars, n)["point_location"])
    assert_rel(dense["density"], ref["density"], what="density")
    # logits of this deliberately large-weight field (weight_gain 2.5) are sums of terms ~100x the smallest |logit|: elements below
    # 2% of the maximum are compared against 1e-3 * 2% * max (one of 9261 sits at 1.2e-5 of the maximum with the default 1% floor)
    assert_rel(dense["semantics"], ref["semantics"], floor=0.02, what="logit")
    assert_rel(dense["rgb"], ref["rgb"], what="rgb")
    counts = buf.counts.cpu()
    keys = buf.keys[2][: int(counts[2])].cpu()
    rows = buf.rows[2][: int(counts[2])].cpu()
    assert torch.equal(rows[:, :3], ref["point_location"].reshape(-1, 3)[keys])
    with pytest.raises(ValueError):
        ops.export_batch(field.kernel_shape(), field.kernel_params(), o.cuda(), [0.0, 0.0, 1.0], bins[:5].cuda().contiguous(), 0.0, 2.0, buf)


@pytest.mark.parametrize("impl", IMPLS, ids=IMPL_IDS)
def test_full_size_properties(native_lib, cuda_device, impl):
    """BASELINE.json workload (4096 rays x 192 samples): size-independent properties --
    weights in [0,1], accumulation = sum(weights) <= 1, rgb is a convex combination, run-to-run
    determinism, and agreement between the two device implementations."""
    sd, spec = make_state("small", table_scale=0.5)
    field = make_field("small", sd, spec, cuda_device).train()
    o, d, s, e, cam = _rays(4096, 192, salt=1, num_images=7)
    with torch.no_grad():
        a = _render_gpu(field, o, d, s, e, cam, impl)
        b = _render_gpu(field, o, d, s, e, cam, impl)
    for k in ("rgb", "accumulation", "semantics", "weights", "depth"):
        assert torch.equal(a[k], b[k]), f"{k} not deterministic"
    w = a["weights"]
    assert float(w.min()) >= 0.0 and float(w.max()) <= 1.0
    assert torch.allclose(w.sum(-1), a["accumulation"], rtol=1e-5, atol=1e-6)
    assert float(a["accumulation"].max()) <= 1.0 + 1e-5
    lo = a["sample_rgb"].min(dim=1).values - 1e-5
    hi = a["sample_rgb"].max(dim=1).values + 1e-5
    assert bool(((a["rgb"] >= lo) & (a["rgb"] <= hi)).all()), "rgb outside the hull of the sample colours"
    if impl != L.FNR_IMPL_SIMT:
        with torch.no_grad():
            ref = _render_gpu(field, o, d, s, e, cam, L.FNR_IMPL_SIMT)
        for k in ("rgb", "accumulation", "semantics", "weights", "sample_density"):
            assert_rel(a[k], ref[k], what=f"tcgen05 vs simt {k}")
    # oracle spot check on a slice of the full batch
    sl = slice(100, 164)
    f = _oracle_field(sd, spec, o[sl], d[sl], s[sl], e[sl], cam[sl], True, "train")
    ref = fr.render(f, s[sl][..., None], e[sl][..., None], training=True)
    assert_rel(a["rgb"][sl], ref["rgb"], what="rgb slice")
    assert_rel(a["semantics"][sl], ref["semantics"], what="semantics slice")
