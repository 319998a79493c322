"""CPU tests of the oracle: golden vectors + independent known-answer checks.

The reference has no tests of its own (SURVEY.md section 4), so the known answers below are derived by
hand / by independent integer arithmetic from the formulas the reference's dependencies publish.
"""
from pathlib import Path

import math

import numpy as np
import pytest
import torch

from fruitnerf_b200 import synthetic as syn
from oracle import fruit_ref as fr
from oracle import ns_torch as ns

GOLD = Path(__file__).resolve().parent / "golden"


def test_scalings_are_float32_floor():
    # float32 pow through Tensor.__rpow__: top level of max_res 2048 is 2047 (SURVEY.md section 7)
    assert ns.hash_scalings(16, 16, 2048).tolist() == [16, 22, 30, 42, 58, 80, 111, 153, 212, 294, 406, 561, 776, 1072, 1482, 2047]
    assert ns.hash_scalings(16, 16, 4096)[-1] == 4095


def _py_hash(x, y, z, T, level):
    return (((x * 1) ^ (y * 2654435761) ^ (z * 805459861)) % (2**T)) + level * 2**T


@pytest.mark.parametrize("T,max_res", [(17, 2048), (19, 2048), (21, 4096)])
def test_hash_rows_against_python_ints_and_golden(T, max_res):
    g = np.load(GOLD / "hash_indices.npz")
    pts = torch.from_numpy(g["points"])
    scal = ns.hash_scalings(16, 16, max_res)
    idx, off = ns.hash_corner_indices(pts, scal, T)
    assert np.array_equal(idx.numpy(), g[f"idx_T{T}"])
    assert np.array_equal(off.numpy(), g[f"off_T{T}"])
    # independent arbitrary-precision check + uint32 wrap-around equivalence
    order = ("ccc", "cfc", "ffc", "fcc", "ccf", "cff", "fff", "fcf")
    for n in range(pts.shape[0]):
        for l in range(16):
            s = (pts[n] * scal[l]).numpy()
            f, c = np.floor(s).astype(np.int64), np.ceil(s).astype(np.int64)
            for k, sel in enumerate(order):
                v = [int(c[i]) if ch == "c" else int(f[i]) for i, ch in enumerate(sel)]
                assert int(idx[n, l, k]) == _py_hash(*v, T, l)
                u32 = ((v[0] & 0xFFFFFFFF) ^ ((v[1] * 2654435761) & 0xFFFFFFFF) ^ ((v[2] * 805459861) & 0xFFFFFFFF)) & (2**T - 1)
                assert int(idx[n, l, k]) == u32 + l * 2**T


def test_hash_encode_is_trilinear_interpolation():
    """On a table that stores an affine function of the corner coordinates the encoding must
    reproduce that function at the query point (trilinear interpolation reproduces affine maps)."""
    T, L = 14, 2
    scal = torch.tensor([4.0, 7.0])
    table = torch.zeros(L * 2**T, 2)
    # fill every reachable corner of both levels
    for l, res in enumerate((4, 7)):
        g = torch.arange(res + 1)
        xyz = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
        rows = ns.hash_fn(xyz[:, None, :].expand(-1, L, 3).to(torch.int32), T, L)[:, l]
        assert rows.unique().numel() == rows.numel(), "test needs a collision-free table"
        vals = xyz.float() / res
        table[rows, 0] = 1.0 + 2.0 * vals[:, 0] - 3.0 * vals[:, 1] + 0.5 * vals[:, 2]
        table[rows, 1] = vals[:, 2]
    p = torch.tensor([[0.3, 0.6, 0.9], [0.01, 0.5, 0.25], [0.5, 0.5, 0.5]])
    enc = ns.hash_encode(p, table, scal, T)
    want0 = 1.0 + 2.0 * p[:, 0] - 3.0 * p[:, 1] + 0.5 * p[:, 2]
    for l in range(L):
        assert torch.allclose(enc[:, 2 * l], want0, atol=1e-5)
        assert torch.allclose(enc[:, 2 * l + 1], p[:, 2], atol=1e-6)


def test_contraction_and_masking():
    x = torch.tensor([[0.5, -0.25, 0.0], [2.0, 0.0, 0.0], [0.0, -4.0, 2.0]])
    c = ns.scene_contraction_inf(x)
    assert torch.allclose(c[0], x[0])
    assert torch.allclose(c[1], torch.tensor([1.5, 0.0, 0.0]))
    assert torch.allclose(c[2], torch.tensor([0.0, -1.75, 0.875]))
    aabb = torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    pos, sel = fr.sample_positions(torch.tensor([[[0.0, 0, 0]], [[5.0, 0, 0]]]), torch.tensor([[[1.0, 0, 0]], [[1.0, 0, 0]]]),
                                   torch.tensor([[[0.0]], [[0.0]]]), torch.tensor([[[1.0]], [[1.0]]]), aabb, contraction=False)
    assert sel.tolist() == [[True], [False]] and pos[1].abs().sum() == 0
    assert torch.allclose(pos[0], torch.tensor([[0.75, 0.5, 0.5]]))


def test_sh_degree4_known_values():
    c = ns.sh_degree4(torch.tensor([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0]]))
    assert torch.allclose(c[:, 0], torch.full((2,), 0.28209479))
    assert abs(float(c[0, 6]) - (0.9461746957575601 - 0.31539156525251999)) < 1e-6
    assert abs(float(c[0, 12]) - 0.3731763325901154 * 2) < 1e-6
    assert abs(float(c[1, 15]) - 0.5900435899266435) < 1e-6 and abs(float(c[1, 3]) - 0.4886025119029199) < 1e-6


def test_compositing_known_answers():
    deltas = torch.full((4, 3, 1), 0.5)
    dens = torch.tensor([[0.0, 0.0, 0.0], [1e9, 0.0, 0.0], [2.0, 2.0, 2.0], [float("nan"), 1.0, 1.0]])[..., None]
    w = ns.get_weights(deltas, dens)
    assert w[0].abs().sum() == 0  # empty space
    assert torch.allclose(w[1, :, 0], torch.tensor([1.0, 0.0, 0.0]))  # opaque first sample
    a = 1 - np.exp(-1.0)
    assert torch.allclose(w[2, :, 0], torch.tensor([a, a * np.exp(-1.0), a * np.exp(-2.0)], dtype=torch.float32), atol=1e-6)
    assert torch.isfinite(w[3]).all() and w[3, 0, 0] == 0  # nan_to_num
    rgb = torch.tensor([[[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]]]).repeat(4, 1, 1)
    out = ns.render_rgb_last_sample(rgb, w, training=True)
    assert torch.allclose(out[0], torch.tensor([0.0, 0.0, 1.0]))  # background = last sample colour
    assert torch.allclose(out[1], torch.tensor([1.0, 0.0, 0.0]))
    starts = torch.tensor([0.0, 0.5, 1.0]).view(1, 3, 1).repeat(4, 1, 1)
    depth, idx = ns.render_depth_median(w, starts, starts + 0.5)
    assert idx[:3, 0].tolist() == [2, 0, 0]  # never reaches 0.5 -> clamped to the last sample
    assert float(depth[2]) == 0.25
    # exact tie: cumulative weight hits 0.5 exactly at index 1 (searchsorted side="left")
    wt = torch.tensor([[[0.25], [0.25], [0.25]]])
    _, it = ns.render_depth_median(wt, starts[:1], starts[:1] + 0.5)
    assert int(it) == 1


def test_trunc_exp_gradient_is_clamped():
    x = torch.tensor([-20.0, 0.0, 20.0], requires_grad=True)
    ns.trunc_exp(x).sum().backward()
    assert torch.allclose(x.grad, torch.exp(torch.tensor([-15.0, 0.0, 15.0])))


def test_export_thresholds_and_selection():
    out = {
        "point_location": torch.arange(18.0).view(1, 6, 3),
        "semantics": torch.tensor([[2.9, 3.0, 5.0, 5.0, 2.0, 2.2]]),
        "density": torch.tensor([[100.0, 69.9, 70.0, 10.0, 80.0, 75.0]]),
        "rgb": torch.rand(1, 6, 3),
    }
    out["semantics_colormap"] = torch.heaviside(torch.sigmoid(out["semantics"]) - 0.9, torch.tensor(0.0)).long()
    assert out["semantics_colormap"].tolist() == [[1, 1, 1, 1, 0, 1]]  # sigmoid(2.2) = 0.9002 > 0.9
    sel = fr.export_select(out)
    assert sel["density"]["points"].shape[0] == 4
    assert sel["semantic"]["points"][:, 0].tolist() == [6.0]  # logit >= 3 and density >= 70
    assert sel["semantic_colormap"]["points"][:, 0].tolist() == [0.0, 6.0, 15.0]
    assert torch.allclose(sel["semantic"]["colors"][:, 3], torch.sigmoid(torch.tensor([5.0])))
    assert torch.allclose(sel["density"]["colors"][:, 3], torch.ones(4))  # sigmoid(density >= 70) == 1


def test_export_grid_golden_and_shapes():
    g = np.load(GOLD / "export_grid.npz")
    for n, aabb, tag in ((4, ((-1, -1, -1), (1, 1, 1)), "n4_cube"), (64, ((-1, -1, -1), (1, 1, 1)), "n64_cube"),
                         (10, ((-1.0, -0.5, -0.25), (1.0, 0.5, 0.75)), "n10_box")):
        pts, plane = ns.surface_points(aabb, n)
        assert np.array_equal(pts.numpy(), g[f"{tag}_points"]) and np.array_equal(plane.numpy(), g[f"{tag}_plane"])
    pts, plane = ns.surface_points(((-1.0, -0.5, -0.25), (1.0, 0.5, 0.75)), 10)
    assert pts.shape == (int(2.0 / 1.0 * 10) * int(1.0 / 1.0 * 10), 3)  # int(dx/dz*n) x int(dy/dz*n), fruit_datamanager.py:100-103
    assert torch.all(pts[:, 2] == -0.25) and torch.allclose(plane, torch.tensor([[0.0, 0.0, 1.0]]))
    assert pts[1, 0] == pts[0, 0] and pts[1, 1] != pts[0, 1]  # meshgrid 'ij', x-major flatten
    o, d, nears, fars = ns.orthographic_rays(pts, plane, batch=150, count=2)
    assert o.shape[0] == 50 and torch.all(nears == 0) and torch.allclose(fars, torch.ones(50, 1))
    starts, ends = ns.uniform_bins(nears, fars, 5)
    assert torch.allclose(starts[0, :, 0], torch.tensor([0.0, 0.2, 0.4, 0.6, 0.8]))


@pytest.mark.parametrize("name", ["small", "big"])
def test_field_forward_golden(name):
    g = np.load(GOLD / "field_forward.npz")
    v = syn.SMALL if name == "small" else syn.BIG
    sd = syn.field_state(geo=v["geo"], sem_dims=v["sem_dims"], log2_hashmap_size=v["log2_hashmap_size"], num_images=7,
                         table_scale=0.5, weight_gain=1.5)
    spec = fr.FieldSpec(max_res=v["max_res"], log2_hashmap_size=v["log2_hashmap_size"], geo_feat_dim=v["geo"])
    o, d, s, e, cam = syn.ray_batch(32, 24, salt=77, far=3.0, num_images=7)
    for mode, contraction in (("train", True), ("mean", False)):
        f = fr.field_forward(sd, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, contraction=contraction, appearance=mode)
        r = fr.render(f, s[..., None], e[..., None], training=True)
        tag = f"{name}_{mode}"
        for k in ("density", "rgb", "semantics"):
            assert np.allclose(f[k].numpy(), g[f"{tag}_{k}"], rtol=1e-5, atol=1e-7), (tag, k)
        for k in ("rgb", "accumulation", "semantics", "weights"):
            assert np.allclose(r[k].numpy(), g[f"{tag}_render_{k}"], rtol=1e-5, atol=1e-7), (tag, k)
        assert np.array_equal(r["depth_index"].numpy(), g[f"{tag}_render_depth_index"])


def test_oracle_gradients_match_finite_differences():
    """Central differences in float64 through the whole oracle path (field + compositing + losses),
    including the semantic detach (fruit_field.py:264-265, fruit_nerf.py:343-345)."""
    torch.manual_seed(0)
    sd = syn.field_state(log2_hashmap_size=8, num_images=3, table_scale=0.5, weight_gain=1.5)
    sd = {k: v.double() for k, v in sd.items()}
    spec = fr.FieldSpec(log2_hashmap_size=8)
    spec.scalings = lambda: ns.hash_scalings(16, 16, 2048).double()
    o, d, s, e, cam = syn.ray_batch(3, 6, salt=2, far=2.0, num_images=3)
    o, d, s, e = o.double(), d.double(), s.double(), e.double()
    img, mask = syn.targets(3)

    def loss_fn(state, with_sem=True):
        f = fr.field_forward(state, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, True, "train")
        r = fr.render(f, s[..., None], e[..., None], training=True)
        ld = fr.loss_dict(r, img.double(), mask.double())
        return ld["rgb_loss"] + (ld["semantics_loss"] if with_sem else 0.0)

    # parameters upstream of the detach points are checked on the rgb loss only: finite differences
    # see through detach(), autograd (by design of the reference) does not
    for key, with_sem in (("mlp_head.layers.1.weight", True), ("mlp_base_mlp.layers.1.bias", False),
                          ("mlp_semantics.layers.0.weight", True), ("mlp_base_grid.hash_table", False)):
        st = {k: v.clone() for k, v in sd.items()}
        st[key].requires_grad_(True)
        loss_fn(st, with_sem).backward()
        g = st[key].grad.reshape(-1)
        flat = sd[key].reshape(-1)
        nz = torch.nonzero(g).reshape(-1)
        for i in (int(nz[0]), int(nz[len(nz) // 2]), int(nz[-1])):
            def at(delta):
                s2 = {k: v.clone() for k, v in sd.items()}
                s2[key].reshape(-1)[i] += delta
                return float(loss_fn(s2, with_sem))
            fd = (at(1e-6) - at(-1e-6)) / 2e-6
            assert abs(fd - float(g[i])) <= 1e-5 * max(1.0, abs(fd)) + 1e-8, (key, i, fd, float(g[i]))
    # the semantic loss must not reach the base MLP (detach) -- compare with a semantics-only loss
    st = {k: v.clone() for k, v in sd.items()}
    st["mlp_base_mlp.layers.0.weight"].requires_grad_(True)
    f = fr.field_forward(st, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, True, "train")
    r = fr.render(f, s[..., None], e[..., None], training=True)
    assert not r["semantics"].sum().requires_grad or torch.autograd.grad(r["semantics"].sum(), st["mlp_base_mlp.layers.0.weight"], allow_unused=True)[0] is None


# ---- golden vectors of the proposal stage / compositing edge cases / gradients -------------------------------------
def _gold(name):
    return {k: v for k, v in np.load(GOLD / name).items()}


def test_proposal_stage_golden():
    g = _gold("proposal.npz")
    R = g["origins"].shape[0]
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd_")}
    spec = fr.DensitySpec(num_levels=5, max_res=128, log2_hashmap_size=12)
    o, d = torch.from_numpy(g["origins"]), torch.from_numpy(g["directions"])
    nears, fars = torch.full((R, 1), 0.05), torch.full((R, 1), 1000.0)
    bins = torch.from_numpy(g["bins0"])
    e = ns.spacing_to_euclidean(bins, nears, fars)
    assert np.array_equal(e.numpy(), g["euclid0"])
    # piecewise map: linear below distance 1 (s = x/2), linear in disparity beyond; monotone, inside [near, far]
    # (the stratified jitter also moves the outermost edges inwards)
    assert bool((e[:, 0] >= 0.05).all()) and bool((e[:, -1] <= 1000.0 * (1 + 1e-6)).all())
    det = ns.spacing_to_euclidean(ns.spaced_bins(1, 64, None), nears[:1], fars[:1])
    assert float(det[0, 0]) == pytest.approx(0.05) and float(det[0, -1]) == pytest.approx(1000.0, rel=1e-4)
    assert bool((e[:, 1:] >= e[:, :-1]).all())
    w = fr.proposal_weights(sd, spec, o, d, e[:, :-1], e[:, 1:], aabb)
    assert np.allclose(w.numpy(), g["weights0"], rtol=1e-6, atol=1e-9)
    w_zero = w.clone()
    w_zero[0] = 0.0
    for tag, anneal in (("eval", 1.0), ("single", 0.37), ("perbin", 1.0)):
        u = torch.from_numpy(g[f"pdf_{tag}_u"]) if f"pdf_{tag}_u" in g else None
        nb = ns.pdf_sample(torch.pow(w_zero, anneal), bins, 24, u)
        assert np.allclose(nb.numpy(), g[f"pdf_{tag}_bins"], rtol=0, atol=1e-7), tag
        assert bool((nb[:, 1:] >= nb[:, :-1]).all()) and float(nb.min()) >= 0.0 and float(nb.max()) <= 1.0
    # an all-zero histogram (ray 0) resamples uniformly over the existing bins' span
    nb0 = torch.from_numpy(g["pdf_eval_bins"])[0]
    assert torch.allclose(nb0[1:] - nb0[:-1], (nb0[1:] - nb0[:-1]).mean().expand(24), atol=2e-3)
    nb = torch.from_numpy(g["pdf_eval_bins"])
    w2 = torch.from_numpy(g["weights1"])
    assert float(ns.interlevel_loss([w, w2], [bins, nb])) == pytest.approx(float(g["interlevel"]), rel=1e-6)
    outer = ns.lossfun_outer(nb, w2, bins, w)
    assert np.allclose(outer.numpy(), g["outer"], rtol=1e-5, atol=1e-9) and float(outer.min()) >= 0.0


def test_compositing_edge_case_golden():
    g = _gold("composite_gradients.npz")
    dens, rgb, sem = (torch.from_numpy(g[k]) for k in ("c_density", "c_rgb", "c_semantics"))
    starts = torch.arange(4, dtype=torch.float32).expand(5, 4)[..., None]
    r = fr.render({"density": dens, "rgb": rgb, "semantics": sem}, starts, starts + 1.0, training=False)
    for k in ("rgb", "accumulation", "depth", "semantics", "weights"):
        assert np.allclose(r[k].numpy(), g[f"c_out_{k}"], rtol=1e-6, atol=1e-7, equal_nan=False), k
    assert np.array_equal(r["depth_index"].numpy(), g["c_out_depth_index"])
    w = r["weights"][..., 0]
    # hand-derived: sigma = 0 -> no weight, colour = last sample; opaque first sample takes everything;
    # NaN density: that sample and everything behind it contribute 0 (nan_to_num); ln2 then opaque: 0.5 / 0.5 tie -> index 0
    assert torch.equal(w[0], torch.zeros(4)) and torch.allclose(r["rgb"][0], rgb[0, -1])
    assert torch.allclose(w[1], torch.tensor([1.0, 0.0, 0.0, 0.0]))
    assert torch.allclose(w[2], torch.tensor([1 - math.exp(-0.5), 0.0, 0.0, 0.0]), atol=1e-7)
    assert torch.allclose(w[3], torch.tensor([0.5, 0.5, 0.0, 0.0]), atol=1e-7) and int(r["depth_index"][3]) == 0
    assert bool(torch.isfinite(r["rgb"]).all())


def test_gradient_golden_is_reproducible():
    g = _gold("composite_gradients.npz")
    v = syn.SMALL
    sd = syn.field_state(geo=v["geo"], sem_dims=v["sem_dims"], log2_hashmap_size=12, num_images=3, table_scale=0.5, weight_gain=1.5)
    spec = fr.FieldSpec(max_res=v["max_res"], log2_hashmap_size=12, geo_feat_dim=v["geo"])
    o, d, s, e, cam = syn.ray_batch(16, 12, salt=931, far=3.0, num_images=3)
    img, mask = syn.targets(16, salt=932)
    sdg = {k: t.clone().requires_grad_(k != "aabb") for k, t in sd.items()}
    f = fr.field_forward(sdg, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, True, "train")
    loss = sum(fr.loss_dict(fr.render(f, s[..., None], e[..., None], training=True), img, mask).values())
    loss.backward()
    assert float(loss) == pytest.approx(float(g["g_loss"]), rel=1e-6)
    for k in g:
        if k.startswith("g_") and k not in ("g_loss", "g_table_rows", "g_table_vals"):
            ref = g[k]
            assert np.allclose(sdg[k[2:]].grad.numpy(), ref, rtol=1e-4, atol=1e-6 * np.abs(ref).max()), k
    assert np.allclose(sdg["mlp_base_grid.hash_table"].grad[torch.from_numpy(g["g_table_rows"])].numpy(), g["g_table_vals"], rtol=1e-4,
                       atol=1e-6 * np.abs(g["g_table_vals"]).max())
    # the semantic branch is detached from the geometry features (fruit_field.py:264-265): the colour loss alone reaches the base MLP


# --------------------------------------------------------------------------------------------------------------
# Independent pins: the oracle's building blocks against third-party implementations of the same mathematics that ARE
# installed here (scipy, numpy) or against brute-force evaluations of the published definitions.  They do not replace
# golden vectors from nerfstudio itself (tools/regen_golden_from_nerfstudio.py), but they are not the oracle checking itself.
# --------------------------------------------------------------------------------------------------------------
def _real_sh_scipy(l: int, m: int, d: np.ndarray) -> np.ndarray:
    """Real spherical harmonic Y_lm (the table convention: positive leading coefficients, no Condon-Shortley sign in the real
    form) built from scipy's complex harmonics."""
    from scipy.special import sph_harm_y

    polar = np.arccos(np.clip(d[:, 2], -1, 1))
    azim = np.arctan2(d[:, 1], d[:, 0])
    if m == 0:
        return sph_harm_y(l, 0, polar, azim).real
    y = sph_harm_y(l, abs(m), polar, azim)
    return math.sqrt(2.0) * (-1) ** m * (y.real if m > 0 else y.imag)


def test_sh_degree4_matches_scipy_real_spherical_harmonics():
    """All 16 components (constants, polynomial forms, ordering l^2 + l + m) on random unit directions."""
    g = torch.Generator().manual_seed(5)
    d = torch.nn.functional.normalize(torch.randn(256, 3, generator=g, dtype=torch.float64), dim=-1)
    got = ns.sh_degree4(d).numpy()
    for l in range(4):
        for m in range(-l, l + 1):
            want = _real_sh_scipy(l, m, d.numpy())
            assert np.allclose(got[:, l * l + l + m], want, atol=1e-9), (l, m)


def test_pdf_sample_matches_numpy_inverse_cdf():
    """PDFSampler = piecewise-linear inverse CDF of the padded histogram: numpy's interp(u, cdf, bins) ray by ray."""
    g = torch.Generator().manual_seed(6)
    R, S, n = 32, 24, 17
    w = torch.rand(R, S, generator=g) ** 3
    w[3] = 0.0  # an empty ray: uniform after the histogram padding
    edges = torch.sort(torch.rand(R, S + 1, generator=g), dim=-1).values
    for u_rand in (None, torch.rand(R, 1, generator=g), torch.rand(R, n + 1, generator=g)):
        got = ns.pdf_sample(w, edges, n, u_rand).double().numpy()
        nb = n + 1
        for r in range(R):
            ww = w[r].double().numpy() + 0.01
            cdf = np.concatenate([[0.0], np.minimum(1.0, np.cumsum(ww / ww.sum()))])
            u = np.linspace(0.0, 1.0 - 1.0 / nb, nb)
            u = u + (1.0 / (2 * nb) if u_rand is None else u_rand[r].double().numpy() / nb)
            want = np.interp(u, cdf, edges[r].double().numpy())
            assert np.allclose(got[r], want, atol=2e-6), r


def test_get_weights_matches_the_product_form():
    """w_i = alpha_i * prod_{j<i} (1 - alpha_j) (the discrete volume-rendering quadrature) in float64 loops."""
    g = torch.Generator().manual_seed(7)
    R, S = 16, 40
    deltas = torch.rand(R, S, 1, generator=g) * 0.1
    dens = torch.rand(R, S, 1, generator=g) ** 4 * 200
    got = ns.get_weights(deltas, dens)[..., 0].double().numpy()
    a = 1.0 - np.exp(-(dens * deltas)[..., 0].double().numpy())
    for r in range(R):
        T = 1.0
        for i in range(S):
            assert got[r, i] == pytest.approx(a[r, i] * T, abs=2e-6)
            T *= 1.0 - a[r, i]


def test_interlevel_loss_matches_the_outer_measure_definition():
    """mip-NeRF 360's proposal loss: for each interval of the fine histogram, the bound is the total proposal weight of every
    proposal interval that overlaps it; loss = mean(max(0, w - bound)^2 / (w + eps)).  Brute force over interval pairs."""
    g = torch.Generator().manual_seed(8)
    R = 6
    fine_t = torch.sort(torch.rand(R, 13, generator=g), dim=-1).values
    fine_w = torch.rand(R, 12, generator=g)
    fine_w = fine_w / fine_w.sum(-1, keepdim=True)
    total = 0.0
    props = []
    for S in (20, 9):
        t = torch.sort(torch.rand(R, S + 1, generator=g), dim=-1).values
        t[:, 0], t[:, -1] = 0.0, 1.0
        w = torch.rand(R, S, generator=g) * 0.1
        props.append((t, w))
        acc = 0.0
        for r in range(R):
            for i in range(12):
                lo, hi = float(fine_t[r, i]), float(fine_t[r, i + 1])
                bound = sum(float(w[r, j]) for j in range(S) if float(t[r, j + 1]) > lo and float(t[r, j]) < hi)
                wi = float(fine_w[r, i])
                acc += max(0.0, wi - bound) ** 2 / (wi + 1e-7)
        total += acc / (R * 12)
    got = ns.interlevel_loss([w for _, w in props] + [fine_w], [t for t, _ in props] + [fine_t])
    assert float(got) == pytest.approx(total, rel=1e-4)
    assert total > 0


def test_scene_contraction_and_lindisp_are_inverses_and_bounded():
    """Published forms: contract(x) = x inside the unit L-inf ball, (2 - 1/|x|) x/|x| outside (mip-NeRF 360, L-inf variant);
    s(t) = t/2 below 1, 1 - 1/(2t) above, and its inverse."""
    g = torch.Generator().manual_seed(9)
    x = torch.randn(512, 3, generator=g) * 4
    c = ns.scene_contraction_inf(x)
    n = x.abs().amax(-1)
    inside = n <= 1
    assert torch.equal(c[inside], x[inside])
    assert float(c.abs().amax()) < 2.0
    assert torch.allclose(c[~inside].abs().amax(-1), 2 - 1 / n[~inside], atol=1e-6)
    assert torch.allclose(torch.nn.functional.normalize(c[~inside], dim=-1), torch.nn.functional.normalize(x[~inside], dim=-1), atol=1e-6)
    t = torch.rand(256, generator=g) * 20 + 1e-3
    s = ns.lindisp_piecewise_fn(t)
    assert float(s.min()) > 0 and float(s.max()) < 1
    assert torch.allclose(ns.lindisp_piecewise_inv(s), t, rtol=2e-4)
    assert torch.allclose(s[t < 1], t[t < 1] / 2) and torch.allclose(s[t >= 1], 1 - 1 / (2 * t[t >= 1]))


def test_distortion_loss_is_the_integral_it_closes():
    """mip-NeRF 360's distortion loss is the closed form of  integral integral p(u) p(v) |u - v| du dv  for the piecewise-constant
    density p = w_i / delta_i: midpoint quadrature of that double integral on a fine grid."""
    g = torch.Generator().manual_seed(10)
    S, G = 9, 3000
    t = torch.sort(torch.rand(1, S + 1, generator=g, dtype=torch.float64), dim=-1).values
    t[:, 0], t[:, -1] = 0.0, 1.0
    w = torch.rand(1, S, generator=g, dtype=torch.float64)
    u = (torch.arange(G, dtype=torch.float64) + 0.5) / G
    idx = torch.clamp(torch.searchsorted(t[0], u, right=True) - 1, 0, S - 1)
    p = (w[0] / (t[0, 1:] - t[0, :-1]))[idx]
    want = float((p[:, None] * p[None, :] * (u[:, None] - u[None, :]).abs()).sum() / (G * G))
    assert float(ns.distortion_loss(w, t)) == pytest.approx(want, rel=2e-3)


def test_median_depth_is_the_first_sample_reaching_half_the_weight():
    g = torch.Generator().manual_seed(11)
    R, S = 64, 30
    w = torch.rand(R, S, 1, generator=g) ** 2
    w = w / w.sum(1, keepdim=True) * torch.rand(R, 1, 1, generator=g) * 1.2  # some rays never reach 0.5
    starts = torch.sort(torch.rand(R, S + 1, generator=g), dim=-1).values
    depth, idx = ns.render_depth_median(w, starts[:, :-1, None], starts[:, 1:, None])
    for r in range(R):
        c, k = 0.0, S - 1
        cum = torch.cumsum(w[r, :, 0], 0)  # the same float32 running sum the renderer thresholds
        for i in range(S):
            if float(cum[i]) >= 0.5:
                k = i
                break
        assert int(idx[r]) == k
        assert float(depth[r]) == pytest.approx(float(starts[r, k] + starts[r, k + 1]) / 2, abs=1e-6)


def test_render_pass_semantic_gradients_flag():
    """fruit_nerf.py:301-305: the semantic renderer's weights are detached unless pass_semantic_gradients.  The flag changes
    the gradients of the density path (base MLP, hash table) under a semantics loss, and no forward value."""
    v = syn.SMALL
    sd = syn.field_state(geo=v["geo"], sem_dims=v["sem_dims"], log2_hashmap_size=10, num_images=3, table_scale=0.5, weight_gain=1.5)
    o, d, s, e, cam = syn.ray_batch(8, 12, salt=17, far=3.0, num_images=3)
    _, mask = syn.targets(8, salt=18)
    res = {}
    for flag in (False, True):
        spec = fr.FieldSpec(max_res=v["max_res"], log2_hashmap_size=10, geo_feat_dim=v["geo"])  # geo stays detached
        st = {k: t.double().requires_grad_(k != "aabb") for k, t in sd.items()}
        f = fr.field_forward(st, spec, o[:, None, :], d[:, None, :], s[..., None], e[..., None], cam, True, "train")
        r = fr.render(f, s[..., None], e[..., None], training=True, pass_semantic_gradients=flag)
        ns.semantic_bce(r["semantics"], mask.double()).backward()
        res[flag] = (r, {k: t.grad for k, t in st.items() if k != "aabb"})
    (r0, g0), (r1, g1) = res[False], res[True]
    for k in ("rgb", "accumulation", "semantics", "weights", "depth"):
        assert torch.equal(r0[k], r1[k]), k
    for k in ("mlp_base_mlp.layers.0.weight", "mlp_base_mlp.layers.1.weight", "mlp_base_mlp.layers.1.bias", "mlp_base_grid.hash_table"):
        assert g0[k] is None or float(g0[k].abs().max()) == 0.0, k  # the semantics loss cannot reach the density path
        assert g1[k] is not None and float(g1[k].abs().max()) > 0.0, k
    for k in ("mlp_semantics.layers.0.weight", "field_head_semantics.net.bias"):
        assert torch.allclose(g0[k], g1[k], rtol=1e-12, atol=0.0), k  # the semantic branch itself sees the same weights
