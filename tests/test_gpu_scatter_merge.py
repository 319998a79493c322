"""fruit_nerf's table-gradient scatter kernel (`level_scatter_kernel`, run alone through `fnr_level_scatter`) against a
float64 `index_add` of weight x gradient at the rows and positions the device itself computes (`fnr_hash_indices`).

The kernel merges the reds of adjacent lanes that add to the same row (a segmented shuffle sum per corner) and sends an
x-neighbour pair of rows r, r ^ 1 as one 16-byte red.  The cases put runs where they are easy to get wrong: one run
across a whole warp, zero corner weights and zero gradients inside runs, rows that collide in a tiny table, a ragged last
warp, floor x odd and even.  Only the summation order differs from the reference, so the bar is a reordered-fp32 one:
1e-5 of the sum of the magnitudes added to a row.
"""
import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn

from .util import make_field, make_state

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("native_lib", "cuda_device")]

LEVELS = 16
CORNER_SEL = (7, 5, 4, 6, 3, 1, 0, 2)  # oracle corner order: x | y << 1 | z << 2, 1 = ceil


def _shape(log2T, contraction):
    sd, spec = make_state("small", log2T=log2T)
    field = make_field("small", sd, spec, "cuda", contraction=contraction)
    with torch.no_grad():
        field.aabb.copy_(torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]]))
    return field.kernel_shape(), field.position_mode()


def _reference(shape, rows, pos, denc):
    """float64 sum of w * g per table row, and of |w * g| (the scale of the row's rounding error)."""
    N = pos.shape[0]
    scal = torch.tensor(list(shape.scalings), dtype=torch.float32)[:LEVELS]
    scaled = pos.float().cpu()[:, None, :] * scal[None, :, None]  # fp32 products, as the kernel forms them
    off = (scaled - torch.floor(scaled)).double()  # [N, L, 3]
    w = torch.ones(N, LEVELS, 8, dtype=torch.float64)
    for k, s in enumerate(CORNER_SEL):
        for a in range(3):
            w[..., k] *= off[..., a] if (s >> a) & 1 else 1.0 - off[..., a]
    g = denc.double().cpu().permute(1, 0, 2)  # [N, L, 2]
    contrib = w[..., None] * g[:, :, None, :]  # [N, L, 8, 2]
    idx = rows.reshape(N, LEVELS, 8).long().cpu().reshape(-1)
    want = torch.zeros(LEVELS << shape.log2_hashmap_size, 2, dtype=torch.float64)
    mag = torch.zeros_like(want)
    want.index_add_(0, idx, contrib.reshape(-1, 2))
    mag.index_add_(0, idx, contrib.abs().reshape(-1, 2))
    return want, mag


def _check(o, d, s, e, log2T=15, contraction=False, denc=None, seed=0):
    shape, mode = _shape(log2T, contraction)
    o, d, s, e = (t.cuda().contiguous() for t in (o, d, s, e))
    R, S = s.shape
    N = R * S
    if denc is None:
        denc = torch.randn(LEVELS, N, 2, generator=torch.Generator().manual_seed(seed))
    denc = denc.cuda().contiguous()
    rows, pos = ops.hash_indices(shape, o, d, s, e, mode)
    got = torch.zeros(LEVELS << log2T, 2, dtype=torch.float32, device="cuda")
    ops.level_scatter(shape, o, d, s, e, mode, denc, got)
    torch.cuda.synchronize()
    want, mag = _reference(shape, rows, pos.reshape(N, 3), denc)
    err = (got.double().cpu() - want).abs()
    bad = err > 1e-5 * mag + 1e-30
    assert not bad.any(), (f"{int(bad.any(-1).sum())} rows off, first {bad.any(-1).nonzero()[:5].flatten().tolist()}, "
                           f"max err {float(err.max()):.3g}")
    assert float(want.abs().sum()) > 0


def _point_rays(points, samples=1):
    """Rays of zero direction: every sample of ray r sits at points[r] (AABB [-1, 1]^3, so position = (x + 1) / 2)."""
    R = points.shape[0]
    o = points * 2.0 - 1.0
    d = torch.zeros(R, 3)
    s = torch.full((R, samples), 0.25)
    return o, d, s, s + 0.5


def test_one_run_across_the_warp():
    """Each ray's 64 samples at one point: a run of 32 lanes at every level, every corner."""
    pts = torch.rand(5, 3, generator=torch.Generator().manual_seed(1)) * 0.9 + 0.05
    _check(*_point_rays(pts, samples=64))


def test_zero_weights_inside_runs():
    """Lanes alternate between a point on a level-0 cell face (x = m / 16: its ceil-x corners weigh 0) and one inside the
    same cell, so every ceil-x run is broken by zero-weight lanes and every floor-x run spans the warp."""
    face = torch.tensor([5 / 16, 0.40625, 0.6875])
    inside = face + torch.tensor([0.01, 0.0, 0.0])
    pts = torch.stack([face if i % 2 == 0 else inside for i in range(96)])
    _check(*_point_rays(pts))


def test_zero_gradient_on_alternate_lanes():
    pts = torch.rand(3, 3, generator=torch.Generator().manual_seed(2)) * 0.9 + 0.05
    o, d, s, e = _point_rays(pts, samples=64)
    denc = torch.randn(LEVELS, 3 * 64, 2, generator=torch.Generator().manual_seed(3))
    denc[:, ::2] = 0.0
    _check(o, d, s, e, denc=denc)


@pytest.mark.parametrize("log2T", [1, 3])
def test_tiny_table_collisions(log2T):
    """With 2 or 8 rows per level, different cells and corners share rows, inside runs and across pairs."""
    o, d, s, e, _ = syn.ray_batch(7, 45, salt=5, far=3.0)
    _check(o, d, s, e, log2T=log2T, contraction=True)


@pytest.mark.parametrize("contraction", [True, False], ids=["contract", "aabb"])
def test_ragged_batch_both_position_modes(contraction):
    """37 x 77 = 2849 points: the last warp has 1 active lane; rays cross chunk boundaries."""
    o, d, s, e, _ = syn.ray_batch(37, 77, salt=7, far=3.0)
    _check(o, d, s, e, contraction=contraction)


def test_odd_and_even_floor_x():
    """Runs in cells with odd and with even floor x at level 0: only even ones pair into 16-byte reds."""
    pts = torch.tensor([[(m + 0.5) / 16, 0.5, 0.5] for m in range(2, 8)])
    _check(*_point_rays(pts, samples=40))


def test_refuses_misaligned_table():
    shape, mode = _shape(15, False)
    o, d, s, e = (t.cuda() for t in _point_rays(torch.full((2, 3), 0.5)))
    flat = torch.zeros((LEVELS << 15) * 2 + 2, device="cuda")
    with pytest.raises(L.FruitNerfNativeError):
        ops.level_scatter(shape, o, d, s, e, mode, torch.zeros(LEVELS, 2, 2, device="cuda"), flat[2:].view(-1, 2))
