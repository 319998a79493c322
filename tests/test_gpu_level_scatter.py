"""The tensor-core backward's hash-table gradient against the simt backward's inline scatter.  For fruit_nerf the field
backward leaves level-major encoding gradients and level_scatter_kernel adds them to the table one level at a time;
fruit_nerf_big's tensor-core backward scatters inline.

The two paths' values differ where their ReLU masks do (tests/test_gpu_backward_resident.py holds them to measured
distances), but which table rows a batch touches depends only on the positions, the levels and the corner weights.  So the
set of nonzero rows must be identical: a wrong level base, a wrong point-to-ray mapping or a skipped level shows there
even when a tolerance would hide it.  fruit_nerf_big at its own table size (log2T = 21) is held against the float64 oracle
on every row by tests/test_gpu_fullsize.py::test_gradients_at_real_table_size_match_oracle.
"""
import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn

from .test_gpu_backward_configs import _gpu_backward
from .util import HASH_KEY, make_field, make_state, mse_bce_loss

pytestmark = pytest.mark.gpu

LOG2T = 15


def _table_grads(name, R, S, contraction, impl):
    sd, spec = make_state(name, log2T=LOG2T)
    rays = syn.ray_batch(R, S, salt=7, far=3.0, num_images=7)
    img, mask = syn.targets(R, salt=7)
    got, _, _ = _gpu_backward(name, sd, spec, rays, mse_bce_loss(img, mask), torch.ones(R), impl, contraction=contraction)
    return got[HASH_KEY].detach().reshape(16, 1 << LOG2T, 2)


def _assert_same_rows(name, R, S, contraction):
    simt = _table_grads(name, R, S, contraction, L.FNR_IMPL_SIMT)
    tc = _table_grads(name, R, S, contraction, L.FNR_IMPL_TCGEN05)
    rows_simt, rows_tc = (simt != 0).any(-1), (tc != 0).any(-1)
    per_level = rows_simt.sum(-1).tolist()
    assert all(n > 0 for n in per_level), f"every level has touched rows: {per_level}"
    diff = (rows_simt != rows_tc).nonzero().tolist()
    assert not diff, f"{len(diff)} (level, row) pairs nonzero on one path only, first {diff[:5]}"


@pytest.mark.parametrize("contraction", [True, False], ids=["contract", "aabb"])
@pytest.mark.parametrize("name", ["small", "big"])
def test_nonzero_table_rows_match_simt(native_lib, cuda_device, name, contraction):
    """A few rays (250 points: less than one scatter CTA), both families and both position modes."""
    _assert_same_rows(name, 5, 50, contraction)


def test_ragged_batch_matches_simt(native_lib, cuda_device):
    """37 x 77 = 2849 points: not a multiple of the scatter kernel's 256-thread CTA, so levels change inside a CTA, and a
    grid stride that spans several levels (each thread's next work item lies past the last level)."""
    _assert_same_rows("small", 37, 77, True)


def test_second_backward_over_retained_graph_adds_the_same_gradient(native_lib, cuda_device):
    """The encoding gradients live in backward scratch, not in the forward's encoding stash: a second backward over the same
    graph reads the same encodings and adds the same table gradient again."""
    sd, spec = make_state("small", log2T=LOG2T)
    field = make_field("small", sd, spec, "cuda").train()
    o, d, s, e, cam = (t.cuda() for t in syn.ray_batch(64, 48, salt=7, far=3.0, num_images=7))
    out = ops.render(field.kernel_shape(), field.kernel_params(), o, d, s, e, cam, field.position_mode(), field.appearance_mode(),
                     impl=L.FNR_IMPL_TCGEN05)
    loss = out["rgb"].square().sum() + out["semantics"].sum()
    loss.backward(retain_graph=True)
    first = field.mlp_base_grid.hash_table.grad.clone()
    loss.backward()
    second = field.mlp_base_grid.hash_table.grad - first
    scale = float(first.abs().max())
    assert scale > 0
    assert float((second - first).abs().max()) <= 1e-5 * scale
