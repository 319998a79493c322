"""The small family's tensor-core forward and export on the resident weight image.  Their CTAs split the six tensor-core
layers once into shared memory and run several warpgroups, each on its own 128-point tiles; the kernels they replaced
(one warpgroup per CTA) staged each layer's weight tile from global memory at every layer step.  The image holds exactly
the bytes the staged kernel staged and every layer runs the same MMA sequence, so the outputs are bit for bit the staged
kernel's.  The backward's recompute relies on that: its ReLU masks are right only while its bits are the forward's.

(a) Per-sample density, semantic logit, rgb and the encoding stash of the render forward, and the export's dense outputs
and selected rows, equal the staged kernel's bits in tests/golden/forward_resident.npz.  Its forward cases are one tile
for a CTA of several warpgroups (R1 x S77), a ragged second tile (R3 x S50) and four tiles, the last ragged (R5 x S100);
its export grid is 11^3 points, ten and a half tiles.
(b) At the bench shape (4096 x 192, 6144 tiles: many per warpgroup) the forward agrees with the exact-fp32 simt forward at
the bars of test_gpu_parity.py.

As a script, writes the fixture of (a) from the library it loads (by default the package's; --lib names another, such as
a build of the staged kernel):

    python tests/test_gpu_forward_resident.py tests/golden/forward_resident.npz [--lib path/to/libfruitnerf_b200.so]
"""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200 import synthetic as syn
from oracle import ns_torch as ns

from tests.util import assert_rel, make_field, make_state

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "forward_resident.npz"
FORWARD_CASES = {"R1xS77": (1, 77), "R3xS50": (3, 50), "R5xS100": (5, 100)}
EXPORT_N = 11  # samples per ray and rays per side of the export grid
TC_IMPLS = [L.FNR_IMPL_AUTO, L.FNR_IMPL_TCGEN05]
TC_IDS = ["auto", "tcgen05"]
SAMPLE_KEYS = ("sample_density", "sample_semantics", "sample_rgb")


def _render(field, rays, impl, train):
    """The render forward; in training mode also the encoding stash it keeps for the backward."""
    dev = torch.device("cuda:0")
    o, d, s, e, cam = (t.to(dev) for t in rays)
    args = (field.kernel_shape(), field.kernel_params(), o, d, s, e, cam.to(torch.int32), field.position_mode(),
            field.appearance_mode())
    if not train:
        with torch.no_grad():
            out = ops.render(*args, impl=impl)
        return {k: out[k].cpu() for k in SAMPLE_KEYS}
    out = ops.render(*args, impl=impl)
    res = {k: out[k].detach().cpu() for k in SAMPLE_KEYS}
    res["stash"] = out["rgb"].grad_fn.saved[9].cpu()  # the _Render node's saved encoding stash
    return res


def forward_outputs(case, impl, train=True):
    R, S = FORWARD_CASES[case]
    sd, spec = make_state("small", log2T=15)
    field = make_field("small", sd, spec, "cuda:0").train()
    return _render(field, syn.ray_batch(R, S, salt=3, far=3.0, num_images=7), impl, train)


def _export_setup():
    sd, spec = make_state("small", log2T=15, table_scale=2.0, weight_gain=2.5)
    field = make_field("small", sd, spec, "cuda:0", contraction=False, test_mode="export").eval()
    pts, plane = ns.surface_points(((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), EXPORT_N)
    o, dirs, nears, fars = ns.orthographic_rays(pts, plane, batch=10_000, count=1)
    return field, o, [float(v) for v in dirs[0]], torch.linspace(0.0, 1.0, EXPORT_N + 1), float(nears[0]), float(fars[0])


def export_outputs(impl, thresholds):
    """Dense export outputs and, per point set, its keys and rows ordered by key (rows are claimed in warp order)."""
    field, o, normal, bins, near, far = _export_setup()
    buf = ops.ExportBuffers(capacity=o.shape[0] * EXPORT_N, device="cuda:0")
    dense = ops.export_batch(field.kernel_shape(), field.kernel_params(), o.cuda(), normal, bins.cuda(), near, far, buf,
                             dense_out=True, thresholds=thresholds, impl=impl)
    res = {f"export_{k}": v.cpu() for k, v in dense.items()}
    counts = buf.counts.cpu()
    for k in range(3):
        keys = buf.keys[k][: int(counts[k])].cpu()
        order = torch.argsort(keys)
        res[f"export_keys{k}"] = keys[order]
        res[f"export_rows{k}"] = buf.rows[k][: int(counts[k])].cpu()[order]
    return res


def _bits(t):
    t = torch.as_tensor(t)
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_bits(got, want, what):
    got, want = torch.as_tensor(got), torch.as_tensor(want)
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    diff = _bits(got) != _bits(want)
    assert not bool(diff.any()), f"{what}: {int(diff.sum())}/{diff.numel()} elements differ from the staged kernel's bits"


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("impl", TC_IMPLS, ids=TC_IDS)
@pytest.mark.parametrize("case", list(FORWARD_CASES))
def test_forward_bits_equal_staged_kernel(native_lib, cuda_device, golden, case, impl):
    """(a) training mode (with the stash) and inference mode."""
    got = forward_outputs(case, impl, train=True)
    for k, v in got.items():
        _assert_bits(v, golden[f"{case}/{k}"], f"{case} {k}")
    inf = forward_outputs(case, impl, train=False)
    for k in SAMPLE_KEYS:
        _assert_bits(inf[k], golden[f"{case}/{k}"], f"{case} inference {k}")


@pytest.mark.parametrize("impl", TC_IMPLS, ids=TC_IDS)
def test_export_bits_equal_staged_kernel(native_lib, cuda_device, golden, impl):
    """(a) the export: dense outputs and the three selected point sets."""
    got = export_outputs(impl, tuple(float(v) for v in golden["export_thresholds"]))
    assert all(len(got[f"export_keys{k}"]) > 0 for k in range(3)), "the thresholds leave a point set empty"
    for k, v in got.items():
        _assert_bits(v, golden[k], k)


def test_bench_shape_against_simt(native_lib, cuda_device):
    """(b) many tiles per warpgroup: the tensor-core forward against the simt forward at test_gpu_parity.py's bars."""
    sd, spec = make_state("small", table_scale=0.5)
    field = make_field("small", sd, spec, cuda_device).train()
    rays = syn.ray_batch(4096, 192, salt=1, num_images=7)
    tc = _render(field, rays, L.FNR_IMPL_AUTO, train=True)
    ref = _render(field, rays, L.FNR_IMPL_SIMT, train=True)
    for k in SAMPLE_KEYS:
        assert_rel(tc[k], ref[k], what=f"tensor cores vs simt {k}")
    assert torch.equal(tc["stash"], ref["stash"]), "the encoding stash is exact fp32 on both paths"


def write_golden(path):
    res = {}
    for case in FORWARD_CASES:
        for k, v in forward_outputs(case, L.FNR_IMPL_TCGEN05).items():
            res[f"{case}/{k}"] = v.numpy()
    # thresholds at the medians of this field's logits and densities, so that every point set is populated
    dense = export_outputs(L.FNR_IMPL_TCGEN05, (3.0, 70.0, 0.9))
    thr = (float(dense["export_semantics"].median()), float(dense["export_density"].median()), 0.5)
    res["export_thresholds"] = np.array(thr, dtype=np.float64)
    res.update({k: v.numpy() for k, v in export_outputs(L.FNR_IMPL_TCGEN05, thr).items()})
    Path(path).parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(path, **res)
    print(f"wrote {path}: " + ", ".join(f"{k} {tuple(v.shape)}" for k, v in res.items()))


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--lib", default=None, help="library to run (default: the package's)")
    a = ap.parse_args()
    if a.lib:
        L.LIB_PATH = Path(a.lib).resolve()
    L.load()
    write_golden(a.out)
