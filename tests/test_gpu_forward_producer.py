"""The small family's tensor-core forward and export with a gather warpgroup: a third warpgroup of the CTA gathers the
fine half of the hash-grid levels and hands it to the two MMA warpgroups through a shared-memory ring; they gather the
coarse half themselves.  The encoding, the stash and every output must keep the bits of the kernels in which each MMA
warpgroup gathered all of its own encodings.

(a) Per-sample density, semantic logit, rgb and (training mode) the encoding stash equal the earlier kernels' bits,
recorded as SHA-256 digests in tests/golden/forward_producer.json: both position modes, training and inference, batches
with fewer tiles than warpgroups, ragged last tiles, and batches where the ring's slots are reused many times.
(b) The export's dense outputs, its three point sets and their keys equal the earlier kernels' bits for three threshold
sets, on a grid of several tiles per warpgroup.
(c) At a shape with many tiles per warpgroup the forward agrees with the exact-fp32 simt forward at test_gpu_parity.py's
bars, and its encoding stash equals the simt stash bit for bit.

As a script, writes the digests of (a) and (b) from the library it loads (--lib names another build, such as the
earlier kernels'):

    python tests/test_gpu_forward_producer.py tests/golden/forward_producer.json [--lib path/to/libfruitnerf_b200.so]
"""
import hashlib
import json
import sys
from pathlib import Path

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

GOLDEN = Path(__file__).resolve().parent / "golden" / "forward_producer.json"
# rays x samples: 1 tile (fewer tiles than warpgroups), 2 tiles with a ragged second, 132 CTAs with several tiles each
# and a ragged last tile (ring slots reused), and many tiles per warpgroup
FORWARD_CASES = {"R1xS77": (1, 77), "R3xS50": (3, 50), "R701xS97": (701, 97), "R2048xS192": (2048, 192)}
POSITION_MODES = {"contract": True, "aabb": False}
EXPORT_N = 41  # samples per ray and rays per side of the export grid: 68 921 points, 539 tiles
EXPORT_QUANTILES = {"q25": 0.25, "q50": 0.5, "q75": 0.75}  # threshold sets at these quantiles of the field's outputs
SAMPLE_KEYS = ("sample_density", "sample_semantics", "sample_rgb")


def _digest(t):
    t = torch.as_tensor(t).contiguous()
    return hashlib.sha256(t.numpy().tobytes()).hexdigest() + f":{t.dtype}:{tuple(t.shape)}"


def _field(contraction):
    sd, spec = make_state("small", log2T=15)
    return make_field("small", sd, spec, "cuda:0", contraction=contraction).train()


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


def forward_outputs(case, mode, train, impl=L.FNR_IMPL_AUTO):
    R, S = FORWARD_CASES[case]
    return _render(_field(POSITION_MODES[mode]), syn.ray_batch(R, S, salt=5, far=3.0, num_images=7), impl, train)


def export_outputs(q, impl=L.FNR_IMPL_AUTO):
    """Dense export outputs and, per point set, its keys and rows ordered by key (rows are claimed in warp order).  The
    thresholds are the q-quantiles of the logits and densities of a first call, the label threshold the sigmoid of the
    logits', so that every point set is populated."""
    sd, spec = make_state("small", log2T=15, table_scale=2.0, weight_gain=2.5)
    field = make_field("small", sd, spec, "cuda:0", contraction=False, test_mode="export").eval()
    pts, plane = ns.surface_points(((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), EXPORT_N)
    o, dirs, nears, fars = ns.orthographic_rays(pts, plane, batch=10_000, count=1)
    bins = torch.linspace(0.0, 1.0, EXPORT_N + 1)

    def run(thresholds):
        buf = ops.ExportBuffers(capacity=o.shape[0] * EXPORT_N, device="cuda:0")
        dense = ops.export_batch(field.kernel_shape(), field.kernel_params(), o.cuda(), [float(v) for v in dirs[0]],
                                 bins.cuda(), float(nears[0]), float(fars[0]), buf, dense_out=True, thresholds=thresholds, impl=impl)
        return buf, dense

    _, first = run((3.0, 70.0, 0.9))
    logit_min = float(torch.quantile(first["semantics"].cpu().double(), q))
    thresholds = (logit_min, float(torch.quantile(first["density"].cpu().double(), q)), float(torch.sigmoid(torch.tensor(logit_min))))
    buf, dense = run(thresholds)
    res = {f"export_{k}": v.cpu() for k, v in dense.items()}
    counts = buf.counts.cpu()
    for k in range(3):
        keys = buf.keys[k][: int(counts[k])].cpu()
        order = torch.argsort(keys)
        res[f"export_keys{k}"] = keys[order]
        res[f"export_rows{k}"] = buf.rows[k][: int(counts[k])].cpu()[order]
    return res


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


def _check(got, golden, prefix):
    bad = [k for k, v in got.items() if _digest(v) != golden[f"{prefix}/{k}"]]
    assert not bad, f"{prefix}: {bad} differ from the earlier kernels' bits"


@pytest.mark.parametrize("train", [True, False], ids=["train", "inference"])
@pytest.mark.parametrize("mode", list(POSITION_MODES))
@pytest.mark.parametrize("case", list(FORWARD_CASES))
def test_forward_bits_equal_earlier_kernels(native_lib, cuda_device, golden, case, mode, train):
    """(a)"""
    got = forward_outputs(case, mode, train)
    assert ("stash" in got) == train
    _check(got, golden, f"{case}/{mode}/{'train' if train else 'inference'}")


@pytest.mark.parametrize("thr", list(EXPORT_QUANTILES))
def test_export_bits_equal_earlier_kernels(native_lib, cuda_device, golden, thr):
    """(b)"""
    got = export_outputs(EXPORT_QUANTILES[thr])
    assert all(len(got[f"export_keys{k}"]) > 0 for k in range(3)), "the thresholds leave a point set empty"
    _check(got, golden, f"export/{thr}")


@pytest.mark.parametrize("mode", list(POSITION_MODES))
def test_many_tiles_against_simt(native_lib, cuda_device, mode):
    """(c)"""
    field = _field(POSITION_MODES[mode])
    rays = syn.ray_batch(2048, 192, salt=2, num_images=7)
    tc = _render(field, rays, L.FNR_IMPL_AUTO, train=True)
    ref = _render(field, rays, L.FNR_IMPL_SIMT, train=True)
    for k in SAMPLE_KEYS:
        assert_rel(tc[k], ref[k], what=f"tensor cores vs simt {k}")
    assert torch.equal(tc["stash"], ref["stash"]), "the encoding stash is exact fp32 on both paths"


def write_golden(path):
    res = {}
    for case in FORWARD_CASES:
        for mode in POSITION_MODES:
            for train in (True, False):
                for k, v in forward_outputs(case, mode, train).items():
                    res[f"{case}/{mode}/{'train' if train else 'inference'}/{k}"] = _digest(v)
    for thr, q in EXPORT_QUANTILES.items():
        got = export_outputs(q)
        print(f"export {thr}: point sets of {[len(got[f'export_keys{k}']) for k in range(3)]}")
        res.update({f"export/{thr}/{k}": _digest(v) for k, v in got.items()})
    Path(path).parent.mkdir(parents=True, exist_ok=True)
    Path(path).write_text(json.dumps(res, indent=1, sort_keys=True) + "\n")
    print(f"wrote {path}: {len(res)} digests")


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
