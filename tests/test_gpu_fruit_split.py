"""Stage 3 of the fruit count on the device (fnr_fruit_split.cu) against the numpy reference of clustering.py.

The fixtures are seeded clouds whose nearest-neighbour and Ward distances have no near ties, so pairings and merge
orders are decided by clear margins: ICP must then reach the same transforms (1e-9) in the same number of iterations,
the Ward sub-centres agree to 1e-12 and the Hausdorff distances are bit-equal."""
import numpy as np
import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import clustering as cl
from fruitnerf_b200 import ops
from fruitnerf_b200.synthetic import sphere_template, touching_fruit_cloud

pytestmark = pytest.mark.gpu

REAL_TREE = dict(eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                 remove_outliers_radius=0.015)  # clustering/config_real.py


def dev(x, cuda_device):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to(cuda_device)


@pytest.fixture(scope="module")
def candidates():
    """Surface samples of the groups to split in a touching-fruit cloud, and the template."""
    pts, _ = touching_fruit_cloud(seed=1)
    tmpl = sphere_template(0.035, 1000)
    groups = _host_groups(pts)
    _, samples = cl.alpha_stage(groups, tmpl, seed=0)
    assert len(samples) >= 4
    return [samples[g] for g in sorted(samples)], tmpl


def _host_groups(pts):
    """The merged groups count_fruits' CPU path hands to stage 3."""
    captured = {}
    orig = cl.split_clusters

    def spy(groups, template, seed=0, device=None):
        captured["groups"] = groups
        return orig(groups, template, seed=seed, device=device)

    cl.split_clusters = spy
    try:
        cl.count_fruits(pts, **REAL_TREE, template=sphere_template(0.035, 200))
    finally:
        cl.split_clusters = orig
    return captured["groups"]


def _offsets(segs):
    return np.concatenate([[0], np.cumsum([s.shape[0] for s in segs])])


def test_icp_matches_host(native_lib, cuda_device, candidates):
    samples, tmpl = candidates
    inits = np.stack([s.mean(axis=0) for s in samples])
    T, fit, rmse, it = ops.icp_scaled(dev(tmpl, cuda_device), dev(np.concatenate(samples), cuda_device), _offsets(samples),
                                      dev(inits, cuda_device))
    for i, s in enumerate(samples):
        init = np.eye(4)
        init[:3, 3] = inits[i]
        Tr, fr, rr, itr = cl.icp_scaled(tmpl, s, init)
        assert int(it[i]) == itr
        np.testing.assert_allclose(T[i].cpu().numpy(), Tr, rtol=0, atol=1e-9)
        assert float(fit[i]) == pytest.approx(fr, abs=1e-12) and float(rmse[i]) == pytest.approx(rr, abs=1e-12)


def test_icp_matches_host_on_similarity_transforms(native_lib, cuda_device):
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(4)
    src = rng.uniform(-1, 1, (400, 3)) * [0.05, 0.03, 0.02]
    truths, targets = [], []
    for b, scale in enumerate((0.8, 1.0, 1.2)):
        t = np.eye(4)
        t[:3, :3] = scale * Rotation.from_euler("xyz", [5 * b, -4, 3], degrees=True).as_matrix()
        t[:3, 3] = [0.3 * b, -0.2, 1.1]
        truths.append(t)
        targets.append(cl.transform_points(src, t))
    # initial translation only: the 5-degree rotations are within reach of the 0.01 correspondence distance
    inits = np.stack([t[:3, 3] for t in truths])
    T, fit, _, _ = ops.icp_scaled(dev(src, cuda_device), dev(np.concatenate(targets), cuda_device), _offsets(targets), dev(inits, cuda_device))
    for i, t in enumerate(truths):
        init = np.eye(4)
        init[:3, 3] = inits[i]
        np.testing.assert_allclose(T[i].cpu().numpy(), cl.icp_scaled(src, targets[i], init)[0], rtol=0, atol=1e-9)


def test_ward_matches_host(native_lib, cuda_device, candidates):
    samples, _ = candidates
    rng = np.random.default_rng(7)
    segs = list(samples) + [rng.uniform(-1, 1, (n, 3)) for n in (1, 3, 7, 4096)]
    got = ops.ward_cut(dev(np.concatenate(segs), cuda_device), _offsets(segs)).cpu().numpy()
    for i, s in enumerate(segs):
        np.testing.assert_allclose(got[i], cl.ward_cut_centres(s), rtol=0, atol=1e-12)


def test_hausdorff_is_bit_equal_to_host(native_lib, cuda_device):
    rng = np.random.default_rng(8)
    a_sets = [rng.uniform(-1, 1, (n, 3)) for n in (1, 300, 1000, 2500)]
    b_sets = [rng.uniform(-1, 1, (n, 3)) * 0.5 for n in (5000, 1, 1025, 700)]
    a_off, b_off = _offsets(a_sets), _offsets(b_sets)
    got = ops.hausdorff(dev(np.concatenate(a_sets), cuda_device), np.stack([a_off[:-1], a_off[1:]], 1),
                        dev(np.concatenate(b_sets), cuda_device), np.stack([b_off[:-1], b_off[1:]], 1)).cpu().numpy()
    want = np.array([cl.hausdorff(a, b) for a, b in zip(a_sets, b_sets)])
    assert np.array_equal(got, want)


def test_count_fruits_on_device_matches_host(native_lib, cuda_device):
    pts, gt = touching_fruit_cloud(seed=2)
    tmpl = sphere_template(0.035, 1000)
    ref = cl.count_fruits(pts, **REAL_TREE, template=tmpl)
    got = cl.count_fruits(dev(pts, cuda_device), **REAL_TREE, template=tmpl)
    for key in ("count", "count_before_merge", "count_after_merge", "num_split_extra", "num_pruned", "num_points"):
        assert got[key] == ref[key], key
    np.testing.assert_allclose(got["centers"], ref["centers"], rtol=0, atol=1e-9)
    assert got["count"] == len(gt)
    plain = cl.count_fruits(dev(pts, cuda_device), **REAL_TREE)
    assert set(plain) == {"count", "count_before_merge", "centers", "num_points"} and plain["count"] == got["count_after_merge"]


def test_repeated_runs_give_identical_bits(native_lib, cuda_device, candidates):
    samples, tmpl = candidates
    t, x, off = dev(tmpl, cuda_device), dev(np.concatenate(samples), cuda_device), _offsets(samples)
    init = dev(np.stack([s.mean(axis=0) for s in samples]), cuda_device)
    r1 = (*ops.icp_scaled(t, x, off, init), ops.ward_cut(x, off), ops.hausdorff(x, np.stack([off[:-1], off[1:]], 1), x[:500].flip(0),
                                                                                   np.tile([0, 500], (len(samples), 1))))
    r2 = (*ops.icp_scaled(t, x, off, init), ops.ward_cut(x, off), ops.hausdorff(x, np.stack([off[:-1], off[1:]], 1), x[:500].flip(0),
                                                                                   np.tile([0, 500], (len(samples), 1))))
    for u, v in zip(r1, r2):
        assert torch.equal(u, v)


def test_bad_inputs_are_refused(native_lib, cuda_device):
    x = dev(np.random.default_rng(9).uniform(-1, 1, (5000, 3)), cuda_device)
    with pytest.raises(L.FruitNerfNativeError, match="at most 4096"):
        ops.ward_cut(x, [0, 4097])
    bad = x[:100].clone()
    bad[7, 1] = float("nan")
    with pytest.raises(ValueError):
        ops.ward_cut(bad, [0, 100])
    with pytest.raises(ValueError):
        ops.icp_scaled(x[:50], bad, [0, 100], x[:1])
    with pytest.raises(ValueError):
        ops.hausdorff(bad, [[0, 100]], x, [[0, 10]])
    with pytest.raises(ValueError):
        ops.hausdorff(x, [[0, 0]], x, [[0, 10]])
    with pytest.raises(ValueError):
        ops.ward_cut(x, [0, 6000])


def test_count_cli_with_template_and_ground_truth(native_lib, cuda_device, tmp_path):
    import json

    from fruitnerf_b200.export.exporter_utils import write_ply
    from fruitnerf_b200.scripts import count as count_cli

    pts, gt = touching_fruit_cloud(seed=3)
    write_ply(tmp_path / "semantic_colormap.ply", pts, np.ones_like(pts))
    tmpl = sphere_template(0.05, 1000)
    write_ply(tmp_path / "template.ply", tmpl, np.ones_like(tmpl))
    np.save(tmp_path / "gt.npy", gt)
    out = count_cli.main(["--pcd", str(tmp_path / "semantic_colormap.ply"), "--template", str(tmp_path / "template.ply"),
                          "--template-size", "0.7", "--gt-centers", str(tmp_path / "gt.npy"), "--json", str(tmp_path / "count.json")])
    assert out["count"] == len(gt) and (out["TP"], out["FP"], out["FN"]) == (len(gt), 0, 0) and out["F1"] == 1.0
    assert out["num_pruned"] == 2 and len(out["centers"]) == out["count"]
    assert json.loads((tmp_path / "count.json").read_text()) == out
