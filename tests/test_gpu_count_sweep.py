"""Parameter sweeps of the fruit count on the device: the multi-radius count (fnr_radius_count_multi) against its
single-radius sibling and scikit-learn, and clustering.count_sweep against per-config count_fruits.

Every fixture is checked to have no pair whose distance lies within 1e-12 relative of a radius it is queried with, so
ties cannot decide a result."""
import ctypes as C
import json

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree
from sklearn.neighbors import NearestNeighbors

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import clustering, ops
from fruitnerf_b200.export.exporter_utils import write_ply
from fruitnerf_b200.scripts import count_sweep as sweep_cli
from fruitnerf_b200.synthetic import sphere_template, touching_fruit_cloud

pytestmark = pytest.mark.gpu

OK, INVALID, UNSUPPORTED = 0, -1, -2  # FNR_OK, FNR_ERR_INVALID_ARGUMENT, FNR_ERR_UNSUPPORTED


def no_ties(pts: np.ndarray, *radii: float) -> None:
    tree = cKDTree(pts)
    for r in radii:
        near = tree.count_neighbors(tree, np.array([r * (1 - 1e-12), r * (1 + 1e-12)]))
        assert near[0] == near[1], f"fixture has a pair at distance {r} within 1e-12"


def dev(pts, cuda_device):
    return torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float64)).to(cuda_device)


def blobs(seed=0, n_blob=300, n_noise=200, spread=0.03):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-1, 1, (6, 3))
    pts = np.concatenate([c + spread * rng.standard_normal((n_blob, 3)) for c in centers] + [rng.uniform(-1.2, 1.2, (n_noise, 3))])
    return pts[rng.permutation(len(pts))]


def test_radius_count_multi_matches_single_and_radius_neighbors(native_lib, cuda_device):
    pts = blobs(1, n_blob=800, n_noise=400)
    radii = [0.02, 0.03, 0.05, 0.079]  # 0.079 / 0.02 = 3.95: 8 rings of the shared grid, more than the single call's 2
    caps = [5, 40, 10_000, 60]  # 5 and 40 / 60 saturate in the blobs, 10_000 never does
    no_ties(pts, *radii)
    x = dev(pts, cuda_device)
    multi = ops.radius_count_multi(x, radii, caps).cpu().numpy()
    assert multi.shape == (len(radii), len(pts))
    for k, (r, cap) in enumerate(zip(radii, caps)):
        single = ops.radius_count(x, r, cap).cpu().numpy()
        np.testing.assert_array_equal(multi[k], single)
        full = np.array([len(ix) for ix in NearestNeighbors(radius=r).fit(pts).radius_neighbors(pts, return_distance=False)])
        np.testing.assert_array_equal(multi[k], np.minimum(full, cap))
        assert (multi[k] == cap).any() == (cap < 10_000)
    again = ops.radius_count_multi(x, radii, caps).cpu().numpy()
    np.testing.assert_array_equal(again, multi)


@pytest.mark.parametrize("num_radii", [6, 13])  # the 8- and 16-radius instantiations of the kernel
def test_radius_count_multi_many_radii(native_lib, cuda_device, num_radii):
    pts = blobs(4, n_blob=600, n_noise=300)
    radii = list(0.02 * 3.9 ** (np.arange(num_radii) / (num_radii - 1)) + 1e-5 * np.arange(num_radii))  # up to 0.078 + ...
    caps = [[4, 30, 10_000, 200][k % 4] for k in range(num_radii)]
    no_ties(pts, *radii)
    x = dev(pts, cuda_device)
    multi = ops.radius_count_multi(x, radii, caps).cpu().numpy()
    assert multi.shape == (num_radii, len(pts))
    for k, (r, cap) in enumerate(zip(radii, caps)):
        np.testing.assert_array_equal(multi[k], ops.radius_count(x, r, cap).cpu().numpy())
    assert (multi == np.array(caps)[:, None]).any(axis=1)[np.array(caps) <= 30].all()  # caps 4 and 30 saturate


def test_radius_count_multi_on_empty_and_single_point(native_lib, cuda_device):
    empty = torch.zeros((0, 3), dtype=torch.float64, device=cuda_device)
    assert ops.radius_count_multi(empty, [0.1, 0.2], [1, 3]).shape == (2, 0)
    one = torch.tensor([[0.5, -1.0, 2.0]], dtype=torch.float64, device=cuda_device)
    np.testing.assert_array_equal(ops.radius_count_multi(one, [0.1, 0.3], [1, 4]).cpu().numpy(), [[1], [1]])


def test_radius_count_multi_rejects_invalid_arguments(native_lib, cuda_device):
    x = dev(blobs(3, n_blob=20, n_noise=10), cuda_device)
    lo, hi = ops._bounds(x)
    scratch = ops._cluster_scratch(x.shape[0], cuda_device)
    out = torch.empty((17, x.shape[0]), dtype=torch.int32, device=cuda_device)

    def count(radii, caps):
        r, c = (C.c_double * max(len(radii), 1))(*radii), (C.c_int32 * max(len(caps), 1))(*caps)
        return native_lib.fnr_radius_count_multi(x.data_ptr(), x.shape[0], lo, hi, r, c, len(radii), out.data_ptr(), scratch.data_ptr(),
                                                 scratch.numel(), None)

    assert count([], []) == INVALID
    assert count([0.1] * 17, [2] * 17) == UNSUPPORTED
    assert count([0.1, 0.0], [2, 2]) == INVALID
    assert count([0.1, -0.2], [2, 2]) == INVALID
    assert count([0.1, 0.2], [2, 0]) == INVALID
    assert count([0.1, 0.41], [2, 2]) == UNSUPPORTED
    assert b"at most 4" in native_lib.fnr_last_error()
    assert count([0.1, 0.4], [2, 2]) == OK
    torch.cuda.synchronize()
    with pytest.raises(L.FruitNerfNativeError):
        ops.radius_count_multi(x, [], [])


SWEEP = dict(nb=(60, 120), eps=(0.02, 0.025), sizes=(0.9, 1.0, 1.1))


def sweep_configs():
    configs, templates = [], []
    for nb in SWEEP["nb"]:
        for eps in SWEEP["eps"]:
            for size in SWEEP["sizes"]:
                configs.append(dict(eps=eps, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=nb,
                                    remove_outliers_radius=0.015))
                templates.append(sphere_template() * size)
    return configs, templates


def assert_same_count(a, b, atol):
    for k in ("count", "count_before_merge", "count_after_merge", "num_split_extra", "num_pruned", "num_points"):
        assert a[k] == b[k], k
    assert a["centers"].shape == b["centers"].shape
    np.testing.assert_allclose(a["centers"], b["centers"], rtol=0, atol=atol)


def test_count_sweep_matches_count_fruits(native_lib, cuda_device):
    pts, truth = touching_fruit_cloud(seed=3)
    no_ties(pts, 0.015, *SWEEP["eps"])
    configs, templates = sweep_configs()
    x = dev(pts, cuda_device)
    stages = []
    sweep = clustering.count_sweep(x, configs, templates, on_stage=stages.append)
    assert stages == ["radius_count", "voxel", "dbscan", "merge", "alpha", "match"]
    host = clustering.count_sweep(pts, configs, templates)
    assert len(sweep) == len(host) == 12
    split_seen = 0
    for c, t, s, h in zip(configs, templates, sweep, host):
        single = clustering.count_fruits(x, **c, template=t)
        assert_same_count(s, single, atol=0)  # the same kernels on the same inputs
        assert_same_count(s, h, atol=1e-9)
        es, e1 = clustering.evaluate_count(s["centers"], truth), clustering.evaluate_count(single["centers"], truth)
        assert (es["TP"], es["FP"], es["FN"]) == (e1["TP"], e1["FP"], e1["FN"])
        split_seen += s["num_split_extra"] + s["num_pruned"]
    assert split_seen > 0, "the fixture should exercise the split / prune stage"
    plain = clustering.count_sweep(x, configs[:3])  # no templates: stage 2 only
    for c, s in zip(configs[:3], plain):
        assert_same_count({**s, "count_after_merge": 0, "num_split_extra": 0, "num_pruned": 0},
                          {**clustering.count_fruits(x, **c), "count_after_merge": 0, "num_split_extra": 0, "num_pruned": 0}, atol=0)


def test_count_fruits_is_the_op_chain(native_lib, cuda_device):
    """Device count_fruits is the one-config count_sweep, so the test above compares the sweep with itself; this holds
    it to the chain of the public ops instead."""
    pts, _ = touching_fruit_cloud(seed=3)
    no_ties(pts, 0.015, 0.02)
    x = dev(pts, cuda_device)
    got = clustering.count_fruits(x, eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                                  remove_outliers_radius=0.015)
    down = ops.voxel_down_sample(clustering.remove_radius_outliers(x, 120, 0.015), 0.001)
    labels, k = ops.dbscan(down, 0.02, 100)
    sums, counts = ops.cluster_sums(down, labels, k)
    want = {**clustering.merge_cluster_centers(sums.cpu().numpy(), counts.cpu().numpy(), 0.04), "num_points": int(down.shape[0])}
    assert got.keys() == want.keys()
    for key in want:
        assert type(got[key]) is type(want[key]), key
    for key in ("count", "count_before_merge", "num_points"):
        assert got[key] == want[key], key
    assert got["centers"].dtype == want["centers"].dtype
    np.testing.assert_array_equal(got["centers"], want["centers"])
    assert got["count"] > 0


def write_obj(path, centres, n=12, radius=0.03):
    with open(path, "w") as f:
        for i, c in enumerate(centres):
            f.write(f"o fruit_{i}\n")
            for p in c + sphere_template(radius, n):
                f.write(f"v {float(p[0])!r} {float(p[1])!r} {float(p[2])!r}\n")


def write_line_set(path, centres, half=0.035):
    corners = np.array([[x, y, z] for x in (-half, half) for y in (-half, half) for z in (-half, half)])
    verts = (centres[:, None, :] + corners[None]).reshape(-1, 3)
    edges = [(8 * b + i, 8 * b + j) for b in range(len(centres)) for i, j in ((0, 1), (0, 2), (1, 3), (2, 3))]
    with open(path, "w") as f:
        f.write(f"ply\nformat ascii 1.0\nelement vertex {len(verts)}\nproperty double x\nproperty double y\nproperty double z\n"
                f"element edge {len(edges)}\nproperty int vertex1\nproperty int vertex2\nend_header\n")
        f.writelines(f"{float(v[0])!r} {float(v[1])!r} {float(v[2])!r}\n" for v in verts)
        f.writelines(f"{a} {b}\n" for a, b in edges)


def test_count_sweep_cli_end_to_end(native_lib, cuda_device, tmp_path):
    pts, truth = touching_fruit_cloud(seed=4)
    write_ply(tmp_path / "cloud.ply", pts, np.zeros_like(pts))
    write_ply(tmp_path / "template.ply", sphere_template(), np.zeros((1000, 3)))
    write_obj(tmp_path / "fruits.obj", truth)
    write_line_set(tmp_path / "lineset.ply", truth)
    base = {"path": str(tmp_path / "cloud.ply"), "remove_outliers_nb_points": [60, 120], "remove_outliers_radius": 0.015, "down_sample": 0.001,
            "eps": [0.02, 0.025], "cluster_merge_distance": 0.04, "minimum_size_factor": 0.3, "min_samples": 100,
            "template_path": str(tmp_path / "template.ply"), "apple_template_size": [0.9, 1.1], "gt_count": len(truth)}
    spec = {"obj": {**base, "gt_cluster": str(tmp_path / "fruits.obj")}, "lines": {**base, "gt_cluster": str(tmp_path / "lineset.ply")},
            "plain": {**base, "gt_cluster": None, "eps": 0.02, "remove_outliers_nb_points": 120, "apple_template_size": 1.0}}
    (tmp_path / "spec.json").write_text(json.dumps(spec))
    out = sweep_cli.main([str(tmp_path / "spec.json"), "--device", str(cuda_device), "--json", str(tmp_path / "res.json")])
    assert json.loads((tmp_path / "res.json").read_text()) == json.loads(json.dumps(out))
    assert list(out["obj"]) == [str(i) for i in range(8)]
    x = dev(pts, cuda_device)
    for i, nb, eps, size in [(0, 60, 0.02, 0.9), (5, 120, 0.02, 1.1), (7, 120, 0.025, 1.1)]:
        e = out["obj"][str(i)]
        assert e["params"] == {"remove_outliers_nb_points": nb, "eps": eps, "apple_template_size": size}
        ref = clustering.count_fruits(x, eps=eps, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=nb,
                                      remove_outliers_radius=0.015, template=clustering.load_template(tmp_path / "template.ply", size))
        score = clustering.evaluate_count(ref["centers"], truth)
        assert e["count"] == ref["count"] and e["TP"] == score["TP"] and e["F1"] == score["F1"] and e["gt"] == len(truth)
        assert out["lines"][str(i)] == e  # both ground truths hold the same centres
    ref = clustering.count_fruits(x, eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                                  remove_outliers_radius=0.015, template=clustering.load_template(tmp_path / "template.ply", 1.0))
    assert out["plain"] == {"0": {"path": str(tmp_path / "cloud.ply"), "count": ref["count"], "gt": len(truth)}}


def test_count_sweep_over_outlier_radii(native_lib, cuda_device):
    """Several outlier radii, 0.025 / 0.006 > 4 apart, so count_sweep needs two multi-radius calls; no template."""
    pts, _ = touching_fruit_cloud(seed=5)
    radii, eps = (0.006, 0.012, 0.025), (0.02, 0.025)
    no_ties(pts, *radii, *eps)
    assert clustering._radius_chunks(list(radii)) == [[0.006, 0.012], [0.025]]
    configs = [dict(eps=e, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=nb,
                    remove_outliers_radius=r) for r in radii for nb in (20, 100) for e in eps]
    configs.append(dict(configs[0]))  # shares stage 2 with configs[0]
    x = dev(pts, cuda_device)
    sweep = clustering.count_sweep(x, configs)
    for c, s in zip(configs, sweep):
        single = clustering.count_fruits(x, **c)
        assert s.keys() == single.keys()
        for k in ("count", "count_before_merge", "num_points"):
            assert s[k] == single[k], (c, k)
        np.testing.assert_array_equal(s["centers"], single["centers"])
    assert len({s["num_points"] for s in sweep}) >= 3, "the radii and nb should filter differently"
    assert sweep[0]["centers"] is not sweep[-1]["centers"]
    sweep[-1]["centers"][:] = np.nan  # results are independent, as separate count_fruits calls are
    assert np.isfinite(sweep[0]["centers"]).all()
