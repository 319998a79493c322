"""Fruit counting on the device (fnr_cluster.cu) against the numpy / scikit-learn path of clustering.py.

Every fixture is checked to have no pair whose distance lies within 1e-12 relative of a radius it is queried with, so
ties cannot decide a result: counts, keep masks, voxel rows and labels must then be identical."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree
from sklearn.cluster import DBSCAN
from sklearn.neighbors import NearestNeighbors

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import clustering, ops
from fruitnerf_b200.synthetic import fruit_shell_cloud

pytestmark = pytest.mark.gpu

REAL_TREE = dict(eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                 remove_outliers_radius=0.015)  # clustering/config_real.py


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


def sk_labels(pts, eps, min_samples):
    return DBSCAN(eps=eps, min_samples=min_samples).fit(pts).labels_


def check_dbscan(pts, eps, min_samples, cuda_device):
    if len(pts) > 1:
        no_ties(pts, eps)
    labels, k = ops.dbscan(dev(pts, cuda_device), eps, min_samples)
    ref = sk_labels(pts, eps, min_samples) if len(pts) else np.zeros(0, dtype=np.int64)
    np.testing.assert_array_equal(labels.cpu().numpy(), ref)
    assert k == (int(ref.max()) + 1 if len(ref) else 0)
    return ref


def test_radius_counts_match_radius_neighbors(native_lib, cuda_device):
    pts = blobs(1, n_blob=800, n_noise=400)
    r = 0.04
    no_ties(pts, r)
    full = np.array([len(ix) for ix in NearestNeighbors(radius=r).fit(pts).radius_neighbors(pts, return_distance=False)])
    assert full.max() > 50 and full.min() == 1
    x = dev(pts, cuda_device)
    for cap in (1, 2, 17, 120, len(pts)):
        np.testing.assert_array_equal(ops.radius_count(x, r, cap).cpu().numpy(), np.minimum(full, cap))


def test_outlier_keep_mask_matches_cpu(native_lib, cuda_device):
    pts = blobs(2)
    for nb, r in ((8, 0.03), (40, 0.05), (1, 0.2)):
        no_ties(pts, r)
        got = clustering.remove_radius_outliers(dev(pts, cuda_device), nb, r).cpu().numpy()
        ref = clustering.remove_radius_outliers(pts, nb, r)
        assert 0 < len(ref) < len(pts)
        np.testing.assert_array_equal(got, ref)


def test_voxel_down_sample_is_bitwise_equal_to_cpu(native_lib, cuda_device):
    rng = np.random.default_rng(4)
    pts = np.concatenate([rng.uniform(-0.3, 0.7, (20000, 3)),  # dense: many points per voxel
                          rng.uniform(5, 9, (50, 3))])          # sparse: single-point voxels
    pts = np.concatenate([pts, pts[rng.integers(0, len(pts), 3000)]])  # exact duplicates
    pts = pts[rng.permutation(len(pts))]
    for voxel in (0.05, 0.013, 1.0):
        ref = clustering.voxel_down_sample(pts, voxel)
        got = clustering.voxel_down_sample(dev(pts, cuda_device), voxel).cpu().numpy()
        assert got.shape == ref.shape and got.shape[0] < len(pts)
        np.testing.assert_array_equal(got.view(np.int64), ref.view(np.int64))
    assert clustering.voxel_down_sample(dev(np.zeros((0, 3)), cuda_device), 0.1).shape == (0, 3)


def test_dbscan_blobs_and_noise(native_lib, cuda_device):
    ref = check_dbscan(blobs(5), 0.05, 10, cuda_device)
    assert ref.max() >= 5 and (ref == -1).sum() > 100


def test_dbscan_chain_linked_only_through_cells_two_apart(native_lib, cuda_device):
    eps = 0.01
    h = 15.0 / 16.0 * eps / math.sqrt(3.0)  # grid cell side of fnr_cluster.cu
    rng = np.random.default_rng(6)
    x = np.arange(60) * 0.93 * eps + 1e-4 * rng.standard_normal(60)
    chain = np.stack([x, 1e-4 * rng.standard_normal(60), 1e-4 * rng.standard_normal(60)], axis=1)
    steps = np.diff(np.floor((chain - chain.min(axis=0)) / h), axis=0)
    assert (np.abs(steps).max(axis=1) == 2).sum() > 20  # most links join cells two apart
    far = chain + np.array([0, 5 * eps, 0])
    pts = np.concatenate([chain, far])[rng.permutation(120)]
    ref = check_dbscan(pts, eps, 2, cuda_device)
    assert ref.max() == 1 and (ref >= 0).all()


def test_dbscan_border_points_take_the_smallest_adjacent_cluster(native_lib, cuda_device):
    eps = 0.1
    rng = np.random.default_rng(7)
    tuft = np.array([[0, 0, 0], [-0.03, 0.01, 0], [-0.03, -0.01, 0.005], [-0.035, 0, -0.01]])
    parts = []
    for k in range(6):
        a = tuft + np.array([5 * k * eps, 0, 0])  # core at x = 5k eps, its tuft behind it
        b = -tuft + np.array([5 * k * eps + 1.9 * eps, 0, 0])  # core 1.9 eps further on, its tuft in front
        border = np.array([[5 * k * eps + 0.95 * eps, 0, 0]])  # within eps of both cores, 3 neighbours itself
        parts += [a, b, border]
    pts = np.concatenate(parts) + 1e-5 * rng.standard_normal((sum(len(p) for p in parts), 3))
    for perm in (np.arange(len(pts)), rng.permutation(len(pts)), np.arange(len(pts))[::-1]):
        ref = check_dbscan(pts[perm], eps, 4, cuda_device)
        assert ref.max() == 11


def test_dbscan_edge_cases(native_lib, cuda_device):
    pts = blobs(8, n_blob=50, n_noise=50)
    check_dbscan(pts, 0.02, 1, cuda_device)  # min_samples = 1: every point is a core
    ref = check_dbscan(pts, 10.0, 5, cuda_device)  # eps larger than the cloud: one cluster
    assert (ref == 0).all()
    ref = check_dbscan(np.random.default_rng(9).uniform(0, 1, (500, 3)), 0.01, 3, cuda_device)  # all noise
    assert (ref == -1).all()
    check_dbscan(np.zeros((0, 3)), 0.1, 3, cuda_device)
    check_dbscan(np.array([[0.5, -2.0, 3.0]]), 0.1, 1, cuda_device)
    check_dbscan(np.array([[0.5, -2.0, 3.0]]), 0.1, 2, cuda_device)


def assert_counts_match(pts, cuda_device, **kw):
    ref = clustering.count_fruits(pts, **kw)
    got = clustering.count_fruits(dev(pts, cuda_device), **kw)
    assert set(got) == set(ref)
    for key in ("count", "count_before_merge", "num_points"):
        assert got[key] == ref[key] and type(got[key]) is type(ref[key]), key
    assert isinstance(got["centers"], np.ndarray) and got["centers"].dtype == np.float64
    np.testing.assert_allclose(got["centers"], ref["centers"], rtol=0, atol=1e-9)
    return got


def test_count_fruits_matches_cpu_on_the_host_test_fixture(native_lib, cuda_device):
    rng = np.random.default_rng(0)  # the cloud of test_training_host.py::test_clustering_counts_blobs_and_merges_fragments
    centers = np.array([[0, 0, 0], [0.5, 0, 0], [0, 0.5, 0.2], [0.4, 0.4, 0.4]], dtype=float)
    pts = np.concatenate([c + 0.02 * rng.standard_normal((400, 3)) for c in centers])
    frag = centers[0] + np.array([0.05, 0, 0]) + 0.004 * rng.standard_normal((60, 3))
    noise = rng.uniform(-1, 1, (30, 3))
    cloud = np.concatenate([pts, frag, noise])
    no_ties(cloud, 0.012)
    got = assert_counts_match(cloud, cuda_device, eps=0.012, min_samples=8, cluster_merge_distance=0.08)
    assert got["count"] == 4
    got = assert_counts_match(cloud.astype(np.float32).astype(np.float64), cuda_device, eps=0.012, min_samples=8,
                              cluster_merge_distance=0.08)
    f32 = clustering.count_fruits(torch.from_numpy(cloud.astype(np.float32)).to(cuda_device), eps=0.012, min_samples=8,
                                  cluster_merge_distance=0.08)  # float32 input is upcast
    assert f32["count"] == got["count"] and np.array_equal(f32["centers"], got["centers"])
    assert clustering.count_fruits(dev(np.zeros((0, 3)), cuda_device), 0.1, 5, 0.1)["count"] == 0


def test_count_fruits_matches_cpu_at_real_tree_parameters(native_lib, cuda_device):
    pts = fruit_shell_cloud(400_000, seed=11)
    no_ties(pts, REAL_TREE["eps"], REAL_TREE["remove_outliers_radius"])
    got = assert_counts_match(pts, cuda_device, **REAL_TREE)
    assert got["count"] == 400_000 // 4000


def test_device_counting_is_deterministic(native_lib, cuda_device):
    x = dev(fruit_shell_cloud(200_000, seed=12), cuda_device)
    runs = []
    for _ in range(2):
        labels, k = ops.dbscan(x, 0.02, 100)
        sums, counts = ops.cluster_sums(x, labels, k)
        res = clustering.count_fruits(x, **REAL_TREE)
        runs.append((labels.cpu().numpy(), sums.cpu().numpy(), counts.cpu().numpy(), res["centers"]))
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_non_finite_points_and_oversized_grids_are_refused(native_lib, cuda_device):
    bad = torch.zeros(10, 3, dtype=torch.float64, device=cuda_device)
    bad[3, 1] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        clustering.count_fruits(bad, 0.1, 2, 0.1)
    pts = dev(np.array([[0.0, 0, 0], [0, 1e5, 0], [1, 2, 3]]), cuda_device)
    with pytest.raises(L.FruitNerfNativeError, match=r"eps 0\.01 over an extent of 100000 on axis 1") as e:
        ops.dbscan(pts, 0.01, 2)
    assert "code -2" in str(e.value)
    with pytest.raises(L.FruitNerfNativeError, match=r"radius 0\.001 over an extent of 100000"):
        ops.radius_count(pts, 0.001, 2)
    with pytest.raises(L.FruitNerfNativeError, match=r"voxel size 0\.01 over an extent of 100000"):
        ops.voxel_down_sample(pts, 0.01)


def test_export_capacity_cloud_labels_agree_with_brute_force(native_lib, cuda_device):
    n, eps, min_samples = 1 << 24, REAL_TREE["eps"], REAL_TREE["min_samples"]
    fruits = n // 4000  # fruit_shell_cloud's default points per fruit; shells on a lattice of pitch 0.15
    x = dev(fruit_shell_cloud(n, seed=13), cuda_device)
    labels, k = ops.dbscan(x, eps, min_samples)
    core = ops.radius_count(x, eps, min_samples) >= min_samples
    assert int(core.sum()) > n // 2
    # no merges and no splits: one cluster per shell, and no cluster wider than one shell plus its border points
    # (<= 2 * (1.15 * 0.035 + eps) = 0.12 per axis; two neighbouring shells together span more than 0.16)
    assert k == fruits
    lab = labels.long()
    keep = lab >= 0
    idx = lab[keep][:, None].expand(-1, 3)
    lo = torch.full((k, 3), float("inf"), dtype=torch.float64, device=cuda_device).scatter_reduce_(0, idx, x[keep], "amin")
    hi = torch.full((k, 3), float("-inf"), dtype=torch.float64, device=cuda_device).scatter_reduce_(0, idx, x[keep], "amax")
    assert float((hi - lo).max()) < 0.14
    assert clustering.count_fruits(x, **REAL_TREE)["count"] == fruits
    # every sampled core shares its label with each core within eps (brute force, axis by axis, 4 queries at a time)
    g = torch.Generator(device="cpu").manual_seed(0)
    sample = torch.nonzero(core).reshape(-1).cpu()[torch.randint(0, int(core.sum()), (10_000,), generator=g)].to(cuda_device)
    cols = [x[:, a].contiguous() for a in range(3)]
    e2 = eps * eps
    for q in sample.split(4):
        d = cols[0][None, :] - cols[0][q][:, None]
        d2 = d * d
        for a in (1, 2):  # (dx*dx + dy*dy) + dz*dz, the kernels' order
            d = cols[a][None, :] - cols[a][q][:, None]
            d2 += d * d
        del d
        mism = (d2 <= e2) & core[None, :] & (labels[None, :] != labels[q][:, None])
        assert not bool(mism.any())
        assert bool((labels[q] >= 0).all())


def test_count_cli_agrees_with_count_fruits(native_lib, cuda_device, tmp_path):
    import json

    from fruitnerf_b200.export.exporter_utils import write_ply
    from fruitnerf_b200.scripts import count as count_cli

    pts = fruit_shell_cloud(100_000, seed=14)
    path = tmp_path / "semantic_colormap.ply"
    write_ply(path, pts, np.ones_like(pts))
    out = count_cli.main(["--pcd", str(path), "--json", str(tmp_path / "count.json")])
    ref = clustering.count_fruits(dev(pts, cuda_device), **REAL_TREE)
    assert (out["count"], out["count_before_merge"], out["num_points"]) == (ref["count"], ref["count_before_merge"], ref["num_points"])
    assert np.array_equal(np.array(out["centers"]).reshape(-1, 3), ref["centers"])
    assert json.loads((tmp_path / "count.json").read_text()) == out
