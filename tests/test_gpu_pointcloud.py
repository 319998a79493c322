"""The `pointcloud` export on the device (fnr_cluster.cu kNN kernels, fnr_backproject_select) against the scipy / numpy
restatement in pointcloud.py, and the CLI end to end on a briefly trained model.

Fixtures are checked for the ties that would let two exact answers differ: no point has its k-th and (k+1)-th neighbour
at the same distance (within 1e-12), no mean distance lies within 1e-9 of an outlier threshold, and normals are only
compared where the two smallest covariance eigenvalues are clearly apart."""
import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops, pointcloud
from fruitnerf_b200.synthetic import fruit_shell_cloud

pytestmark = pytest.mark.gpu


def dev(pts, cuda_device):
    return torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float64)).to(cuda_device)


def no_kth_ties(pts, k):
    n = len(pts)
    if n <= k:
        return
    d, _ = cKDTree(pts).query(pts, k=k + 1)
    gap = d[:, k] - d[:, k - 1]
    assert (gap > 1e-12 * np.maximum(d[:, k], 1e-300)).all(), "fixture has a tie at the k-th neighbour distance"


def clouds():
    rng = np.random.default_rng(0)
    blob_c = rng.uniform(-1, 1, (5, 3))
    blobs = np.concatenate([c + 0.02 * rng.standard_normal((800, 3)) for c in blob_c])
    isolated = np.concatenate([rng.uniform(-0.5, 0.5, (3000, 3)), [[40.0, -35.0, 12.0], [-60.0, 2.0, 0.5], [41.0, -35.5, 12.3]]])
    return {
        "uniform": rng.uniform(-1, 1, (6000, 3)),
        "blobs": blobs[rng.permutation(len(blobs))],
        "shell": fruit_shell_cloud(40_000, seed=1),
        "far_isolated": isolated[rng.permutation(len(isolated))],
        "small": rng.standard_normal((17, 3)),
        "one": np.array([[0.3, -0.2, 5.0]]),
    }


@pytest.mark.parametrize("k", [20, 30, 1, 32])
def test_mean_distances_match_ckdtree(native_lib, cuda_device, k):
    for name, pts in clouds().items():
        got = ops.knn_mean_distance(dev(pts, cuda_device), k).cpu().numpy()
        ref = pointcloud.knn_mean_distance(pts, k)
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=0, err_msg=name)


def test_k_above_32_is_refused(native_lib, cuda_device):
    with pytest.raises(L.FruitNerfNativeError, match="at most 32") as e:
        ops.knn_mean_distance(dev(np.zeros((4, 3)), cuda_device), 33)
    assert "code -2" in str(e.value)


@pytest.mark.parametrize("std_ratio", [0.5, 2.0, 10.0])
def test_outlier_keep_masks_are_array_equal(native_lib, cuda_device, std_ratio):
    for name, pts in clouds().items():
        if len(pts) < 2:
            continue
        avg = pointcloud.knn_mean_distance(pts, 20)
        n = len(pts)
        mean = avg[avg > 0].sum() / n
        thr = mean + std_ratio * np.sqrt(((avg[avg > 0] - mean) ** 2).sum() / (n - 1))
        assert (np.abs(avg - thr) > 1e-9 * thr).all(), f"{name}: a mean distance lies at its threshold"
        kept, idx = pointcloud.remove_statistical_outliers(dev(pts, cuda_device), 20, std_ratio, return_index=True)
        ref_pts, ref_idx = pointcloud.remove_statistical_outliers(pts, 20, std_ratio, return_index=True)
        np.testing.assert_array_equal(idx.cpu().numpy(), ref_idx, err_msg=name)
        np.testing.assert_array_equal(kept.cpu().numpy(), ref_pts, err_msg=name)


def clear_gap(pts, k):
    """Points whose neighbour covariance has its two smallest eigenvalues clearly apart (gap > 1e-3 of the largest)."""
    kk = min(k, len(pts))
    _, idx = cKDTree(pts).query(pts, k=kk)
    nb = pts[np.asarray(idx).reshape(len(pts), kk)]
    c = nb - nb.mean(axis=1, keepdims=True)
    w = np.linalg.eigvalsh(np.einsum("nki,nkj->nij", c, c) / kk)
    return (w[:, 1] - w[:, 0]) > 1e-3 * np.maximum(w[:, 2], 1e-300)


def angle_up_to_sign(a, b):
    c = np.abs(np.sum(a * b, axis=1)) / (np.linalg.norm(a, axis=1) * np.linalg.norm(b, axis=1))
    return np.arccos(np.clip(c, -1, 1))


def test_normals_match_eigh_up_to_sign(native_lib, cuda_device):
    rng = np.random.default_rng(5)
    uv = rng.uniform(-1, 1, (3000, 2))
    plane = np.stack([uv[:, 0], 0.3 * uv[:, 1], 0.2 * uv[:, 0] - 0.1 * uv[:, 1]], axis=1)
    sets = dict(clouds(), plane=plane)
    for name, pts in sets.items():
        if len(pts) < 31:
            continue
        no_kth_ties(pts, 30)
        got = ops.estimate_normals(dev(pts, cuda_device), 30).cpu().numpy()
        ref = pointcloud.estimate_normals(pts, 30)
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-12, err_msg=name)
        ok = clear_gap(pts, 30)
        assert ok.mean() > 0.5, name
        ang = angle_up_to_sign(got[ok], ref[ok])
        assert ang.max() < 1e-6, (name, float(ang.max()))
    for pts in (np.array([[0.0, 0, 0]]), np.array([[0.0, 0, 0], [1, 2, 3]]), np.ones((6, 3))):
        got = ops.estimate_normals(dev(pts, cuda_device), 30).cpu().numpy()
        np.testing.assert_array_equal(got, np.tile([0.0, 0, 1], (len(pts), 1)))


def test_reoriented_normals_face_against_the_view(native_lib, cuda_device):
    pts = fruit_shell_cloud(20_000, seed=2)
    rng = np.random.default_rng(6)
    view = rng.standard_normal((len(pts), 3)).astype(np.float32)
    got = ops.estimate_normals(dev(pts, cuda_device), 30, torch.from_numpy(view).to(cuda_device)).cpu().numpy()
    dot = np.sum(got.astype(np.float32) * view, axis=1)
    assert (dot[np.abs(dot) > 1e-4] <= 0).all()
    ref = pointcloud.estimate_normals(pts, 30, view_dirs=view)
    ok = clear_gap(pts, 30) & (np.abs(dot) > 1e-4)
    cos = np.sum(got[ok] * ref[ok], axis=1)
    assert (cos > np.cos(1e-6)).all()  # same sign after reorientation


def test_backprojection_rows_are_bitwise_torch(native_lib, cuda_device):
    g = torch.Generator(device="cpu").manual_seed(7)
    R = 5000
    o = torch.rand(R, 3, generator=g) - 0.5
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    depth = torch.rand(R, 1, generator=g) * 1.5
    rgb = torch.rand(R, 3, generator=g)
    acc = torch.rand(R, 1, generator=g)
    acc[::7] = 0.5  # exactly at the threshold: rejected
    o[:10], d[:10], depth[:10], acc[:10] = torch.tensor([0.25, 0.0, 0.0]), torch.tensor([1.0, 0.0, 0.0]), 0.5, 1.0  # x = 0.75
    o[5:10, 0] = 0.0  # x = 0.5: on the face of the box
    o, d, depth, rgb, acc = (t.to(cuda_device) for t in (o, d, depth, rgb, acc))
    box = ((-0.7, -0.6, -0.8), (0.5, 0.9, 0.6))
    for b in (box, None):
        buf = ops.PointBuffers(2 * R, cuda_device)
        ops.backproject_select(o[:3000], d[:3000], depth[:3000], rgb[:3000], acc[:3000], buf, b)
        ops.backproject_select(o[3000:], d[3000:], depth[3000:], rgb[3000:], acc[3000:], buf, b)
        point = o + d * depth
        mask = acc[:, 0] > 0.5
        if b is not None:
            lo, hi = torch.tensor(b[0], device=cuda_device), torch.tensor(b[1], device=cuda_device)
            mask &= torch.all(torch.cat([point > lo, point < hi], dim=-1), dim=-1)
            assert not bool(mask[:10].any())
        n = int(buf.count.item())
        assert n == int(mask.sum()) and 0 < n < R
        for got, want in ((buf.points, point), (buf.colors, rgb), (buf.view_dirs, d)):
            assert torch.equal(got[:n].view(torch.int32), want[mask].contiguous().view(torch.int32))


def test_repeat_runs_give_identical_bits(native_lib, cuda_device):
    x = dev(fruit_shell_cloud(100_000, seed=3), cuda_device)
    view = torch.randn(x.shape[0], 3, device=cuda_device)
    runs = [(ops.knn_mean_distance(x, 20), ops.estimate_normals(x, 30, view)) for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_2p24_shell_cloud_matches_ckdtree_on_samples(native_lib, cuda_device):
    n = 1 << 24
    pts = fruit_shell_cloud(n, seed=4)
    x = dev(pts, cuda_device)
    avg = ops.knn_mean_distance(x, 20).cpu().numpy()
    nrm = ops.estimate_normals(x, 30).cpu().numpy()
    del x
    torch.cuda.empty_cache()
    q = np.random.default_rng(0).choice(n, 10_000, replace=False)
    tree = cKDTree(pts)
    d, _ = tree.query(pts[q], k=20)
    np.testing.assert_allclose(avg[q], np.cumsum(d, axis=1)[:, -1] / 20, rtol=1e-12, atol=0)
    d31, idx = tree.query(pts[q], k=31)
    tie_free = (d31[:, 30] - d31[:, 29]) > 1e-12 * d31[:, 30]
    nb = pts[idx[:, :30]]
    c = nb - nb.mean(axis=1, keepdims=True)
    w, v = np.linalg.eigh(np.einsum("nki,nkj->nij", c, c) / 30)
    ok = tie_free & ((w[:, 1] - w[:, 0]) > 1e-3 * w[:, 2])
    assert ok.mean() > 0.9
    assert angle_up_to_sign(nrm[q][ok], v[ok, :, 0]).max() < 1e-6


# ---- end to end --------------------------------------------------------------------------------------------------
def _tiny_spec(seed=0):  # as test_gpu_training.py
    from fruitnerf_b200.scripts.train import synthetic_spec

    spec = synthetic_spec("fruit_nerf", num_images=20, image_size=64, num_fruits=5, seed=seed, rays_per_batch=2048)
    m = spec.pipeline.model
    m.log2_hashmap_size = 17
    m.proposal_weights_anneal_max_num_iters = 100
    return spec


def test_pointcloud_cli_end_to_end(native_lib, cuda_device, tmp_path):
    from fruitnerf_b200.export.exporter_utils import read_ply
    from fruitnerf_b200.scripts.exporter import entrypoint, eval_setup
    from fruitnerf_b200.trainer import Trainer

    torch.manual_seed(0)
    run = tmp_path / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    out = tmp_path / "exports"
    lo, hi = (-0.8, -0.8, -0.8), (0.8, 0.8, 0.8)
    box_args = ["--bounding-box-min", *map(str, lo), "--bounding-box-max", *map(str, hi)]
    args = ["pointcloud", "--load-config", str(run / "config.yml"), "--output-dir", str(out), "--normal-method", "open3d",
            "--num-points", "20000", "--num-rays-per-batch", "4096", *box_args]
    torch.manual_seed(11)
    pcd = entrypoint(args)
    path = out / "point_cloud.ply"
    assert pcd["path"] == str(path)
    pts, col = read_ply(path)
    head, body = path.read_bytes().split(b"end_header\n", 1)
    rec = np.frombuffer(body, dtype=[("p", "<f8", 3), ("n", "<f8", 3), ("c", "u1", 3)])
    assert len(rec) == len(pts) > 1000
    assert ((pts > np.array(lo, dtype=np.float32)) & (pts < np.array(hi, dtype=np.float32))).all()

    # the same batches again, restated with torch on the device and the host reference
    torch.manual_seed(11)
    _, pipeline, _, _ = eval_setup(run / "config.yml")
    pipeline.datamanager.config.train_num_rays_per_batch = 4096
    lo_t, hi_t = torch.tensor(lo, device=cuda_device), torch.tensor(hi, device=cuda_device)
    points, colors, views, count = [], [], [], 0
    with torch.no_grad():
        while count < 20000:
            bundle, _ = pipeline.datamanager.next_train(0)
            outputs = pipeline.model(bundle)
            rgba = torch.cat([outputs["rgb"], outputs["accumulation"]], dim=-1)
            point = bundle.origins + bundle.directions * outputs["depth"]
            mask = (rgba[..., -1] > 0.5) & torch.all(torch.cat([point > lo_t, point < hi_t], dim=-1), dim=-1)
            points.append(point[mask])
            colors.append(rgba[mask][:, :3])
            views.append(bundle.directions[mask])
            count += int(mask.sum())
    points = torch.cat(points).double().cpu().numpy()
    colors = torch.cat(colors).double().cpu().numpy()
    views = torch.cat(views).cpu().numpy()
    avg = pointcloud.knn_mean_distance(points, 20)
    n = len(points)
    mean = avg[avg > 0].sum() / n
    thr = mean + 10.0 * np.sqrt(((avg[avg > 0] - mean) ** 2).sum() / (n - 1))
    assert (np.abs(avg - thr) > 1e-9 * thr).all()
    kept, idx = pointcloud.remove_statistical_outliers(points, 20, 10.0, return_index=True)
    assert np.array_equal(pts, kept) and np.array_equal(pcd["points"], kept)
    assert np.array_equal(rec["c"], np.clip(colors[idx] * 255, 0, 255).astype(np.uint8))
    assert np.array_equal(pcd["colors"], colors[idx])
    ref = pointcloud.estimate_normals(kept, 30, view_dirs=views[idx]).astype(np.float32).astype(np.float64)
    ok = clear_gap(kept, 30)
    d31, _ = cKDTree(kept).query(kept, k=31)
    ok &= (d31[:, 30] - d31[:, 29]) > 1e-12 * d31[:, 30]
    assert ok.mean() > 0.5
    ang = angle_up_to_sign(rec["n"][ok], ref[ok])
    assert ang.max() < 1e-6, float(ang.max())
    dot = np.sum(rec["n"].astype(np.float32) * views[idx], axis=1)
    assert (dot[np.abs(dot) > 1e-4] <= 0).all()

    with pytest.raises(SystemExit) as e:
        entrypoint(["pointcloud", "--load-config", str(run / "config.yml"), "--output-dir", str(out / "m"), "--normal-method",
                    "model_output", "--num-points", "100"])
    assert e.value.code == 1
