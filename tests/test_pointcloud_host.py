"""Host side of the `pointcloud` export: the scipy / numpy restatement of open3d's statistical outlier removal and normal
estimation against brute force, the PLY normals, the CLI defaults and the sm_90a build (no GPU needed)."""
import dataclasses
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from fruitnerf_b200 import _build
from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops, pointcloud
from fruitnerf_b200.export.exporter_utils import read_ply, write_ply
from fruitnerf_b200.scripts import exporter


def brute_mean_distance(pts, k):
    """Full distance matrix; neighbours ordered by (distance, index)."""
    n = len(pts)
    kk = min(k, n)
    d = np.sqrt(((pts[:, None, :] - pts[None, :, :]) ** 2).sum(-1))
    order = np.lexsort((np.broadcast_to(np.arange(n), (n, n)), d), axis=1)[:, :kk]
    near = np.take_along_axis(d, order, axis=1)
    return np.array([sum(row) for row in near]) / kk  # sequential sum in ascending order


def test_mean_distance_matches_brute_force():
    rng = np.random.default_rng(0)
    for n, k in ((200, 20), (57, 30), (20, 20), (7, 20), (1, 20), (300, 1)):
        pts = rng.standard_normal((n, 3))
        np.testing.assert_allclose(pointcloud.knn_mean_distance(pts, k), brute_mean_distance(pts, k), rtol=1e-13, atol=0)
    assert pointcloud.knn_mean_distance(np.zeros((0, 3)), 20).shape == (0,)


def test_statistical_outlier_edge_cases():
    rng = np.random.default_rng(1)
    assert pointcloud.remove_statistical_outliers(np.zeros((0, 3)), 20, 2.0).shape == (0, 3)
    assert pointcloud.remove_statistical_outliers(np.ones((1, 3)), 20, 2.0).shape == (0, 3)  # avg = 0: dropped
    # n <= k: every point sees the whole cloud
    pts = rng.standard_normal((12, 3))
    _, idx = pointcloud.remove_statistical_outliers(pts, 20, 10.0, return_index=True)
    assert np.array_equal(idx, np.arange(12))
    # a far point is removed at a tight ratio, kept points stay in input order
    pts = np.concatenate([rng.uniform(-1, 1, (300, 3)), [[30.0, 30.0, 30.0]], rng.uniform(-1, 1, (50, 3))])
    kept, idx = pointcloud.remove_statistical_outliers(pts, 20, 2.0, return_index=True)
    assert 300 not in idx and np.all(np.diff(idx) > 0) and np.array_equal(kept, pts[idx])
    # duplicates: a group of >= k identical points has avg = 0 and is dropped, and counts in n but not in the mean
    dup = np.concatenate([rng.uniform(-1, 1, (100, 3)), np.tile([[5.0, 5.0, 5.0]], (25, 1))])
    avg = pointcloud.knn_mean_distance(dup, 20)
    assert np.all(avg[100:] == 0) and np.all(avg[:100] > 0)
    mean = avg[:100].sum() / 125
    std = np.sqrt(((avg[:100] - mean) ** 2).sum() / 124)
    want = (avg > 0) & (avg < mean + 1.5 * std)
    np.testing.assert_array_equal(pointcloud.statistical_outlier_mask(avg, 1.5), want)
    _, idx = pointcloud.remove_statistical_outliers(dup, 20, 1.5, return_index=True)
    np.testing.assert_array_equal(idx, np.flatnonzero(want))


def test_normals_of_planes_and_spheres():
    rng = np.random.default_rng(2)
    uv = rng.uniform(-1, 1, (400, 2))
    n = np.array([1.0, -2.0, 0.5]) / np.linalg.norm([1.0, -2.0, 0.5])
    a = np.cross(n, [0, 0, 1.0])
    a /= np.linalg.norm(a)
    b = np.cross(n, a)
    plane = uv[:, :1] * a + uv[:, 1:] * b + 0.3
    got = pointcloud.estimate_normals(plane, 30)
    np.testing.assert_allclose(np.abs(got @ n), 1.0, atol=1e-9)
    d = rng.standard_normal((3000, 3))
    sphere = d / np.linalg.norm(d, axis=1, keepdims=True) * 2.0 + np.array([1.0, 0, -1])
    got = pointcloud.estimate_normals(sphere, 30)
    radial = (sphere - np.array([1.0, 0, -1])) / 2.0
    assert np.abs(np.sum(got * radial, axis=1)).min() > 0.99
    np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-12)
    # fewer than 3 neighbours, and a zero covariance, give (0, 0, 1)
    for pts in (np.array([[0.0, 0, 0]]), np.array([[0.0, 0, 0], [1, 1, 1]]), np.ones((5, 3))):
        np.testing.assert_array_equal(pointcloud.estimate_normals(pts, 30), np.tile([0.0, 0, 1], (len(pts), 1)))


def test_reorientation_flips_normals_facing_the_view_direction():
    rng = np.random.default_rng(3)
    uv = rng.uniform(-1, 1, (200, 2))
    plane = np.stack([uv[:, 0], uv[:, 1], np.zeros(200)], axis=1)
    view = np.tile(np.array([0.1, 0.2, -1.0], dtype=np.float32), (200, 1))
    view[::2] *= -1
    got = pointcloud.estimate_normals(plane, 30, view_dirs=view)
    assert np.all(np.sum(got * view, axis=1) <= 0)


def test_write_ply_normals_layout(tmp_path):
    rng = np.random.default_rng(4)
    pts, nrm, col = rng.standard_normal((9, 3)), rng.standard_normal((9, 3)), rng.uniform(0, 1, (9, 3))
    path = tmp_path / "point_cloud.ply"
    write_ply(path, pts, col, normals=nrm)
    raw = path.read_bytes()
    head, body = raw.split(b"end_header\n", 1)
    props = [line.split()[-1] for line in head.decode().splitlines() if line.startswith("property")]
    assert props == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    rec = np.frombuffer(body, dtype=[("p", "<f8", 3), ("n", "<f8", 3), ("c", "u1", 3)])
    assert np.array_equal(rec["p"], pts) and np.array_equal(rec["n"], nrm)
    assert np.array_equal(rec["c"], (np.clip(col * 255, 0, 255)).astype(np.uint8))
    p, c = read_ply(path)
    assert np.array_equal(p, pts) and c.shape == (9, 3)
    # without normals the bytes are those of the plain writer
    write_ply(tmp_path / "a.ply", pts, col)
    write_ply(tmp_path / "b.ply", pts, col, normals=None)
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()
    assert b"nx" not in (tmp_path / "a.ply").read_bytes().split(b"end_header")[0]


def test_pointcloud_subparser_defaults_equal_the_dataclass():
    import argparse

    ap = argparse.ArgumentParser()
    p = exporter.add_pointcloud_parser(ap.add_subparsers(dest="command"))
    a = p.parse_args(["--load-config", "c.yml", "--output-dir", "out"])
    for f in dataclasses.fields(exporter.ExportPointCloud):
        if f.name in ("load_config", "output_dir"):
            continue
        got = getattr(a, f.name)
        assert (tuple(got) if isinstance(got, list) else got) == f.default, f.name
    d = exporter.ExportPointCloud(load_config=None, output_dir=Path("."))
    assert (d.num_points, d.remove_outliers, d.reorient_normals, d.normal_method, d.normal_output_name, d.depth_output_name,
            d.rgb_output_name, d.use_bounding_box, d.bounding_box_min, d.bounding_box_max, d.num_rays_per_batch, d.std_ratio) == (
        1000000, True, True, "model_output", "normals", "depth", "rgb", True, (-1, -1, -1), (1, 1, 1), 32768, 10.0)
    a = p.parse_args(["--load-config", "c.yml", "--output-dir", "o", "--normal-method", "open3d", "--num-points", "5", "--remove-outliers",
                      "false", "--std-ratio", "2.5", "--bounding-box-min", "-2", "-2", "-2"])
    assert (a.normal_method, a.num_points, a.remove_outliers, a.std_ratio, a.bounding_box_min) == ("open3d", 5, False, 2.5, [-2.0, -2.0, -2.0])
    with pytest.raises(SystemExit):
        p.parse_args(["--load-config", "c.yml", "--output-dir", "o", "--normal-method", "pca"])


def test_pointcloud_ops_refuse_cpu_tensors():
    pts = torch.zeros(4, 3, dtype=torch.float64)
    f = torch.zeros(4, 3)
    calls = (lambda: ops.knn_mean_distance(pts, 2), lambda: ops.estimate_normals(pts, 3),
             lambda: ops.backproject_select(f, f, f[:, 0], f, f[:, 0], None))
    for call in calls:
        with pytest.raises(L.FruitNerfNativeError, match="no CPU fallback"):
            call()


def test_new_kernels_compile_for_sm_90a():
    lib = _build.build()
    assert "arch=compute_90a,code=sm_90a" in _build.NVCC_FLAGS and "fnr_cluster.cu" in _build.SOURCES
    cuobjdump = Path(_build._nvcc()).with_name("cuobjdump")
    if cuobjdump.exists():
        out = subprocess.run([str(cuobjdump), "--list-elf", str(lib)], capture_output=True, text=True)
        assert out.returncode == 0 and "sm_90a" in out.stdout
    h = L.load()
    for sym in ("fnr_knn_mean_distance", "fnr_estimate_normals", "fnr_backproject_select"):
        assert getattr(h, sym) is not None
