"""Host side of fruit counting: PLY reading, the count CLI's arguments, and the device wrappers' refusal of CPU tensors
(no GPU needed)."""
import numpy as np
import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200.export.exporter_utils import read_ply, write_ply
from fruitnerf_b200.scripts import count as count_cli


def test_read_ply_round_trips_write_ply(tmp_path):
    rng = np.random.default_rng(3)
    pts = rng.standard_normal((257, 3))
    col = rng.uniform(0, 1, (257, 3))
    path = tmp_path / "cloud.ply"
    write_ply(path, pts, col)
    p, c = read_ply(path)
    assert p.dtype == np.float64 and np.array_equal(p, pts)
    assert np.array_equal(np.round(c * 255).astype(np.uint8), np.clip(col * 255, 0, 255).astype(np.uint8))
    write_ply(path, np.zeros((0, 3)), np.zeros((0, 3)))
    p, c = read_ply(path)
    assert p.shape == (0, 3) and c.shape == (0, 3)


def test_read_ply_reads_open3d_style_float_cloud_with_extra_properties(tmp_path):
    n = 5
    rec = np.zeros(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                             ("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1"), ("q", "<f8")])
    rec["x"], rec["y"], rec["z"] = np.arange(n), 2 * np.arange(n), -np.arange(n) / 4
    rec["nx"], rec["red"], rec["green"], rec["blue"], rec["alpha"], rec["q"] = 7, 255, 0, 51, 9, 1e300
    header = ("ply\nformat binary_little_endian 1.0\ncomment Created by Open3D\nelement vertex 5\n"
              "property float x\nproperty float y\nproperty float z\nproperty float nx\nproperty float ny\nproperty float nz\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\nproperty double q\n"
              "element face 0\nproperty list uchar int vertex_indices\nend_header\n")
    path = tmp_path / "o3d.ply"
    path.write_bytes(header.encode("ascii") + rec.tobytes())
    with pytest.raises(ValueError, match="list property"):
        read_ply(path)
    header = header.replace("element face 0\nproperty list uchar int vertex_indices\n", "")
    path.write_bytes(header.encode("ascii") + rec.tobytes())
    p, c = read_ply(path)
    assert np.array_equal(p, np.stack([np.arange(n), 2 * np.arange(n), -np.arange(n) / 4], axis=1).astype(np.float64))
    assert np.array_equal(c, np.tile([1.0, 0.0, 0.2], (n, 1)))
    path.write_bytes(header.replace("binary_little_endian", "ascii").encode("ascii"))
    with pytest.raises(ValueError, match="binary_little_endian"):
        read_ply(path)


def test_count_cli_arguments():
    a = count_cli.parse_args(["--pcd", "x.ply"])
    # the reference's real-tree parameters (clustering/config_real.py)
    assert (a.eps, a.min_samples, a.remove_outliers_nb_points, a.remove_outliers_radius, a.down_sample, a.cluster_merge_distance) == (
        0.02, 100, 120, 0.015, 0.001, 0.04)
    a = count_cli.parse_args(["--pcd", "y.ply", "--eps", "0.5", "--min-samples", "3", "--remove-outliers-nb-points", "0",
                              "--remove-outliers-radius", "0.1", "--down-sample", "0", "--cluster-merge-distance", "0.25", "--json",
                              "out/c.json"])
    assert (a.pcd, a.eps, a.min_samples, a.remove_outliers_nb_points, a.remove_outliers_radius, a.down_sample,
            a.cluster_merge_distance, a.json) == ("y.ply", 0.5, 3, 0, 0.1, 0.0, 0.25, "out/c.json")
    with pytest.raises(SystemExit):
        count_cli.parse_args([])


def test_count_cli_fails_without_a_gpu(tmp_path, monkeypatch):
    path = tmp_path / "c.ply"
    write_ply(path, np.zeros((3, 3)), np.zeros((3, 3)))
    with pytest.raises(ValueError, match="no CPU fallback"):  # a CPU device is refused whether or not a GPU exists
        count_cli.main(["--pcd", str(path), "--device", "cpu"])
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        count_cli.main(["--pcd", str(path)])


def test_cluster_ops_refuse_cpu_tensors():
    pts = torch.zeros(4, 3, dtype=torch.float64)
    calls = (lambda: ops.radius_count(pts, 0.1, 2), lambda: ops.voxel_down_sample(pts, 0.1), lambda: ops.dbscan(pts, 0.1, 2),
             lambda: ops.cluster_sums(pts, torch.zeros(4, dtype=torch.int32), 1))
    for call in calls:
        with pytest.raises(L.FruitNerfNativeError, match="no CPU fallback"):
            call()
