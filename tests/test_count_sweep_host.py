"""Host side of the count sweeps: ground truth in the reference's formats, the sweep spec (checks, expansion, output
shape), the count CLI's --gt-cluster, and the numpy count_sweep (no GPU needed)."""
import json

import numpy as np
import pytest
import torch

from fruitnerf_b200 import clustering
from fruitnerf_b200.export.exporter_utils import read_line_set_points, read_ply, write_ply
from fruitnerf_b200.scripts import count as count_cli
from fruitnerf_b200.scripts import count_sweep as sweep_cli
from fruitnerf_b200.synthetic import sphere_template

FUJI = {  # run_clustering_sweep.py's Fuji_sam_sweep, paths replaced
    "path": "cloud.ply", "remove_outliers_nb_points": [50, 60, 75], "remove_outliers_radius": 0.025, "down_sample": 0.001,
    "eps": [0.015, 0.02], "cluster_merge_distance": 0.04, "minimum_size_factor": 0.2, "min_samples": 100,
    "template_path": "template.ply", "apple_template_size": [0.9, 1, 1.1], "gt_cluster": "lineset.ply", "gt_count": 1455,
}


@pytest.fixture
def files(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    write_ply(tmp_path / "cloud.ply", np.zeros((4, 3)), np.zeros((4, 3)))
    write_ply(tmp_path / "template.ply", sphere_template(), np.zeros((1000, 3)))
    write_line_set(tmp_path / "lineset.ply", np.array([[0.0, 0.0, 0.0]]), "ascii")
    return tmp_path


BOX = np.array([[x, y, z] for x in (-1.0, 1.0) for y in (-2.0, 2.0) for z in (-0.5, 0.5)])


def write_line_set(path, centres, fmt, extra_vertices=0, vertex_type="double"):
    """An open3d-style line set of axis-aligned boxes: vertex x/y/z, then an edge element (and an edge colour)."""
    verts = np.concatenate([(centres[:, None, :] + BOX[None]).reshape(-1, 3), np.ones((extra_vertices, 3))])
    edges = np.array([(8 * b + i, 8 * b + j) for b in range(len(centres)) for i, j in ((0, 1), (1, 3), (3, 2), (2, 0))], dtype="<i4")
    header = (f"ply\nformat {fmt} 1.0\ncomment Created by Open3D\nelement vertex {len(verts)}\nproperty {vertex_type} x\n"
              f"property {vertex_type} y\nproperty {vertex_type} z\nelement edge {len(edges)}\nproperty int vertex1\nproperty int vertex2\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n").encode("ascii")
    if fmt == "ascii":
        body = "".join(f"{float(v[0])!r} {float(v[1])!r} {float(v[2])!r}\n" for v in verts) + "".join(f"{a} {b} 255 0 0\n" for a, b in edges)
        path.write_bytes(header + body.encode("ascii"))
    else:
        vt = "<f8" if vertex_type == "double" else "<f4"
        rec = np.zeros(len(edges), dtype=[("a", "<i4"), ("b", "<i4"), ("r", "u1"), ("g", "u1"), ("bl", "u1")])
        rec["a"], rec["b"], rec["r"] = edges[:, 0], edges[:, 1], 255
        path.write_bytes(header + verts.astype(vt).tobytes() + rec.tobytes())


@pytest.mark.parametrize("fmt,vertex_type", [("ascii", "double"), ("binary_little_endian", "double"), ("binary_little_endian", "float")])
def test_line_set_ground_truth(tmp_path, fmt, vertex_type):
    centres = np.array([[0.25, 1.5, -3.0], [10.0, 20.0, 30.0], [-0.5, 0.0, 0.125]])
    path = tmp_path / "lineset.ply"
    write_line_set(path, centres, fmt, vertex_type=vertex_type)
    assert read_line_set_points(path).shape == (24, 3)
    np.testing.assert_array_equal(clustering.load_gt_centres(path), centres)
    with pytest.raises(ValueError, match="not a point cloud|only binary_little_endian"):  # read_ply keeps refusing line sets
        read_ply(path)
    write_line_set(path, centres, fmt, extra_vertices=3, vertex_type=vertex_type)
    with pytest.raises(ValueError, match="8-corner boxes"):
        clustering.load_gt_centres(path)


def test_obj_ground_truth(tmp_path):
    path = tmp_path / "fruits.obj"
    path.write_text("# three fruit\nmtllib fruits.mtl\no apple_0\nv 0 0 0\nv 2 0 0\nv 1 3 0\nvn 0 0 1\nf 1 2 3\n"
                    "o apple_1\nv 10 10 10\nv 12 10 10\nusemtl red\nf 4 5 4\no apple_2\nv -1 -1 -1\n")
    np.testing.assert_allclose(clustering.load_gt_centres(path), [[1, 1, 0], [11, 10, 10], [-1, -1, -1]], rtol=0, atol=0)
    path.write_text("v 0 0 0\nv 1 1 1\nf 1 2 1\n")
    with pytest.raises(ValueError, match="no 'o' line"):
        clustering.load_gt_centres(path)
    path.write_text("v 0 0 0\no apple_0\nv 1 1 1\n")
    with pytest.raises(ValueError, match="before the first 'o'"):
        clustering.load_gt_centres(path)
    np.save(tmp_path / "c.npy", np.arange(6.0))
    np.testing.assert_array_equal(clustering.load_gt_centres(tmp_path / "c.npy"), [[0, 1, 2], [3, 4, 5]])
    with pytest.raises(ValueError, match="must be"):
        clustering.load_gt_centres(tmp_path / "c.txt")


def test_count_cli_gt_cluster():
    a = count_cli.parse_args(["--pcd", "x.ply", "--gt-cluster", "fruits.obj"])
    assert (a.gt_cluster, a.gt_centers) == ("fruits.obj", None)
    a = count_cli.parse_args(["--pcd", "x.ply", "--gt-centers", "c.npy"])
    assert (a.gt_cluster, a.gt_centers) == (None, "c.npy")
    with pytest.raises(SystemExit):
        count_cli.parse_args(["--pcd", "x.ply", "--gt-centers", "c.npy", "--gt-cluster", "fruits.obj"])


def test_spec_expansion_order_and_size(files):
    run = sweep_cli.check_run("fuji", FUJI)
    combos = sweep_cli.expand(run)
    assert len(combos) == 18
    keys = [(c["remove_outliers_nb_points"], c["eps"], c["apple_template_size"]) for c in combos]
    # nb outermost, then eps, then the template size, as the reference's nested loops
    assert keys == [(nb, eps, s) for nb in (50, 60, 75) for eps in (0.015, 0.02) for s in (0.9, 1, 1.1)]
    assert all(c["remove_outliers_radius"] == 0.025 and c["min_samples"] == 100 for c in combos)
    assert sweep_cli.swept_keys(run) == ["remove_outliers_nb_points", "eps", "apple_template_size"]
    assert list(sweep_cli.PARAMETERS).index("remove_outliers_nb_points") < list(sweep_cli.PARAMETERS).index("eps") \
        < list(sweep_cli.PARAMETERS).index("apple_template_size")


def test_spec_scalars_make_one_count_and_minimum_size_factor_is_ignored(files):
    scalar = {k: (v[0] if isinstance(v, list) else v) for k, v in FUJI.items()}
    run = sweep_cli.check_run("one", scalar)
    assert len(sweep_cli.expand(run)) == 1 and sweep_cli.swept_keys(run) == []
    other = sweep_cli.check_run("one", {**scalar, "minimum_size_factor": 0.9})
    assert sweep_cli.expand(other) == sweep_cli.expand(run)
    without = {k: v for k, v in scalar.items() if k != "minimum_size_factor"}
    assert sweep_cli.expand(sweep_cli.check_run("one", without)) == sweep_cli.expand(run)


@pytest.mark.parametrize("change,match", [
    ({"colour": 1}, "unknown keys"),
    ({"path": "missing.ply"}, "does not exist"),
    ({"template_path": "missing.ply"}, "does not exist"),
    ({"template_path": ["template.ply", "missing.ply"]}, "does not exist"),
    ({"gt_cluster": "missing.obj"}, "does not exist"),
    ({"eps": [0.02, 0.0]}, "eps"),
    ({"eps": -0.1}, "eps"),
    ({"remove_outliers_radius": 0.0}, "remove_outliers_radius"),
    ({"remove_outliers_radius": [0.02, -0.01]}, "remove_outliers_radius"),
    ({"apple_template_size": 0}, "apple_template_size"),
    ({"min_samples": 0}, "min_samples"),
    ({"eps": []}, "empty list"),
    ({"gt_count": [1, 2]}, "cannot be a list"),
])
def test_spec_refusals(files, change, match):
    with pytest.raises(ValueError, match=match):
        sweep_cli.check_run("bad", {**FUJI, **change})


def test_spec_refused_before_any_count(files, monkeypatch):
    called = []
    monkeypatch.setattr(sweep_cli, "run_sweep", lambda *a: called.append(a))
    (files / "spec.json").write_text(json.dumps({"good": FUJI, "bad": {**FUJI, "eps": 0}}))
    with pytest.raises(SystemExit):
        sweep_cli.main([str(files / "spec.json")])
    assert called == []
    ok = sweep_cli.check_run("none", {**FUJI, "template_path": None, "gt_cluster": None, "remove_outliers_nb_points": 0,
                                      "remove_outliers_radius": 0.0})
    assert ok["template_path"] is None and ok["gt_cluster"] is None


def test_sweep_cli_fails_cleanly_without_a_gpu(files, monkeypatch, capsys):
    (files / "spec.json").write_text(json.dumps({"fuji": FUJI}))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit) as e:
        sweep_cli.main([str(files / "spec.json")])
    assert e.value.code == 2
    assert "no CPU fallback" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        sweep_cli.main([str(files / "spec.json"), "--device", "cpu"])


def test_json_shape_matches_the_reference(files, monkeypatch):
    """{run: {"<i>": {"path", "count", "TP", "gt", "precision", "recall", "F1", "params"}}} with ground truth (FP / FN
    added), {"path", "count", "gt"} without -- what run_clustering_sweep.py writes."""
    centres = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]])

    def fake_sweep(points, configs, templates):
        return [{"count": 2 + i, "centers": np.concatenate([centres, np.full((i, 3), 5.0)])} for i in range(len(configs))]

    monkeypatch.setattr(sweep_cli, "count_sweep", fake_sweep)
    write_line_set(files / "lineset.ply", centres, "binary_little_endian")
    run = sweep_cli.check_run("fuji", FUJI)
    out = sweep_cli.run_sweep("fuji", run, "cpu")
    assert list(out) == [str(i) for i in range(18)]
    e = out["3"]
    assert set(e) == {"path", "count", "TP", "FP", "FN", "gt", "precision", "recall", "F1", "params"}
    assert e["params"] == {"remove_outliers_nb_points": 50, "eps": 0.02, "apple_template_size": 0.9}
    assert (e["count"], e["TP"], e["FP"], e["FN"], e["gt"]) == (5, 2, 3, 0, 1455)
    assert (e["precision"], e["recall"], e["F1"]) == pytest.approx((0.4, 1.0, 2 * 0.4 / 1.4))
    plain = sweep_cli.run_sweep("fuji", sweep_cli.check_run("fuji", {**FUJI, "gt_cluster": None}), "cpu")
    assert plain["0"] == {"path": "cloud.ply", "count": 2, "gt": 1455}
    json.dumps(out)


def test_numpy_count_sweep_is_the_count_fruits_loop():
    rng = np.random.default_rng(7)
    centres = np.array([[0.0, 0.0, 0.0], [0.3, 0.0, 0.0], [0.3665, 0.0, 0.0], [0.0, 0.3, 0.0]])  # two touch
    d = rng.standard_normal((3000, 3))
    pts = centres[rng.integers(0, 4, 3000)] + 0.035 * d / np.linalg.norm(d, axis=1, keepdims=True)
    configs = [dict(eps=eps, min_samples=ms, cluster_merge_distance=0.04, down_sample=0.002, remove_outliers_nb_points=nb,
                    remove_outliers_radius=0.02) for nb in (4, 8) for eps in (0.015, 0.03) for ms in (5,)]
    templates = [sphere_template(0.035, 300) * s for s in (1.0, 0.9, 1.0, 1.1)]
    sweep = clustering.count_sweep(pts, configs, templates)
    for c, t, s in zip(configs, templates, sweep):
        ref = clustering.count_fruits(pts, **c, template=t)
        assert s.keys() == ref.keys()
        for k in ref:
            np.testing.assert_array_equal(s[k], ref[k])
    assert clustering.count_sweep(pts, configs[:1])[0]["count"] == clustering.count_fruits(pts, **configs[0])["count"]
    with pytest.raises(ValueError, match="unknown"):
        clustering.count_sweep(pts, [{**configs[0], "colour": 1}])
    with pytest.raises(ValueError, match="templates"):
        clustering.count_sweep(pts, configs, templates[:1])


def test_radius_chunks():
    assert clustering._radius_chunks([0.4, 0.1, 0.41, 0.2]) == [[0.1, 0.2, 0.4], [0.41]]
    assert [len(c) for c in clustering._radius_chunks([1.0 + i / 100 for i in range(20)])] == [16, 4]
