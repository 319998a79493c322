"""Stage 3 of the fruit count (clustering.py's numpy / scipy reference: alpha shapes, scaled ICP, Ward sub-centres,
Hausdorff distances, the split decision and the ground-truth score) against independent results.  CPU only."""
import math

import numpy as np
import pytest
from scipy.spatial import ConvexHull
from scipy.spatial.distance import directed_hausdorff
from scipy.spatial.transform import Rotation
from sklearn.cluster import AgglomerativeClustering

from fruitnerf_b200 import clustering as cl
from fruitnerf_b200.synthetic import sphere_template, touching_fruit_cloud

REAL_TREE = dict(eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                 remove_outliers_radius=0.015)  # clustering/config_real.py


def test_alpha_volume_tends_to_the_convex_hull():
    pts = np.random.default_rng(0).uniform(-1, 1, (400, 3))
    vol = cl.alpha_shape(pts, (1e-9,))[0][0]
    assert vol == pytest.approx(ConvexHull(pts).volume, rel=1e-12)


def test_alpha_volume_of_a_dense_ball():
    rng = np.random.default_rng(1)
    r = 0.035
    d = rng.standard_normal((30000, 3))
    pts = d / np.linalg.norm(d, axis=1, keepdims=True) * (r * rng.uniform(0, 1, (30000, 1)) ** (1 / 3))
    vol = cl.alpha_shape(pts, (cl.ALPHA_VOLUME,))[0][0]
    assert vol == pytest.approx(4 / 3 * math.pi * r**3, rel=0.03)


def test_single_tetrahedron_boundary_is_its_four_faces():
    pts = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    vols, tris, sample = cl.alpha_shape(pts, (0.1,), num_samples=50)
    assert vols[0] == pytest.approx(1 / 6)
    assert sorted(map(tuple, tris[0])) == [(0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)]
    assert sample.shape == (50, 3) and bool((sample >= -1e-12).all()) and bool((sample.sum(axis=1) <= 1 + 1e-12).all())
    on_face = np.isclose(sample, 0).any(axis=1) | np.isclose(sample.sum(axis=1), 1)
    assert bool(on_face.all())
    # alpha too large for the one tetrahedron: nothing kept, no boundary, no sample
    vols, tris, sample = cl.alpha_shape(pts, (10.0,))
    assert vols[0] == 0 and tris[0].shape == (0, 3) and sample is None


def test_degenerate_groups_have_no_volume():
    assert cl.alpha_shape(np.zeros((3, 3)))[2] is None
    flat = np.random.default_rng(2).uniform(0, 1, (50, 3)) * [1, 1, 0]
    vols, tris, sample = cl.alpha_shape(flat)
    assert (vols == 0).all() and sample is None


def test_circumradii_match_brute_force():
    rng = np.random.default_rng(3)
    pts = rng.uniform(-1, 1, (40, 3))
    tets = np.stack([rng.choice(40, 4, replace=False) for _ in range(100)])
    r, vol = cl.tetra_circumradii(pts, tets)
    for t, rr, vv in zip(tets, r, vol):
        a, rest = pts[t[0]], pts[t[1:]]
        centre = np.linalg.solve(2 * (rest - a), (rest * rest).sum(1) - a @ a)
        assert rr == pytest.approx(np.linalg.norm(centre - a), rel=1e-9)
        assert vv == pytest.approx(abs(np.linalg.det(rest - a)) / 6, rel=1e-9)


def test_surface_sample_is_a_pure_function_of_seed_and_group():
    pts = touching_fruit_cloud(seed=5, singles=1, pairs=0, triples=0, fragments=0)[0]
    s1 = cl.alpha_shape(pts, seed=3, group=7)[2]
    assert np.array_equal(s1, cl.alpha_shape(pts, seed=3, group=7)[2])
    assert not np.array_equal(s1, cl.alpha_shape(pts, seed=3, group=8)[2])
    assert s1.shape == (cl.SURFACE_SAMPLES, 3)


def _asymmetric_cloud(seed=4, n=400):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, (n, 3)) * [0.05, 0.03, 0.02]


@pytest.mark.parametrize("scale", [0.8, 1.0, 1.2])
def test_icp_recovers_a_similarity_transform(scale):
    src = _asymmetric_cloud()
    truth = np.eye(4)
    truth[:3, :3] = scale * Rotation.from_euler("xyz", [20, -35, 50], degrees=True).as_matrix()
    truth[:3, 3] = [0.3, -0.2, 1.1]
    tgt = cl.transform_points(src, truth)
    init = np.eye(4)
    init[:3, :3] = Rotation.from_euler("z", 0.3, degrees=True).as_matrix() @ truth[:3, :3]
    init[:3, 3] = truth[:3, 3] + [4e-4, -3e-4, 2e-4]
    T, fitness, rmse, it = cl.icp_scaled(src, tgt, init)
    np.testing.assert_allclose(T, truth, rtol=0, atol=1e-9)
    assert fitness == 1.0 and rmse < 1e-9 and 1 <= it < 50


def test_icp_without_correspondences_is_the_identity_update():
    src = _asymmetric_cloud()
    init = np.eye(4)
    init[:3, 3] = [5.0, 0, 0]
    T, fitness, rmse, it = cl.icp_scaled(src, src, init)
    assert np.array_equal(T, init) and fitness == 0 and rmse == 0 and it == 1


def _blobs(seed, n=240):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-1, 1, (6, 3))
    return np.concatenate([c + 0.15 * rng.standard_normal((n // 6, 3)) for c in centres])[rng.permutation(n)]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ward_cut_centres_match_sklearn(seed):
    pts = _blobs(seed)
    got = cl.ward_cut_centres(pts)
    for k in range(2, 7):
        labels = AgglomerativeClustering(n_clusters=k, linkage="ward").fit_predict(pts)
        want = np.stack([pts[labels == lab].mean(axis=0) for lab in np.unique(labels)])
        mine = got[cl.CUT_OFFSETS[k - 2]:cl.CUT_OFFSETS[k - 1]]
        np.testing.assert_allclose(np.array(sorted(map(tuple, mine))), np.array(sorted(map(tuple, want))), rtol=0, atol=1e-12)
        # ordered by each sub-cluster's smallest point index
        first = [int(np.flatnonzero(labels == labels[np.argmin(np.linalg.norm(pts - c, axis=1))])[0]) for c in mine]
        assert first == sorted(first)


def test_ward_cut_of_tiny_segments_leaves_missing_cuts_nan():
    got = cl.ward_cut_centres(np.array([[0.0, 0, 0], [1, 0, 0], [5, 0, 0]]))
    np.testing.assert_array_equal(got[0:2], [[0.5, 0, 0], [5, 0, 0]])
    np.testing.assert_array_equal(got[2:5], [[0, 0, 0], [1, 0, 0], [5, 0, 0]])
    assert np.isnan(got[5:]).all()


def test_hausdorff_matches_scipy():
    rng = np.random.default_rng(6)
    a, b = rng.uniform(-1, 1, (700, 3)), rng.uniform(-1, 1, (1300, 3)) + 0.2
    assert cl.hausdorff(a, b) == max(directed_hausdorff(a, b)[0], directed_hausdorff(b, a)[0])
    with pytest.raises(ValueError):
        cl.hausdorff(a, np.zeros((0, 3)))


def test_evaluate_count_is_greedy_in_centre_order():
    gt = np.array([[0.0, 0, 0], [0.25, 0, 0]])
    c1, c2 = [0.13, 0, 0], [0.27, 0, 0]  # c1 takes the far ground truth first, leaving c2 unmatched
    r = cl.evaluate_count(np.array([c1, c2]), gt)
    assert (r["TP"], r["FP"], r["FN"]) == (1, 1, 1)
    assert r["precision"] == 0.5 and r["recall"] == 0.5 and r["F1"] == 0.5
    r = cl.evaluate_count(np.array([c2, c1]), gt)
    assert (r["TP"], r["FP"], r["FN"]) == (2, 0, 0) and r["F1"] == 1.0


def test_evaluate_count_boundary_and_empty_inputs():
    gt = np.zeros((1, 3))
    assert cl.evaluate_count(np.array([[0.5, 0, 0]]), gt, max_distance=0.5)["TP"] == 0  # strictly closer
    assert cl.evaluate_count(np.array([[0.149, 0, 0]]), gt)["TP"] == 1
    assert cl.evaluate_count(np.array([[0.151, 0, 0]]), gt)["TP"] == 0
    r = cl.evaluate_count(np.zeros((0, 3)), gt)
    assert (r["TP"], r["FP"], r["FN"], r["precision"], r["recall"], r["F1"]) == (0, 0, 1, 0.0, 0.0, 0.0)
    r = cl.evaluate_count(np.zeros((2, 3)), np.zeros((0, 3)))
    assert (r["TP"], r["FP"], r["FN"], r["F1"]) == (0, 2, 0, 0.0)
    r = cl.evaluate_count(np.zeros((0, 3)), np.zeros((0, 3)))
    assert (r["TP"], r["FP"], r["FN"], r["precision"], r["recall"], r["F1"]) == (0, 0, 0, 0.0, 0.0, 0.0)


def test_count_fruits_splits_touching_fruit_and_prunes_fragments():
    pts, gt = touching_fruit_cloud(seed=0)
    base = cl.count_fruits(pts, **REAL_TREE)
    assert set(base) == {"count", "count_before_merge", "centers", "num_points"}
    res = cl.count_fruits(pts, **REAL_TREE, template=sphere_template(0.035, 1000))
    assert res["count"] == len(gt) == res["centers"].shape[0]
    assert res["count_after_merge"] == base["count"] and res["count_before_merge"] == base["count_before_merge"]
    assert (res["num_split_extra"], res["num_pruned"]) == (3 * 1 + 2 * 2, 2)
    score = cl.evaluate_count(res["centers"], gt)
    assert (score["TP"], score["FP"], score["FN"]) == (len(gt), 0, 0)


def test_load_template_scales_then_centres(tmp_path):
    from fruitnerf_b200.export.exporter_utils import write_ply

    t = sphere_template(0.05, 500) + [1.0, 2.0, 3.0]
    write_ply(tmp_path / "t.ply", t, np.ones_like(t))
    got = cl.load_template(tmp_path / "t.ply", 0.7)
    np.testing.assert_allclose(got, t * 0.7 - (t * 0.7).mean(axis=0), atol=1e-15)


def test_count_cli_parses_the_stage3_options():
    from fruitnerf_b200.scripts import count as count_cli

    a = count_cli.parse_args(["--pcd", "c.ply"])
    assert (a.template, a.template_size, a.gt_centers) == (None, 1.0, None)
    a = count_cli.parse_args(["--pcd", "c.ply", "--template", "apple.ply", "--template-size", "0.7", "--gt-centers", "gt.npy"])
    assert (a.template, a.template_size, a.gt_centers) == ("apple.ply", 0.7, "gt.npy")
