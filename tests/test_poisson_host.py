"""The `poisson` mesh export without a GPU: the numpy / scipy restatement in poisson.py (splat, assembled operator, solve,
trim), the CLI's options and refusals, and the C-ABI refusal codes (no compute calls)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

from fruitnerf_b200 import poisson as P


def sphere_cloud(n, radius=0.3, centre=(0.5, 0.5, 0.5), seed=0):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return np.asarray(centre) + radius * v, v.astype(np.float32)


def test_cube_of():
    pts = np.array([[0.0, 0.0, 0.0], [2.0, 1.0, 0.5]])
    origin, side = P.cube_of(pts)
    assert side == pytest.approx(2.2)
    np.testing.assert_allclose(origin, [1.0 - 1.1, 0.5 - 1.1, 0.25 - 1.1])
    with pytest.raises(ValueError):
        P.cube_of(np.zeros((3, 3)))
    with pytest.raises(ValueError):
        P.cube_of(np.array([[0.0, np.nan, 0.0], [1.0, 1.0, 1.0]]))


def test_splat_equals_brute_force():
    rng = np.random.default_rng(0)
    n, depth = 400, 3
    pts = rng.uniform(-1, 1, (n, 3))
    nrm = rng.standard_normal((n, 3)).astype(np.float32)
    col = rng.uniform(size=(n, 3)).astype(np.float32)
    fr = rng.uniform(size=n).astype(np.float32)
    origin, side = P.cube_of(pts)
    got = P.restated_splat(pts, nrm, depth, origin, side, col, fr)
    R, Nn = 2 ** depth, 2 ** depth + 1
    rho, nsum, csum, fsum = np.zeros(Nn ** 3), np.zeros((Nn ** 3, 3)), np.zeros((Nn ** 3, 3)), np.zeros(Nn ** 3)
    cells = set()
    for p in range(n):  # per point, per node: phi = prod max(0, 1 - |q - I|)
        q = (pts[p] - origin) / (side / R)
        cells.add(tuple(np.floor(q).astype(int)))
        for i in range(Nn):
            for j in range(Nn):
                for k in range(Nn):
                    phi = np.prod(np.maximum(0.0, 1.0 - np.abs(q - [i, j, k])))
                    if phi > 0:
                        node = (i * Nn + j) * Nn + k
                        rho[node] += phi
                        nsum[node] += phi * nrm[p]
                        csum[node] += phi * col[p]
                        fsum[node] += phi * fr[p]
    h = 1.0 / R
    a = h * h * len(cells) / n
    assert got["occupied"] == len(cells) and got["area"] == pytest.approx(a, rel=1e-15)
    np.testing.assert_allclose(got["density"], rho, rtol=1e-6, atol=1e-12)
    np.testing.assert_allclose(got["normal_field"], a / h ** 3 * nsum, rtol=1e-5, atol=1e-6 * np.abs(a / h ** 3 * nsum).max())
    safe = np.where(rho > 0, rho, 1)
    np.testing.assert_allclose(got["colors"], np.where(rho[:, None] > 0, csum / safe[:, None], 0), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got["fruit"], np.where(rho > 0, fsum / safe, 0), rtol=1e-5, atol=1e-6)


def test_operator_is_symmetric_positive_definite():
    pts, nrm = sphere_cloud(2000)
    origin, side = P.cube_of(pts)
    sp = P.restated_splat(pts, nrm, 3, origin, side)
    A = P.operator(pts, 3, origin, side, sp["area"])
    assert A.shape == (9 ** 3, 9 ** 3)
    D = A.toarray()
    np.testing.assert_array_equal(D, D.T)
    assert np.linalg.eigvalsh(D).min() > 0
    K = P.assemble(3)["K"].toarray()
    np.testing.assert_allclose(K @ np.ones(len(K)), 0, atol=1e-12)  # Neumann: constants are in K's null space
    # the gradient-mass matrices integrate to the boundary flux: sum_ij G_ij = 0 per axis (phi sums to one)
    for a in range(3):
        assert abs(P.assemble(3)[f"G{a}"].sum()) < 1e-12


def test_restated_solve_gives_a_sphere_at_33():
    r = 0.3
    pts, nrm = sphere_cloud(20000, r)
    col = np.tile(np.float32([0.2, 0.4, 0.6]), (len(pts), 1))
    out = P.reconstruct(pts, nrm, colors=col, depth=5)
    vox = out["side"] / 32
    v = out["mesh"]["vertices"].astype(np.float64)
    d = np.abs(np.linalg.norm(v - 0.5, axis=1) - r) / vox
    assert len(v) > 1000 and d.max() <= 0.5
    assert (np.sum(out["mesh"]["normals"] * (v - 0.5), axis=1) > 0).all()  # outward
    np.testing.assert_allclose(out["mesh"]["colors"], np.broadcast_to([0.2, 0.4, 0.6], v.shape), atol=1e-6)
    assert len(out["full"]["vertices"]) > len(v)


def test_trim_matches_quantile_and_open3d_rule():
    rng = np.random.default_rng(0)
    nv = 50
    mesh = {"vertices": rng.standard_normal((nv, 3)).astype(np.float32), "normals": rng.standard_normal((nv, 3)).astype(np.float32),
            "colors": rng.uniform(size=(nv, 3)).astype(np.float32), "fruit": rng.uniform(size=nv).astype(np.float32),
            "faces": rng.integers(0, nv, (80, 3))}
    density = rng.uniform(size=nv).astype(np.float32)
    out = P.trim_by_density(mesh, density, 0.1)
    q = np.quantile(density, 0.1)  # numpy's linear rule
    drop = density < q
    assert drop.sum() == 5
    keep_idx = np.flatnonzero(~drop)
    np.testing.assert_array_equal(out["vertices"], mesh["vertices"][keep_idx])
    np.testing.assert_array_equal(out["fruit"], mesh["fruit"][keep_idx])
    # open3d remove_vertices_by_mask: drop every face that touches a removed vertex, renumber the rest
    want = [[int(np.searchsorted(keep_idx, v)) for v in f] for f in mesh["faces"] if not drop[f].any()]
    np.testing.assert_array_equal(out["faces"], np.asarray(want, np.int64).reshape(-1, 3))


def test_depth_range():
    for d in (1, 11):
        with pytest.raises(ValueError, match="depth"):
            P.check_depth(d)
    assert P.check_depth(2) == 2 and P.check_depth(10) == 10


# ---- the CLI -------------------------------------------------------------------------------------------------------------
def test_cli_options_mirror_export_poisson_mesh():
    import argparse

    from fruitnerf_b200.scripts.exporter import ExportPoissonMesh, add_poisson_parser, poisson_exporter_from_args

    d = ExportPoissonMesh(load_config=None, output_dir=Path("."))
    assert (d.num_points, d.remove_outliers, d.reorient_normals, d.normal_method, d.save_point_cloud, d.use_bounding_box,
            d.bounding_box_min, d.bounding_box_max, d.num_rays_per_batch, d.std_ratio, d.texture_method, d.depth) == (
        1000000, True, True, "model_output", False, True, (-1, -1, -1), (1, 1, 1), 32768, 10.0, "point_cloud", 9)
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="command")
    add_poisson_parser(sub)
    a = ap.parse_args(["poisson", "--load-config", "c.yml", "--output-dir", "o"])
    e = poisson_exporter_from_args(a)
    assert e == ExportPoissonMesh(load_config=Path("c.yml"), output_dir=Path("o"))
    a = ap.parse_args(["poisson", "--load-config", "c.yml", "--output-dir", "o", "--depth", "7", "--num-points", "5000",
                       "--remove-outliers", "false", "--save-point-cloud", "true", "--normal-method", "open3d", "--std-ratio", "3"])
    e = poisson_exporter_from_args(a)
    assert (e.depth, e.num_points, e.remove_outliers, e.save_point_cloud, e.normal_method, e.std_ratio) == (7, 5000, False, True, "open3d", 3.0)


@pytest.mark.parametrize("extra,msg", [
    (["--texture-method", "nerf"], "xatlas"),
    (["--depth", "11"], "depth"),
    (["--depth", "1"], "depth"),
    (["--bounding-box-min", "0", "0", "0", "--bounding-box-max", "1", "-1", "1"], "Bounding box"),
])
def test_cli_refusals(tmp_path, capsys, extra, msg):
    from fruitnerf_b200.scripts.exporter import entrypoint

    with pytest.raises(SystemExit) as e:
        entrypoint(["poisson", "--load-config", str(tmp_path / "missing.yml"), "--output-dir", str(tmp_path / "o"), *extra])
    assert e.value.code == 2
    assert msg in capsys.readouterr().err
    assert not (tmp_path / "o").exists()


# ---- the C ABI -------------------------------------------------------------------------------------------------------------
def test_cabi_refusals(native_lib):
    lib = native_lib
    n = C.c_size_t(0)
    for num, depth in ((0, 5), (-1, 5), (1000, 1), (1000, 11), (2 ** 31, 5)):
        assert lib.fnr_poisson_scratch_bytes(num, depth, C.byref(n)) == -1, (num, depth)
    assert lib.fnr_poisson_scratch_bytes(1000, 5, None) == -1
    origin = (C.c_double * 3)(0.0, 0.0, 0.0)
    fake = C.c_void_p(16)  # never dereferenced: every call below is refused before any device work
    assert lib.fnr_poisson_splat(None, fake, None, None, 1000, 5, origin, 1.0, fake, 1 << 30, fake, fake, None, None, fake, None) == -1
    assert b"fnr_poisson_splat" in lib.fnr_last_error()
    assert lib.fnr_poisson_splat(fake, fake, None, None, 1000, 11, origin, 1.0, fake, 1 << 30, fake, fake, None, None, fake, None) == -1
    assert lib.fnr_poisson_splat(fake, fake, None, None, 1000, 5, origin, 0.0, fake, 1 << 30, fake, fake, None, None, fake, None) == -1
    nan = (C.c_double * 3)(0.0, float("nan"), 0.0)
    assert lib.fnr_poisson_splat(fake, fake, None, None, 1000, 5, nan, 1.0, fake, 1 << 30, fake, fake, None, None, fake, None) == -1
    assert lib.fnr_poisson_splat(fake, fake, fake, None, 1000, 5, origin, 1.0, fake, 1 << 30, fake, fake, None, None, fake, None) == -1
    assert lib.fnr_poisson_apply(1000, 5, 2.0, fake, 1 << 30, None, fake, None) == -1
    assert lib.fnr_poisson_apply(1000, 5, -1.0, fake, 1 << 30, fake, fake, None) == -1
    it = (C.c_int64 * 2)()
    res = C.c_double(0.0)
    assert lib.fnr_poisson_solve(fake, fake, None, None, 0, 5, origin, 1.0, 2.0, 100, 1e-5, fake, 1 << 30, fake, fake, None, None, it,
                                 C.byref(res), None) == -1
    assert lib.fnr_poisson_solve(fake, fake, None, None, 1000, 5, origin, 1.0, 2.0, -1, 1e-5, fake, 1 << 30, fake, fake, None, None, it,
                                 C.byref(res), None) == -1
    assert lib.fnr_poisson_solve(fake, fake, None, None, 1000, 5, origin, 1.0, 2.0, 100, 1e-5, fake, 1 << 30, fake, fake, None, None, None,
                                 C.byref(res), None) == -1
    assert lib.fnr_poisson_sample(None, 1000, 5, origin, 1.0, fake, fake, None) == -1
    assert lib.fnr_poisson_sample(fake, 1000, 12, origin, 1.0, fake, fake, None) == -1
