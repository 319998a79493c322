"""The `poisson` mesh export on the device: fnr_poisson_splat against the numpy restatement in poisson.py (bit for bit),
the operator against scipy, the coarse-to-fine CG solve against spsolve, analytic clouds (sphere, torus, two spheres,
colours and fruit), the traced apple scene, 2^24 points at depth 9, and the CLI end to end on a briefly trained model."""

import numpy as np
import pytest
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

from fruitnerf_b200 import mesh as M
from fruitnerf_b200 import ops
from fruitnerf_b200 import poisson as P

pytestmark = pytest.mark.gpu


def sphere_cloud(n, radius=0.3, centre=(0.1, -0.2, 0.05), seed=0):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return np.asarray(centre) + radius * v, v.astype(np.float32)


def torus_cloud(n, R0=0.3, r0=0.12, seed=0):
    rng = np.random.default_rng(seed)
    u, v = rng.uniform(0, 2 * np.pi, 4 * n), rng.uniform(0, 2 * np.pi, 4 * n)
    keep = rng.uniform(size=4 * n) < (R0 + r0 * np.cos(v)) / (R0 + r0)  # uniform by area
    u, v = u[keep][:n], v[keep][:n]
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    pts = np.stack([(R0 + r0 * np.cos(v)) * np.cos(u), (R0 + r0 * np.cos(v)) * np.sin(u), r0 * np.sin(v)], 1)
    return pts, nrm.astype(np.float32)


def random_cloud(n, seed):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-0.7, 1.3, (n, 3)) * np.array([1.0, 0.6, 0.8])
    nrm = rng.standard_normal((n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return pts, nrm.astype(np.float32), rng.uniform(size=(n, 3)).astype(np.float32), rng.uniform(size=n).astype(np.float32)


def cuda(*arrays, dev):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


def components(faces, nv):
    f = np.asarray(faces)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(nv, nv))
    return connected_components(g, directed=False)[1]


def closed_and_euler(faces):
    """(every edge in exactly two faces, V - E + F) of a face set."""
    f = np.asarray(faces)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    return bool((counts == 2).all()), len(np.unique(f)) - len(counts) + len(f)


def face_components(faces, nv):
    """[(faces of the component)] by decreasing size, over the vertices the faces use."""
    lab = components(faces, nv)[np.asarray(faces)[:, 0]]
    ids, counts = np.unique(lab, return_counts=True)
    return [np.asarray(faces)[lab == i] for i in ids[np.argsort(-counts)]]


# ---- against the restatement -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,depth,n", [(0, 4, 3000), (1, 5, 20000), (2, 6, 1000)])
def test_splat_is_array_equal_to_restatement(native_lib, cuda_device, seed, depth, n):
    pts, nrm, col, fr = random_cloud(n, seed)
    origin, side = P.cube_of(pts)
    ref = P.restated_splat(pts, nrm, depth, origin, side, col, fr)
    dp, dn, dc, df = cuda(pts, nrm, col, fr, dev=cuda_device)
    got = [ops.poisson_splat(dp, dn, depth, origin, side, dc, df) for _ in range(2)]
    for key in ("density", "normal_field", "colors", "fruit", "rhs"):
        np.testing.assert_array_equal(got[0][key].cpu().numpy().reshape(ref[key].shape), ref[key], err_msg=key)
        assert torch.equal(got[0][key].view(torch.int32), got[1][key].view(torch.int32)), key
    assert float(np.abs(ref["rhs"]).max()) > 0
    # the rhs stencil is G v with the assembled gradient-mass matrices
    G = P.assemble(depth)
    v = ref["normal_field"].astype(np.float64)
    b = sum(G[f"G{a}"] @ v[:, a] for a in range(3))
    np.testing.assert_allclose(ref["rhs"], b, rtol=0, atol=1e-6 * np.abs(b).max())


@pytest.mark.parametrize("depth", [3, 5])
def test_operator_matches_scipy(native_lib, cuda_device, depth):
    pts, nrm = sphere_cloud(5000, seed=depth)
    origin, side = P.cube_of(pts)
    ref = P.restated_splat(pts, nrm, depth, origin, side)
    A = P.operator(pts, depth, origin, side, ref["area"])
    assert abs(A - A.T).max() == 0
    dp, dn = cuda(pts, nrm, dev=cuda_device)
    sp = ops.poisson_splat(dp, dn, depth, origin, side)
    rng = np.random.default_rng(depth)
    for x in (rng.standard_normal(A.shape[0]).astype(np.float32), np.linspace(-1, 1, A.shape[0], dtype=np.float32)):
        y = ops.poisson_apply(torch.from_numpy(x).to(cuda_device), len(pts), depth, sp["scratch"]).cpu().numpy().astype(np.float64)
        want = A @ x.astype(np.float64)
        assert np.abs(y - want).max() <= 1e-6 * np.abs(want).max()


@pytest.mark.parametrize("depth,cloud", [(4, "sphere"), (5, "sphere"), (5, "torus")])
def test_solve_matches_spsolve(native_lib, cuda_device, depth, cloud):
    pts, nrm = sphere_cloud(20000, seed=3) if cloud == "sphere" else torus_cloud(20000, seed=3)
    origin, side = P.cube_of(pts)
    ref = P.restated_solve(pts, nrm, depth, origin, side)
    dp, dn = cuda(pts, nrm, dev=cuda_device)
    got = ops.poisson_solve(dp, dn, depth, origin, side, tolerance=1e-6, max_iters=5000)
    chi = got["chi"].cpu().numpy().astype(np.float64)
    b = ref["rhs"].astype(np.float64)
    res = np.linalg.norm(b - ref["operator"] @ chi) / np.linalg.norm(b)
    diff = np.abs(chi - ref["chi"]).max() / np.abs(ref["chi"]).max()
    print(f"\ndepth {depth} {cloud}: {got['iterations']} iterations ({got['total_iterations']} in all), CG residual {got['residual']:.3g}, "
          f"fp64 residual {res:.3g}, max |chi - spsolve| / max |chi| {diff:.3g}")
    assert res <= 1e-5 and diff <= 1e-3
    Nn = 2 ** depth + 1
    vox = side / (Nn - 1)
    verts = []
    for c in (chi.astype(np.float32), ref["chi"].astype(np.float32)):
        iso = P.restated_sample(pts, c, depth, origin, side).astype(np.float64).mean()
        verts.append(M.marching_cubes_numpy((c - np.float32(iso)).reshape(Nn, Nn, Nn), origin.astype(np.float32), np.float32(vox))["vertices"])
    d01 = cKDTree(verts[1]).query(verts[0])[0].max() / vox
    d10 = cKDTree(verts[0]).query(verts[1])[0].max() / vox
    assert max(d01, d10) <= 0.05, (d01, d10)


# ---- analytic clouds --------------------------------------------------------------------------------------------------
def test_sphere_depth7(native_lib, cuda_device):
    r, c = 0.3, np.array([0.1, -0.2, 0.05])
    pts, nrm = sphere_cloud(100000, r, c, seed=7)
    out = P.reconstruct(*cuda(pts, nrm, dev=cuda_device), depth=7)
    vox = out["side"] / 128
    kept = out["mesh"]["vertices"].astype(np.float64)
    dev_r = np.abs(np.linalg.norm(kept - c, axis=1) - r) / vox
    comps = face_components(out["full"]["faces"], len(out["full"]["vertices"]))
    closed, chi = closed_and_euler(comps[0])
    print(f"\nsphere d=7: {out['iterations']} iterations, residual {out['residual']:.3g}, {len(kept)} kept vertices, worst {dev_r.max():.3f} "
          f"voxels, {len(comps)} components")
    assert out["residual"] <= 1e-5
    assert len(kept) > 1000 and dev_r.max() <= 0.5
    assert closed and chi == 2
    # outward normals
    assert (np.sum(out["mesh"]["normals"] * (kept - c), axis=1) > 0).all()


def test_torus_and_two_spheres(native_lib, cuda_device):
    pts, nrm = torus_cloud(100000, seed=1)
    out = P.reconstruct(*cuda(pts, nrm, dev=cuda_device), depth=7)
    comps = face_components(out["full"]["faces"], len(out["full"]["vertices"]))
    closed, chi = closed_and_euler(comps[0])
    assert closed and chi == 0
    a, na = sphere_cloud(50000, 0.2, (-0.35, 0.0, 0.0), seed=2)
    b, nb = sphere_cloud(50000, 0.2, (0.35, 0.0, 0.0), seed=3)
    out = P.reconstruct(*cuda(np.concatenate([a, b]), np.concatenate([na, nb]), dev=cuda_device), depth=7)
    comps = face_components(out["full"]["faces"], len(out["full"]["vertices"]))
    assert len(comps) == 2
    for f in comps:
        assert closed_and_euler(f) == (True, 2)


def test_colours_and_fruit(native_lib, cuda_device, tmp_path):
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply, write_mesh_ply

    c = np.array([0.1, -0.2, 0.05])
    pts, nrm = sphere_cloud(100000, 0.3, c, seed=4)
    colour = np.array([0.25, 0.5, 0.75], np.float32)
    col = np.tile(colour, (len(pts), 1))
    fr = (pts[:, 2] > c[2]).astype(np.float32)
    out = P.reconstruct(*cuda(pts, nrm, col, fr, dev=cuda_device), depth=6)
    m = out["mesh"]
    np.testing.assert_allclose(m["colors"], np.broadcast_to(colour, m["colors"].shape), rtol=0, atol=1e-6)
    fv, fn, fc, ff, fidx = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    vox = out["side"] / 64
    assert len(fidx) > 100
    assert (fv[:, 2] >= c[2] - 1.5 * vox).all()
    write_mesh_ply(tmp_path / "f.ply", fv, fn, fc, fidx)
    v2, _, _, f2 = read_mesh_ply(tmp_path / "f.ply")
    np.testing.assert_array_equal(v2, fv.astype(v2.dtype))
    np.testing.assert_array_equal(f2, fidx)


# ---- the traced apple scene ---------------------------------------------------------------------------------------------
def test_ground_truth_apple_scene(native_lib, cuda_device):
    from fruitnerf_b200 import pointcloud
    from fruitnerf_b200.data.synthetic_scene import camera_rays, make_apple_scene, trace

    from .test_gpu_mesh import fruit_distance, surface_distance

    size = 160  # as test_gpu_mesh.py::test_ground_truth_apple_scene
    train, ev = make_apple_scene(num_images=40, height=size, width=size, noise_std=0.0)
    geom, cams = train.geometry, train.cameras
    pts, col, fruit, view = [], [], [], []
    ys, xs = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    for c2w in torch.cat([train.cameras.camera_to_worlds, ev.cameras.camera_to_worlds]):
        o, d = camera_rays(c2w, cams.fx, cams.fy, cams.cx, cams.cy, ys.reshape(-1), xs.reshape(-1))
        rgb, m, t = trace(geom, o, d)
        p = o + d * torch.where(torch.isfinite(t), t, torch.zeros_like(t))[:, None]
        keep = torch.isfinite(t) & (p.abs() < 1).all(dim=1)
        pts.append(p[keep])
        col.append(rgb[keep])
        fruit.append(m[keep, 0])
        view.append(d[keep])
    pts, col, fruit, view = (torch.cat(a) for a in (pts, col, fruit, view))
    sel = torch.randperm(pts.shape[0], generator=torch.Generator().manual_seed(0))[:1000000]
    pts, col, fruit, view = (a[sel].to(cuda_device) for a in (pts, col, fruit, view))
    pts = pts.double()
    nrm = pointcloud.estimate_normals(pts, 30, view).float()
    out = P.reconstruct(pts, nrm, col.float(), fruit.float(), depth=8)
    vox = out["side"] / 256
    m = out["mesh"]
    dist = surface_distance(geom, m["vertices"]).numpy() / vox
    # As the TSDF test measures the vertices on observed edges, this measures the vertices with samples around them
    # (nearest-node density > 0).  The rest is surface that closes unobserved space: it has zero density, so the 0.1
    # quantile trim keeps it once more than a tenth of the vertices are unsupported.
    supported = m["density"] > 0
    frac = float((dist[supported] <= 2).mean())
    fv = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])[0]
    print(f"\napple scene d=8: {len(pts)} points, {out['iterations']} iterations ({out['total_iterations']} in all), residual "
          f"{out['residual']:.3g}; {len(m['vertices'])} kept vertices, {int(supported.sum())} with density > 0, of which {frac:.5f} "
          f"within 2 voxels (p99 {np.quantile(dist[supported], 0.99):.3f}); of all kept vertices {float((dist <= 2).mean()):.5f}; "
          f"fruit mesh {len(fv)} vertices")
    assert supported.sum() > 10000 and frac >= 0.99
    cent = geom.fruit_centers.double()
    near = (torch.from_numpy(fv).double()[:, None] - cent[None]).norm(dim=-1) <= geom.fruit_radius + 2 * vox
    for k in range(cent.shape[0]):
        assert bool(near[:, k].any()), f"fruit {k} has no fruit-mesh vertex"
    print(f"fruit mesh: {float((fruit_distance(geom, fv).numpy() / vox <= 2).mean()):.5f} of its vertices within 2 voxels of a fruit")


def test_refuses_bad_points(native_lib, cuda_device):
    from fruitnerf_b200 import _lib as L

    pts, nrm = sphere_cloud(1000)
    origin, side = P.cube_of(pts)
    bad = pts.copy()
    bad[17, 1] = np.nan
    dp, dn = cuda(bad, nrm, dev=cuda_device)
    with pytest.raises(L.FruitNerfNativeError, match="not finite or lies outside"):
        ops.poisson_splat(dp, dn, 5, origin, side)
    dp, dn = cuda(pts, nrm, dev=cuda_device)
    with pytest.raises(L.FruitNerfNativeError, match="not finite or lies outside"):
        ops.poisson_solve(dp, dn, 5, origin + 0.1 * side, side)
    with pytest.raises(ValueError, match="all finite"):
        P.reconstruct(*cuda(bad, nrm, dev=cuda_device), depth=5)


def test_2p24_points_depth9(native_lib, cuda_device):
    n = 2 ** 24
    g = torch.Generator(device=cuda_device).manual_seed(0)
    v = torch.nn.functional.normalize(torch.randn(n, 3, device=cuda_device, generator=g, dtype=torch.float64), dim=1)
    k = torch.randint(0, 4, (n,), device=cuda_device, generator=g)
    centres = torch.tensor([[-0.4, -0.4, 0.0], [0.4, -0.4, 0.1], [-0.4, 0.4, -0.1], [0.4, 0.4, 0.0]], dtype=torch.float64, device=cuda_device)
    pts = centres[k] + 0.3 * v
    out = P.reconstruct(pts, v.float(), depth=9)
    print(f"\n2^24 points d=9: {out['iterations']} iterations ({out['total_iterations']} in all), residual {out['residual']:.3g}, "
          f"{len(out['mesh']['vertices'])} kept vertices")
    assert out["iterations"] > 0 and out["residual"] <= 1e-4
    vox = out["side"] / 512
    kept = torch.from_numpy(out["mesh"]["vertices"]).double().to(cuda_device)
    d = ((kept[:, None] - centres[None]).norm(dim=-1) - 0.3).abs().min(dim=1).values / vox
    assert len(kept) > 100000 and float(d.max()) <= 1.0


# ---- end to end ---------------------------------------------------------------------------------------------------------
def test_poisson_cli_end_to_end(native_lib, cuda_device, tmp_path):
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply
    from fruitnerf_b200.scripts.exporter import entrypoint
    from fruitnerf_b200.trainer import Trainer

    from .test_gpu_mesh import _tiny_spec

    torch.manual_seed(0)
    run = tmp_path / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    base = ["poisson", "--load-config", str(run / "config.yml"), "--num-points", "30000", "--depth", "6"]
    res = entrypoint([*base, "--output-dir", str(tmp_path / "a"), "--normal-method", "open3d", "--save-point-cloud", "true"])
    v, nrm, col, f = read_mesh_ply(tmp_path / "a" / "poisson_mesh.ply")
    fv, fn, fc, ff = read_mesh_ply(tmp_path / "a" / "fruit_poisson_mesh.ply")
    assert (tmp_path / "a" / "point_cloud.ply").exists()
    assert len(f) > 100 and col is not None
    assert f.min() >= 0 and f.max() < len(v) and (len(ff) == 0 or (ff.min() >= 0 and ff.max() < len(fv)))
    np.testing.assert_array_equal(v, res["mesh"]["vertices"].astype(v.dtype))
    full_tris = {tuple(map(tuple, v[t])) for t in f}
    assert all(tuple(map(tuple, fv[t])) in full_tris for t in ff)
    pc = res["point_cloud"]["points"]
    centre, half = (pc.min(0) + pc.max(0)) / 2, 0.55 * (pc.max(0) - pc.min(0)).max()  # the Poisson cube
    assert (np.abs(v - centre) <= half * (1 + 1e-5)).all()
    assert len(res["point_cloud"]["fruit"]) == len(pc)
    with pytest.raises(SystemExit) as e:
        entrypoint([*base, "--output-dir", str(tmp_path / "b")])  # --normal-method model_output: FruitModel renders no normals
    assert e.value.code == 1
    assert not (tmp_path / "b" / "poisson_mesh.ply").exists()
