"""The `tsdf` mesh export on the device: fnr_tsdf_integrate and fnr_marching_cubes_count / _emit against the torch / numpy
restatement in mesh.py (bit for bit), a grid of more than 2^31 points, the ground-truth apple scene fused from traced
depth, and the CLI end to end on a briefly trained model."""

import numpy as np
import pytest
import torch
from scipy import ndimage

from fruitnerf_b200 import mesh as M

pytestmark = pytest.mark.gpu


def look_at(eye, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    from fruitnerf_b200.data.synthetic_scene import look_at_c2w

    return look_at_c2w(torch.tensor(eye, dtype=torch.float32), torch.tensor(target, dtype=torch.float32), up)


def random_frames(seed, B, H, W):
    g = torch.Generator().manual_seed(seed)
    c2w = []
    for _ in range(B):
        d = torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0)
        c2w.append(look_at((d * (1.3 + 0.4 * torch.rand(1, generator=g))).tolist(), (0.1 * torch.randn(3, generator=g)).tolist()))
    c2w = torch.stack(c2w)
    fx = 0.9 * W * (1 + 0.1 * torch.rand(B, generator=g))
    fy = 0.9 * W * (1 + 0.1 * torch.rand(B, generator=g))
    cx = W / 2 + torch.randn(B, generator=g)
    cy = H / 2 + torch.randn(B, generator=g)
    depth = 0.9 + 0.8 * torch.rand(B, H, W, generator=g)
    depth[torch.rand(B, H, W, generator=g) < 0.05] = 0.0  # misses
    return c2w, fx, fy, cx, cy, depth, torch.rand(B, H, W, 3, generator=g), torch.rand(B, H, W, generator=g)


def boundary_ties(tsdf, c2w, fx, fy, cx, cy):
    """Grid points whose fp64 projection in some frame lies within 1e-5 px of a pixel boundary."""
    X, Y, Z = tsdf.dims
    idx = torch.stack(torch.meshgrid(*(torch.arange(n, dtype=torch.float64) for n in (X, Y, Z)), indexing="ij"), -1).reshape(-1, 3)
    x = tsdf.origin.double() + idx * tsdf.voxel_size.double()
    tie = torch.zeros(x.shape[0], dtype=torch.bool)
    for b in range(c2w.shape[0]):
        m = c2w[b].double()
        p = (x - m[:, 3]) @ m[:, :3]
        zc = -p[:, 2]
        u = float(cx[b]) + float(fx[b]) * p[:, 0] / zc
        v = float(cy[b]) - float(fy[b]) * p[:, 1] / zc
        tie |= ((u - u.round()).abs() < 1e-5) | ((v - v.round()).abs() < 1e-5)
    return tie.reshape(X, Y, Z)


def test_fusion_is_bitwise_the_restatement(native_lib, cuda_device):
    H, W = 48, 64
    box = [[-0.6, -0.5, -0.55], [0.6, 0.5, 0.45]]
    host = M.TSDF.from_aabb(box, [40, 36, 33])
    dev = M.TSDF.from_aabb(box, [40, 36, 33], device=cuda_device)
    ties = torch.zeros(host.dims, dtype=torch.bool)
    for seed in range(3):  # three batches, the last without fruit
        c2w, fx, fy, cx, cy, depth, rgb, fruit = random_frames(seed, 4, H, W)
        fr = fruit if seed < 2 else None
        host.integrate(c2w, fx, fy, cx, cy, depth, rgb, fr)
        dev.integrate(*(t.to(cuda_device) for t in (c2w, fx, fy, cx, cy, depth, rgb)), None if fr is None else fr.to(cuda_device))
        ties |= boundary_ties(host, c2w, fx, fy, cx, cy)
    torch.cuda.synchronize()
    assert int(ties.sum()) < 0.01 * ties.numel()
    keep = ~ties
    assert int((host.weights[keep] >= 4).sum()) > 1000
    for name in ("values", "weights", "colors", "fruit"):
        a, b = getattr(host, name), getattr(dev, name).cpu()
        assert torch.equal(a[keep].view(torch.int32), b[keep].view(torch.int32)), name


def smooth_field(shape, seed, sigma=2.5):
    rng = np.random.default_rng(seed)
    v = ndimage.gaussian_filter(rng.standard_normal(shape), sigma)
    return (v / v.std()).astype(np.float32)


def fields():
    n = 48
    g = np.linspace(-0.5, 0.5, n)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    q = np.sqrt(X ** 2 + Y ** 2) - 0.3
    shape = (37, 64, 129)
    a = np.arange(max(shape), dtype=np.float32)
    return {
        "sphere": ((np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.37).astype(np.float32), (-0.5,) * 3, 1 / (n - 1)),
        "torus": ((np.sqrt(q ** 2 + Z ** 2) - 0.1).astype(np.float32), (-0.5,) * 3, 1 / (n - 1)),
        "smooth": (smooth_field((56, 50, 61), 0), (0.1, -0.2, 0.3), (0.02, 0.03, 0.025)),
        "cell": (np.array([-1, 2, 0.5, -3, 1, -0.25, 4, -2], np.float32).reshape(2, 2, 2), (0.0, 0.0, 0.0), 1.0),
        "noncubic": ((np.sin(a[:37, None, None] / 5) + np.cos(a[None, :64, None] / 7) * np.sin(a[None, None, :129] / 11) - 0.2).astype(np.float32),
                     (-1.0, -2.0, -3.0), (0.05, 0.04, 0.03)),
    }


@pytest.mark.parametrize("name", ["sphere", "torus", "smooth", "cell", "noncubic"])
def test_marching_cubes_is_array_equal_to_numpy(native_lib, cuda_device, name):
    v, origin, vs = fields()[name]
    rng = np.random.default_rng(1)
    col = rng.uniform(size=v.shape + (3,)).astype(np.float32)
    fr = rng.uniform(size=v.shape).astype(np.float32)
    ref = M.marching_cubes_numpy(v, origin, vs, col, fr)
    got = M.marching_cubes(torch.from_numpy(v).to(cuda_device), origin, vs, torch.from_numpy(col).to(cuda_device),
                           torch.from_numpy(fr).to(cuda_device))
    assert len(ref["faces"]) > 0
    for key in ("vertices", "normals", "colors", "fruit", "faces"):
        np.testing.assert_array_equal(got[key].cpu().numpy(), ref[key], err_msg=key)
    bare = M.marching_cubes(torch.from_numpy(v).to(cuda_device), origin, vs)
    assert bare["colors"] is None and bare["fruit"] is None and torch.equal(bare["faces"], got["faces"])


def test_more_than_2p31_grid_points(native_lib, cuda_device):
    """A mostly constant 2100 x 1024 x 1025 grid (2.2e9 points) with a small sphere past point index 2^31: the same
    mesh as the numpy reference on a crop around it."""
    dims = (2100, 1024, 1025)
    vs = 1e-3
    c = np.array([2080, 600, 700])
    n = 24
    lo = c - n // 2
    ii = [np.arange(lo[a], lo[a] + n) for a in range(3)]
    X, Y, Z = np.meshgrid(*ii, indexing="ij")
    crop = (np.sqrt((X - c[0] - 0.3) ** 2 + (Y - c[1] + 0.2) ** 2 + (Z - c[2]) ** 2) - 7.5).astype(np.float32)
    assert ((lo[0] * dims[1] + lo[1]) * dims[2] + lo[2]) > 2 ** 31
    v = torch.ones(dims, dtype=torch.float32, device=cuda_device)
    v[lo[0]:lo[0] + n, lo[1]:lo[1] + n, lo[2]:lo[2] + n] = torch.from_numpy(crop).to(cuda_device)
    got = M.marching_cubes(v, (0.0, 0.0, 0.0), vs)
    del v
    torch.cuda.empty_cache()
    ref = M.marching_cubes_numpy(crop, (lo * np.float32(vs)).astype(np.float32), vs)
    np.testing.assert_array_equal(got["faces"].cpu().numpy(), ref["faces"])
    np.testing.assert_array_equal(got["normals"].cpu().numpy(), ref["normals"])
    np.testing.assert_allclose(got["vertices"].cpu().numpy(), ref["vertices"], atol=2e-6, rtol=0)
    assert len(ref["faces"]) > 500


# ---- the ground-truth apple scene -------------------------------------------------------------------------------------
def surface_distance(geom, p):
    """Distance of points [N,3] (fp64) to the nearest analytic surface: fruit and leaf spheres, trunk, ground."""
    p = torch.as_tensor(p, dtype=torch.float64)
    centres = torch.cat([geom.fruit_centers, geom.leaf_centers]).double()
    radii = torch.cat([torch.full((geom.fruit_centers.shape[0],), geom.fruit_radius), geom.leaf_radii]).double()
    d_s = ((p[:, None] - centres[None]).norm(dim=-1) - radii).abs().min(dim=1).values
    rho = p[:, :2].norm(dim=-1)
    z0, z1 = geom.trunk_z
    dz = torch.clamp(torch.maximum(z0 - p[:, 2], p[:, 2] - z1), min=0)
    d_c = torch.sqrt((rho - geom.trunk_radius) ** 2 + dz ** 2)
    d_g = (p[:, 2] - geom.ground_z).abs()
    return torch.minimum(torch.minimum(d_s, d_c), d_g)


def fruit_distance(geom, p):
    p = torch.as_tensor(p, dtype=torch.float64)
    return ((p[:, None] - geom.fruit_centers.double()[None]).norm(dim=-1) - geom.fruit_radius).abs().min(dim=1).values


def traced_views(cuda_device, size=160):
    from fruitnerf_b200.data.synthetic_scene import make_apple_scene, trace

    train, ev = make_apple_scene(num_images=40, height=size, width=size, noise_std=0.0)
    geom = train.geometry
    c2w = torch.cat([train.cameras.camera_to_worlds, ev.cameras.camera_to_worlds])
    cams = train.cameras
    depth, rgb, fruit, hits = [], [], [], []
    for i in range(c2w.shape[0]):
        from fruitnerf_b200.data.synthetic_scene import camera_rays

        ys, xs = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
        o, d = camera_rays(c2w[i], cams.fx, cams.fy, cams.cx, cams.cy, ys.reshape(-1), xs.reshape(-1))
        col, m, t = trace(geom, o, d)
        depth.append(torch.where(torch.isfinite(t), t, torch.zeros_like(t)).reshape(size, size))
        rgb.append(col.reshape(size, size, 3))
        fruit.append(m.reshape(size, size))
        hits.append((o + d * torch.where(torch.isfinite(t), t, torch.zeros_like(t))[:, None])[m[:, 0] > 0])
    B = c2w.shape[0]
    fx = torch.full((B,), float(cams.fx))
    cy = torch.full((B,), float(cams.cy))
    frames = (c2w, fx, fx.clone(), torch.full((B,), float(cams.cx)), cy, torch.stack(depth), torch.stack(rgb), torch.stack(fruit))
    return geom, tuple(t.to(cuda_device) for t in frames), torch.cat(hits)


def test_ground_truth_apple_scene(native_lib, cuda_device, tmp_path):
    from fruitnerf_b200.export.exporter_utils import write_mesh_ply

    geom, frames, fruit_hits = traced_views(cuda_device)
    n = 192
    voxel = 2.0 / n
    paths = []
    for run in range(2):
        tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], n, device=cuda_device)
        for b0 in range(0, 40, 10):
            tsdf.integrate(*(t[b0:b0 + 10] for t in frames))
        m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
        fm = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
        for name, mm in (("full", (m["vertices"], m["normals"], m["colors"], m["faces"])), ("fruit", (fm[0], fm[1], fm[2], fm[4]))):
            paths.append(tmp_path / f"{name}{run}.ply")
            write_mesh_ply(paths[-1], *mm)
    assert paths[0].read_bytes() == paths[2].read_bytes() and paths[1].read_bytes() == paths[3].read_bytes()
    # vertices on edges whose two endpoints were observed
    w = tsdf.weights.cpu().numpy()
    vals = tsdf.values.cpu().numpy()
    inside = vals < 0
    act = np.zeros(vals.shape + (3,), bool)
    act[:-1, :, :, 0] = inside[:-1] != inside[1:]
    act[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    act[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    keys = np.flatnonzero(act.reshape(-1))
    assert len(keys) == len(m["vertices"])
    pa = np.stack(np.unravel_index(keys // 3, vals.shape), 1)
    pb = pa.copy()
    pb[np.arange(len(keys)), keys % 3] += 1
    observed = (w[tuple(pa.T)] > 0) & (w[tuple(pb.T)] > 0)
    dist = surface_distance(geom, m["vertices"][observed]).numpy() / voxel
    frac_full = float((dist <= 2).mean())
    fv = fm[0]
    fdist = fruit_distance(geom, fv).numpy() / voxel
    frac_fruit = float((fdist <= 2).mean())
    print(f"\n192^3 ground truth: {observed.sum()} observed vertices of {len(observed)}, {frac_full:.5f} within 2 voxels "
          f"(p99 {np.quantile(dist, 0.99):.3f}, worst {dist.max():.3f} voxels); fruit mesh {len(fv)} vertices, {frac_fruit:.5f} within 2 "
          f"voxels (p99 {np.quantile(fdist, 0.99):.3f}, worst {fdist.max():.3f} voxels)")
    assert observed.sum() > 10000 and frac_full >= 0.99
    assert len(fv) > 100 and frac_fruit >= 0.99
    # every fruit seen by >= 50 pixels has fruit-mesh vertices near it
    cent = geom.fruit_centers.double()
    owner = (fruit_hits.double()[:, None] - cent[None]).norm(dim=-1).argmin(dim=1)
    seen = torch.bincount(owner, minlength=cent.shape[0])
    near = (torch.from_numpy(fv).double()[:, None] - cent[None]).norm(dim=-1) <= geom.fruit_radius + 2 * voxel
    for k in range(cent.shape[0]):
        if int(seen[k]) >= 50:
            assert bool(near[:, k].any()), f"fruit {k} seen by {int(seen[k])} pixels has no fruit-mesh vertex"


# ---- end to end ---------------------------------------------------------------------------------------------------------
def _tiny_spec(seed=0):  # as test_gpu_pointcloud.py
    from fruitnerf_b200.scripts.train import synthetic_spec

    spec = synthetic_spec("fruit_nerf", num_images=20, image_size=64, num_fruits=5, seed=seed, rays_per_batch=2048)
    m = spec.pipeline.model
    m.log2_hashmap_size = 17
    m.proposal_weights_anneal_max_num_iters = 100
    return spec


def test_tsdf_cli_end_to_end(native_lib, cuda_device, tmp_path):
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply
    from fruitnerf_b200.scripts.exporter import entrypoint
    from fruitnerf_b200.trainer import Trainer

    torch.manual_seed(0)
    run = tmp_path / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    lo, hi = np.array([-0.8] * 3), np.array([0.8] * 3)
    base = ["tsdf", "--load-config", str(run / "config.yml"), "--resolution", "64", "--bounding-box-min", *map(str, lo),
            "--bounding-box-max", *map(str, hi)]
    res = entrypoint([*base, "--output-dir", str(tmp_path / "a")])
    v, nrm, col, f = read_mesh_ply(tmp_path / "a" / "tsdf_mesh.ply")
    fv, fn, fc, ff = read_mesh_ply(tmp_path / "a" / "fruit_mesh.ply")
    voxel = (hi - lo) / 64
    assert len(f) > 100 and col is not None
    assert ((v >= lo - voxel) & (v <= hi + voxel)).all()
    np.testing.assert_allclose(np.linalg.norm(nrm, axis=1), 1.0, atol=1e-5)
    assert f.min() >= 0 and f.max() < len(v) and (len(ff) == 0 or (ff.min() >= 0 and ff.max() < len(fv)))
    full_tris = {tuple(map(tuple, v[t])) for t in f}
    assert all(tuple(map(tuple, fv[t])) in full_tris for t in ff)
    np.testing.assert_array_equal(v, res["mesh"]["vertices"].astype(np.float64))
    # refinement: the second grid spans the first mesh's vertex box widened by epsilon
    eps = 0.02
    ref = entrypoint([*base, "--output-dir", str(tmp_path / "b"), "--refine-mesh-using-initial-aabb-estimate", "true",
                      "--refinement-epsilon", str(eps)])
    v32 = res["mesh"]["vertices"]
    want = np.stack([v32.min(0) - eps, v32.max(0) + eps]).astype(np.float32)
    np.testing.assert_allclose(ref["aabb"], want, atol=1e-6)
    rv = ref["mesh"]["vertices"]
    assert (rv >= want[0] - 1e-6).all() and (rv <= want[1] + (want[1] - want[0]) / 64 + 1e-6).all()
    # a box the cameras never see: an empty mesh, exit status 1, nothing written
    with pytest.raises(SystemExit) as e:
        entrypoint(["tsdf", "--load-config", str(run / "config.yml"), "--output-dir", str(tmp_path / "c"), "--resolution", "16",
                    "--bounding-box-min", "5", "5", "5", "--bounding-box-max", "6", "6", "6"])
    assert e.value.code == 1
    assert not (tmp_path / "c" / "tsdf_mesh.ply").exists()
