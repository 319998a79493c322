"""NeRF textures of exported meshes on the device: fnr_texel_rays bit for bit against the numpy restatement in texture.py,
fnr_mesh_mean_edge's repeatability, the traced apple scene as the model (its shading is view-independent, so the right
texture is known) for a TSDF and a Poisson mesh, and the CLI end to end on a briefly trained model."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

from fruitnerf_b200 import mesh as M
from fruitnerf_b200 import ops
from fruitnerf_b200 import texture as T

pytestmark = pytest.mark.gpu


def random_mesh(seed, F, V):
    rng = np.random.default_rng(seed)
    v = rng.uniform(-1, 1, (V, 3)).astype(np.float32)
    n = rng.standard_normal((V, 3)).astype(np.float32)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    n[rng.uniform(size=V) < 0.05] = 0  # vanishing normals: the face-normal fallback
    f = rng.integers(0, V, (F, 3))
    f[: F // 50, 1] = f[: F // 50, 0]  # degenerate faces
    if F > 10:
        f[-1, 1] = f[-1, 0]
        f[-1, 2] = f[-1, 0]  # a point face whose normals vanish too: +z
        n[f[-1, 0]] = 0
    return v, n, f


def cuda(*arrays, dev):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


@pytest.mark.parametrize("F, p, chunk", [(1, 2, 3), (7, 4, 5), (1001, 7, 4097), (99999, 4, 65536), (12345, 2, 1 << 20)])
def test_texel_rays_are_the_restatement(native_lib, cuda_device, F, p, chunk):
    v, n, f = random_mesh(F, F, max(3, F // 2))
    W, H = T.atlas_size(F, p)
    raylen = float(np.float32(0.0371))
    ro, rd = T.restated_texel_rays(v, n, f, p, W, H, raylen)
    dv, dn, df = cuda(v, n, f, dev=cuda_device)
    o_buf = torch.empty((chunk, 3), dtype=torch.float32, device=cuda_device)
    d_buf = torch.empty((chunk, 3), dtype=torch.float32, device=cuda_device)
    go, gd = [], []
    for t0 in range(0, W * H, chunk):  # chunk boundaries anywhere in the atlas
        m = min(chunk, W * H - t0)
        o, d = ops.texel_rays(dv, dn, df, p, W, H, raylen, t0, m, out=(o_buf, d_buf))
        go.append(o.cpu().numpy().copy())
        gd.append(d.cpu().numpy().copy())
    go, gd = np.concatenate(go), np.concatenate(gd)
    assert np.array_equal(go.view(np.int32), ro.view(np.int32))
    assert np.array_equal(gd.view(np.int32), rd.view(np.int32))
    if F > 10:  # the point face's texels take +z
        assert (gd == np.float32([0, 0, -1])).all(axis=1).any()


def test_mean_edge_is_repeatable(native_lib, cuda_device):
    for F in (1, 255, 257, 1000003):
        v, _, f = random_mesh(F, F, max(3, F // 3))
        dv, df = cuda(v, f, dev=cuda_device)
        a, b = ops.mesh_mean_edge(dv, df), ops.mesh_mean_edge(dv, df)
        assert a.dtype == torch.float64 and a.view(torch.int64).item() == b.view(torch.int64).item()
        assert float(a) == pytest.approx(T.restated_mean_edge(v, f), rel=1e-12)


# ---- the traced apple scene as the model --------------------------------------------------------------------------------
class TraceModel(torch.nn.Module):
    """A model whose forward is synthetic_scene.trace of the given rays: its 'rgb' is the analytic scene's colour."""

    def __init__(self, geom, device, chunk):
        super().__init__()
        self.geom = geom
        self.anchor = torch.nn.Parameter(torch.zeros(1, device=device))
        self.config = SimpleNamespace(eval_num_rays_per_chunk=chunk)

    @property
    def device(self):
        return self.anchor.device

    def forward(self, bundle):
        from fruitnerf_b200.data.synthetic_scene import trace

        assert bool((bundle.nears == 0).all()) and bundle.fars is not None
        return {"rgb": trace(self.geom, bundle.origins, bundle.directions)[0]}


def quantised_trace(model, mesh, p, W, H, raylen, dev):
    """trace() of the texel rays, chunk by chunk as the export renders them, quantised as fnr_compose_frame does."""
    v, n, f = cuda(np.asarray(mesh["vertices"], np.float32), np.asarray(mesh["normals"], np.float32), np.asarray(mesh["faces"], np.int64), dev=dev)
    chunk = model.config.eval_num_rays_per_chunk
    out = []
    for t0 in range(0, W * H, chunk):
        o, d = ops.texel_rays(v, n, f, p, W, H, raylen, t0, min(chunk, W * H - t0))
        out.append((model(SimpleNamespace(origins=o, directions=d, nears=torch.zeros_like(o[:, :1]), fars=o[:, :1]))["rgb"]
                    .clamp(0, 1) * 255 + 0.5).to(torch.uint8))
    return torch.cat(out).reshape(H, W, 3).cpu().numpy()


def bilinear(image, uv):
    H, W, _ = image.shape
    x = np.clip(uv[:, 0] * W - 0.5, 0, W - 1)
    y = np.clip((1 - uv[:, 1]) * H - 0.5, 0, H - 1)
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    img = image.astype(np.float64) / 255
    return ((img[y0, x0] * (1 - fx) + img[y0, x1] * fx) * (1 - fy) + (img[y1, x0] * (1 - fx) + img[y1, x1] * fx) * fy)


def check_textured(model, geom, mesh, fruit_mesh, out_dir, vox, dev, what, fraction):
    """Texture both meshes, then: the PNG is trace() of the texel rays exactly; the texture at each face's vt centroid
    matches the traced colour at its 3D centroid; the fruit mesh's texel origins lie outside the fruit spheres."""
    from fruitnerf_b200.data.synthetic_scene import trace
    from fruitnerf_b200.export.exporter_utils import export_textured_meshes

    from .test_gpu_mesh import surface_distance

    pipeline = SimpleNamespace(model=model)
    res = {"mesh": mesh, "fruit_mesh": fruit_mesh}
    paths = export_textured_meshes(pipeline, res, out_dir, px_per_uv_triangle=4)
    assert set(paths) == {f"{k}_{kind}" for k in ("mesh", "fruit_mesh") for kind in ("obj", "mtl", "png")}
    stats = {}
    for key, prefix in (("mesh", ""), ("fruit_mesh", "fruit_")):
        m = res[key]
        F = len(m["faces"])
        W, H = T.atlas_size(F, 4)
        image = np.asarray(Image.open(paths[f"{key}_png"]).convert("RGB"))
        assert image.shape == (H, W, 3)
        raylen = float(np.float32(2 * float(ops.mesh_mean_edge(*cuda(np.asarray(m["vertices"], np.float32), m["faces"], dev=dev)))))
        assert np.array_equal(image, quantised_trace(model, m, 4, W, H, raylen, dev)), key
        obj = T.read_textured_obj(paths[f"{key}_obj"])
        assert len(obj["v"]) == len(m["vertices"]) and len(obj["f"]) == F
        # the texture at the vt centroid against the traced colour at the 3D centroid (from 2 voxels outside along the face
        # normal), on the faces whose centroid lies within 2 voxels of the analytic surfaces
        vt = obj["vt"][obj["f"][:, :, 1] - 1].mean(axis=1)
        tri = np.asarray(m["vertices"], np.float64)[m["faces"]]
        cen = tri.mean(axis=1)
        fn = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
        ok = np.linalg.norm(fn, axis=1) > 0
        fn[ok] /= np.linalg.norm(fn[ok], axis=1, keepdims=True)
        near = ok & (surface_distance(geom, cen).numpy() <= 2 * vox)
        o = torch.from_numpy(cen[near] + 2 * vox * fn[near]).float()
        want = trace(geom, o, -torch.from_numpy(fn[near]).float())[0].double().numpy()
        err = np.abs(bilinear(image, vt[near]) - want).max(axis=1)
        stats[key] = (int(near.sum()), F, float((err <= TOLERANCE).mean()), float(np.median(err)))
    # texel origins of the fruit mesh (owned texels) lie outside the fruit spheres: the normals point out of the fruit
    fm = res["fruit_mesh"]
    F = len(fm["faces"])
    W, H = T.atlas_size(F, 4)
    raylen = float(np.float32(2 * float(ops.mesh_mean_edge(*cuda(np.asarray(fm["vertices"], np.float32), fm["faces"], dev=dev)))))
    o, _ = ops.texel_rays(*cuda(np.asarray(fm["vertices"], np.float32), np.asarray(fm["normals"], np.float32), fm["faces"], dev=dev), 4, W, H,
                          raylen, 0, W * H)
    owned = torch.from_numpy(T.texel_owners(F, 4).reshape(-1) >= 0)
    o = o.cpu().double()[owned]
    face, w = T.texel_barycentrics(F, 4)
    x = torch.from_numpy(np.einsum("tk,tkd->td", w.astype(np.float64), np.asarray(fm["vertices"], np.float64)[fm["faces"][face]]))[owned]
    cent = geom.fruit_centers.double()
    k = (x[:, None] - cent[None]).norm(dim=-1).argmin(dim=1)
    r_o, r_x = (o - cent[k]).norm(dim=-1), (x - cent[k]).norm(dim=-1)
    outward = float((r_o > r_x).float().mean())
    outside = float((r_o > geom.fruit_radius).float().mean())
    print(f"\n{what}: faces near the surface / all, fraction within {TOLERANCE} of the traced colour, median error: {stats}; fruit texel "
          f"origins farther out than their surface point {outward:.5f}, outside their fruit sphere {outside:.5f}")
    for key, (_, _, frac, _) in stats.items():
        assert frac >= fraction[key], (key, frac)
    assert outward >= 0.99 and outside >= 0.99  # first H100 run: 0.9987 / 0.99999 (TSDF), 0.99997 / 1.0 (Poisson)


# Set from the first H100 run (an H100 80GB HBM3): within 0.05, the TSDF meshes had 0.9971 (scene) and 0.9993 (fruit) of
# their faces, the Poisson meshes 0.9346 and 0.9981; the median errors were 0.0016 and below.  Faces that straddle a colour
# edge (a fruit against a leaf, the ground's checker) take a mixture of the two colours, and the Poisson scene mesh has
# more faces that bridge two surfaces.
TOLERANCE = 0.05


def test_traced_apple_scene_tsdf(native_lib, cuda_device, tmp_path):
    from .test_gpu_mesh import traced_views

    geom, frames, _ = traced_views(cuda_device)
    n = 192
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], n, device=cuda_device)
    for b0 in range(0, 40, 10):
        tsdf.integrate(*(t[b0:b0 + 10] for t in frames))
    m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
    fv, fn, fc, ff, fidx = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    model = TraceModel(geom, cuda_device, 1 << 16)
    check_textured(model, geom, m, {"vertices": fv, "normals": fn, "faces": fidx}, tmp_path, 2.0 / n, cuda_device, "tsdf 192^3",
                   {"mesh": 0.99, "fruit_mesh": 0.99})


def test_traced_apple_scene_poisson(native_lib, cuda_device, tmp_path):
    from fruitnerf_b200 import pointcloud
    from fruitnerf_b200 import poisson as P
    from fruitnerf_b200.data.synthetic_scene import camera_rays, make_apple_scene, trace

    size = 160  # the traced surface cloud of test_gpu_poisson.py::test_ground_truth_apple_scene
    train, ev = make_apple_scene(num_images=40, height=size, width=size, noise_std=0.0)
    geom, cams = train.geometry, train.cameras
    pts, col, fruit, view = [], [], [], []
    ys, xs = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    for c2w in torch.cat([train.cameras.camera_to_worlds, ev.cameras.camera_to_worlds]):
        o, d = camera_rays(c2w, cams.fx, cams.fy, cams.cx, cams.cy, ys.reshape(-1), xs.reshape(-1))
        rgb, mk, t = trace(geom, o, d)
        p = o + d * torch.where(torch.isfinite(t), t, torch.zeros_like(t))[:, None]
        keep = torch.isfinite(t) & (p.abs() < 1).all(dim=1)
        pts.append(p[keep])
        col.append(rgb[keep])
        fruit.append(mk[keep, 0])
        view.append(d[keep])
    pts, col, fruit, view = (torch.cat(a) for a in (pts, col, fruit, view))
    sel = torch.randperm(pts.shape[0], generator=torch.Generator().manual_seed(0))[:1000000]
    pts, col, fruit, view = (a[sel].to(cuda_device) for a in (pts, col, fruit, view))
    pts = pts.double()
    nrm = pointcloud.estimate_normals(pts, 30, view).float()
    out = P.reconstruct(pts, nrm, col.float(), fruit.float(), depth=8)
    m = out["mesh"]
    fv, fn, fc, ff, fidx = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    model = TraceModel(geom, cuda_device, 1 << 16)
    check_textured(model, geom, m, {"vertices": fv, "normals": fn, "faces": fidx}, tmp_path, out["side"] / 256, cuda_device, "poisson d=8",
                   {"mesh": 0.9, "fruit_mesh": 0.99})


# ---- end to end ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def trained_run(tmp_path_factory, native_lib, cuda_device):
    from fruitnerf_b200.trainer import Trainer

    from .test_gpu_mesh import _tiny_spec

    torch.manual_seed(0)
    run = tmp_path_factory.mktemp("texture") / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    return run


@pytest.mark.parametrize("command, args, plys", [
    ("tsdf", ["--resolution", "64", "--bounding-box-min", "-0.8", "-0.8", "-0.8", "--bounding-box-max", "0.8", "0.8", "0.8"],
     ("tsdf_mesh.ply", "fruit_mesh.ply")),
    ("poisson", ["--num-points", "30000", "--depth", "6", "--normal-method", "open3d"], ("poisson_mesh.ply", "fruit_poisson_mesh.ply")),
])
def test_cli_end_to_end(trained_run, tmp_path, command, args, plys):
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply
    from fruitnerf_b200.scripts.exporter import entrypoint

    base = [command, "--load-config", str(trained_run / "config.yml"), *args]
    torch.manual_seed(0)
    entrypoint([*base, "--output-dir", str(tmp_path / "plain")])
    runs = []
    for k in range(2):
        torch.manual_seed(0)
        out = tmp_path / f"nerf{k}"
        res = entrypoint([*base, "--output-dir", str(out), "--texture-method", "nerf", "--unwrap-method", "custom"])
        runs.append(out)
        for ply in plys:  # the PLYs are those of a run without texturing
            assert (out / ply).read_bytes() == (tmp_path / "plain" / ply).read_bytes(), ply
        assert not list((tmp_path / "plain").glob("*.obj"))
        for ply, prefix, key in ((plys[0], "", "mesh"), (plys[1], "fruit_", "fruit_mesh")):
            v, _, _, f = read_mesh_ply(out / ply)
            if len(f) == 0:
                assert not (out / f"{prefix}mesh.obj").exists()
                continue
            obj = T.read_textured_obj(out / f"{prefix}mesh.obj")
            assert len(obj["v"]) == len(v) and len(obj["f"]) == len(f) and len(obj["vt"]) == 3 * len(f)
            np.testing.assert_array_equal(obj["f"][:, :, 0] - 1, f)
            assert obj["mtllib"] == f"{prefix}material_0.mtl"
            assert f"map_Kd {prefix}material_0.png" in (out / f"{prefix}material_0.mtl").read_text()
            with Image.open(out / f"{prefix}material_0.png") as im:
                assert im.size == T.atlas_size(len(f), 4)
                pix = np.asarray(im)
            assert pix.std() > 0  # a rendered texture, not a constant image
            assert res["paths"][f"{key}_png"] == str(out / f"{prefix}material_0.png")
    for png in runs[0].glob("*.png"):  # two runs give the same textures
        assert png.read_bytes() == (runs[1] / png.name).read_bytes(), png.name
