"""The `charts` UV unwrap on the device (DESIGN section 4.3r): fnr_chart_unwrap and fnr_chart_texel_rays bit for bit against
the numpy restatement in texture.py on the 192^3 TSDF mesh, the depth-8 Poisson mesh and the decimated TSDF mesh of the
traced apple scene and on a self-overlapping helicoid; the traced scene as the model; the CLI end to end."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

from fruitnerf_b200 import mesh as M
from fruitnerf_b200 import ops
from fruitnerf_b200 import texture as T

from .test_gpu_texture import TOLERANCE, TraceModel, bilinear, cuda, trained_run  # noqa: F401
from .test_unwrap_host import helicoid

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene_meshes(native_lib, cuda_device):
    """{name: (vertices fp32, normals fp32, faces int64)} and the scene geometry."""
    from fruitnerf_b200 import pointcloud
    from fruitnerf_b200 import poisson as P
    from fruitnerf_b200.data.synthetic_scene import camera_rays, make_apple_scene, trace
    from fruitnerf_b200.export.exporter_utils import decimate_for_texture

    from .test_gpu_mesh import traced_views

    geom, frames, _ = traced_views(cuda_device)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], 192, device=cuda_device)
    for b0 in range(0, 40, 10):
        tsdf.integrate(*(t[b0:b0 + 10] for t in frames))
    m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
    out = {"tsdf": m}
    out["tsdf_20k"] = decimate_for_texture(m, 20000, cuda_device)
    size = 160  # the traced surface cloud of test_gpu_texture.py::test_traced_apple_scene_poisson
    train, ev = make_apple_scene(num_images=40, height=size, width=size, noise_std=0.0)
    cams = train.cameras
    pts, col, fruit, view = [], [], [], []
    ys, xs = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    for c2w in torch.cat([train.cameras.camera_to_worlds, ev.cameras.camera_to_worlds]):
        o, d = camera_rays(c2w, cams.fx, cams.fy, cams.cx, cams.cy, ys.reshape(-1), xs.reshape(-1))
        rgb, mk, t = trace(train.geometry, o, d)
        p = o + d * torch.where(torch.isfinite(t), t, torch.zeros_like(t))[:, None]
        keep = torch.isfinite(t) & (p.abs() < 1).all(dim=1)
        pts.append(p[keep])
        col.append(rgb[keep])
        fruit.append(mk[keep, 0])
        view.append(d[keep])
    pts, col, fruit, view = (torch.cat(a) for a in (pts, col, fruit, view))
    sel = torch.randperm(pts.shape[0], generator=torch.Generator().manual_seed(0))[:1000000]
    pts, col, fruit, view = (a[sel].to(cuda_device) for a in (pts, col, fruit, view))
    nrm = pointcloud.estimate_normals(pts.double(), 30, view).float()
    out["poisson"] = P.reconstruct(pts.double(), nrm, col.float(), fruit.float(), depth=8)["mesh"]
    hv, hf = helicoid()
    out["helicoid"] = {"vertices": hv, "normals": np.tile(np.float32([0, 0, 1]), (len(hv), 1)), "faces": hf}
    meshes = {k: (np.asarray(m["vertices"], np.float32), np.asarray(m["normals"], np.float32), np.asarray(m["faces"], np.int64))
              for k, m in out.items()}
    return meshes, geom, m


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.int64, 4: np.int32}[a.dtype.itemsize])


@pytest.mark.parametrize("N", [256, 1024])
@pytest.mark.parametrize("name", ["tsdf", "poisson", "tsdf_20k", "helicoid"])
def test_device_is_the_restatement(scene_meshes, cuda_device, name, N):
    meshes, _, _ = scene_meshes
    v, n, f = meshes[name]
    dv, dn, df = cuda(v, n, f, dev=cuda_device)
    try:
        want = T.restated_chart_unwrap(v, f, N)
    except T.AtlasTooLargeError as e:
        with pytest.raises(T.AtlasTooLargeError, match=str(e).split(" ")[0] + " charts"):
            ops.chart_unwrap(dv, df, N)
        print(f"\n{name} N={N}: {e}")
        return
    got = ops.chart_unwrap(dv, df, N)
    assert got["rounds"] == want["rounds"] and got["num_charts"] == want["num_charts"]
    assert bits(np.float64(got["scale"])) == bits(np.float64(want["scale"]))
    for key in ("labels", "charts", "offsets", "owner", "texels", "texel_faces"):
        assert np.array_equal(got[key].cpu().numpy(), want[key]), key
    for key in ("uv", "barycentrics"):
        assert np.array_equal(bits(got[key].cpu().numpy()), bits(want[key])), key
    n_owned = got["num_owned"]
    print(f"\n{name} N={N}: {len(f)} faces, {got['num_charts']} charts, {got['rounds']} rounds, s = {got['scale']:.6g}, owned "
          f"{n_owned / N / N:.4f} of the atlas")
    if name == "helicoid":
        assert got["rounds"] >= 1
    raylen = float(np.float32(0.0123))
    ro, rd = T.restated_chart_texel_rays(v, n, f, want["texel_faces"], want["barycentrics"], raylen)
    for chunk in (4097, 65536):  # chunk boundaries anywhere in the owned texels
        o_buf = torch.empty((chunk, 3), dtype=torch.float32, device=cuda_device)
        d_buf = torch.empty((chunk, 3), dtype=torch.float32, device=cuda_device)
        go, gd = [], []
        for t0 in range(0, n_owned, chunk):
            o, d = ops.chart_texel_rays(dv, dn, df, got["texel_faces"], got["barycentrics"], raylen, t0, min(chunk, n_owned - t0),
                                        out=(o_buf, d_buf))
            go.append(o.cpu().numpy().copy())
            gd.append(d.cpu().numpy().copy())
        assert np.array_equal(bits(np.concatenate(go)), bits(ro)) and np.array_equal(bits(np.concatenate(gd)), bits(rd))


def test_repeatable_and_refusals(scene_meshes, cuda_device):
    meshes, _, _ = scene_meshes
    v, n, f = meshes["tsdf_20k"]
    dv, df = cuda(v, f, dev=cuda_device)
    a, b = ops.chart_unwrap(dv, df, 1024, timing=True), ops.chart_unwrap(dv, df, 1024)
    assert len(a["stage_ms"]) == 5 and all(t >= 0 for t in a["stage_ms"])
    for key in ("charts", "owner", "uv", "barycentrics"):
        assert torch.equal(a[key], b[key]), key
    bad = df.clone()
    bad[7, 1] = len(v)
    with pytest.raises(Exception, match="outside"):
        ops.chart_unwrap(dv, bad, 256)


def test_traced_apple_scene(scene_meshes, cuda_device, tmp_path):
    """Texture the TSDF scene and fruit meshes with the charts unwrap: every owned texel is trace() of its ray, unowned
    texels are black, the texture at each face's vt centroid matches the traced colour at its 3D centroid, and the fruit
    mesh's texel origins lie outside the fruit spheres."""
    from fruitnerf_b200.data.synthetic_scene import trace
    from fruitnerf_b200.export.exporter_utils import export_textured_meshes

    from .test_gpu_mesh import surface_distance

    _, geom, m = scene_meshes
    N, vox = 1024, 2.0 / 192
    fv, fn, fc, ff, fidx = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    res = {"mesh": m, "fruit_mesh": {"vertices": fv, "normals": fn, "faces": fidx}}
    model = TraceModel(geom, cuda_device, 1 << 16)
    paths = export_textured_meshes(SimpleNamespace(model=model), res, tmp_path, unwrap_method="charts", num_pixels_per_side=N)
    stats = {}
    for key, prefix in (("mesh", ""), ("fruit_mesh", "fruit_")):
        mm = res[key]
        v, nrm, f = (np.asarray(mm[k], dt) for k, dt in (("vertices", np.float32), ("normals", np.float32), ("faces", np.int64)))
        image = np.asarray(Image.open(paths[f"{key}_png"]).convert("RGB"))
        assert image.shape == (N, N, 3)
        dv, dn, df = cuda(v, nrm, f, dev=cuda_device)
        u = ops.chart_unwrap(dv, df, N)
        raylen = float(np.float32(2 * float(ops.mesh_mean_edge(dv, df))))
        o, d = ops.chart_texel_rays(dv, dn, df, u["texel_faces"], u["barycentrics"], raylen, 0, u["num_owned"])
        chunk = model.config.eval_num_rays_per_chunk  # as the export renders them
        want = np.concatenate([(model(SimpleNamespace(origins=o[t0:t0 + chunk], directions=d[t0:t0 + chunk], nears=torch.zeros_like(o[t0:t0 + chunk, :1]),
                                                      fars=o[t0:t0 + chunk, :1]))["rgb"].clamp(0, 1) * 255 + 0.5).to(torch.uint8).cpu().numpy()
                               for t0 in range(0, u["num_owned"], chunk)])
        flat = image.reshape(-1, 3)
        owned = u["owner"].cpu().numpy() >= 0
        assert np.array_equal(flat[u["texels"].cpu().numpy()], want), key
        assert (flat[~owned] == 0).all(), key
        obj = T.read_textured_obj(paths[f"{key}_obj"])
        assert len(obj["v"]) == len(v) and len(obj["f"]) == len(f)
        vt = obj["vt"][obj["f"][:, :, 1] - 1].mean(axis=1)
        tri = v.astype(np.float64)[f]
        cen = tri.mean(axis=1)
        fnn = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
        ok = np.linalg.norm(fnn, axis=1) > 0
        fnn[ok] /= np.linalg.norm(fnn[ok], axis=1, keepdims=True)
        near = ok & (surface_distance(geom, cen).numpy() <= 2 * vox)
        ref = trace(geom, torch.from_numpy(cen[near] + 2 * vox * fnn[near]).float(), -torch.from_numpy(fnn[near]).float())[0].double().numpy()
        err = np.abs(bilinear(image, vt[near]) - ref).max(axis=1)
        stats[key] = (int(near.sum()), len(f), float((err <= TOLERANCE).mean()), float(np.median(err)), float(owned.mean()))
        if key == "fruit_mesh":  # texel origins lie outside the fruit spheres
            x = torch.from_numpy(np.einsum("tk,tkd->td", u["barycentrics"].cpu().numpy().astype(np.float64),
                                           v.astype(np.float64)[f[u["texel_faces"].cpu().numpy()]]))
            oo = o.cpu().double()
            cent = geom.fruit_centers.double()
            k = (x[:, None] - cent[None]).norm(dim=-1).argmin(dim=1)
            outside = float(((oo - cent[k]).norm(dim=-1) > geom.fruit_radius).float().mean())
            stats["fruit_origins_outside"] = outside
    print(f"\ncharts N={N}: faces near the surface / all, fraction within {TOLERANCE}, median error, owned fraction: {stats}")
    assert stats["mesh"][2] >= 0.97 and stats["fruit_mesh"][2] >= 0.97
    assert stats["fruit_origins_outside"] >= 0.99


@pytest.mark.parametrize("command, args, plys", [
    ("tsdf", ["--resolution", "64", "--bounding-box-min", "-0.8", "-0.8", "-0.8", "--bounding-box-max", "0.8", "0.8", "0.8"],
     ("tsdf_mesh.ply", "fruit_mesh.ply")),
    ("poisson", ["--num-points", "30000", "--depth", "6", "--normal-method", "open3d"], ("poisson_mesh.ply", "fruit_poisson_mesh.ply")),
])
@pytest.mark.parametrize("target", [None, 2000])
def test_cli_end_to_end(trained_run, tmp_path, command, args, plys, target):  # noqa: F811
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply
    from fruitnerf_b200.scripts.exporter import entrypoint

    N = 2048  # the briefly trained model's noisy surfaces make many small charts
    base = [command, "--load-config", str(trained_run / "config.yml"), *args]
    torch.manual_seed(0)
    entrypoint([*base, "--output-dir", str(tmp_path / "plain")])
    extra = ["--texture-method", "nerf", "--unwrap-method", "charts", "--num-pixels-per-side", str(N)]
    if target is not None:
        extra += ["--target-num-faces", str(target)]
    runs = []
    for k in range(2):
        torch.manual_seed(0)
        out = tmp_path / f"nerf{k}"
        entrypoint([*base, "--output-dir", str(out), *extra])
        runs.append(out)
        for ply in plys:  # the PLYs are those of a run without texturing
            assert (out / ply).read_bytes() == (tmp_path / "plain" / ply).read_bytes(), ply
        for ply, prefix in ((plys[0], ""), (plys[1], "fruit_")):
            _, _, _, f = read_mesh_ply(out / ply)
            if len(f) == 0:
                assert not (out / f"{prefix}mesh.obj").exists()
                continue
            obj = T.read_textured_obj(out / f"{prefix}mesh.obj")
            F = len(obj["f"])
            assert len(obj["vt"]) == 3 * F
            if target is None or len(f) <= target:  # the mesh of the PLY, as it is
                np.testing.assert_array_equal(obj["f"][:, :, 0] - 1, f)
            else:  # decimated: to the target or one more, or where no edge could collapse any more
                assert target <= F < len(f)
            with Image.open(out / f"{prefix}material_0.png") as im:
                assert im.size == (N, N)
                assert np.asarray(im).std() > 0
    for png in runs[0].glob("*.png"):  # two runs give the same textures
        assert png.read_bytes() == (runs[1] / png.name).read_bytes(), png.name
