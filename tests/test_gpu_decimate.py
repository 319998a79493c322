"""Mesh decimation on the device: fnr_mesh_decimate bit for bit against the numpy restatement in decimate.py (faces,
round counts, vertices and normals) on the host test's marched meshes and on the TSDF and Poisson meshes of the traced
apple scene, repeatability, a mesh of about two million faces, NeRF texturing of decimated meshes and both export commands
end to end with --target-num-faces."""
import numpy as np
import pytest
import torch
from PIL import Image

from fruitnerf_b200 import decimate as D
from fruitnerf_b200 import mesh as M
from fruitnerf_b200 import ops
from fruitnerf_b200 import texture as T

from .test_decimate_host import FRACTIONS, MESHES, boundary_loops, check_manifold, components_euler
from .test_gpu_texture import TraceModel, quantised_trace, trained_run  # noqa: F401  (trained_run is a fixture)

pytestmark = pytest.mark.gpu


def device_decimate(v, f, N, dev):
    r = ops.mesh_decimate(torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(dev), torch.from_numpy(np.ascontiguousarray(f, np.int64)).to(dev), N)
    return {k: (x.cpu().numpy() if torch.is_tensor(x) else x) for k, x in r.items()}


def assert_same(got, want):
    assert got["rounds"] == want["rounds"]
    assert np.array_equal(got["faces"], want["faces"])
    assert np.array_equal(got["vertices"].view(np.int64), want["vertices"].view(np.int64))
    assert np.array_equal(got["normals"].view(np.int64), want["normals"].view(np.int64))


@pytest.mark.parametrize("frac", FRACTIONS)
@pytest.mark.parametrize("name", list(MESHES))
def test_device_is_the_restatement(native_lib, cuda_device, name, frac):
    v, f = MESHES[name][0]()
    N = max(1, int(round(len(f) * frac)))
    assert_same(device_decimate(v, f, N, cuda_device), D.restated_decimate(v, f, N))


def test_two_calls_give_identical_bits(native_lib, cuda_device):
    v, f = MESHES["torus"][0]()
    a, b = device_decimate(v, f, 300, cuda_device), device_decimate(v, f, 300, cuda_device)
    assert_same(a, b)


def test_mesh_at_the_target_and_refusals(native_lib, cuda_device):
    v, f = MESHES["sphere"][0]()
    r = device_decimate(v, f, len(f), cuda_device)
    assert r["rounds"] == 0 and np.array_equal(r["faces"], f) and np.array_equal(r["vertices"], v)
    bad = f.copy()
    bad[5, 1] = len(v)
    with pytest.raises(RuntimeError, match="outside"):
        device_decimate(v, bad, 100, cuda_device)


def apple_meshes(dev):
    """The TSDF (128^3) and Poisson (depth 7) scene and fruit meshes of the traced apple scene, as test_gpu_texture.py
    builds them at larger sizes."""
    from fruitnerf_b200 import pointcloud
    from fruitnerf_b200 import poisson as P
    from fruitnerf_b200.data.synthetic_scene import camera_rays, make_apple_scene, trace

    from .test_gpu_mesh import traced_views

    geom, frames, _ = traced_views(dev)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], 128, device=dev)
    for b0 in range(0, 40, 10):
        tsdf.integrate(*(t[b0:b0 + 10] for t in frames))
    out = {}
    m = {k: (None if x is None else x.cpu().numpy()) for k, x in tsdf.get_mesh().items()}
    fv, fn, _, _, fidx = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    out["tsdf"], out["tsdf_fruit"] = m, {"vertices": fv, "normals": fn, "faces": fidx}
    size = 96
    train, _ = make_apple_scene(num_images=20, height=size, width=size, noise_std=0.0)
    cams = train.cameras
    ys, xs = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    pts, col, fruit, view = [], [], [], []
    for c2w in cams.camera_to_worlds:
        o, d = camera_rays(c2w, cams.fx, cams.fy, cams.cx, cams.cy, ys.reshape(-1), xs.reshape(-1))
        rgb, mk, t = trace(train.geometry, o, d)
        p = o + d * torch.where(torch.isfinite(t), t, torch.zeros_like(t))[:, None]
        keep = torch.isfinite(t) & (p.abs() < 1).all(dim=1)
        pts.append(p[keep])
        col.append(rgb[keep])
        fruit.append(mk[keep, 0])
        view.append(d[keep])
    pts, col, fruit, view = (torch.cat(a).to(dev) for a in (pts, col, fruit, view))
    nrm = pointcloud.estimate_normals(pts.double(), 30, view).float()
    pm = P.reconstruct(pts.double(), nrm, col.float(), fruit.float(), depth=7)["mesh"]
    pm = {k: (x.cpu().numpy() if torch.is_tensor(x) else x) for k, x in pm.items()}
    fv, fn, _, _, fidx = M.fruit_submesh(pm["vertices"], pm["normals"], pm["colors"], pm["fruit"], pm["faces"])
    out["poisson"], out["poisson_fruit"] = pm, {"vertices": fv, "normals": fn, "faces": fidx}
    return geom, out


@pytest.fixture(scope="module")
def apple(native_lib, cuda_device):
    return apple_meshes(cuda_device)


@pytest.mark.parametrize("key", ["tsdf", "tsdf_fruit", "poisson", "poisson_fruit"])
def test_apple_scene_meshes_are_the_restatement(apple, cuda_device, key):
    m = apple[1][key]
    v, f = np.asarray(m["vertices"], np.float64), np.asarray(m["faces"], np.int64)
    assert len(f) > 1000
    N = len(f) // 3
    got = device_decimate(v, f, N, cuda_device)
    assert_same(got, D.restated_decimate(v, f, N))
    assert len(got["faces"]) in (N, N + 1)
    print(f"\n{key}: {len(f)} -> {len(got['faces'])} faces in {got['rounds']} rounds")


def test_two_million_faces(native_lib, cuda_device):
    n = 800
    x = torch.linspace(-1, 1, n, device=cuda_device)
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    sdf = torch.sqrt(X * X + Y * Y + Z * Z) - 0.7
    m = M.marching_cubes(sdf, (-1.0, -1.0, -1.0), (2.0 / (n - 1),) * 3)
    del X, Y, Z, sdf
    v, f = m["vertices"].double(), m["faces"]
    F = int(f.shape[0])
    assert F > 2_000_000
    N = F // 50
    a = ops.mesh_decimate(v, f, N)
    b = ops.mesh_decimate(v, f, N)
    for k in ("vertices", "normals", "faces"):
        assert torch.equal(a[k], b[k]), k
    ov, of = a["vertices"].cpu().numpy(), a["faces"].cpu().numpy()
    assert len(of) in (N, N + 1)
    check_manifold(of, len(ov))
    assert boundary_loops(of) == 0 and components_euler(ov, of) == [2]
    assert np.abs(np.linalg.norm(ov, axis=1) - 0.7).max() < 4 * 2.0 / (n - 1)
    print(f"\n{F} faces -> {len(of)} in {a['rounds']} rounds")


def test_traced_apple_scene_textured_with_a_target(apple, cuda_device, tmp_path):
    from types import SimpleNamespace

    from fruitnerf_b200.export.exporter_utils import decimate_for_texture, export_textured_meshes

    geom, meshes = apple
    model = TraceModel(geom, cuda_device, 1 << 16)
    res = {"mesh": meshes["tsdf"], "fruit_mesh": meshes["tsdf_fruit"]}
    N = 12000  # reachable on the 113 898-face scene mesh; the 2280-face fruit mesh stays as it is
    paths = export_textured_meshes(SimpleNamespace(model=model), res, tmp_path, 4, target_num_faces=N)
    for key, prefix in (("mesh", ""), ("fruit_mesh", "fruit_")):
        d = decimate_for_texture(res[key], N, cuda_device)
        F = len(d["faces"])
        assert F in (N, N + 1) if len(res[key]["faces"]) > N else d is res[key]
        W, H = T.atlas_size(F, 4)
        image = np.asarray(Image.open(paths[f"{key}_png"]).convert("RGB"))
        assert image.shape == (H, W, 3)
        raylen = float(np.float32(2 * float(ops.mesh_mean_edge(torch.from_numpy(d["vertices"]).to(cuda_device),
                                                               torch.from_numpy(d["faces"]).to(cuda_device)))))
        assert np.array_equal(image, quantised_trace(model, d, 4, W, H, raylen, cuda_device)), key
        obj = T.read_textured_obj(paths[f"{key}_obj"])
        assert len(obj["f"]) == F and len(obj["v"]) == len(d["vertices"])
    # the fruit texel origins of a decimated fruit mesh lie outside their fruit spheres
    d = decimate_for_texture(res["fruit_mesh"], len(res["fruit_mesh"]["faces"]) // 3, cuda_device)
    F = len(d["faces"])
    W, H = T.atlas_size(F, 4)
    raylen = float(np.float32(2 * float(ops.mesh_mean_edge(torch.from_numpy(d["vertices"]).to(cuda_device), torch.from_numpy(d["faces"]).to(cuda_device)))))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)  # noqa: E731
    o, _ = ops.texel_rays(t(d["vertices"]), t(d["normals"]), t(d["faces"]), 4, W, H, raylen, 0, W * H)
    owned = torch.from_numpy(T.texel_owners(F, 4).reshape(-1) >= 0)
    o = o.cpu().double()[owned]
    cent = geom.fruit_centers.double().cpu()
    k = (o[:, None] - cent[None]).norm(dim=-1).argmin(dim=1)
    outside = float(((o - cent[k]).norm(dim=-1) > float(geom.fruit_radius)).float().mean())
    print(f"\nfruit texel origins outside their sphere: {outside:.5f}")
    assert outside >= 0.99


@pytest.mark.parametrize("command, args, plys", [
    ("tsdf", ["--resolution", "64", "--bounding-box-min", "-0.8", "-0.8", "-0.8", "--bounding-box-max", "0.8", "0.8", "0.8"],
     ("tsdf_mesh.ply", "fruit_mesh.ply")),
    ("poisson", ["--num-points", "30000", "--depth", "6", "--normal-method", "open3d"], ("poisson_mesh.ply", "fruit_poisson_mesh.ply")),
])
def test_cli_end_to_end_with_a_target(trained_run, tmp_path, command, args, plys):  # noqa: F811
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply
    from fruitnerf_b200.scripts.exporter import entrypoint

    base = [command, "--load-config", str(trained_run / "config.yml"), *args]
    torch.manual_seed(0)
    entrypoint([*base, "--output-dir", str(tmp_path / "plain")])
    runs = []
    for k in range(2):
        torch.manual_seed(0)
        out = tmp_path / f"nerf{k}"
        _, _, _, f = read_mesh_ply(tmp_path / "plain" / plys[0])
        N = max(1, len(f) // 4)
        entrypoint([*base, "--output-dir", str(out), "--texture-method", "nerf", "--unwrap-method", "custom", "--target-num-faces", str(N)])
        runs.append(out)
        for ply in plys:  # the PLYs are never decimated
            assert (out / ply).read_bytes() == (tmp_path / "plain" / ply).read_bytes(), ply
        obj = T.read_textured_obj(out / "mesh.obj")
        assert len(obj["f"]) in (N, N + 1)
        with Image.open(out / "material_0.png") as im:
            assert im.size == T.atlas_size(len(obj["f"]), 4)
    for name in [p.name for p in runs[0].glob("*.obj")] + [p.name for p in runs[0].glob("*.png")]:
        assert (runs[0] / name).read_bytes() == (runs[1] / name).read_bytes(), name
