"""Per-fruit measurement on the device: fnr_mesh_components / _assign_centers / _measure_groups against the restatement in
measure.py (labels and counts array-equal, fp64 within 1e-12, repeated calls bit-identical), a mesh of more than 2^24
faces, the fruit meshes of the traced apple scene against its analytic fruit, and tsdf -> count -> measure end to end."""

import math

import numpy as np
import pytest
import torch

from fruitnerf_b200 import measure as ME
from fruitnerf_b200 import mesh as M
from fruitnerf_b200 import ops
from fruitnerf_b200.synthetic import sphere_lattice

from .test_measure_host import clip_above, ellipsoid, random_mesh, sphere, torus, two_spheres

pytestmark = pytest.mark.gpu

F64_KEYS = {"area": 2, "centroid": 1, "sphere": 1, "volume": 3, "coverage": 0}  # key: power of the length unit
INT_KEYS = ("faces", "boundary_edges", "nonmanifold_edges", "fit_ok", "unassigned_faces")


def meshes():
    v, f, c = two_spheres()
    cap = clip_above(*sphere(20.3, (21.7, 22.2, 22.1), 48), 22.1 + 0.3 * 20.3)
    out = {"sphere": (*sphere(), None, None), "torus": (*torus(), None, None), "ellipsoid": (*ellipsoid(), None, None),
           "cap": (*cap, None, None), "two_spheres": (v, f, None, None), "two_centres": (v, f, c, None), "two_centres_near": (v, f, c, 9.6)}
    for seed in range(3):
        rv, rf = random_mesh(seed)
        out[f"random{seed}"] = (rv, rf, None, None)
        out[f"random{seed}_centres"] = (rv, rf, np.random.default_rng(seed + 10).normal(size=(7, 3)), 1.2)
    return out


def device_labels(v, f, centres, md, dev):
    dv, df = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    if centres is None:
        lab, G = ops.mesh_components(df, len(v))
    else:
        lab, G = ops.mesh_assign_centers(dv, df, torch.from_numpy(centres).to(dev), math.inf if md is None else md), len(centres)
    return dv, df, lab, G


def bits(t):
    return t.view(torch.int64) if t.dtype == torch.float64 else t


@pytest.mark.parametrize("name", list(meshes()))
def test_kernels_match_restatement(native_lib, cuda_device, name):
    v, f, centres, md = meshes()[name]
    dv, df, lab, G = device_labels(v, f, centres, md, cuda_device)
    if centres is None:
        ref_lab, ref_G = ME.restated_components(f, len(v))
    else:
        ref_lab, ref_G = ME.restated_assign(v, f, centres, math.inf if md is None else md), len(centres)
    assert G == ref_G
    np.testing.assert_array_equal(lab.cpu().numpy(), ref_lab)
    got = ops.mesh_measure_groups(dv, df, lab, G)
    again = ops.mesh_measure_groups(dv, df, lab, G)
    for k in got:
        assert torch.equal(bits(got[k]), bits(again[k])), k
    ref = ME.restated_measure(v, f, ref_lab, ref_G)
    for k in INT_KEYS:
        np.testing.assert_array_equal(got[k].cpu().numpy(), ref[k], err_msg=k)
    L = float(np.ptp(v, axis=0).max())
    for k, p in F64_KEYS.items():
        np.testing.assert_allclose(got[k].cpu().numpy(), ref[k], rtol=1e-12, atol=1e-12 * L ** p, err_msg=k)
    np.testing.assert_allclose(got["unassigned_area"].cpu().numpy(), ref["unassigned_area"], rtol=1e-12, atol=1e-12 * L ** 2)
    if name == "two_centres_near":
        assert int(got["unassigned_faces"][0]) > 0


def test_refusals(native_lib, cuda_device):
    from fruitnerf_b200 import _lib as L

    v, f = sphere()
    dv, df = torch.from_numpy(v).to(cuda_device), torch.from_numpy(f).to(cuda_device)
    bad = df.clone()
    bad[17, 1] = len(v)
    with pytest.raises(L.FruitNerfNativeError, match="face index"):
        ops.mesh_components(bad, len(v))
    with pytest.raises(L.FruitNerfNativeError, match="face index"):
        ops.mesh_measure_groups(dv, bad, torch.zeros(len(f), dtype=torch.int32, device=cuda_device), 1)
    centre = torch.tensor([[24.2, 23.7, 24.5]], dtype=torch.float64, device=cuda_device)
    with pytest.raises(L.FruitNerfNativeError, match="face index"):
        ops.mesh_assign_centers(dv, bad, centre, 1.0)
    neg = df.clone()
    neg[3, 0] = -1
    with pytest.raises(L.FruitNerfNativeError, match="face index"):
        ME.measure_fruits(dv, neg, centre)
    lab = torch.zeros(len(f), dtype=torch.int32, device=cuda_device)
    lab[5] = 1
    with pytest.raises(L.FruitNerfNativeError, match="label"):
        ops.mesh_measure_groups(dv, df, lab, 1)
    lab[5] = -2
    with pytest.raises(L.FruitNerfNativeError, match="label"):
        ops.mesh_measure_groups(dv, df, lab, 1)
    c = torch.tensor([[0.0, float("nan"), 0.0]], dtype=torch.float64, device=cuda_device)
    with pytest.raises(L.FruitNerfNativeError, match="not finite"):
        ops.mesh_assign_centers(dv, df, c, 1.0)
    with pytest.raises(L.FruitNerfNativeError, match="max_distance"):
        ops.mesh_assign_centers(dv, df, c[:, :] * 0, 0.0)


def test_more_than_2p24_faces(native_lib, cuda_device):
    v, f, cen, radii = sphere_lattice(cuda_device)
    F, K = int(f.shape[0]), cen.shape[0]
    assert F >= 2 ** 24
    comp = ME.measure_fruits(v, f)
    assert comp["num_groups"] == K and comp["closed"].all() and (comp["fit_ok"] == 1).all()
    # components are numbered by smallest vertex index, the lattice by cell: match them through the fitted centres
    owner = np.linalg.norm(comp["center"][:, None] - cen.numpy()[None], axis=2).argmin(1)
    assert sorted(owner.tolist()) == list(range(K))
    r = radii.numpy()[owner]
    err = comp["radius"] / r - 1
    verr = comp["volume"] / (4 / 3 * math.pi * r ** 3) - 1
    print(f"\n{F} faces, {K} spheres: radius error {np.abs(err).max():.2e} max, volume error {verr.min():.2e} .. {verr.max():.2e}")
    assert np.abs(err).max() <= 0.01 and np.abs(verr).max() <= 0.01 and np.abs(comp["coverage"] - 1).max() <= 1e-9
    byc = ME.measure_fruits(v, f, cen.to(cuda_device))
    assert byc["unassigned_faces"] == 0
    np.testing.assert_array_equal(byc["faces"][owner], comp["faces"])
    np.testing.assert_allclose(byc["volume"][owner], comp["volume"], rtol=1e-9)
    lab, G = ops.mesh_components(f, v.shape[0])
    ref_lab, _ = ME.restated_components(f.cpu().numpy(), v.shape[0])
    np.testing.assert_array_equal(lab.cpu().numpy(), ref_lab)


# ---- the traced apple scene ---------------------------------------------------------------------------------------------
def traced_cloud(cuda_device, size=160):
    """The traced surface cloud of test_gpu_poisson.py::test_ground_truth_apple_scene: 10^6 points with view-oriented
    normals, colours and fruit labels."""
    from fruitnerf_b200 import pointcloud
    from fruitnerf_b200.data.synthetic_scene import camera_rays, make_apple_scene, trace

    train, ev = make_apple_scene(num_images=40, height=size, width=size, noise_std=0.0)
    cams = train.cameras
    pts, col, fruit, view = [], [], [], []
    ys, xs = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    for c2w in torch.cat([train.cameras.camera_to_worlds, ev.cameras.camera_to_worlds]):
        o, d = camera_rays(c2w, cams.fx, cams.fy, cams.cx, cams.cy, ys.reshape(-1), xs.reshape(-1))
        rgb, m, t = trace(train.geometry, o, d)
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
    return pts, pointcloud.estimate_normals(pts, 30, view).float(), col.float(), fruit.float()


def check_fruit(name, fm, geom, seen, voxel, cuda_device):
    cent = geom.fruit_centers.double()
    R = float(geom.fruit_radius)
    res = ME.measure_fruits(torch.from_numpy(np.ascontiguousarray(fm[0], np.float64)).to(cuda_device), torch.from_numpy(fm[4]).to(cuda_device),
                            cent.to(cuda_device), 2 * R)
    truth = 4 / 3 * math.pi * R ** 3
    checked = 0
    print(f"\n{name}: {len(fm[4])} faces, {res['unassigned_faces']} unassigned, voxel {voxel:.5f}")
    for k in range(cent.shape[0]):
        line = (f"  fruit {k}: {int(seen[k])} px, {res['faces'][k]} faces, coverage {res['coverage'][k]:.3f}, radius "
                f"{res['radius'][k]:.5f} ({(res['radius'][k] - R) / voxel:+.2f} voxel), rms {res['rms'][k]:.5f}, volume_extrapolated "
                f"error {100 * (res['volume_extrapolated'][k] / truth - 1):+.1f} %")
        print(line)
        if int(seen[k]) >= 50 and res["coverage"][k] >= 0.25:
            checked += 1
            assert abs(res["radius"][k] - R) <= voxel, line
            assert res["volume"][k] > 0 and res["fit_ok"][k] == 1, line
    assert checked >= 3
    return res


def test_ground_truth_apple_scene(native_lib, cuda_device):
    from fruitnerf_b200 import poisson as P

    from .test_gpu_mesh import traced_views

    geom, frames, fruit_hits = traced_views(cuda_device)
    cent = geom.fruit_centers.double()
    owner = (fruit_hits.double()[:, None] - cent[None]).norm(dim=-1).argmin(dim=1)
    seen = torch.bincount(owner, minlength=cent.shape[0])
    n = 192
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], n, device=cuda_device)
    for b0 in range(0, 40, 10):
        tsdf.integrate(*(t[b0:b0 + 10] for t in frames))
    m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
    fm = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    check_fruit("tsdf 192^3 fruit mesh", fm, geom, seen, 2.0 / n, cuda_device)
    out = P.reconstruct(*traced_cloud(cuda_device), depth=8)
    pm = out["mesh"]
    fm = M.fruit_submesh(pm["vertices"], pm["normals"], pm["colors"], pm["fruit"], pm["faces"])
    check_fruit("poisson depth 8 fruit mesh", fm, geom, seen, out["side"] / 256, cuda_device)


# ---- end to end ---------------------------------------------------------------------------------------------------------
def test_tsdf_count_measure_end_to_end(native_lib, cuda_device, tmp_path):
    import json

    from fruitnerf_b200.scripts import count as count_cli
    from fruitnerf_b200.scripts import measure as measure_cli
    from fruitnerf_b200.scripts.exporter import entrypoint
    from fruitnerf_b200.trainer import Trainer

    from .test_gpu_mesh import _tiny_spec

    torch.manual_seed(0)
    run = tmp_path / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    box = ["--bounding-box-min", "-0.8", "-0.8", "-0.8", "--bounding-box-max", "0.8", "0.8", "0.8"]
    entrypoint(["tsdf", "--load-config", str(run / "config.yml"), "--resolution", "64", *box, "--output-dir", str(tmp_path / "mesh")])
    pcds = entrypoint(["semantic-pointcloud", "--load-config", str(run / "config.yml"), "--output-dir", str(tmp_path / "pcd"),
                       "--num-points-per-side", "192", "--stratified-jitter", "false", *box])
    # the briefly trained model exports a sparse fruit cloud: count it with a wide radius and small clusters
    count = count_cli.main(["--pcd", pcds["semantic_colormap"]["path"], "--eps", "0.1", "--min-samples", "3", "--remove-outliers-nb-points", "0",
                            "--down-sample", "0", "--json", str(tmp_path / "count.json")])
    # The chain as a user runs it.  How many centres count finds, and whether the fruit mesh has faces, depends on how well
    # the briefly trained model learned the fruit; the scene mesh always has faces (the export refuses an empty one).
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply

    mesh = tmp_path / "mesh" / "fruit_mesh.ply"
    if len(read_mesh_ply(mesh)[3]) == 0:
        mesh = tmp_path / "mesh" / "tsdf_mesh.ply"
    v, _, _, f = read_mesh_ply(mesh)
    common = ["--mesh", str(mesh), "--transform-json", str(run / "dataparser_transforms.json")]
    out = measure_cli.main([*common, "--count-json", str(tmp_path / "count.json"), "--json", str(tmp_path / "measure.json"),
                            "--csv", str(tmp_path / "measure.csv")])
    print(f"\n{count['count']} count centres, {out['num_groups']} rows, {out['unassigned_faces']} unassigned faces of {len(f)}")
    assert out["mode"] == "centers" and out["num_groups"] == len(count["centers"]) == len(out["groups"])
    assert [r["id"] for r in out["groups"]] == list(range(len(count["centers"])))
    assert json.loads((tmp_path / "measure.json").read_text()) == out
    assert len((tmp_path / "measure.csv").read_text().splitlines()) == 1 + len(count["centers"])
    # Known centres in count's frame (2 / scale times the mesh's): three mesh vertices.  Every face goes to one of them.
    scale = json.loads((run / "dataparser_transforms.json").read_text())["scale"]
    known = v[f[[0, len(f) // 2, len(f) - 1], 0]] * 2 / scale
    (tmp_path / "known.json").write_text(json.dumps({"count": 3, "centers": known.tolist()}))
    out = measure_cli.main([*common, "--count-json", str(tmp_path / "known.json")])
    assert out["num_groups"] == 3 and out["unassigned_faces"] == 0
    assert sum(r["faces"] for r in out["groups"]) == len(f)
    direct = ME.measure_fruits(v, f, known * scale / 2)
    np.testing.assert_array_equal([r["faces"] for r in out["groups"]], direct["faces"])
    np.testing.assert_allclose([r["area"] for r in out["groups"]], direct["area"] / scale ** 2, rtol=1e-9)
