"""The `charts` UV unwrap (`--unwrap-method charts`, DESIGN section 4.3r) against the `custom` atlas: the TSDF mesh of the
traced apple scene (the frames of tools/bench_tsdf.py fused into a 256^3 grid), as it is and decimated to
--target-num-faces.

    python tools/bench_unwrap.py --json out/bench_unwrap.json

Reported per mesh: the wall time of each unwrap stage (fnr_chart_unwrap with stage timing: labels and edge sort, charts,
packing, raster and conflict rounds, owners and compaction; the stream drained between stages), the whole unwrap without
stage timing, the texel rays of all owned texels (CUDA events), the whole textured export with a freshly initialised
fruit_nerf model (the field's cost does not depend on its weights) for `charts` and `custom`, the chart count, rounds,
scale and owned fraction, and the largest / smallest face area.  Then the texture error: both meshes textured with the
analytic scene as the model, and the mean absolute difference between the texture (bilinear at the vt of the point) and
trace() at 100 000 area-uniform random surface points, for `charts` at N and for `custom` at the --px-per-uv-triangle
whose atlas has the nearest texel count.  The card's name and power limit are written next to the numbers.
"""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_tsdf import card, frames, fuse  # noqa: E402

from fruitnerf_b200 import mesh as M  # noqa: E402
from fruitnerf_b200 import ops  # noqa: E402
from fruitnerf_b200 import texture as T  # noqa: E402
from fruitnerf_b200.data.synthetic_scene import make_geometry, trace  # noqa: E402
from fruitnerf_b200.export.exporter_utils import decimate_for_texture, export_textured_mesh  # noqa: E402


class TraceModel(torch.nn.Module):
    """A model whose 'rgb' is the analytic scene's colour along each ray."""

    def __init__(self, geom, device, chunk):
        super().__init__()
        self.geom = geom
        self.anchor = torch.nn.Parameter(torch.zeros(1, device=device))
        self.config = SimpleNamespace(eval_num_rays_per_chunk=chunk)

    @property
    def device(self):
        return self.anchor.device

    def forward(self, bundle):
        return {"rgb": trace(self.geom, bundle.origins, bundle.directions)[0]}


def timed(fn, iters: int) -> float:
    fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def wall(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def bilinear(image, uv):
    H, W, _ = image.shape
    x = np.clip(uv[:, 0] * W - 0.5, 0, W - 1)
    y = np.clip((1 - uv[:, 1]) * H - 0.5, 0, H - 1)
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    img = image.astype(np.float64) / 255
    return (img[y0, x0] * (1 - fx) + img[y0, x1] * fx) * (1 - fy) + (img[y1, x0] * (1 - fx) + img[y1, x1] * fx) * fy


def texture_error(geom, mesh, png, obj_path, points: int, offset: float) -> float:
    """Mean absolute difference (over points and channels) between the texture and trace() at area-uniform points."""
    from PIL import Image

    image = np.asarray(Image.open(png).convert("RGB"))
    obj = T.read_textured_obj(obj_path)
    v = np.asarray(mesh["vertices"], np.float64)
    f = np.asarray(mesh["faces"], np.int64)
    tri = v[f]
    cr = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    area = 0.5 * np.linalg.norm(cr, axis=1)
    rng = np.random.default_rng(0)
    face = rng.choice(len(f), points, p=area / area.sum())
    w = rng.dirichlet(np.ones(3), points)
    x = np.einsum("pk,pkd->pd", w, tri[face])
    n = cr[face] / np.linalg.norm(cr[face], axis=1, keepdims=True)
    vt = np.einsum("pk,pkd->pd", w, obj["vt"][obj["f"][face, :, 1] - 1])
    ref = trace(geom, torch.from_numpy(x + offset * n).float(), -torch.from_numpy(n).float())[0].double().numpy()
    return float(np.abs(bilinear(image, vt) - ref).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--num-pixels-per-side", type=int, default=1024)
    ap.add_argument("--target-num-faces", type=int, default=50000)
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    N = a.num_pixels_per_side
    fr = frames(a.views, a.size, dev)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], a.grid, device=dev)
    fuse(tsdf, fr, 10)
    m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
    del fr, tsdf
    torch.cuda.empty_cache()
    full = {"vertices": m["vertices"], "normals": m["normals"], "faces": m["faces"]}
    meshes = {"full": full, "decimated": decimate_for_texture(full, a.target_num_faces, dev)}
    from fruitnerf_b200.scripts.train import synthetic_spec

    spec = synthetic_spec("fruit_nerf", num_images=4, image_size=32)
    pipeline = spec.pipeline.setup(device=dev, test_mode="test")
    pipeline.eval()
    geom = make_geometry(12, 0)
    tracer = SimpleNamespace(model=TraceModel(geom, dev, 1 << 16))
    out = {"card": card(), "grid": a.grid, "num_pixels_per_side": N, "target_num_faces": a.target_num_faces}
    for name, mesh in meshes.items():
        F = len(mesh["faces"])
        v, n, f = (torch.from_numpy(np.ascontiguousarray(mesh[k], dt)).to(dev) for k, dt in
                   (("vertices", np.float32), ("normals", np.float32), ("faces", np.int64)))
        try:
            ops.chart_unwrap(v, f, N)  # warm-up
        except T.AtlasTooLargeError as e:
            out[name] = {"faces": F, "refused": str(e)}
            print(json.dumps({name: out[name]}), flush=True)
            continue
        u = ops.chart_unwrap(v, f, N, timing=True)
        whole = wall(lambda: ops.chart_unwrap(v, f, N))
        raylen = float(np.float32(2 * float(ops.mesh_mean_edge(v, f))))
        n_owned = u["num_owned"]
        o = torch.empty((n_owned, 3), dtype=torch.float32, device=dev)
        d = torch.empty((n_owned, 3), dtype=torch.float32, device=dev)
        rays_ms = timed(lambda: ops.chart_texel_rays(v, n, f, u["texel_faces"], u["barycentrics"], raylen, 0, n_owned, out=(o, d)), a.iters)
        tri = np.asarray(mesh["vertices"], np.float64)[np.asarray(mesh["faces"])]
        area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
        # custom's atlas nearest in texel count to N^2
        p = min(range(2, 33), key=lambda q: abs(T.atlas_layout(F, q)[1] * T.atlas_layout(F, q)[2] - N * N))
        r = {"faces": F, "stage_ms": dict(zip(("labels_and_edge_sort", "charts", "packing", "raster_and_conflicts", "owners_and_compaction"),
                                                u["stage_ms"])),
             "unwrap_ms": whole * 1e3, "charts": u["num_charts"], "rounds": u["rounds"], "scale": u["scale"], "owned": n_owned,
             "owned_fraction": n_owned / (N * N), "chart_texel_rays_ms": rays_ms, "face_area_max": float(area.max()),
             "face_area_min": float(area.min()), "face_area_min_nonzero": float(area[area > 0].min()), "custom_px_per_uv_triangle": p,
             "custom_texels": int(T.atlas_layout(F, p)[1] * T.atlas_layout(F, p)[2])}
        with tempfile.TemporaryDirectory() as tmp:
            export_textured_mesh(pipeline, mesh, tmp, "warm_", unwrap_method="charts", num_pixels_per_side=N)
            r["export_charts_s"] = wall(lambda: export_textured_mesh(pipeline, mesh, tmp, "c_", unwrap_method="charts", num_pixels_per_side=N))
            r["export_custom_p4_s"] = wall(lambda: export_textured_mesh(pipeline, mesh, tmp, "p4_", 4))
            export_textured_mesh(tracer, mesh, tmp, "tc_", unwrap_method="charts", num_pixels_per_side=N)
            export_textured_mesh(tracer, mesh, tmp, "tu_", p)
            off = 2.0 * 2.0 / a.grid
            r["mae_charts"] = texture_error(geom, mesh, Path(tmp) / "tc_material_0.png", Path(tmp) / "tc_mesh.obj", a.points, off)
            r["mae_custom"] = texture_error(geom, mesh, Path(tmp) / "tu_material_0.png", Path(tmp) / "tu_mesh.obj", a.points, off)
        out[name] = r
        print(json.dumps({name: r}), flush=True)
    if a.json:
        a.json.parent.mkdir(parents=True, exist_ok=True)
        a.json.write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
