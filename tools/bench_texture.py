"""Time of the NeRF-textured mesh export (`--texture-method nerf --unwrap-method custom`): the TSDF mesh of the traced apple
scene (the frames of tools/bench_tsdf.py fused into a 256^3 grid), textured at --px-per-uv-triangle texels per face by a
fruit_nerf model at its eval sample counts.  The model is freshly initialised: the field's cost does not depend on its
weights.

    python tools/bench_texture.py --json out/bench_texture.json

Reported: fnr_texel_rays alone over the whole atlas, in one launch and in the export's chunks (CUDA events over --iters
repeats after a warm-up); the whole export_textured_mesh call (host clock around it: rays, forward, composition, the one
device-to-host copy, PNG and OBJ / MTL writing), and the OBJ / MTL writing alone.  Texel counts, texels/s and the card's
name and power limit are written next to the numbers.
"""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_tsdf import card, frames, fuse  # noqa: E402

from fruitnerf_b200 import mesh as M  # noqa: E402
from fruitnerf_b200 import ops  # noqa: E402
from fruitnerf_b200 import texture as T  # noqa: E402
from fruitnerf_b200.export.exporter_utils import export_textured_mesh  # noqa: E402


def timed(fn, iters: int) -> float:
    """Mean ms per call of ``fn`` over ``iters`` calls, CUDA events, after one warm-up."""
    fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--px-per-uv-triangle", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    p = a.px_per_uv_triangle
    fr = frames(a.views, a.size, dev)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], a.grid, device=dev)
    fuse(tsdf, fr, 10)
    m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
    del fr, tsdf
    torch.cuda.empty_cache()
    F = len(m["faces"])
    W, H = T.atlas_size(F, p)
    P = W * H
    out = {"card": card(), "grid": a.grid, "faces": F, "px_per_uv_triangle": p, "atlas": [W, H], "texels": P,
           "owned_texels": int((T.texel_owners(F, p) >= 0).sum())}
    v, n, f = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (m["vertices"], m["normals"], m["faces"]))
    raylen = float(np.float32(2 * float(ops.mesh_mean_edge(v, f))))
    out["mean_edge_ms"] = timed(lambda: ops.mesh_mean_edge(v, f), a.iters)
    o = torch.empty((P, 3), dtype=torch.float32, device=dev)
    d = torch.empty((P, 3), dtype=torch.float32, device=dev)
    whole = timed(lambda: ops.texel_rays(v, n, f, p, W, H, raylen, 0, P, out=(o, d)), a.iters)
    from fruitnerf_b200.scripts.train import synthetic_spec

    spec = synthetic_spec("fruit_nerf", num_images=4, image_size=32)
    pipeline = spec.pipeline.setup(device=dev, test_mode="test")
    pipeline.eval()
    chunk = int(pipeline.model.config.eval_num_rays_per_chunk)

    def chunked():
        for t0 in range(0, P, chunk):
            ops.texel_rays(v, n, f, p, W, H, raylen, t0, min(chunk, P - t0), out=(o, d))

    per_chunks = timed(chunked, max(1, a.iters // 4))
    out["texel_rays"] = {"one_launch_ms": whole, "texels_per_s": P / whole * 1e3, "in_chunks_ms": per_chunks, "chunk": chunk,
                         "bytes_written": P * 24}
    print(json.dumps(out), flush=True)
    mesh = {"vertices": m["vertices"], "normals": m["normals"], "faces": m["faces"]}
    with tempfile.TemporaryDirectory() as tmp:
        export_textured_mesh(pipeline, mesh, tmp, "warm_", p)  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = export_textured_mesh(pipeline, mesh, tmp, "", p)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        T.write_textured_obj(Path(tmp) / "again.obj", "again.mtl", "again.png", m["vertices"], m["normals"], m["faces"], T.uv_coordinates(F, p))
        t2 = time.perf_counter()
        sizes = {k: Path(r[k]).stat().st_size for k in ("obj", "png")}
    out["export"] = {"whole_s": t1 - t0, "texels_per_s": P / (t1 - t0), "obj_mtl_write_s": t2 - t1, "obj_bytes": sizes["obj"],
                     "png_bytes": sizes["png"], "raylen": r["raylen"]}
    print(json.dumps(out["export"]), flush=True)
    if a.json:
        a.json.parent.mkdir(parents=True, exist_ok=True)
        a.json.write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
