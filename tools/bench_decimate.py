"""Time of mesh decimation before NeRF texturing (`--target-num-faces`): the TSDF mesh of the traced apple scene (the frames
of tools/bench_tsdf.py fused into a 256^3 grid) decimated to --target faces by fnr_mesh_decimate, and the whole textured
export (export_textured_meshes of the scene mesh, a freshly initialised fruit_nerf model at its eval sample counts) with
and without that target.

    python tools/bench_decimate.py --json out/bench_decimate.json

Reported: fnr_mesh_decimate alone (host clock around the call, which ends in a device synchronise; mean of --iters calls
after a warm-up), its rounds and the mean faces removed per round; the two exports (host clock, one warm-up each) with
their OBJ and PNG sizes; and the card's name and power limit, read in the same run.
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
from fruitnerf_b200.export.exporter_utils import export_textured_meshes  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--target", type=int, default=50000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    fr = frames(a.views, a.size, dev)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], a.grid, device=dev)
    fuse(tsdf, fr, 10)
    m = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
    del fr, tsdf
    torch.cuda.empty_cache()
    F = len(m["faces"])
    v = torch.from_numpy(m["vertices"].astype(np.float64)).to(dev)
    f = torch.from_numpy(m["faces"]).to(dev)
    r = ops.mesh_decimate(v, f, a.target)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        r = ops.mesh_decimate(v, f, a.target)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / a.iters * 1e3
    Fo = int(r["faces"].shape[0])
    out = {"card": card(), "grid": a.grid, "faces": F, "vertices": len(m["vertices"]), "target": a.target,
           "decimate": {"ms": ms, "faces_out": Fo, "vertices_out": int(r["vertices"].shape[0]), "rounds": r["rounds"],
                        "faces_removed_per_round": (F - Fo) / max(r["rounds"], 1)}}
    print(json.dumps(out), flush=True)
    from fruitnerf_b200.scripts.train import synthetic_spec

    spec = synthetic_spec("fruit_nerf", num_images=4, image_size=32)
    pipeline = spec.pipeline.setup(device=dev, test_mode="test")
    pipeline.eval()
    empty = {"vertices": np.zeros((0, 3), np.float32), "normals": np.zeros((0, 3), np.float32), "faces": np.zeros((0, 3), np.int64)}
    result = {"mesh": {"vertices": m["vertices"], "normals": m["normals"], "faces": m["faces"]}, "fruit_mesh": empty}
    out["export"] = {}
    for name, target in (("full", None), ("decimated", a.target)):
        with tempfile.TemporaryDirectory() as tmp:
            export_textured_meshes(pipeline, result, Path(tmp) / "warm", 4, target_num_faces=target)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            paths = export_textured_meshes(pipeline, result, tmp, 4, target_num_faces=target)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            out["export"][name] = {"s": t1 - t0, "obj_bytes": Path(paths["mesh_obj"]).stat().st_size,
                                   "png_bytes": Path(paths["mesh_png"]).stat().st_size}
        print(json.dumps({name: out["export"][name]}), flush=True)
    out["export"]["saved_s"] = out["export"]["full"]["s"] - out["export"]["decimated"]["s"]
    if a.json:
        a.json.parent.mkdir(parents=True, exist_ok=True)
        a.json.write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
