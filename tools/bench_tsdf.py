"""Time of the `tsdf` mesh export's kernels: fusion of ground-truth frames of the synthetic apple scene (100 views traced at
512x512 with `synthetic_scene.trace`: hit distance as depth, misses 0, the fruit mask as fruit probability) into 256^3 and
512^3 grids in batches of 10, then marching cubes of the fused grid; the torch restatement of the fusion (mesh.py on CPU
tensors) and the numpy marching cubes at 128^3 in the same run.

    python tools/bench_tsdf.py --json out/bench_tsdf.json

GPU stages are timed with CUDA events after one warm-up of the same stage; marching cubes includes its one host read
(the vertex and face counts).  The card's name and power limit are written next to the numbers.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from fruitnerf_b200 import mesh as M  # noqa: E402
from fruitnerf_b200.data.synthetic_scene import camera_rays, look_at_c2w, make_geometry, trace  # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def frames(num_views: int, size: int, dev):
    """The apple scene's orbit (three elevation rings, as make_apple_scene) traced on the device."""
    import math

    geom = make_geometry(12, 0)
    target = torch.tensor([0.0, 0.0, 0.02])
    f = 1.1 * size
    c2w, depth, rgb, fruit = [], [], [], []
    ys, xs = torch.meshgrid(torch.arange(size, device=dev), torch.arange(size, device=dev), indexing="ij")
    for i in range(num_views):
        az = 2 * math.pi * i / num_views + 0.37 * (i % 3)
        el = math.radians((12.0, 30.0, 50.0)[i % 3])
        eye = target + torch.tensor([math.cos(az) * math.cos(el), math.sin(az) * math.cos(el), math.sin(el)])
        m = look_at_c2w(eye, target).to(dev)
        o, d = camera_rays(m, f, f, size / 2, size / 2, ys.reshape(-1), xs.reshape(-1))
        col, mask, t = trace(geom, o, d)
        c2w.append(m)
        depth.append(torch.where(torch.isfinite(t), t, torch.zeros_like(t)).reshape(size, size))
        rgb.append(col.reshape(size, size, 3))
        fruit.append(mask.reshape(size, size))
    B = num_views
    full = lambda v: torch.full((B,), float(v), device=dev)  # noqa: E731
    return (torch.stack(c2w), full(f), full(f), full(size / 2), full(size / 2), torch.stack(depth), torch.stack(rgb), torch.stack(fruit))


def fuse(tsdf, fr, batch):
    for b0 in range(0, fr[0].shape[0], batch):
        tsdf.integrate(*(t[b0:b0 + batch] for t in fr))


def gpu_run(fr, n: int, batch: int, dev) -> dict:
    box = [[-1, -1, -1], [1, 1, 1]]
    fuse(M.TSDF.from_aabb(box, n, device=dev), fr, batch)  # warm-up
    tsdf = M.TSDF.from_aabb(box, n, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    fuse(tsdf, fr, batch)
    ev[1].record()
    torch.cuda.synchronize()
    fuse_ms = ev[0].elapsed_time(ev[1])
    M.marching_cubes(tsdf.values, tsdf.origin, tsdf.voxel_size, tsdf.colors, tsdf.fruit)  # warm-up
    torch.cuda.synchronize()
    ev[0].record()
    m = tsdf.get_mesh()
    ev[1].record()
    torch.cuda.synchronize()
    B = fr[0].shape[0]
    return {"grid": n, "frames": B, "batch": batch, "fuse_ms": fuse_ms, "ms_per_frame": fuse_ms / B, "ms_per_batch": fuse_ms / -(-B // batch),
            "marching_cubes_ms": ev[0].elapsed_time(ev[1]), "vertices": int(m["vertices"].shape[0]), "faces": int(m["faces"].shape[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=100)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--grids", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--host-grid", type=int, default=128)
    ap.add_argument("--host-views", type=int, default=10, help="frames the torch restatement fuses (its time is per frame)")
    ap.add_argument("--json", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "views": a.views, "size": a.size, "gpu": []}
    fr = frames(a.views, a.size, dev)
    for n in a.grids:
        out["gpu"].append(gpu_run(fr, n, a.batch, dev))
        print(json.dumps(out["gpu"][-1]), flush=True)
        torch.cuda.empty_cache()
    host = tuple(t[: a.host_views].cpu() for t in fr)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], a.host_grid)
    t0 = time.perf_counter()
    fuse(tsdf, host, a.batch)
    t1 = time.perf_counter()
    m = tsdf.get_mesh()
    t2 = time.perf_counter()
    out["host"] = {"grid": a.host_grid, "frames": a.host_views, "ms_per_frame": 1e3 * (t1 - t0) / a.host_views,
                   "marching_cubes_ms": 1e3 * (t2 - t1), "faces": int(m["faces"].shape[0]), "threads": torch.get_num_threads()}
    dtsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], a.host_grid, device=dev)
    fuse(dtsdf, tuple(t[: a.host_views] for t in fr), a.batch)
    out["host"]["gpu_equal"] = bool(torch.equal(dtsdf.values.cpu(), tsdf.values))
    print(json.dumps(out["host"]), flush=True)
    if a.json:
        a.json.parent.mkdir(parents=True, exist_ok=True)
        a.json.write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
