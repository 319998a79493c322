"""Time of the `poisson` mesh export's stages on 10^6 points of the synthetic apple scene (ground-truth hits of 60 traced
256x256 views inside [-1, 1]^3, normals estimated from 30 neighbours and flipped against the view direction) at depths 8
and 9, and of the numpy / scipy restatement at depth 5 on 10^5 of the points in the same run (its sparse direct solve at
depth 6, 274 625 unknowns, did not finish within 10 minutes on a CPU).

    python tools/bench_poisson.py --json out/bench_poisson.json

Per depth, after one warm-up of the whole reconstruction:
- sort + splat + rhs: CUDA events around ops.poisson_splat (it includes the one host read of the point check), and the
  kernel split from a torch.profiler run of the same call (sort = the grid kernels and CUB, splat_kernel, rhs_kernel);
- solve: CUDA events around ops.poisson_solve (it reads the residual back once per iteration); its iterations; ms per
  iteration = the device time of the finest depth's CG kernels (`finest_cg_ms`, from a profiler run) over its
  iterations; bytes per iteration from the shapes (`cg_bytes`) over 3.35 TB/s;
- iso-value (ops.poisson_sample and the fp64 mean), marching cubes (the two passes of the mesh and of the density) and
  the trim (host), each with events or a host clock after a device synchronise;
- vertex and face counts before and after the trim.
The card's name and power limit are written next to the numbers.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from fruitnerf_b200 import ops, pointcloud  # noqa: E402
from fruitnerf_b200 import poisson as P  # noqa: E402
from fruitnerf_b200.data.synthetic_scene import camera_rays, look_at_c2w, make_geometry, trace  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def cloud(num_points: int, views: int, size: int, dev):
    """Ground-truth hits of the apple scene's orbit inside [-1, 1]^3: points (fp64), estimated normals, colours, fruit."""
    import math

    geom = make_geometry(12, 0)
    target = torch.tensor([0.0, 0.0, 0.02])
    f = 1.1 * size
    ys, xs = torch.meshgrid(torch.arange(size, device=dev), torch.arange(size, device=dev), indexing="ij")
    pts, col, fr, view = [], [], [], []
    for i in range(views):
        az = 2 * math.pi * i / views + 0.37 * (i % 3)
        el = math.radians((12.0, 30.0, 50.0)[i % 3])
        eye = target + torch.tensor([math.cos(az) * math.cos(el), math.sin(az) * math.cos(el), math.sin(el)])
        o, d = camera_rays(look_at_c2w(eye, target).to(dev), f, f, size / 2, size / 2, ys.reshape(-1), xs.reshape(-1))
        rgb, m, t = trace(geom, o, d)
        p = o + d * torch.where(torch.isfinite(t), t, torch.zeros_like(t))[:, None]
        keep = torch.isfinite(t) & (p.abs() < 1).all(dim=1)
        pts.append(p[keep])
        col.append(rgb[keep])
        fr.append(m[keep, 0])
        view.append(d[keep])
    pts, col, fr, view = (torch.cat(a) for a in (pts, col, fr, view))
    sel = torch.randperm(pts.shape[0], generator=torch.Generator().manual_seed(0))[:num_points].to(dev)
    pts, col, fr, view = (a[sel] for a in (pts, col, fr, view))
    pts = pts.double()
    return pts, pointcloud.estimate_normals(pts, 30, view).float(), col.float(), fr.float()


def cg_bytes(n: int, depth: int) -> int:
    """Least DRAM bytes of one CG iteration at one depth, every array read or written once per kernel: point_sample
    (t 24 B, key 8 B, 8 grid values 32 B, sample 8 B per point), apply (x, y, the cell map, and per point 8 visits of t
    and its sample, 32 B), update (p, Ap, D, x, r read; x, r, z written) and direction (z, p read; p written)."""
    R = 2 ** depth
    M = (R + 1) ** 3
    point_sample = n * (24 + 8 + 32 + 8)
    apply = 4 * M + 4 * M + 4 * R ** 3 + 8 * n * 32
    update = 8 * 4 * M
    direction = 3 * 4 * M
    return point_sample + apply + update + direction


def kernel_events(fn) -> list:
    """(name, device ms) of every kernel of one call of fn, in launch order."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == "CUDA"]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, e.device_time_total / 1e3) for e in ev]


def kernel_times(fn) -> dict:
    """Device time (ms) per kernel name of one call of fn."""
    out = defaultdict(float)
    for name, ms in kernel_events(fn):
        out[name] += ms
    return dict(out)


def finest_cg_ms(events: list, iters: int) -> float:
    """Device time of the finest level's CG loop: its last `iters` iterations are the last launches of the loop's
    kernels (point_sample + apply, two scalar steps and the update per iteration, a direction update on all but the last)."""
    want = {"point_sample_kernel": iters, "apply_kernel": iters, "cg_scalars_kernel": 2 * iters, "cg_update_kernel": iters,
            "cg_direction_kernel": max(iters - 1, 0)}
    total = 0.0
    for key, k in want.items():
        ms = [t for name, t in events if key in name]
        total += sum(ms[len(ms) - k:]) if k else 0.0
    return total


def grouped(times: dict) -> dict:
    g = defaultdict(float)
    for name, ms in times.items():
        if "splat_kernel" in name:
            g["splat"] += ms
        elif "rhs_kernel" in name:
            g["rhs"] += ms
        elif any(k in name for k in ("apply_kernel", "point_sample_kernel", "cg_", "diag_kernel", "prolong_kernel")):
            g["cg"] += ms
        else:
            g["sort"] += ms
    return dict(g)


def timed(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    r = fn()
    ev[1].record()
    torch.cuda.synchronize()
    return r, ev[0].elapsed_time(ev[1])


def gpu_run(pts, nrm, col, fr, depth: int) -> dict:
    P.reconstruct(pts, nrm, col, fr, depth=depth)  # warm-up
    origin, side = P.cube_of(pts)
    n = int(pts.shape[0])
    _, splat_ms = timed(lambda: ops.poisson_splat(pts, nrm, depth, origin, side, col, fr))
    splat_split = grouped(kernel_times(lambda: ops.poisson_splat(pts, nrm, depth, origin, side, col, fr)))
    s, solve_ms = timed(lambda: ops.poisson_solve(pts, nrm, depth, origin, side, col, fr))
    events = kernel_events(lambda: ops.poisson_solve(pts, nrm, depth, origin, side, col, fr))
    fine_ms_per_iter = finest_cg_ms(events, s["iterations"]) / max(s["iterations"], 1)
    iso, iso_ms = timed(lambda: float(ops.poisson_sample(pts, s["chi"], depth, origin, side).double().mean()))
    R = 2 ** depth
    dims = (R + 1,) * 3
    values = (s["chi"] - iso).reshape(dims)
    org32, vox32 = np.asarray(origin, np.float32), np.float32(side / R)

    def mc():
        m = ops.marching_cubes(values, org32, vox32, s["colors"].reshape(dims + (3,)), s["fruit"].reshape(dims))
        m["density"] = ops.marching_cubes(values, org32, vox32, None, s["density"].reshape(dims))["fruit"]
        return m

    m, mc_ms = timed(mc)
    t0 = time.perf_counter()
    full = {k: v.cpu().numpy() for k, v in m.items() if k != "fruit" or v is not None}
    kept = P.trim_by_density(full, full["density"])
    trim_ms = 1e3 * (time.perf_counter() - t0)
    bpi = cg_bytes(n, depth)
    return {"depth": depth, "points": n, "nodes": (R + 1) ** 3, "sort_splat_rhs_ms": splat_ms, "kernel_ms": splat_split,
            "solve_ms": solve_ms, "iterations": s["iterations"], "total_iterations": s["total_iterations"], "residual": s["residual"],
            "ms_per_iteration": fine_ms_per_iter, "bytes_per_iteration": bpi,
            "bytes_per_iteration_at_3.35TB/s_ms": 1e3 * bpi / HBM_BYTES_PER_S, "iso_ms": iso_ms, "marching_cubes_ms": mc_ms,
            "trim_ms": trim_ms, "vertices": int(full["vertices"].shape[0]), "faces": int(full["faces"].shape[0]),
            "kept_vertices": int(kept["vertices"].shape[0]), "kept_faces": int(kept["faces"].shape[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--views", type=int, default=60)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--depths", type=int, nargs="+", default=[8, 9])
    ap.add_argument("--host-depth", type=int, default=5)
    ap.add_argument("--host-points", type=int, default=100000)
    ap.add_argument("--json", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "gpu": []}
    pts, nrm, col, fr = cloud(a.points, a.views, a.size, dev)
    for d in a.depths:
        out["gpu"].append(gpu_run(pts, nrm, col, fr, d))
        print(json.dumps(out["gpu"][-1]), flush=True)
        torch.cuda.empty_cache()
    hp = [t[: a.host_points].cpu().numpy() for t in (pts, nrm, col, fr)]
    t0 = time.perf_counter()
    host = P.reconstruct(*hp, depth=a.host_depth)
    out["host"] = {"depth": a.host_depth, "points": len(hp[0]), "ms": 1e3 * (time.perf_counter() - t0),
                   "faces": int(host["full"]["faces"].shape[0])}
    dev_out = P.reconstruct(*(torch.from_numpy(x).to(dev) for x in hp), depth=a.host_depth)
    out["host"]["gpu_faces"] = int(dev_out["full"]["faces"].shape[0])
    print(json.dumps(out["host"]), flush=True)
    if a.json:
        a.json.parent.mkdir(parents=True, exist_ok=True)
        a.json.write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
