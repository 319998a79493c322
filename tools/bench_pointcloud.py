"""Per-stage time of the `pointcloud` export (exporter_utils.generate_point_cloud): render + back-projection of
10^6 points from a briefly trained synthetic model, then statistical outlier removal (k = 20) and normal estimation
(k = 30, reoriented) on seeded fruit-shell clouds (`synthetic.fruit_shell_cloud`) of 10^6 and 2^24 points, and the
scipy / numpy path (`pointcloud.py` on numpy arrays) at 10^6 in the same run.

    python tools/bench_pointcloud.py --json out/bench_pointcloud.json

GPU stages are timed with CUDA events after one warm-up at the same size; every stage ends in a host read (the kept
count or the kept rows), so its window covers all of its work.  The card's name and power limit are written next to the
numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from fruitnerf_b200 import ops, pointcloud  # noqa: E402
from fruitnerf_b200.synthetic import fruit_shell_cloud  # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def gpu_knn_stages(x: torch.Tensor, view: torch.Tensor):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    kept, idx = pointcloud.remove_statistical_outliers(x, 20, 10.0, return_index=True)
    ev[1].record()
    normals = pointcloud.estimate_normals(kept, 30, view[idx])
    ev[2].record()
    torch.cuda.synchronize()
    return {"outliers": ev[0].elapsed_time(ev[1]), "normals": ev[1].elapsed_time(ev[2])}, int(kept.shape[0]), normals


def cpu_knn_stages(pts: np.ndarray, view: np.ndarray):
    t0 = time.perf_counter()
    kept, idx = pointcloud.remove_statistical_outliers(pts, 20, 10.0, return_index=True)
    t1 = time.perf_counter()
    pointcloud.estimate_normals(kept, 30, view_dirs=view[idx])
    t2 = time.perf_counter()
    return {"outliers": 1e3 * (t1 - t0), "normals": 1e3 * (t2 - t1)}, int(kept.shape[0])


def render_stage(num_points: int, train_steps: int, rays_per_batch: int, repeats: int):
    """Render + back-projection of generate_point_cloud (no outlier removal, no normals) on a briefly trained model."""
    from fruitnerf_b200.export.exporter_utils import generate_point_cloud
    from fruitnerf_b200.scripts.train import synthetic_spec
    from fruitnerf_b200.trainer import Trainer

    spec = synthetic_spec("fruit_nerf", num_images=20, image_size=64, num_fruits=5, seed=0, rays_per_batch=2048)
    spec.pipeline.model.log2_hashmap_size = 17
    spec.pipeline.model.proposal_weights_anneal_max_num_iters = 100
    torch.manual_seed(0)
    trainer = Trainer(spec, device=torch.device("cuda:0"), use_cuda_graph=True)
    trainer.train(train_steps, log_every=10**9, eval_every=10**9)
    pipeline = trainer.pipeline
    pipeline.eval()
    pipeline.datamanager.config.train_num_rays_per_batch = rays_per_batch
    kw = dict(remove_outliers=False, estimate_normals=False, reorient_normals=False)
    generate_point_cloud(pipeline, num_points=rays_per_batch, **kw)  # warm-up
    times, n = [], 0
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = generate_point_cloud(pipeline, num_points=num_points, **kw)["points"].shape[0]
        times.append(1e3 * (time.perf_counter() - t0))
    batches = -(-num_points // rays_per_batch)
    return {"render_backproject_ms_all_runs": times, "render_backproject_ms_median": float(np.median(times)), "points": n,
            "rays_per_batch": rays_per_batch, "train_steps": train_steps, "min_batches": batches}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,16777216")
    ap.add_argument("--cpu-max", type=int, default=1000000, help="largest size the CPU path is also timed at")
    ap.add_argument("--render-points", type=int, default=1000000)
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("bench_pointcloud needs a CUDA device")
    out = {"card": card(), "rows": []}
    print(json.dumps(out["card"]), flush=True)
    if a.render_points > 0:
        out["render"] = render_stage(a.render_points, a.train_steps, 32768, a.repeats)
        print(json.dumps(out["render"]), flush=True)
    for n in map(int, a.sizes.split(",")):
        cloud = fruit_shell_cloud(n, seed=0)
        view = np.random.default_rng(1).standard_normal((n, 3)).astype(np.float32)
        x = torch.from_numpy(cloud).cuda()
        v = torch.from_numpy(view).cuda()
        gpu_knn_stages(x, v)  # warm-up: module loads, allocator
        runs = [gpu_knn_stages(x, v) for _ in range(a.repeats)]
        ms = {s: float(np.median([r[0][s] for r in runs])) for s in ("outliers", "normals")}
        row = {"points": n, "gpu_ms_median": ms, "gpu_ms_total": sum(ms.values()), "gpu_ms_all_runs": [r[0] for r in runs],
               "kept": runs[0][1]}
        if n <= a.cpu_max:
            cms, ckept = cpu_knn_stages(cloud, view)
            row["cpu_ms"] = cms
            row["cpu_ms_total"] = sum(cms.values())
            row["cpu_kept"] = ckept
            row["speedup"] = row["cpu_ms_total"] / row["gpu_ms_total"]
        print(json.dumps(row), flush=True)
        out["rows"].append(row)
        del x, v, runs
        torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
