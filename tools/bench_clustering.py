"""Per-stage time of fruit counting (clustering.count_fruits) on seeded synthetic fruit-shell clouds at the reference's
real-tree parameters (clustering/config_real.py), GPU path and -- where it finishes in reasonable time -- the
numpy / scikit-learn path in the same run.

    python tools/bench_clustering.py --json out/bench_clustering.json

GPU stages are the stages of ``count_sweep`` with one config, which is what a device ``count_fruits`` runs, timed with
CUDA events after one warm-up run at the same size; each stage ends in a host read, so its window covers all of its
work.  The card's name and power limit are written next to the numbers.
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

from fruitnerf_b200 import clustering  # noqa: E402
from fruitnerf_b200.synthetic import fruit_shell_cloud  # noqa: E402

REAL_TREE = dict(eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                 remove_outliers_radius=0.015)
STAGES = ("radius_count", "voxel", "dbscan", "sums_merge")


def gpu_stages(x: torch.Tensor, p=REAL_TREE):
    """clustering.count_sweep with the one config of a device count_fruits, one CUDA-event window per stage (its
    'merge' reported as 'sums_merge')."""
    ev = {"start": torch.cuda.Event(enable_timing=True)}
    ev["start"].record()

    def mark(stage):
        ev[stage] = torch.cuda.Event(enable_timing=True)
        ev[stage].record()

    res = clustering.count_sweep(x, [p], on_stage=mark)[0]
    torch.cuda.synchronize()
    names = ["start", "radius_count", "voxel", "dbscan", "merge"]
    return {s: ev[names[i]].elapsed_time(ev[names[i + 1]]) for i, s in enumerate(STAGES)}, res, res["num_points"]


def cpu_stages(pts: np.ndarray, p=REAL_TREE):
    """clustering.count_fruits' numpy / scikit-learn path split at the same stage boundaries."""
    t = [time.perf_counter()]
    pts = clustering.remove_radius_outliers(pts, p["remove_outliers_nb_points"], p["remove_outliers_radius"])
    t.append(time.perf_counter())
    pts = clustering.voxel_down_sample(pts, p["down_sample"])
    t.append(time.perf_counter())
    res = clustering.count_fruits(pts, eps=p["eps"], min_samples=p["min_samples"], cluster_merge_distance=p["cluster_merge_distance"])
    t.append(time.perf_counter())
    ms = {s: 1e3 * (t[i + 1] - t[i]) for i, s in enumerate(STAGES[:2])}
    ms["dbscan_sums_merge"] = 1e3 * (t[3] - t[2])
    return ms, res


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,400000,1000000,16777216")
    ap.add_argument("--cpu-max", type=int, default=400000, help="largest size the CPU path is also timed at")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("bench_clustering needs a CUDA device")
    out = {"card": card(), "parameters": REAL_TREE, "rows": []}
    print(json.dumps(out["card"]), flush=True)
    for n in map(int, a.sizes.split(",")):
        cloud = fruit_shell_cloud(n, seed=0)
        x = torch.from_numpy(cloud).cuda()
        gpu_stages(x)  # warm-up: module loads, allocator
        runs = [gpu_stages(x) for _ in range(a.repeats)]
        ms = {s: float(np.median([r[0][s] for r in runs])) for s in STAGES}
        row = {"points": n, "gpu_ms_median": ms, "gpu_ms_total": sum(ms.values()), "gpu_ms_all_runs": [r[0] for r in runs],
               "count": runs[0][1]["count"], "count_before_merge": runs[0][1]["count_before_merge"], "points_after_voxel": runs[0][2]}
        if n <= a.cpu_max:
            cms, cres = cpu_stages(cloud)
            row["cpu_ms"] = cms
            row["cpu_ms_total"] = sum(cms.values())
            row["cpu_count"] = cres["count"]
            row["cpu_count_before_merge"] = cres["count_before_merge"]
        print(json.dumps(row), flush=True)
        out["rows"].append(row)
        del x
        torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
