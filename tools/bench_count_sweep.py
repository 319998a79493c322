"""Time of a Fuji-shaped parameter sweep of the fruit count (clustering/run_clustering_sweep.py: remove_outliers_nb_points
x3, eps x3, template size x3 = 27 counts) on a seeded synthetic fruit-shell cloud, GPU path:

(a) a loop of device count_fruits, one call per config;
(b) device count_sweep, end to end and per stage (outlier counts, voxel, DBSCAN, merge, host alpha stage, ICP / Ward /
    Hausdorff);
(c) the E = 3 DBSCAN calls of one down-sampled set, as count_sweep makes them.

    python tools/bench_count_sweep.py --json out/bench_count_sweep.json

The host alpha shapes take most of a count with a template (about a minute per count at 2·10^6 points), so (a) runs
``--loop-configs`` of the 27 configs and reports their mean per count next to 27 times it.  The default sample holds
every nb, every eps and every template size (index = 9 nb + 3 eps + size).  GPU windows are CUDA events after a warm-up
of every kernel, stage 3 included, on a small cloud; stages ending on the host (merge, alpha) end in a host read, so
their windows cover all of their work.  The card's name and power limit are written next to the numbers.
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

from fruitnerf_b200 import clustering, ops  # noqa: E402
from fruitnerf_b200.synthetic import fruit_shell_cloud, sphere_template, touching_fruit_cloud  # noqa: E402

FUJI = dict(nb=(50, 60, 75), radius=0.025, down_sample=0.001, eps=(0.015, 0.02, 0.025), min_samples=100, merge=0.04,
            sizes=(0.9, 1.0, 1.1))  # run_clustering_sweep.py's Fuji_unet_sweep
STAGES = ("radius_count", "voxel", "dbscan", "merge", "alpha", "match")


def sweep_configs():
    configs, templates = [], []
    for nb in FUJI["nb"]:
        for eps in FUJI["eps"]:
            for size in FUJI["sizes"]:
                configs.append(dict(eps=eps, min_samples=FUJI["min_samples"], cluster_merge_distance=FUJI["merge"],
                                    down_sample=FUJI["down_sample"], remove_outliers_nb_points=nb, remove_outliers_radius=FUJI["radius"]))
                templates.append(sphere_template() * size)
    return configs, templates


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def timed_sweep(x, configs, templates):
    """count_sweep with one CUDA-event window per stage (ms) and its end-to-end wall time (ms)."""
    ev = {"start": torch.cuda.Event(enable_timing=True)}
    t0 = time.perf_counter()
    ev["start"].record()

    def mark(stage):
        ev[stage] = torch.cuda.Event(enable_timing=True)
        ev[stage].record()

    res = clustering.count_sweep(x, configs, templates, on_stage=mark)
    torch.cuda.synchronize()
    wall = 1e3 * (time.perf_counter() - t0)
    names = ["start", *STAGES]
    return {s: ev[names[i]].elapsed_time(ev[s]) for i, s in enumerate(STAGES)}, wall, res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--loop-configs", default="0,7,13,20,26", help="indices of the configs timed as separate count_fruits calls")
    ap.add_argument("--repeats", type=int, default=5, help="repeats of the DBSCAN timing (c)")
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("bench_count_sweep needs a CUDA device")
    out = {"card": card(), "points": a.points, "sweep": {k: list(v) if isinstance(v, tuple) else v for k, v in FUJI.items()}}
    print(json.dumps(out["card"]), flush=True)
    x = torch.from_numpy(fruit_shell_cloud(a.points, seed=0)).cuda()
    configs, templates = sweep_configs()

    # (c) on the first outlier filter's down-sampled set
    c0 = configs[0]
    pts = ops.voxel_down_sample(clustering.remove_radius_outliers(x, c0["remove_outliers_nb_points"], c0["remove_outliers_radius"]),
                                c0["down_sample"])
    eps = list(FUJI["eps"])
    for e in eps:
        ops.dbscan(pts, e, FUJI["min_samples"])
    runs = []
    for _ in range(a.repeats):
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for e in eps:
            ops.dbscan(pts, e, FUJI["min_samples"])
        t.record()
        torch.cuda.synchronize()
        runs.append(s.elapsed_time(t))
    out["dbscan"] = {"points": int(pts.shape[0]), "eps": eps, "ms_median": float(np.median(runs)), "ms_all": runs}
    print(json.dumps(out["dbscan"]), flush=True)

    # (b) the whole sweep, after a warm-up of every kernel (ICP, Ward and Hausdorff too) on a small cloud with a template
    small, _ = touching_fruit_cloud(seed=0)
    clustering.count_sweep(torch.from_numpy(small).cuda(), configs[:2], templates[:2])
    stages, wall, res = timed_sweep(x, configs, templates)
    out["count_sweep"] = {"ms_total": wall, "stage_ms": stages, "counts": [int(r["count"]) for r in res]}
    print(json.dumps(out["count_sweep"]), flush=True)

    # (a) separate count_fruits calls
    loop = [int(i) for i in a.loop_configs.split(",")]
    per = []
    for i in loop:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = clustering.count_fruits(x, **configs[i], template=templates[i])
        torch.cuda.synchronize()
        per.append(1e3 * (time.perf_counter() - t0))
        assert r["count"] == res[i]["count"] and np.array_equal(r["centers"], res[i]["centers"])
    out["count_fruits_loop"] = {"configs": loop, "ms_each": per, "ms_mean": float(np.mean(per)),
                                "ms_27_estimate": len(configs) * float(np.mean(per))}
    print(json.dumps(out["count_fruits_loop"]), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
