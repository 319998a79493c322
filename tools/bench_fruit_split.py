"""Time of stage 3 of the fruit count (clustering.split_clusters) on a seeded touching-fruit cloud the size of an export
(`synthetic.touching_fruit_cloud`, about 3.5·10^5 points at the defaults): the host alpha-shape step, each kernel
(ICP, Ward, Hausdorff), the whole stage on the device path and the same stage on the numpy path, plus the ICP iteration
counts.  Stage 3 runs on the merged groups of the device count at the reference's real-tree parameters.

    python tools/bench_fruit_split.py --json out/bench_fruit_split.json

Kernels are timed with CUDA events after one warm-up with the same inputs; the stage timings are host clocks around
work that ends in a host read.  The card's name and power limit are written next to the numbers.
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

from fruitnerf_b200 import clustering as cl  # noqa: E402
from fruitnerf_b200 import ops  # noqa: E402
from fruitnerf_b200.synthetic import sphere_template, touching_fruit_cloud  # noqa: E402

REAL_TREE = dict(eps=0.02, min_samples=100, cluster_merge_distance=0.04, down_sample=0.001, remove_outliers_nb_points=120,
                 remove_outliers_radius=0.015)  # clustering/config_real.py


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def timed(fn, reps: int) -> float:
    """Mean milliseconds of ``fn`` over ``reps`` launches, CUDA events, after one warm-up call."""
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--singles", type=int, default=30)
    ap.add_argument("--pairs", type=int, default=15)
    ap.add_argument("--triples", type=int, default=8)
    ap.add_argument("--fragments", type=int, default=6)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true", help="skip the numpy path of the matching step")
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise RuntimeError("bench_fruit_split measures the GPU path and no CUDA device is available")
    dev = torch.device("cuda:0")
    pts, gt = touching_fruit_cloud(seed=0, singles=a.singles, pairs=a.pairs, triples=a.triples, fragments=a.fragments)
    tmpl = sphere_template(0.035, 1000)
    x = torch.from_numpy(pts).to(dev)

    captured = {}
    orig = cl.split_clusters

    def spy(groups, template, seed=0, device=None):
        captured["groups"] = groups
        t0 = time.perf_counter()
        out = orig(groups, template, seed=seed, device=device)
        captured["ms"] = 1e3 * (time.perf_counter() - t0)
        return out

    cl.split_clusters = spy
    try:
        cl.count_fruits(x, **REAL_TREE, template=tmpl)  # warm-up of every kernel
        t0 = time.perf_counter()
        res = cl.count_fruits(x, **REAL_TREE, template=tmpl)
        total_ms = 1e3 * (time.perf_counter() - t0)
    finally:
        cl.split_clusters = orig
    groups = captured["groups"]
    stage3_gpu_ms = captured["ms"]

    t0 = time.perf_counter()
    _, samples = cl.alpha_stage(groups, tmpl)
    alpha_ms = 1e3 * (time.perf_counter() - t0)
    samp = [samples[g] for g in sorted(samples)]
    f64 = dict(dtype=torch.float64, device=dev)
    offs = np.concatenate([[0], np.cumsum([s.shape[0] for s in samp])])
    tg, xs = torch.from_numpy(tmpl).to(**f64), torch.from_numpy(np.concatenate(samp)).to(**f64)
    init = torch.from_numpy(np.stack([s.mean(axis=0) for s in samp])).to(**f64)
    _, _, _, its = ops.icp_scaled(tg, xs, offs, init)
    cuts = ops.ward_cut(xs, offs)
    kernels = {"icp": timed(lambda: ops.icp_scaled(tg, xs, offs, init), a.reps), "ward": timed(lambda: ops.ward_cut(xs, offs), a.reps)}
    # the k = 6 hypothesis of every sample: the largest Hausdorff pair of the stage
    hyp = torch.cat([(tg[None] + cuts[i, 14:20][:, None]).reshape(-1, 3) for i in range(len(samp))])
    ar = np.stack([offs[:-1], offs[1:]], 1)
    br = np.stack([np.arange(len(samp)) * 6 * tmpl.shape[0], (np.arange(len(samp)) + 1) * 6 * tmpl.shape[0]], 1)
    kernels["hausdorff_k6"] = timed(lambda: ops.hausdorff(xs, ar, hyp, br), a.reps)

    out = {"card": card(), "points": int(pts.shape[0]), "true_fruit": int(len(gt)), "groups": len(groups), "candidates": len(samp),
           "count": int(res["count"]), "num_split_extra": int(res["num_split_extra"]), "num_pruned": int(res["num_pruned"]),
           "score": cl.evaluate_count(res["centers"], gt), "icp_iterations": {"mean": float(its.float().mean()), "max": int(its.max())},
           "ms": {"count_fruits_gpu_total": total_ms, "stage3_gpu": stage3_gpu_ms, "alpha_shapes_host": alpha_ms,
                  **{f"kernel_{k}": v for k, v in kernels.items()}}}
    if not a.no_cpu:
        t0 = time.perf_counter()
        host = cl.match_candidates(samp, tmpl)
        out["ms"]["matching_cpu"] = 1e3 * (time.perf_counter() - t0)
        out["ms"]["stage3_cpu"] = alpha_ms + out["ms"]["matching_cpu"]
        out["cpu_same_choice"] = bool((np.argmin(host[2], axis=1) == np.argmin(ops_distances(samp, tmpl, dev), axis=1)).all())
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


def ops_distances(samp, tmpl, dev):
    return cl.match_candidates(samp, tmpl, device=dev)[2]


if __name__ == "__main__":
    main()
