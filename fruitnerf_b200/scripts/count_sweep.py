"""Count the fruit of several data sets and parameter sweeps on the GPU, scored against ground truth: the reference's
clustering drivers (clustering/run_clustering.py, clustering/run_clustering_sweep.py).

The spec is a JSON object of named runs; each run is one data set with the reference's keys (clustering/config_real.py,
config_synthetic.py), so such a dict pasted as JSON is a valid run of one count:

    {"Fuji_sam_sweep": {
        "path": "eval/fuji/sam/semantic_colormap_cropped.ply",
        "remove_outliers_nb_points": [50, 60, 75], "remove_outliers_radius": 0.025, "down_sample": 0.001,
        "eps": [0.015, 0.02], "min_samples": 100, "cluster_merge_distance": 0.04, "minimum_size_factor": 0.2,
        "template_path": "apple_template.ply", "apple_template_size": [0.9, 1, 1.1],
        "gt_cluster": "eval/fuji/data/lineset_aligned.ply", "gt_count": 1455}}

    python -m fruitnerf_b200.scripts.count_sweep spec.json --json results.json

Any parameter in ``PARAMETERS`` may be a list; a run counts every combination, the cartesian product in the order of
``PARAMETERS`` with the first key outermost (so remove_outliers_nb_points is outside eps, and eps outside
apple_template_size, as in the reference's nested loops), and the result index is the position in that product.
``template_path`` null means no stage 3 (template matching).  ``gt_cluster`` (null allowed) is the ground truth: an OBJ
of fruit objects, a PLY line set of boxes or a .npy of centres (clustering.load_gt_centres); ``gt_count`` is reported
as "gt".  ``minimum_size_factor`` is accepted and ignored, as the reference ignores it.  Relative paths are taken
from the working directory, as the reference's configs take them.  Unknown keys, missing files and non-positive radii are refused before any count runs.

The output has the reference's shape, {run: {"<i>": {"path", "count", "TP", "FP", "FN", "gt", "precision", "recall",
"F1", "params": {the swept keys}}}}, or {"path", "count", "gt"} per count when gt_cluster is null.  Each run's counts
share their common work on the device (clustering.count_sweep).  The kernels need a CUDA device; without one the
script fails (there is no CPU fallback).
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import sys
from typing import Dict, List

import torch

from ..clustering import count_sweep, evaluate_count, load_gt_centres, load_template
from ..export.exporter_utils import read_ply

PARAMETERS = ("remove_outliers_nb_points", "remove_outliers_radius", "down_sample", "eps", "min_samples", "cluster_merge_distance",
              "template_path", "apple_template_size")
FIXED = ("path", "gt_cluster", "gt_count", "minimum_size_factor")
REQUIRED = ("path", "eps", "min_samples", "cluster_merge_distance")
DEFAULTS = {"remove_outliers_nb_points": 0, "remove_outliers_radius": 0.0, "down_sample": 0.0, "template_path": None,
            "apple_template_size": 1.0, "gt_cluster": None, "gt_count": None}


def _values(run: Dict, key: str) -> List:
    v = run.get(key, DEFAULTS.get(key))
    return list(v) if isinstance(v, list) else [v]


def check_run(name: str, run: Dict) -> Dict:
    """The run with defaults filled in; raises ValueError on unknown or missing keys,
    empty lists, out-of-range values and files that do not exist."""
    if not isinstance(run, dict):
        raise ValueError(f"{name}: a run must be a JSON object")
    unknown = sorted(set(run) - set(PARAMETERS) - set(FIXED))
    if unknown:
        raise ValueError(f"{name}: unknown keys {unknown}")
    missing = [k for k in REQUIRED if k not in run]
    if missing:
        raise ValueError(f"{name}: missing keys {missing}")
    out = {**DEFAULTS, **run}
    for k in FIXED:
        if isinstance(out.get(k), list):
            raise ValueError(f"{name}: '{k}' cannot be a list")
    for k in PARAMETERS:
        vals = _values(out, k)
        if not vals:
            raise ValueError(f"{name}: '{k}' is an empty list")
        for v in vals:
            if k == "template_path":
                if v is not None and not isinstance(v, str):
                    raise ValueError(f"{name}: template_path must be a path or null, got {v!r}")
                continue
            if isinstance(v, bool) or not isinstance(v, (int, float)):
                raise ValueError(f"{name}: '{k}' must be a number, got {v!r}")
            if k in ("eps", "apple_template_size") and not v > 0:
                raise ValueError(f"{name}: '{k}' must be positive, got {v}")
            if k in ("remove_outliers_nb_points", "min_samples") and v != int(v):
                raise ValueError(f"{name}: '{k}' must be an integer, got {v}")
            if k == "min_samples" and v < 1:
                raise ValueError(f"{name}: min_samples must be >= 1, got {v}")
            if k in ("remove_outliers_nb_points", "down_sample", "cluster_merge_distance", "remove_outliers_radius") and v < 0:
                raise ValueError(f"{name}: '{k}' must not be negative, got {v}")
    if any(nb > 0 for nb in _values(out, "remove_outliers_nb_points")) and not all(r > 0 for r in _values(out, "remove_outliers_radius")):
        raise ValueError(f"{name}: remove_outliers_radius must be positive when remove_outliers_nb_points > 0")
    for what, p in [("path", out["path"]), ("gt_cluster", out["gt_cluster"])] + [("template_path", t) for t in _values(out, "template_path")]:
        if p is not None and not (isinstance(p, str) and os.path.isfile(p)):
            raise ValueError(f"{name}: {what} {p} does not exist")
    return out


def expand(run: Dict) -> List[Dict]:
    """Every combination of the run's list-valued PARAMETERS, first key outermost: [{parameter: value}]."""
    return [dict(zip(PARAMETERS, combo)) for combo in itertools.product(*(_values(run, k) for k in PARAMETERS))]


def swept_keys(run: Dict) -> List[str]:
    return [k for k in PARAMETERS if isinstance(run.get(k), list)]


def load_spec(path) -> Dict[str, Dict]:
    """The runs of a spec file, each checked and resolved (``check_run``) before any count starts."""
    with open(path) as f:
        spec = json.load(f)
    if not isinstance(spec, dict) or not spec:
        raise ValueError(f"{path}: the spec must be a non-empty JSON object of named runs")
    return {name: check_run(name, run) for name, run in spec.items()}


def run_sweep(name: str, run: Dict, device) -> Dict[str, Dict]:
    """All counts of one run on ``device``: {"<i>": entry} in the reference's shape."""
    points, _ = read_ply(run["path"])
    gt = load_gt_centres(run["gt_cluster"]) if run["gt_cluster"] else None
    combos = expand(run)
    templates, cache = [], {}
    for c in combos:
        key = (c["template_path"], float(c["apple_template_size"]))
        if c["template_path"] is not None and key not in cache:
            cache[key] = load_template(*key)
        templates.append(cache.get(key) if c["template_path"] is not None else None)
    configs = [{"eps": float(c["eps"]), "min_samples": int(c["min_samples"]), "cluster_merge_distance": float(c["cluster_merge_distance"]),
                "down_sample": float(c["down_sample"]), "remove_outliers_nb_points": int(c["remove_outliers_nb_points"]),
                "remove_outliers_radius": float(c["remove_outliers_radius"])} for c in combos]
    results = count_sweep(torch.from_numpy(points).to(device), configs, templates)
    swept, out = swept_keys(run), {}
    for i, (c, res) in enumerate(zip(combos, results)):
        entry = {"path": run["path"], "count": int(res["count"])}
        if gt is not None:
            score = evaluate_count(res["centers"], gt)
            entry.update({"TP": score["TP"], "FP": score["FP"], "FN": score["FN"], "gt": run["gt_count"], "precision": score["precision"],
                          "recall": score["recall"], "F1": score["F1"], "params": {k: c[k] for k in swept}})
        else:
            entry["gt"] = run["gt_count"]
        out[str(i)] = entry
        params = " ".join(f"{k}={c[k]}" for k in swept)
        scored = f" TP={entry['TP']} precision={entry['precision']:.4f} recall={entry['recall']:.4f} F1={entry['F1']:.4f}" if gt is not None else ""
        print(f"{name}[{i}] {params + ' ' if params else ''}count={entry['count']} gt={entry['gt']}{scored}", flush=True)
    return out


def parse_args(argv=None) -> argparse.Namespace:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("spec", help="JSON object of named runs (see the module docstring)")
    ap.add_argument("--device", default="cuda:0", help="CUDA device to count on (cuda or cuda:N)")
    ap.add_argument("--json", default=None, help="write the results to this file")
    return ap.parse_args(argv)


def main(argv=None) -> Dict:
    a = parse_args(argv)
    try:
        runs = load_spec(a.spec)
        if torch.device(a.device).type != "cuda":
            raise ValueError(f"--device {a.device}: fruit counting runs on a CUDA device (there is no CPU fallback)")
        if not torch.cuda.is_available():
            raise RuntimeError("fruit counting runs on the GPU and no CUDA device is available (there is no CPU fallback)")
    except (ValueError, RuntimeError, OSError) as e:
        print(f"count_sweep: {e}", file=sys.stderr)
        raise SystemExit(2)
    results = {name: run_sweep(name, run, a.device) for name, run in runs.items()}
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w", encoding="utf-8") as f:
            json.dump(results, f, ensure_ascii=False, indent=4)
    return results


if __name__ == "__main__":
    main()
