"""Count the fruit in an exported semantic point cloud on the GPU: the reference's clustering driver
(clustering/run_clustering.py with clustering/clustering_base.py), i.e. radius-outlier removal, voxel down-sampling,
DBSCAN and the merge of cluster centres closer than ``--cluster-merge-distance``, then, with ``--template``, the split of
groups of touching fruit and the pruning of fragments by template matching (stage 3).  ``--gt-centers`` scores the
centres against ground truth (TP / FP / FN, precision, recall, F1).  The defaults are the reference's real-tree
parameters (clustering/config_real.py).

    python -m fruitnerf_b200.scripts.count --pcd OUT/semantic_colormap.ply --json OUT/count.json
    python -m fruitnerf_b200.scripts.count --pcd OUT/semantic_colormap.ply --template apple.ply --template-size 0.7 \
        --gt-centers gt_centers.npy

The kernels need a CUDA device; without one the script fails (there is no CPU fallback).
"""
from __future__ import annotations

import argparse
import json
import os

import numpy as np
import torch

from ..clustering import count_fruits, evaluate_count, load_template
from ..export.exporter_utils import read_ply


def parse_args(argv=None) -> argparse.Namespace:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pcd", required=True, help="binary little-endian PLY point cloud (the exporter's semantic_colormap.ply)")
    ap.add_argument("--eps", type=float, default=0.02, help="DBSCAN neighbourhood radius")
    ap.add_argument("--min-samples", type=int, default=100, help="DBSCAN core-point threshold (the point itself included)")
    ap.add_argument("--remove-outliers-nb-points", type=int, default=120, help="radius-outlier removal: neighbours required (0: off)")
    ap.add_argument("--remove-outliers-radius", type=float, default=0.015, help="radius-outlier removal: radius (0: off)")
    ap.add_argument("--down-sample", type=float, default=0.001, help="voxel size of the down-sampling (0: off)")
    ap.add_argument("--cluster-merge-distance", type=float, default=0.04, help="clusters whose centres are closer are merged")
    ap.add_argument("--template", default=None, help="fruit template PLY point cloud; stage 3 (split / prune by template matching) runs only "
                    "when it is given")
    ap.add_argument("--template-size", type=float, default=1.0, help="scale of the template about the origin (the reference uses "
                    "e.g. 0.7 for apples and 1.1 for pears)")
    ap.add_argument("--gt-centers", default=None, help=".npy of ground-truth fruit centres [K,3]: adds TP / FP / FN / precision / "
                    "recall / F1 (a centre matches the nearest unmatched one closer than 0.15)")
    ap.add_argument("--device", default="cuda:0", help="CUDA device to count on (cuda or cuda:N)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    return ap.parse_args(argv)


def count_cloud(a: argparse.Namespace) -> dict:
    if torch.device(a.device).type != "cuda":
        raise ValueError(f"--device {a.device}: fruit counting runs on a CUDA device (there is no CPU fallback)")
    if not torch.cuda.is_available():
        raise RuntimeError("fruit counting runs on the GPU and no CUDA device is available (there is no CPU fallback)")
    points, _ = read_ply(a.pcd)
    template = load_template(a.template, a.template_size) if a.template else None
    gt = np.load(a.gt_centers).astype(np.float64).reshape(-1, 3) if a.gt_centers else None
    res = count_fruits(torch.from_numpy(points).to(a.device), eps=a.eps, min_samples=a.min_samples,
                       cluster_merge_distance=a.cluster_merge_distance, down_sample=a.down_sample,
                       remove_outliers_nb_points=a.remove_outliers_nb_points, remove_outliers_radius=a.remove_outliers_radius,
                       template=template)
    out = {"count": int(res["count"]), "count_before_merge": int(res["count_before_merge"]), "num_points": int(res["num_points"])}
    if template is not None:
        out.update({k: int(res[k]) for k in ("count_after_merge", "num_split_extra", "num_pruned")})
    out["centers"] = res["centers"].tolist()
    if gt is not None:
        out.update(evaluate_count(res["centers"], gt))
    return out


def main(argv=None) -> dict:
    a = parse_args(argv)
    out = count_cloud(a)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    return out


if __name__ == "__main__":
    main()
