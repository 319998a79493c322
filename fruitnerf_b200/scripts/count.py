"""Count the fruit in an exported semantic point cloud on the GPU: stages 1-2 of the reference's clustering driver
(clustering/run_clustering.py with clustering/clustering_base.py:138-259), i.e. radius-outlier removal, voxel
down-sampling, DBSCAN and the merge of cluster centres closer than ``--cluster-merge-distance``.  The defaults are the
reference's real-tree parameters (clustering/config_real.py).

    python -m fruitnerf_b200.scripts.count --pcd OUT/semantic_colormap.ply --json OUT/count.json

The kernels need a CUDA device; without one the script fails (there is no CPU fallback).
"""
from __future__ import annotations

import argparse
import json
import os

import torch

from ..clustering import count_fruits
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
    ap.add_argument("--device", default="cuda:0", help="CUDA device to count on (cuda or cuda:N)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    return ap.parse_args(argv)


def count_cloud(a: argparse.Namespace) -> dict:
    if torch.device(a.device).type != "cuda":
        raise ValueError(f"--device {a.device}: fruit counting runs on a CUDA device (there is no CPU fallback)")
    if not torch.cuda.is_available():
        raise RuntimeError("fruit counting runs on the GPU and no CUDA device is available (there is no CPU fallback)")
    points, _ = read_ply(a.pcd)
    res = count_fruits(torch.from_numpy(points).to(a.device), eps=a.eps, min_samples=a.min_samples,
                       cluster_merge_distance=a.cluster_merge_distance, down_sample=a.down_sample,
                       remove_outliers_nb_points=a.remove_outliers_nb_points, remove_outliers_radius=a.remove_outliers_radius)
    return {"count": int(res["count"]), "count_before_merge": int(res["count_before_merge"]), "num_points": int(res["num_points"]),
            "centers": res["centers"].tolist()}


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
