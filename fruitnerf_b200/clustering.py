"""Fruit counting on the exported semantic point cloud: stages 1-2 of the reference's clustering
(clustering/clustering_base.py:138-143 radius-outlier removal + voxel down-sampling, :183-207 DBSCAN,
:209-259 merging of cluster centres closer than ``cluster_merge_distance``).  The template-matching split of
oversized clusters (stage 3, :261-) needs open3d / alphashape and the LFS fruit templates, none of which exist
offline; it is not restated.

Where each stage runs depends on the input:
- a CUDA ``torch.Tensor`` runs on the GPU (fnr_cluster.cu through ``ops``): radius-outlier removal, voxel
  down-sampling, DBSCAN and the per-cluster sums are kernels; only the centre merge, a loop over the K cluster sums,
  runs on the host.  Labels, counts and down-sampled points are identical to the CPU path; centres agree to rounding.
- anything else (a numpy array) runs the numpy / scikit-learn code below, which is the reference of the GPU path.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
from sklearn.cluster import DBSCAN
from sklearn.neighbors import NearestNeighbors

from . import ops


def _on_device(points) -> bool:
    return isinstance(points, torch.Tensor) and points.is_cuda


def remove_radius_outliers(points: np.ndarray, nb_points: int, radius: float) -> np.ndarray:
    """open3d remove_radius_outlier: keep points with at least ``nb_points`` neighbours within ``radius``."""
    if _on_device(points):
        return _device_remove_radius_outliers(points, nb_points, radius)
    if points.shape[0] == 0:
        return points
    nn = NearestNeighbors(radius=radius).fit(points)
    counts = np.array([len(ix) for ix in nn.radius_neighbors(points, return_distance=False)])
    return points[counts - 1 >= nb_points]  # the query point itself is excluded, as in open3d


def voxel_down_sample(points: np.ndarray, voxel: float) -> np.ndarray:
    """open3d voxel_down_sample: one point (the mean) per occupied voxel."""
    if _on_device(points):
        return ops.voxel_down_sample(points, voxel)
    if points.shape[0] == 0 or voxel <= 0:
        return points
    keys = np.floor((points - points.min(axis=0)) / voxel).astype(np.int64)
    _, inv, cnt = np.unique(keys, axis=0, return_inverse=True, return_counts=True)
    out = np.zeros((cnt.shape[0], 3))
    np.add.at(out, inv.reshape(-1), points)
    return out / cnt[:, None]


def count_fruits(points: np.ndarray, eps: float, min_samples: int, cluster_merge_distance: float, down_sample: float = 0.0,
                 remove_outliers_nb_points: int = 0, remove_outliers_radius: float = 0.0) -> Dict:
    """Returns {'count', 'count_before_merge', 'centers' [count,3], 'num_points'}."""
    if _on_device(points):
        return _device_count_fruits(points, eps, min_samples, cluster_merge_distance, down_sample, remove_outliers_nb_points,
                                    remove_outliers_radius)
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    if remove_outliers_nb_points > 0 and remove_outliers_radius > 0:
        pts = remove_radius_outliers(pts, remove_outliers_nb_points, remove_outliers_radius)
    pts = voxel_down_sample(pts, down_sample)
    if pts.shape[0] == 0:
        return {"count": 0, "count_before_merge": 0, "centers": np.zeros((0, 3)), "num_points": 0}
    labels = DBSCAN(eps=eps, min_samples=min_samples, n_jobs=-1).fit(pts).labels_
    centers, members = [], []
    first_stage = 0
    for lab in np.unique(labels):
        if lab == -1:
            continue
        first_stage += 1
        cluster = pts[labels == lab]
        c = cluster.mean(axis=0)
        if centers:
            d = np.linalg.norm(np.vstack(centers) - c, axis=1)
            j = int(np.argmin(d))
            if d[j] < cluster_merge_distance:  # fuse with the nearest earlier cluster: centre = midpoint of the two
                centers[j] = (members[j].mean(axis=0) + c) / 2
                members[j] = np.vstack([members[j], cluster])
                continue
        centers.append(c)
        members.append(cluster)
    return {"count": len(centers), "count_before_merge": first_stage, "centers": np.vstack(centers) if centers else np.zeros((0, 3)),
            "num_points": int(pts.shape[0])}


# ---- GPU path ------------------------------------------------------------------------------------------------------

def _device_remove_radius_outliers(points, nb_points: int, radius: float):
    pts = ops.cluster_points(points)
    if pts.shape[0] == 0:
        return pts
    counts = ops.radius_count(pts, radius, cap=nb_points + 1)  # nb_points neighbours + the point itself
    return pts[counts - 1 >= nb_points]


def _device_count_fruits(points, eps: float, min_samples: int, cluster_merge_distance: float, down_sample: float,
                         remove_outliers_nb_points: int, remove_outliers_radius: float) -> Dict:
    pts = ops.cluster_points(points)
    if remove_outliers_nb_points > 0 and remove_outliers_radius > 0:
        pts = _device_remove_radius_outliers(pts, remove_outliers_nb_points, remove_outliers_radius)
    pts = ops.voxel_down_sample(pts, down_sample)
    if pts.shape[0] == 0:
        return {"count": 0, "count_before_merge": 0, "centers": np.zeros((0, 3)), "num_points": 0}
    labels, k = ops.dbscan(pts, eps, min_samples)
    sums, counts = ops.cluster_sums(pts, labels, k)
    return {**merge_cluster_centers(sums.cpu().numpy(), counts.cpu().numpy(), cluster_merge_distance), "num_points": int(pts.shape[0])}


def merge_cluster_centers(sums: np.ndarray, counts: np.ndarray, cluster_merge_distance: float) -> Dict:
    """The centre merge of ``count_fruits`` from per-cluster coordinate sums and point counts, in label order: a cluster
    whose mean lies within ``cluster_merge_distance`` of the nearest earlier centre fuses with it (new centre = midpoint
    of that group's mean and this cluster's mean), otherwise it starts a new centre."""
    k = len(counts)
    centers, group_sum, group_cnt = np.zeros((k, 3)), np.zeros((k, 3)), np.zeros(k)
    m = 0  # centres so far (rows of the arrays above)
    for s, n in zip(sums, counts):
        c = s / n
        if m:
            d = np.linalg.norm(centers[:m] - c, axis=1)
            j = int(np.argmin(d))
            if d[j] < cluster_merge_distance:
                centers[j] = (group_sum[j] / group_cnt[j] + c) / 2
                group_sum[j] += s
                group_cnt[j] += n
                continue
        centers[m], group_sum[m], group_cnt[m] = c, s, n
        m += 1
    return {"count": m, "count_before_merge": int(k), "centers": centers[:m].copy()}
