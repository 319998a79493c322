"""Point-cloud post-processing of the `pointcloud` export (nerfstudio generate_point_cloud): open3d's
remove_statistical_outlier and estimate_normals, restated.  open3d is not a dependency; DESIGN section 4.3g lists the
semantics as recalled from its sources.

Where each step runs depends on the input:
- a CUDA ``torch.Tensor`` runs on the GPU (fnr_cluster.cu through ``ops``): the k-nearest-neighbour queries, mean
  distances and normals are kernels; the mean / std / threshold of the outlier test are fp64 torch reductions on the
  device.
- anything else (a numpy array) runs the scipy / numpy code below, which is the reference of the GPU path.
"""
from __future__ import annotations

import numpy as np
import torch
from scipy.spatial import cKDTree

from . import ops


def _on_device(points) -> bool:
    return isinstance(points, torch.Tensor) and points.is_cuda


def knn_mean_distance(points: np.ndarray, k: int) -> np.ndarray:
    """Mean distance of every point to its min(k, n) nearest neighbours, itself included, summed in ascending order."""
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    n = pts.shape[0]
    if n == 0:
        return np.zeros(0)
    kk = min(k, n)
    d, _ = cKDTree(pts).query(pts, k=kk)
    d = np.asarray(d, dtype=np.float64).reshape(n, kk)
    return np.cumsum(d, axis=1)[:, -1] / kk  # cumsum: the sequential order of the sum


def statistical_outlier_mask(avg, std_ratio: float):
    """Keep mask of remove_statistical_outlier from the per-point mean distances: the mean and (n - 1) std of the
    positive averages, both divided by the full n; a point is kept iff 0 < avg < mean + std_ratio * std."""
    if isinstance(avg, torch.Tensor):
        n = avg.shape[0]
        valid = avg > 0
        mean = torch.where(valid, avg, 0).sum() / n
        std = torch.sqrt(torch.where(valid, (avg - mean) ** 2, 0).sum() / (n - 1)) if n > 1 else avg.new_tensor(float("nan"))
        return valid & (avg < mean + std_ratio * std)
    n = avg.shape[0]
    valid = avg > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = avg[valid].sum() / n if n else np.nan
        std = np.sqrt(((avg[valid] - mean) ** 2).sum() / (n - 1)) if n > 1 else np.nan
        return valid & (avg < mean + std_ratio * std)


def remove_statistical_outliers(points, nb_neighbors: int = 20, std_ratio: float = 2.0, return_index: bool = False):
    """open3d remove_statistical_outlier: the kept points in input order (and their indices with ``return_index``)."""
    if _on_device(points):
        pts = ops.cluster_points(points)
        avg = ops.knn_mean_distance(pts, nb_neighbors) if pts.shape[0] else pts.new_zeros(0)
        idx = torch.nonzero(statistical_outlier_mask(avg, std_ratio)).reshape(-1)
        return (pts[idx], idx) if return_index else pts[idx]
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    idx = np.flatnonzero(statistical_outlier_mask(knn_mean_distance(pts, nb_neighbors), std_ratio))
    return (pts[idx], idx) if return_index else pts[idx]


def _normals_from_neighbours(nbrs: np.ndarray) -> np.ndarray:
    """[n,k,3] neighbour coordinates -> [n,3] smallest-eigenvalue eigenvectors of their two-pass covariance."""
    n, k = nbrs.shape[:2]
    out = np.tile(np.array([0.0, 0.0, 1.0]), (n, 1))
    if k < 3 or n == 0:
        return out
    c = nbrs - nbrs.mean(axis=1, keepdims=True)
    cov = np.einsum("nki,nkj->nij", c, c) / k
    ok = np.abs(cov).reshape(n, -1).max(axis=1) > 0
    if ok.any():
        _, vec = np.linalg.eigh(cov[ok])
        out[ok] = vec[:, :, 0]
    return out


def estimate_normals(points, knn: int = 30, view_dirs=None):
    """open3d estimate_normals (KDTreeSearchParamKNN(knn)): the unit eigenvector of the smallest eigenvalue of the
    covariance of the min(knn, n) nearest neighbours, self included; (0, 0, 1) with fewer than 3 neighbours or a zero
    covariance.  The sign is the solver's.  With ``view_dirs`` [n,3], a normal whose fp32 dot product with its view
    direction is positive is flipped (generate_point_cloud's reorientation)."""
    if _on_device(points):
        return ops.estimate_normals(points, knn, view_dirs)
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    n = pts.shape[0]
    if n == 0:
        return np.zeros((0, 3))
    kk = min(knn, n)
    _, idx = cKDTree(pts).query(pts, k=kk)
    normals = _normals_from_neighbours(pts[np.asarray(idx).reshape(n, kk)])
    if view_dirs is not None:
        v = np.asarray(view_dirs, dtype=np.float32).reshape(-1, 3)
        f = normals.astype(np.float32)
        dot = (v[:, 0] * f[:, 0] + v[:, 1] * f[:, 1]) + v[:, 2] * f[:, 2]
        normals[dot > 0] *= -1
    return normals
