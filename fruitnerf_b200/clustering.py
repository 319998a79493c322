"""Fruit counting on the exported semantic point cloud: the reference's clustering (clustering/clustering_base.py).

- Stages 1-2: radius-outlier removal + voxel down-sampling (:138-143), DBSCAN (:183-207) and the merging of cluster
  centres closer than ``cluster_merge_distance`` (:209-259).
- Stage 3, run when a fruit template is given (:261-511): each merged group's alpha-shape volume is compared with the
  template's.  A group much larger than one fruit is split into the k = 1..6 fruit whose template copies (scaled ICP
  for k = 1, Ward sub-centres for k >= 2) lie nearest to its surface in the Hausdorff sense; a group smaller than 0.3 of
  a fruit is pruned.  ``evaluate_count`` scores centres against ground truth (:464-506).

Where each stage runs depends on the input:
- a CUDA ``torch.Tensor`` runs on the GPU (fnr_cluster.cu and fnr_fruit_split.cu through ``ops``): radius-outlier
  removal, voxel down-sampling, DBSCAN, the per-cluster sums, ICP, Ward clustering and the Hausdorff distances are
  kernels.  The centre merge (a loop over the K cluster sums) and the alpha shapes (qhull's Delaunay, as in the
  reference) run on the host.  Labels, counts and down-sampled points are identical to the CPU path; centres agree to
  rounding.
- anything else (a numpy array) runs the numpy / scipy / scikit-learn code below, which is the reference of the GPU path.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

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
                 remove_outliers_nb_points: int = 0, remove_outliers_radius: float = 0.0, template: Optional[np.ndarray] = None,
                 seed: int = 0) -> Dict:
    """Returns {'count', 'count_before_merge', 'centers' [count,3], 'num_points'}.

    With ``template`` (a [m,3] fruit point cloud, see ``load_template``) stage 3 runs on the merged groups and the result
    also holds 'count_after_merge' (the stage-2 count), 'num_split_extra' and 'num_pruned'; 'count' and 'centers' are then
    the stage-3 values.  ``seed`` selects the hashed surface samples of ``alpha_shape``.

    On a CUDA tensor this is ``count_sweep`` with one config."""
    if _on_device(points):
        config = dict(eps=eps, min_samples=min_samples, cluster_merge_distance=cluster_merge_distance, down_sample=down_sample,
                      remove_outliers_nb_points=remove_outliers_nb_points, remove_outliers_radius=remove_outliers_radius, seed=seed)
        return _device_count_sweep(points, [config], [template], lambda stage: None)[0]
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    if remove_outliers_nb_points > 0 and remove_outliers_radius > 0:
        pts = remove_radius_outliers(pts, remove_outliers_nb_points, remove_outliers_radius)
    pts = voxel_down_sample(pts, down_sample)
    if pts.shape[0] == 0:
        return _with_stage3({"count": 0, "count_before_merge": 0, "centers": np.zeros((0, 3)), "num_points": 0}, [], template, seed)
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
    res = {"count": len(centers), "count_before_merge": first_stage, "centers": np.vstack(centers) if centers else np.zeros((0, 3)),
           "num_points": int(pts.shape[0])}
    return _with_stage3(res, members, template, seed)


def _with_stage3(res: Dict, groups: List[np.ndarray], template, seed: int) -> Dict:
    """Stage 3 on the merged ``groups`` when a template is given; ``res`` unchanged otherwise."""
    if template is None:
        return res
    return _with_split(res, split_clusters(groups, template, seed=seed, device=None))


def _with_split(res: Dict, split: Dict) -> Dict:
    """The stage-2 result ``res`` after stage 3, ``split`` being what ``split_clusters`` returned for its groups."""
    return {**res, "count_after_merge": res["count"], "count": res["count"] + split["num_split_extra"] - split["num_pruned"],
            "num_split_extra": split["num_split_extra"], "num_pruned": split["num_pruned"], "centers": split["centers"]}


# ---- GPU path ------------------------------------------------------------------------------------------------------

def _device_remove_radius_outliers(points, nb_points: int, radius: float):
    pts = ops.cluster_points(points)
    if pts.shape[0] == 0:
        return pts
    counts = ops.radius_count(pts, radius, cap=nb_points + 1)  # nb_points neighbours + the point itself
    return pts[counts - 1 >= nb_points]


def _device_groups(pts, labels, group_of: np.ndarray) -> List[np.ndarray]:
    """The points of each merged group on the host, in the order of the CPU path: the group's clusters in label order,
    each cluster's points in input order (noise left out)."""
    lab = labels.cpu().numpy().astype(np.int64)
    keep = np.flatnonzero(lab >= 0)
    order = keep[np.lexsort((lab[keep], group_of[lab[keep]]))]  # stable: input order inside a cluster
    host = pts.cpu().numpy()[order]
    bounds = np.searchsorted(group_of[lab[order]], np.arange(int(group_of.max(initial=-1)) + 2))
    return [host[bounds[g]:bounds[g + 1]] for g in range(len(bounds) - 1)]


def merge_cluster_centers(sums: np.ndarray, counts: np.ndarray, cluster_merge_distance: float) -> Dict:
    """The centre merge of ``count_fruits`` from per-cluster coordinate sums and point counts, in label order: a cluster
    whose mean lies within ``cluster_merge_distance`` of the nearest earlier centre fuses with it (new centre = midpoint
    of that group's mean and this cluster's mean), otherwise it starts a new centre."""
    return _merge_groups(sums, counts, cluster_merge_distance)[0]


def _merge_groups(sums: np.ndarray, counts: np.ndarray, cluster_merge_distance: float) -> Tuple[Dict, np.ndarray]:
    """``merge_cluster_centers`` and the group (row of 'centers') each cluster label joined, int64 [K]."""
    k = len(counts)
    centers, group_sum, group_cnt = np.zeros((k, 3)), np.zeros((k, 3)), np.zeros(k)
    group_of = np.zeros(k, dtype=np.int64)
    m = 0  # centres so far (rows of the arrays above)
    for i, (s, n) in enumerate(zip(sums, counts)):
        c = s / n
        if m:
            d = np.linalg.norm(centers[:m] - c, axis=1)
            j = int(np.argmin(d))
            if d[j] < cluster_merge_distance:
                centers[j] = (group_sum[j] / group_cnt[j] + c) / 2
                group_sum[j] += s
                group_cnt[j] += n
                group_of[i] = j
                continue
        centers[m], group_sum[m], group_cnt[m] = c, s, n
        group_of[i] = m
        m += 1
    return {"count": m, "count_before_merge": int(k), "centers": centers[:m].copy()}, group_of


# ---- stage 3: template matching of the merged groups (clustering_base.py:261-511) ------------------------------------

ALPHA_VOLUME = 10.0  # alphashape(G, 10): the volume of a group (:331) and of the template (run_clustering.py:43)
ALPHA_SURFACE = 100.0  # alphashape(G, 100): the surface the sample is drawn from (:343)
SURFACE_SAMPLES = 1000  # sample_points_uniformly(1000) (:365)
SPLIT_RATIO, PRUNE_RATIO = 0.9, 0.3  # (:372, :422)
ICP_MAX_DISTANCE, ICP_MAX_ITERATION, ICP_RELATIVE = 0.01, 2000, 1e-6  # (:266-269), open3d's default criteria
MAX_FRUIT_PER_GROUP = 6  # k = 1..6 (:380-407)
WARD_MAX_POINTS = 4096  # the per-segment limit of the Ward kernel
CUT_OFFSETS = (0, 2, 5, 9, 14, 20)  # rows of the k = 2..6 sub-centres in ward_cut_centres' [20,3] output


def load_template(path, size: float = 1.0) -> np.ndarray:
    """A fruit template as the reference prepares it (run_clustering.py:40-42): the PLY's points scaled by ``size``
    about the origin, then translated so that their mean is the origin.  [m,3] float64."""
    from .export.exporter_utils import read_ply

    pts, _ = read_ply(path)
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3) * float(size)
    if pts.shape[0] == 0:
        raise ValueError(f"{path}: the template has no points")
    return pts - pts.mean(axis=0)


def _hash_unit(n: int, *key: int) -> np.ndarray:
    """n float64 values in [0, 1), a pure function of (key, index): splitmix64 over a counter, like
    ``synthetic.hash_uniform`` a hash rather than a random stream, so every run and machine draws the same values."""
    def mix(z):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))

    h = np.uint64(0x9E3779B97F4A7C15)
    with np.errstate(over="ignore"):
        for k in key:
            h = mix(np.uint64(h + np.uint64(k & 0xFFFFFFFFFFFFFFFF) * np.uint64(0x9E3779B97F4A7C15)))
        z = mix(h + np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
    return (z >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def tetra_circumradii(points: np.ndarray, tets: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(circumradius, volume) of each tetrahedron [T,4] of ``points``; a flat tetrahedron has radius inf."""
    a = points[tets[:, 0]]
    u, v, w = points[tets[:, 1]] - a, points[tets[:, 2]] - a, points[tets[:, 3]] - a
    vw, wu, uv = np.cross(v, w), np.cross(w, u), np.cross(u, v)
    det = np.einsum("ij,ij->i", u, vw)
    num = (u * u).sum(1)[:, None] * vw + (v * v).sum(1)[:, None] * wu + (w * w).sum(1)[:, None] * uv
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.linalg.norm(num, axis=1) / np.abs(2.0 * det)
    r[~np.isfinite(r)] = np.inf
    return r, np.abs(det) / 6.0


def alpha_shape(points: np.ndarray, alphas: Sequence[float] = (ALPHA_VOLUME, ALPHA_SURFACE), seed: int = 0, group: int = 0,
                num_samples: int = SURFACE_SAMPLES):
    """3-D alpha shapes of ``points`` from one Delaunay tetrahedralisation (qhull, as alphashape 1.3.1 uses): for each
    alpha the tetrahedra with circumradius < 1/alpha are kept.

    Returns (volumes [len(alphas)], boundary triangles, sample):
    - volume: the sum of the kept tetrahedra's volumes (what trimesh reports for the consistently oriented boundary);
    - boundary triangles: per alpha, int64 [t,3] vertex indices of the faces that belong to exactly one kept
      tetrahedron, in lexicographic order;
    - sample: ``num_samples`` points on the boundary of the last alpha, triangles chosen by area and barycentric
      coordinates uniform (open3d sample_points_uniformly), drawn from a hash of (seed, group, sample); None when that
      boundary is empty.
    Fewer than 4 points, or a set qhull rejects as degenerate, gives volume 0 and empty boundaries."""
    from scipy.spatial import Delaunay, QhullError

    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    empty = (np.zeros(len(alphas)), [np.zeros((0, 3), dtype=np.int64) for _ in alphas], None)
    if pts.shape[0] < 4:
        return empty
    if pts.shape[0] >= 1 << 21:
        raise ValueError(f"alpha_shape: {pts.shape[0]} points; at most 2^21 - 1 are supported")
    try:
        tets = Delaunay(pts).simplices.astype(np.int64)
    except QhullError:
        return empty
    radius, vol = tetra_circumradii(pts, tets)
    volumes, boundaries = np.zeros(len(alphas)), []
    for i, alpha in enumerate(alphas):
        kept = tets[radius < 1.0 / alpha]
        volumes[i] = vol[radius < 1.0 / alpha].sum()
        faces = np.sort(np.concatenate([kept[:, [1, 2, 3]], kept[:, [0, 2, 3]], kept[:, [0, 1, 3]], kept[:, [0, 1, 2]]]), axis=1)
        if faces.shape[0] == 0:
            boundaries.append(np.zeros((0, 3), dtype=np.int64))
            continue
        n = np.int64(pts.shape[0])  # one int64 key per sorted face: its order is the lexicographic one
        keys, cnt = np.unique((faces[:, 0] * n + faces[:, 1]) * n + faces[:, 2], return_counts=True)
        keys = keys[cnt == 1]
        boundaries.append(np.stack([keys // (n * n), keys // n % n, keys % n], axis=1))
    return volumes, boundaries, _surface_sample(pts, boundaries[-1], num_samples, seed, group)


def _surface_sample(pts: np.ndarray, tri: np.ndarray, num: int, seed: int, group: int) -> Optional[np.ndarray]:
    if tri.shape[0] == 0:
        return None
    a, b, c = pts[tri[:, 0]], pts[tri[:, 1]], pts[tri[:, 2]]
    cdf = np.cumsum(0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1))
    if not cdf[-1] > 0.0:
        return None
    u = _hash_unit(3 * num, seed, group).reshape(3, num)
    t = np.minimum(np.searchsorted(cdf, u[0] * cdf[-1], side="right"), tri.shape[0] - 1)
    r1, r2 = np.sqrt(u[1])[:, None], u[2][:, None]
    return a[t] * (1.0 - r1) + b[t] * (r1 * (1.0 - r2)) + c[t] * (r1 * r2)


def _sq_dist(p: np.ndarray, q: np.ndarray) -> np.ndarray:
    """[len(p), len(q)] squared distances in the kernels' order, (dx*dx + dy*dy) + dz*dz."""
    d2 = None
    for a in range(3):
        d = q[None, :, a] - p[:, None, a]
        d2 = d * d if d2 is None else d2 + d * d
    return d2


def _chunks(n: int, q: int):
    step = max(1, (1 << 22) // max(q, 1))
    return range(0, n, step), step


def transform_points(points: np.ndarray, T: np.ndarray) -> np.ndarray:
    """x' = ((T00 x + T01 y) + T02 z) + T03 per row, without fused multiply-adds (the kernels' order)."""
    x, y, z = points[:, 0], points[:, 1], points[:, 2]
    return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], axis=1)


def _correspond(src: np.ndarray, target: np.ndarray, max_distance: float):
    """Each source point's nearest target (lowest index on ties) when its squared distance is < max_distance**2."""
    idx, best = np.empty(src.shape[0], dtype=np.int64), np.empty(src.shape[0])
    starts, step = _chunks(src.shape[0], target.shape[0])
    for s in starts:
        d2 = _sq_dist(src[s:s + step], target)
        idx[s:s + step] = np.argmin(d2, axis=1)
        best[s:s + step] = d2[np.arange(d2.shape[0]), idx[s:s + step]]
    return idx, best, best < max_distance * max_distance


def _umeyama(p: np.ndarray, q: np.ndarray) -> np.ndarray:
    """Eigen::umeyama(p, q, with_scaling=true): the similarity x -> c R x + t that maps p onto q in least squares.
    Fewer than 3 pairs, zero source spread or a cross-covariance of rank < 2 give the identity."""
    U4 = np.eye(4)
    n = p.shape[0]
    if n < 3:
        return U4
    mp, mq = p.sum(axis=0) / n, q.sum(axis=0) / n
    pd, qd = p - mp, q - mq
    var = (pd * pd).sum() / n
    if not var > 0.0:
        return U4
    sigma = qd.T @ pd / n
    u, s, vt = np.linalg.svd(sigma)
    if not s[1] > 1e-12 * s[0]:
        return U4
    S = np.ones(3)
    if np.linalg.det(u) * np.linalg.det(vt) < 0:
        S[2] = -1.0
    R = (u * S) @ vt
    c = float(s @ S) / var
    U4[:3, :3] = c * R
    U4[:3, 3] = mq - c * R @ mp
    return U4


def icp_scaled(source: np.ndarray, target: np.ndarray, init: np.ndarray, max_distance: float = ICP_MAX_DISTANCE,
               max_iteration: int = ICP_MAX_ITERATION, relative_fitness: float = ICP_RELATIVE, relative_rmse: float = ICP_RELATIVE):
    """open3d registration_icp with TransformationEstimationPointToPoint(with_scaling=True) (clustering_base.py:262-269).

    Each iteration pairs every transformed source point with its nearest target closer than ``max_distance``, solves
    Umeyama with scale on the pairs and left-multiplies the update onto the transform; it stops when both the fitness
    (pairs / source points) and the inlier rmse change by less than their thresholds.  The source is transformed from the
    original points every iteration.  Returns (T [4,4], fitness, rmse, iterations)."""
    src, tgt = np.asarray(source, dtype=np.float64), np.asarray(target, dtype=np.float64)
    T = np.array(init, dtype=np.float64)

    def evaluate(T):
        p = transform_points(src, T)
        idx, d2, ok = _correspond(p, tgt, max_distance)
        cnt = int(ok.sum())
        return p, idx, ok, (cnt / src.shape[0] if cnt else 0.0), (float(np.sqrt(d2[ok].sum() / cnt)) if cnt else 0.0)

    p, idx, ok, fitness, rmse = evaluate(T)
    it = 0
    while it < max_iteration:
        T = _umeyama(p[ok], tgt[idx[ok]]) @ T
        p, idx, ok, f, r = evaluate(T)
        it += 1
        done = abs(fitness - f) < relative_fitness and abs(rmse - r) < relative_rmse
        fitness, rmse = f, r
        if done:
            break
    return T, fitness, rmse, it


def _ward_merges(points: np.ndarray):
    """Ward's agglomerative clustering by the nearest-neighbour chain in centroid form.  Clusters live in slots
    0..n-1 (slot i starts as point i); a merge keeps the lower slot, so a cluster's slot is its smallest point index.
    The Ward distance of clusters a, b is sqrt(2 na nb / (na + nb)) * |ca - cb|.  Ties: the chain's predecessor wins,
    then the lower slot.  Returns [(slot_lo, slot_hi, height)] in execution order."""
    n = points.shape[0]
    c, size = points.astype(np.float64).copy(), np.ones(n)
    active = np.ones(n, dtype=bool)
    merges, chain = [], []
    for _ in range(n - 1):
        while True:
            if not chain:
                chain.append(int(np.flatnonzero(active)[0]))
            a = chain[-1]
            d = c - c[a]
            dist = np.sqrt((2.0 * size[a] * size) / (size[a] + size)) * np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
            dist[~active] = np.inf
            dist[a] = np.inf
            b = int(np.argmin(dist))
            if len(chain) >= 2 and dist[chain[-2]] == dist[b]:
                b = chain[-2]
            if len(chain) >= 2 and b == chain[-2]:
                break
            chain.append(b)
        chain.pop()
        chain.pop()
        lo, hi = min(a, b), max(a, b)
        nl, nh = size[lo], size[hi]
        c[lo] = (nl * c[lo] + nh * c[hi]) / (nl + nh)
        size[lo] = nl + nh
        active[hi] = False
        merges.append((lo, hi, float(dist[b])))
    return merges


def _ward_top(merges) -> List[int]:
    """The up to 5 highest merges as cuts see them: the root, then repeatedly the highest (height, then later merge) of
    the merges directly below those taken.  Cutting at k undoes the first k - 1 of them."""
    if not merges:
        return []

    def children(m):
        lo, hi, _ = merges[m]
        out = []
        for s in (lo, hi):  # the subtree on slot s is the latest earlier merge that kept slot s, else the leaf s
            prev = [j for j in range(m - 1, -1, -1) if merges[j][0] == s]
            if prev:
                out.append(prev[0])
        return out

    top, frontier = [len(merges) - 1], children(len(merges) - 1)
    while len(top) < MAX_FRUIT_PER_GROUP - 1 and frontier:
        m = max(frontier, key=lambda j: (merges[j][2], j))
        frontier.remove(m)
        top.append(m)
        frontier += children(m)
    return top


def ward_cut_centres(points: np.ndarray) -> np.ndarray:
    """Sub-centres of ``AgglomerativeClustering(n_clusters=k, linkage="ward")`` for k = 2..6 from one Ward tree:
    [20,3], rows CUT_OFFSETS[k-2]:CUT_OFFSETS[k-1] hold the k sub-cluster means ordered by their smallest point index.
    A cut with more clusters than points is NaN."""
    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    n = pts.shape[0]
    out = np.full((CUT_OFFSETS[-1], 3), np.nan)
    if n == 0:
        return out
    merges = _ward_merges(pts)
    top = _ward_top(merges)
    parent = np.arange(n)
    topset = set(top)
    for m, (lo, hi, _) in enumerate(merges):
        if m not in topset:
            parent[hi] = lo
    root = parent.copy()
    for i in range(n):  # parent[i] <= i: one pass in slot order resolves every root
        root[i] = i if parent[i] == i else root[parent[i]]
    base = sorted(set(root.tolist()))
    sums = {r: pts[root == r].sum(axis=0) for r in base}
    cnts = {r: float((root == r).sum()) for r in base}
    clusters = list(base)
    for k in range(len(base), 1, -1):  # len(base) = len(top) + 1 clusters, then undo the splits from the lowest up
        if k <= MAX_FRUIT_PER_GROUP:
            rows = slice(CUT_OFFSETS[k - 2], CUT_OFFSETS[k - 1])
            out[rows] = np.stack([sums[r] / cnts[r] for r in sorted(clusters)])
        lo, hi, _ = merges[top[k - 2]]
        sums[lo], cnts[lo] = sums[lo] + sums[hi], cnts[lo] + cnts[hi]
        clusters.remove(hi)
    return out


def hausdorff(a: np.ndarray, b: np.ndarray) -> float:
    """Symmetric Hausdorff distance max(h(a, b), h(b, a)) of two non-empty point sets, exact (brute force)."""
    def directed2(p, q):
        worst = 0.0
        starts, step = _chunks(p.shape[0], q.shape[0])
        for s in starts:
            worst = max(worst, float(_sq_dist(p[s:s + step], q).min(axis=1).max()))
        return worst

    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape[0] == 0 or b.shape[0] == 0:
        raise ValueError("hausdorff needs two non-empty point sets")
    return float(np.sqrt(max(directed2(a, b), directed2(b, a))))


def _decide(vt: float, volume: float, sample: Optional[np.ndarray]) -> str:
    """'split', 'prune' or 'one' for a group of alpha = 10 volume ``volume`` and surface ``sample``, the template's
    volume being ``vt`` (clustering_base.py:372, :422)."""
    if sample is None:  # empty alpha = 100 boundary: nothing to sample, the group counts as one fruit
        return "one"
    if vt < SPLIT_RATIO * volume:
        return "split"
    return "prune" if PRUNE_RATIO * vt > abs(volume) else "one"


def _alpha(jobs) -> Tuple[List[Tuple[List[str], Dict[int, tuple]]], Dict[tuple, np.ndarray]]:
    """The host half of stage 3 for every job (groups, template [m,3] float64, seed).  The template volume is computed
    once per template, the alpha shapes once per group content and the surface sample once per (content, seed, group
    index), since the sample's hash includes the group index.  Returns, per job, (decisions [G], {group to split: sample
    key}) and the samples {sample key: [SURFACE_SAMPLES,3]}."""
    template_vol, shapes, samples, plans = {}, {}, {}, []  # template bytes -> V_t; content -> (V, boundary)
    for groups, tmpl, seed in jobs:
        tkey = tmpl.tobytes()
        if tkey not in template_vol:
            template_vol[tkey] = float(alpha_shape(tmpl, (ALPHA_VOLUME,))[0][0])
        decisions, picks = [], {}
        for g, grp in enumerate(groups):
            p64 = np.asarray(grp, dtype=np.float64).reshape(-1, 3)
            content = (p64.shape[0], p64.tobytes())
            skey = (content, seed, g)
            if content not in shapes:
                volumes, boundaries, samples[skey] = alpha_shape(p64, (ALPHA_VOLUME, ALPHA_SURFACE), seed=seed, group=g)
                shapes[content] = (volumes[0], boundaries[-1])
            elif skey not in samples:
                samples[skey] = _surface_sample(p64, shapes[content][1], SURFACE_SAMPLES, seed, g)
            decisions.append(_decide(template_vol[tkey], shapes[content][0], samples[skey]))
            if decisions[-1] == "split":
                picks[g] = skey
        plans.append((decisions, picks))
    return plans, samples


def alpha_stage(groups: Sequence[np.ndarray], template: np.ndarray, seed: int = 0):
    """The host half of stage 3 (clustering_base.py:350-429): per group 'one', 'prune' or 'split' and, for each group
    to split, its surface sample.  Returns (decisions [G], samples {group: [SURFACE_SAMPLES,3]})."""
    plans, samples = _alpha([(groups, np.asarray(template, dtype=np.float64), seed)])
    decisions, picks = plans[0]
    return decisions, {g: samples[k] for g, k in picks.items()}


def match_candidates(samples: Sequence[np.ndarray], template: np.ndarray, device=None):
    """ICP (k = 1), Ward sub-centres (k = 2..6) and the six Hausdorff distances of each surface sample.  Returns
    (T [B,4,4], sub-centres [B,20,3], distances [B,6], ICP iterations [B]) as numpy arrays; ``device`` (a CUDA device)
    runs one launch of each kernel over all samples, None the numpy code."""
    return _match(list(samples), [(np.asarray(template, dtype=np.float64), list(range(len(samples))))], device)


def _match(samples: List[np.ndarray], fits: List[Tuple[np.ndarray, List[int]]], device):
    """``match_candidates`` for several templates: ``fits`` holds (template [m,3] float64, the indices of the samples it
    is fitted to) per template.  Returns (T [P,4,4], sub-centres [S,20,3], distances [P,6], ICP iterations [P]): the
    sub-centres of each sample, the rest for the P (template, sample) pairs in the order of ``fits``.  ``device`` runs
    one ICP launch per template, one Ward launch over all samples and one Hausdorff launch over all pairs."""
    if not samples:
        return np.zeros((0, 4, 4)), np.zeros((0, 20, 3)), np.zeros((0, MAX_FRUIT_PER_GROUP)), np.zeros(0, dtype=np.int64)
    inits = [s.mean(axis=0) for s in samples]  # ICP starts from a translation to the sample's mean
    if device is None:
        cuts = np.stack([ward_cut_centres(s) for s in samples])
        T, d, its = [], [], []
        for tmpl, rows in fits:
            for j in rows:
                Tj, _, _, it = icp_scaled(tmpl, samples[j], _translation(inits[j]))
                T.append(Tj)
                its.append(it)
                d.append([hausdorff(samples[j], copies) for copies in _template_copies(tmpl, Tj, cuts[j])])
        return np.stack(T), cuts, np.array(d), np.array(its, dtype=np.int64)
    f64 = dict(dtype=torch.float64, device=device)
    offsets = _offsets(samples)
    targets = torch.from_numpy(np.concatenate(samples)).to(**f64)
    cuts = ops.ward_cut(targets, offsets)
    T, its, hyp, a_ranges = [], [], [], []
    for tmpl, rows in fits:
        t = torch.from_numpy(tmpl).to(**f64)
        sub = [samples[j] for j in rows]
        Tt, _, _, it = ops.icp_scaled(t, torch.from_numpy(np.concatenate(sub)).to(**f64), _offsets(sub),
                                      torch.from_numpy(np.stack([inits[j] for j in rows])).to(**f64))
        # the six hypotheses of every sample as segments of one array, in the order (sample, k)
        x, y, z = t[:, 0], t[:, 1], t[:, 2]
        R = Tt[:, :3, :]
        fitted = torch.stack([((R[:, r, 0:1] * x + R[:, r, 1:2] * y) + R[:, r, 2:3] * z) + R[:, r, 3:4] for r in range(3)], dim=2)
        for b, j in enumerate(rows):
            hyp.append(fitted[b])
            for k in range(2, MAX_FRUIT_PER_GROUP + 1):
                centres = cuts[j, CUT_OFFSETS[k - 2]:CUT_OFFSETS[k - 1]]
                hyp.append((t[None, :, :] + centres[:, None, :]).reshape(-1, 3))
            a_ranges += [offsets[j:j + 2]] * MAX_FRUIT_PER_GROUP
        T.append(Tt)
        its.append(it)
    b_offsets = _offsets(hyp)
    d = ops.hausdorff(targets, np.stack(a_ranges), torch.cat(hyp), np.stack([b_offsets[:-1], b_offsets[1:]], axis=1))
    return (torch.cat(T).cpu().numpy(), cuts.cpu().numpy(), d.view(-1, MAX_FRUIT_PER_GROUP).cpu().numpy(),
            torch.cat(its).cpu().numpy().astype(np.int64))


def _offsets(segments) -> np.ndarray:
    """Ascending int64 offsets [len + 1] of consecutive segments (arrays or tensors) of one concatenation."""
    return np.concatenate([[0], np.cumsum([s.shape[0] for s in segments], dtype=np.int64)])


def _translation(t) -> np.ndarray:
    T = np.eye(4)
    T[:3, 3] = t
    return T


def _template_copies(tmpl: np.ndarray, T: np.ndarray, cuts: np.ndarray) -> List[np.ndarray]:
    """The k = 1..6 fruit hypotheses: the ICP-transformed template, then k copies translated to the sub-centres."""
    out = [transform_points(tmpl, T)]
    for k in range(2, MAX_FRUIT_PER_GROUP + 1):
        centres = cuts[CUT_OFFSETS[k - 2]:CUT_OFFSETS[k - 1]]
        out.append((tmpl[None, :, :] + centres[:, None, :]).reshape(-1, 3))
    return out


def _assemble(groups: Sequence[np.ndarray], tmpl: np.ndarray, decisions: List[str], matched: Dict[int, tuple]) -> Dict:
    """``split_clusters``' result from the decisions of the alpha stage and the match of each group to split:
    ``matched`` {group: (T [4,4], sub-centres [20,3], distances [6], ICP iterations)}."""
    centers, per_group, its = [], np.zeros(len(groups), dtype=np.int64), []
    for g, (pts, dec) in enumerate(zip(groups, decisions)):
        if dec == "one":
            centers.append(np.asarray(pts, dtype=np.float64).mean(axis=0)[None])
            per_group[g] = 1
        elif dec == "split":
            T, cuts, d, it = matched[g]
            k = int(np.argmin(d)) + 1
            per_group[g] = k
            centers.append(transform_points(tmpl, T).mean(axis=0)[None] if k == 1 else cuts[CUT_OFFSETS[k - 2]:CUT_OFFSETS[k - 1]])
            its.append(it)
    split = per_group[np.array([dec == "split" for dec in decisions], dtype=bool)]
    return {"centers": np.concatenate(centers) if centers else np.zeros((0, 3)), "fruit_per_group": per_group,
            "num_split_extra": int((split - 1).sum()), "num_pruned": int(sum(dec == "prune" for dec in decisions)),
            "icp_iterations": np.array(its, dtype=np.int64)}


def split_clusters(groups: Sequence[np.ndarray], template: np.ndarray, seed: int = 0, device=None) -> Dict:
    """Stage 3 of the reference clustering (clustering_base.py:261-511) on the merged groups, in group order.

    A group whose alpha = 10 volume V satisfies V_t < 0.9 V (V_t: the template's) is split: it counts argmin_k d_k
    fruit (lowest k on ties), where d_1 is the Hausdorff distance of its surface sample S to the ICP-fitted template and
    d_k (k = 2..6) that of S to k template copies at S's Ward sub-centres.  Otherwise a group with 0.3 V_t > |V| is
    pruned, and any other group is one fruit centred at its mean.  Returns {'centers' [m,3], 'fruit_per_group' [G]
    (0 = pruned), 'num_split_extra', 'num_pruned', 'icp_iterations' (per split group)}; ``device`` as in
    ``match_candidates``."""
    return _stage3([(groups, np.asarray(template, dtype=np.float64), seed)], device)[0]


def _stage3(jobs, device, on_stage: Callable[[str], None] = lambda stage: None) -> List[Dict]:
    """``split_clusters`` for every job (groups, template [m,3] float64, seed), sharing the host work of ``_alpha`` and
    the launches of ``_match`` between the jobs.  ``on_stage`` is called with 'alpha' and 'match' as they end."""
    plans, samples = _alpha(jobs)
    on_stage("alpha")
    keys = list(dict.fromkeys(k for _, picks in plans for k in picks.values()))  # the distinct samples to split
    row = {k: j for j, k in enumerate(keys)}
    fits: Dict[bytes, Tuple[np.ndarray, Dict[int, None]]] = {}  # template bytes -> (template, rows fitted to it), in first use
    for (_, tmpl, _), (_, picks) in zip(jobs, plans):
        fits.setdefault(tmpl.tobytes(), (tmpl, {}))[1].update(dict.fromkeys(row[k] for k in picks.values()))
    pair = {p: i for i, p in enumerate((tkey, j) for tkey, (_, rows) in fits.items() for j in rows)}
    T, cuts, d, its = _match([samples[k] for k in keys], [(tmpl, list(rows)) for tmpl, rows in fits.values() if rows], device)
    on_stage("match")
    out = []
    for (groups, tmpl, _), (decisions, picks) in zip(jobs, plans):
        matched = {}
        for g, k in picks.items():
            i = pair[(tmpl.tobytes(), row[k])]
            matched[g] = (T[i], cuts[row[k]], d[i], its[i])
        out.append(_assemble(groups, tmpl, decisions, matched))
    return out


def load_obj_centres(path) -> np.ndarray:
    """Ground-truth fruit centres from an OBJ file with one object per fruit (the synthetic trees' ``fruits.obj``,
    clustering_base.py:67-111 load_obj_file): an ``o`` line starts a new object, each ``v`` line adds a vertex to the
    current object, and a fruit's centre is the mean of its object's vertices.  [K,3] float64 in object order.

    A file without any ``o`` line, a vertex before the first ``o`` line or an object without vertices raises
    ValueError.  The reference crashes on the first (its vertex list does not exist yet), silently counts the vertices
    before the first ``o`` as part of the first object, and takes the mean of an empty object as NaN."""
    objects: List[List[List[float]]] = []
    stray = 0  # line of the first vertex before any 'o' line
    with open(path, "r") as f:
        for num, line in enumerate(f, 1):
            parts = line.split()
            if not parts:
                continue
            if parts[0] == "o":
                objects.append([])
            elif parts[0] == "v":
                if len(parts) < 4:
                    raise ValueError(f"{path}:{num}: vertex with fewer than 3 coordinates")
                if not objects:
                    stray = stray or num
                    continue
                objects[-1].append([float(v) for v in parts[1:4]])
    if not objects:
        raise ValueError(f"{path}: no 'o' line: the file holds no fruit objects")
    if stray:
        raise ValueError(f"{path}:{stray}: vertex before the first 'o' line")
    empty = [i for i, o in enumerate(objects) if not o]
    if empty:
        raise ValueError(f"{path}: object {empty[0]} has no vertices")
    return np.stack([np.asarray(o, dtype=np.float64).mean(axis=0) for o in objects])


def load_gt_centres(path) -> np.ndarray:
    """Ground-truth fruit centres [K,3] float64 in the reference's formats, by file suffix:
    - ``.obj``: one object per fruit (``load_obj_centres``);
    - ``.ply``: a line set of 8-corner boxes as open3d writes it (Fuji's ``lineset_aligned.ply``), ascii or binary; the
      centres are the means of each 8 consecutive vertices (clustering_base.py:459-462).  A vertex count that is not a
      multiple of 8 raises ValueError;
    - ``.npy``: an array of centres, as ``count --gt-centers`` reads it."""
    from pathlib import Path

    suffix = Path(path).suffix.lower()
    if suffix == ".obj":
        return load_obj_centres(path)
    if suffix == ".ply":
        from .export.exporter_utils import read_line_set_points

        pts = read_line_set_points(path)
        if pts.shape[0] % 8:
            raise ValueError(f"{path}: {pts.shape[0]} line-set vertices are not whole 8-corner boxes")
        return pts.reshape(-1, 8, 3).mean(axis=1)
    if suffix == ".npy":
        return np.load(path).astype(np.float64).reshape(-1, 3)
    raise ValueError(f"{path}: ground truth must be .obj (fruit objects), .ply (line set of boxes) or .npy (centres)")


def evaluate_count(centres: np.ndarray, gt_centres: np.ndarray, max_distance: float = 0.15) -> Dict:
    """The reference's score of a count (clustering_base.py:464-506): centres are visited in order and each takes the
    nearest remaining ground-truth centre if that is closer than ``max_distance`` (a true positive; the ground-truth
    centre is then used up), else it is a false positive.  Unmatched ground-truth centres are false negatives.
    Precision, recall and F1 are 0 where their denominator is 0."""
    remaining = np.asarray(gt_centres, dtype=np.float64).reshape(-1, 3)
    tp = fp = 0
    for c in np.asarray(centres, dtype=np.float64).reshape(-1, 3):
        if remaining.shape[0]:
            dist = np.linalg.norm(remaining - c, axis=1)
            j = int(np.argmin(dist))
            if dist[j] < max_distance:
                tp += 1
                remaining = np.delete(remaining, j, axis=0)
                continue
        fp += 1
    fn = int(remaining.shape[0])
    precision = tp / (tp + fp) if tp + fp else 0.0
    recall = tp / (tp + fn) if tp + fn else 0.0
    f1 = 2 * precision * recall / (precision + recall) if precision + recall else 0.0
    return {"TP": tp, "FP": fp, "FN": fn, "precision": precision, "recall": recall, "F1": f1}


# ---- parameter sweeps: many counts of one cloud (clustering/run_clustering_sweep.py) -----------------------------------

COUNT_ARGS = ("eps", "min_samples", "cluster_merge_distance", "down_sample", "remove_outliers_nb_points", "remove_outliers_radius", "seed")
_COUNT_DEFAULTS = {"down_sample": 0.0, "remove_outliers_nb_points": 0, "remove_outliers_radius": 0.0, "seed": 0}
MAX_RADIUS_RATIO, MAX_RADII = 4.0, 16  # what one ops.radius_count_multi call accepts


def count_sweep(points, configs: Sequence[Dict], templates: Optional[Sequence[Optional[np.ndarray]]] = None,
                on_stage: Optional[Callable[[str], None]] = None) -> List[Dict]:
    """``count_fruits(points, **configs[i], template=templates[i])`` for every i: each result is exactly what that call
    returns alone.  ``configs``: dicts of count_fruits' keyword arguments (``COUNT_ARGS``); ``templates``: one fruit
    template (or None: no stage 3) per config, all None when omitted.

    numpy input runs that loop; on a CUDA tensor ``count_fruits`` is this function with one config.  A CUDA tensor
    shares the work the configs have in common: the radius counts of each distinct outlier radius (one walk per run
    of radii ``_radius_chunks`` makes, cap = the largest nb_points + 1), the voxel down-sampling of each
    distinct filtered set, DBSCAN once per distinct (set, eps, min_samples), stage 2 once per distinct (set, eps,
    min_samples, merge distance); stage 3's alpha shapes once per group content, its surface sample
    once per (content, seed, group index), and one ICP launch per template, one Ward launch over every distinct sample
    and one Hausdorff launch over every (template, sample) pair.  ``on_stage`` (device path only) is called with the
    name of each stage as it ends: 'radius_count', 'voxel', 'dbscan', 'merge', 'alpha', 'match'."""
    configs = [dict(c) for c in configs]
    templates = [None] * len(configs) if templates is None else list(templates)
    if len(templates) != len(configs):
        raise ValueError(f"{len(templates)} templates for {len(configs)} configs")
    for c in configs:
        unknown = sorted(set(c) - set(COUNT_ARGS))
        if unknown:
            raise ValueError(f"count_sweep: unknown count_fruits arguments {unknown}")
    if not _on_device(points):
        return [count_fruits(points, **c, template=t) for c, t in zip(configs, templates)]
    return _device_count_sweep(points, [{**_COUNT_DEFAULTS, **c} for c in configs], templates, on_stage or (lambda stage: None))


def _radius_chunks(values: Sequence) -> List[List]:
    """Ascending radii cut into runs one ``ops.radius_count_multi`` call accepts: at most MAX_RADII entries, the largest at
    most MAX_RADIUS_RATIO times the first."""
    chunks: List[List] = []
    for r in sorted(values):
        if chunks and len(chunks[-1]) < MAX_RADII and not r > MAX_RADIUS_RATIO * chunks[-1][0]:
            chunks[-1].append(r)
        else:
            chunks.append([r])
    return chunks


def _device_count_sweep(points, configs: List[Dict], templates: List, on_stage) -> List[Dict]:
    pts = ops.cluster_points(points)

    def outlier_key(c):  # None: no outlier removal (an empty cloud has no outliers to count)
        nb, r = c["remove_outliers_nb_points"], c["remove_outliers_radius"]
        return (int(nb), float(r)) if nb > 0 and r > 0 and pts.shape[0] else None

    # radius counts: each distinct radius once, saturated at the largest nb_points + 1 it is used with
    caps: Dict[float, int] = {}
    for c in configs:
        k = outlier_key(c)
        if k is not None:
            caps[k[1]] = max(caps.get(k[1], 0), k[0] + 1)
    counts = {}
    for chunk in _radius_chunks(list(caps)):
        if len(chunk) == 1:  # fnr_radius_count: bit-equal to a one-radius fnr_radius_count_multi, and its errors name it
            counts[chunk[0]] = ops.radius_count(pts, chunk[0], caps[chunk[0]])
        else:
            counts.update(zip(chunk, ops.radius_count_multi(pts, chunk, [caps[r] for r in chunk])))
    filtered = {None: pts}
    for c in configs:
        k = outlier_key(c)
        if k is not None and k not in filtered:
            filtered[k] = pts[counts[k[1]] - 1 >= k[0]]  # = _device_remove_radius_outliers: min(count, cap) - 1 >= nb
    on_stage("radius_count")

    down = {}
    for c in configs:
        key = (outlier_key(c), float(c["down_sample"]))
        if key not in down:
            down[key] = ops.voxel_down_sample(filtered[key[0]], key[1])
    on_stage("voxel")

    # one DBSCAN per distinct (set, eps, min_samples); separate calls beat one shared-grid walk over several eps (DESIGN 4.3k)
    labels = {}
    for c in configs:
        key = (outlier_key(c), float(c["down_sample"]))
        prob = (float(c["eps"]), int(c["min_samples"]))
        if down[key].shape[0] and (key, prob) not in labels:
            labels[(key, prob)] = ops.dbscan(down[key], *prob)
    on_stage("dbscan")

    stage2, results, jobs = {}, [None] * len(configs), []
    for i, (c, t) in enumerate(zip(configs, templates)):
        key = (outlier_key(c), float(c["down_sample"]))
        prob = (float(c["eps"]), int(c["min_samples"]))
        s2 = (key, prob, float(c["cluster_merge_distance"]))
        if s2 not in stage2:
            dpts = down[key]
            if dpts.shape[0] == 0:
                stage2[s2] = [{"count": 0, "count_before_merge": 0, "centers": np.zeros((0, 3)), "num_points": 0}, None, []]
            else:
                lab, k = labels[(key, prob)]
                sums, cnt = ops.cluster_sums(dpts, lab, k)
                res, group_of = _merge_groups(sums.cpu().numpy(), cnt.cpu().numpy(), s2[2])
                res["num_points"] = int(dpts.shape[0])
                stage2[s2] = [res, (dpts, lab, group_of), None]
        entry = stage2[s2]
        if t is None:
            results[i] = {**entry[0], "centers": entry[0]["centers"].copy()}  # as independent as separate calls
            continue
        if entry[2] is None:
            entry[2] = _device_groups(*entry[1])
        jobs.append((i, entry[0], (entry[2], np.asarray(t, dtype=np.float64), int(c["seed"]))))
    on_stage("merge")
    for (i, res, _), split in zip(jobs, _stage3([job for _, _, job in jobs], pts.device, on_stage)):
        results[i] = _with_split(res, split)
    return results
