"""Per-fruit measurement of the fruit meshes (``fruit_mesh.ply`` of ``tsdf``, ``fruit_poisson_mesh.ply`` of ``poisson``;
DESIGN section 4.3n): each face gets a group, and each group its face count, area, area-weighted centroid, fitted
sphere, volume, solid-angle coverage and edge counts.

Where it runs depends on the input, as ``clustering.count_fruits``: CUDA tensors run the kernels of fnr_measure.cu through
``ops``; anything else runs the numpy / scipy restatement below.  Labels and integer counts agree exactly, fp64 values to
summation order.

Grouping is by connected components of the faces (shared vertex indices; marching cubes shares one vertex per grid
edge, so an exported fruit is one component) or, given centres such as ``count``'s, by the centre nearest each face
centroid, which separates touching fruit.
"""
from __future__ import annotations

import json
import math
from typing import Dict, Optional

import numpy as np
import torch

from . import ops

PIVOT_TOL = 1e-12  # fnr_measure.cu kPivotTol
_CHUNK = 1 << 16


def _on_device(x) -> bool:
    return isinstance(x, torch.Tensor) and x.is_cuda


# ---- the restatement --------------------------------------------------------------------------------------------------
def _mesh(vertices, faces):
    v = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
    f = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError(f"face indices must lie in [0, {len(v)})")
    return v, f


def restated_components(faces, num_vertices: int):
    """(int32 [F] labels, G): connected components through shared vertex indices (scipy ``connected_components``),
    vertices that no face uses dropped, components numbered by their smallest vertex index."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    f = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)
    V = int(num_vertices)
    if len(f) == 0:
        return np.zeros(0, np.int32), 0
    if f.min() < 0 or f.max() >= V:
        raise ValueError(f"face indices must lie in [0, {V})")
    rows, cols = np.concatenate([f[:, 0], f[:, 1]]), np.concatenate([f[:, 1], f[:, 2]])
    graph = coo_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(V, V)).tocsr()
    _, comp = connected_components(graph, directed=False)
    used = np.zeros(V, bool)
    used[f.reshape(-1)] = True
    minv = np.full(comp.max() + 1, V, np.int64)
    np.minimum.at(minv, comp[used], np.flatnonzero(used))
    kept = np.flatnonzero(minv < V)
    rank = np.full(len(minv), -1, np.int64)
    rank[kept[np.argsort(minv[kept], kind="stable")]] = np.arange(len(kept))
    return rank[comp[f[:, 0]]].astype(np.int32), int(len(kept))


def face_centroids(v: np.ndarray, f: np.ndarray) -> np.ndarray:
    """(v0 + v1 + v2) / 3, summed left to right."""
    return ((v[f[:, 0]] + v[f[:, 1]]) + v[f[:, 2]]) / 3.0


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def face_areas(v: np.ndarray, f: np.ndarray) -> np.ndarray:
    """|e1 x e2| / 2."""
    n = _cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    return np.sqrt(_dot(n, n)) * 0.5


def restated_assign(vertices, faces, centers, max_distance: float = math.inf) -> np.ndarray:
    """int32 [F]: the index of the centre nearest each face centroid in fp64 squared distance, ties to the lower index,
    -1 when the distance exceeds ``max_distance``."""
    v, f = _mesh(vertices, faces)
    c = np.ascontiguousarray(centers, dtype=np.float64).reshape(-1, 3)
    _check_assign_args(c, max_distance)
    md2 = float(max_distance) * float(max_distance)
    out = np.full(len(f), -1, np.int32)
    for s in range(0, len(f), _CHUNK):
        p = face_centroids(v, f[s:s + _CHUNK])
        best, bi = np.full(len(p), np.inf), np.full(len(p), -1, np.int64)
        for k0 in range(0, len(c), 256):
            d = p[:, None, :] - c[None, k0:k0 + 256, :]
            d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
            d2 = np.where(np.isnan(d2), np.inf, d2)
            j = np.argmin(d2, axis=1)
            m = d2[np.arange(len(p)), j]
            upd = m < best
            best[upd], bi[upd] = m[upd], j[upd] + k0
        out[s:s + _CHUNK] = np.where((bi >= 0) & (best <= md2), bi, -1)
    return out


def _check_assign_args(centers: np.ndarray, max_distance: float) -> None:
    if not np.isfinite(centers).all():
        raise ValueError("centres must be finite")
    if not float(max_distance) > 0:
        raise ValueError(f"max_distance must be > 0, got {max_distance}")


def kasa_solve(A: float, S, s1, t, T: float):
    """The fit of fnr_measure.cu's kasa_solve, operation for operation: (ok, x [3] relative to the centroid, r)."""
    if not A > 0.0:
        return False, None, None
    s2 = T / A
    if not s2 > 0.0:
        return False, None, None
    sc = math.sqrt(s2)
    as2, as1 = A * s2, A * sc
    as3 = as2 * sc
    ij = ((0, 1, 2), (1, 3, 4), (2, 4, 5))
    M = [[0.0] * 5 for _ in range(4)]
    for i in range(3):
        for j in range(3):
            M[i][j] = (4.0 * float(S[ij[i][j]])) / as2
        M[i][3] = (2.0 * float(s1[i])) / as1
        M[3][i] = M[i][3]
        M[i][4] = (2.0 * float(t[i])) / as3
    M[3][3] = 1.0
    M[3][4] = float(T) / as2
    for k in range(4):
        p = k
        for i in range(k + 1, 4):
            if abs(M[i][k]) > abs(M[p][k]):
                p = i
        if not abs(M[p][k]) > PIVOT_TOL:
            return False, None, None
        M[k], M[p] = M[p], M[k]
        for i in range(k + 1, 4):
            fct = M[i][k] / M[k][k]
            for j in range(k, 5):
                M[i][j] = M[i][j] - fct * M[k][j]
    u = [0.0] * 4
    for k in range(3, -1, -1):
        acc = M[k][4]
        for j in range(k + 1, 4):
            acc = acc - M[k][j] * u[j]
        u[k] = acc / M[k][k]
    rr = u[3] + ((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2])
    if not rr > 0.0:
        return False, None, None
    return True, np.array(u[:3]) * sc, math.sqrt(rr) * sc


def restated_edges(faces, face_group, num_groups: int):
    """(boundary [G], nonmanifold [G]) int64: per (edge key, group), one half-edge is a boundary edge and three or more a
    non-manifold edge; edge key = (min, max) vertex id."""
    f = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)
    g = np.repeat(np.asarray(face_group, np.int64).reshape(-1), 3)
    a, b = f.reshape(-1), np.roll(f, -1, axis=1).reshape(-1)
    pairs = np.stack([np.minimum(a, b), np.maximum(a, b), g], axis=1)[g >= 0]
    G = int(num_groups)
    if len(pairs) == 0:
        return np.zeros(G, np.int64), np.zeros(G, np.int64)
    uniq, counts = np.unique(pairs, axis=0, return_counts=True)
    return (np.bincount(uniq[counts == 1, 2], minlength=G).astype(np.int64), np.bincount(uniq[counts >= 3, 2], minlength=G).astype(np.int64))


def restated_measure(vertices, faces, face_group, num_groups: int) -> Dict[str, np.ndarray]:
    """fnr_mesh_measure_groups in numpy fp64 (the keys of ``ops.mesh_measure_groups``)."""
    v, f = _mesh(vertices, faces)
    lab = np.asarray(face_group, np.int64).reshape(-1)
    G = int(num_groups)
    if len(lab) != len(f):
        raise ValueError(f"{len(lab)} face labels for {len(f)} faces")
    if len(lab) and (lab.min() < -1 or lab.max() >= G):
        raise ValueError(f"face labels must lie in [-1, {G})")
    area_f, cent_f = face_areas(v, f), face_centroids(v, f)
    un = lab < 0
    sel = ~un
    g, a, c, fs = lab[sel], area_f[sel], cent_f[sel], f[sel]
    bsum = lambda w: np.bincount(g, weights=w, minlength=G)  # noqa: E731
    n = np.bincount(g, minlength=G).astype(np.int64)
    A = bsum(a)
    with np.errstate(invalid="ignore", divide="ignore"):
        m = np.where((A > 0)[:, None], np.stack([bsum(a * c[:, k]) for k in range(3)], 1) / A[:, None],
                     np.stack([bsum(c[:, k]) for k in range(3)], 1) / n[:, None])
    p = c - m[g]
    wp = a[:, None] * p
    pp = _dot(p, p)
    S = np.stack([bsum(wp[:, i] * p[:, j]) for i, j in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))], 1)
    s1 = np.stack([bsum(wp[:, k]) for k in range(3)], 1)
    t = np.stack([bsum(wp[:, k] * pp) for k in range(3)], 1)
    T = bsum(a * pp)
    ctr, r, ok = m.copy(), np.full(G, np.nan), np.zeros(G, np.int32)
    for k in np.flatnonzero(n > 0):
        good, x, rad = kasa_solve(float(A[k]), S[k], s1[k], t[k], float(T[k]))
        if good:
            ctr[k], r[k], ok[k] = m[k] + x, rad, 1
        else:
            r[k] = math.sqrt(T[k] / A[k]) if A[k] > 0 else 0.0
    d = [v[fs[:, k]] - ctr[g] for k in range(3)]
    pc = c - ctr[g]
    e = np.sqrt(_dot(pc, pc)) - r[g]
    det = _dot(d[0], _cross(d[1], d[2]))
    la, lb, lc = (np.sqrt(_dot(x, x)) for x in d)
    den = ((la * lb * lc + _dot(d[0], d[1]) * lc) + _dot(d[0], d[2]) * lb) + _dot(d[1], d[2]) * la
    with np.errstate(invalid="ignore", divide="ignore"):
        rms = np.where(A > 0, np.sqrt(bsum(a * (e * e)) / A), 0.0)
    rms[n == 0] = np.nan
    boundary, nonmanifold = restated_edges(f, lab, G)
    return {"faces": n, "boundary_edges": boundary, "nonmanifold_edges": nonmanifold, "area": A, "centroid": m,
            "sphere": np.concatenate([ctr, r[:, None], rms[:, None]], axis=1), "volume": bsum(det) / 6.0,
            "coverage": bsum(2.0 * np.arctan2(det, den)) / (4.0 * math.pi), "fit_ok": ok,
            "unassigned_faces": np.array([int(un.sum())], np.int64), "unassigned_area": np.array([float(area_f[un].sum())])}


# ---- the driver -------------------------------------------------------------------------------------------------------
def measure_fruits(vertices, faces, centers=None, max_distance: Optional[float] = None) -> Dict[str, np.ndarray]:
    """Measure each group of faces of a triangle mesh (``vertices`` [V,3], ``faces`` [F,3]).  Without ``centers`` the
    groups are the connected components; with ``centers`` [K,3] group k holds the faces whose centroid is nearest centre
    k and within ``max_distance`` (None: no limit).  CUDA tensors run on the GPU, anything else on the host.

    Returns numpy arrays per group: 'faces', 'area', 'centroid' [G,3], 'center' [G,3], 'radius', 'rms', 'fit_ok',
    'volume', 'coverage', 'volume_extrapolated' (the volume of a closed group, whose star volume is exact about any point;
    of an open one volume / coverage, NaN when coverage <= 0), 'equivalent_diameter'
    ((6 volume_extrapolated / pi)^(1/3), NaN when that volume is not positive), 'boundary_edges', 'nonmanifold_edges',
    'closed'; and 'face_group' [F], 'num_groups', 'unassigned_faces', 'unassigned_area'."""
    md = math.inf if max_distance is None else float(max_distance)
    if centers is not None:
        _check_assign_args(np.asarray(centers.detach().cpu() if torch.is_tensor(centers) else centers, np.float64), md)
    if _on_device(vertices):
        dev = vertices.device
        faces = torch.as_tensor(faces, device=dev)
        if centers is None:
            labels, G = ops.mesh_components(faces, int(vertices.reshape(-1, 3).shape[0]))
        else:
            c = torch.as_tensor(centers, dtype=torch.float64, device=dev).reshape(-1, 3)
            labels, G = ops.mesh_assign_centers(vertices, faces, c, md), int(c.shape[0])
        res = {k: t.cpu().numpy() for k, t in ops.mesh_measure_groups(vertices, faces, labels, G).items()}
        labels = labels.cpu().numpy()
    else:
        v, f = _mesh(vertices, faces)
        if centers is None:
            labels, G = restated_components(f, len(v))
        else:
            c = np.asarray(centers, np.float64).reshape(-1, 3)
            labels, G = restated_assign(v, f, c, md), len(c)
        res = restated_measure(v, f, labels, G)
    vol, cov = res["volume"], res["coverage"]
    closed = (res["boundary_edges"] == 0) & (res["nonmanifold_edges"] == 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        # a closed surface needs no extrapolation, and its coverage is 0 when the fitted centre lies outside it (a torus)
        vext = np.where(closed, vol, np.where(cov > 0, vol / np.where(cov > 0, cov, 1.0), np.nan))
        diam = np.where(vext > 0, np.cbrt(6.0 * np.where(vext > 0, vext, 0.0) / math.pi), np.nan)
    return {"faces": res["faces"], "area": res["area"], "centroid": res["centroid"], "center": res["sphere"][:, :3],
            "radius": res["sphere"][:, 3], "rms": res["sphere"][:, 4], "fit_ok": res["fit_ok"], "volume": vol, "coverage": cov,
            "volume_extrapolated": vext, "equivalent_diameter": diam, "boundary_edges": res["boundary_edges"],
            "nonmanifold_edges": res["nonmanifold_edges"], "closed": closed,
            "face_group": labels, "num_groups": G, "unassigned_faces": int(res["unassigned_faces"][0]),
            "unassigned_area": float(res["unassigned_area"][0])}


# ---- frames -----------------------------------------------------------------------------------------------------------
def load_transform(path) -> Dict:
    """A run's ``dataparser_transforms.json``: {'transform': [3,4] (R | t), 'scale'}.  A capture point p lies at
    scale * (R p + t) in the dataparser frame."""
    with open(path) as fh:
        tj = json.load(fh)
    scale = float(tj["scale"])
    m = np.asarray(tj["transform"], np.float64).reshape(3, 4)
    if not (np.isfinite(scale) and scale > 0 and np.isfinite(m).all()):
        raise ValueError(f"{path}: the transform must be finite and its scale > 0")
    return {"transform": m, "scale": scale}


def count_to_mesh_scale(transform: Dict) -> float:
    """Factor from ``count``'s frame to the mesh (dataparser) frame.  ``count`` runs on the semantic point cloud, which
    ``sample_volume`` writes at 2 / scale times the dataparser frame."""
    return transform["scale"] / 2.0


LENGTHS = ("radius", "rms", "equivalent_diameter")
VOLUMES = ("volume", "volume_extrapolated")


def to_capture_frame(res: Dict, transform: Dict) -> Dict:
    """``measure_fruits`` output from the dataparser frame to the capture's: positions mapped back through the transform,
    lengths divided by scale, areas by scale^2 and volumes by scale^3 (rotation and translation keep sizes)."""
    s, m = transform["scale"], transform["transform"]
    out = dict(res)
    for k in ("centroid", "center"):
        p = np.asarray(res[k], np.float64).reshape(-1, 3)
        out[k] = np.linalg.solve(m[:, :3], (p / s - m[:, 3]).T).T
    for k in LENGTHS:
        out[k] = res[k] / s
    out["area"] = res["area"] / s ** 2
    out["unassigned_area"] = res["unassigned_area"] / s ** 2
    for k in VOLUMES:
        out[k] = res[k] / s ** 3
    return out
