"""Screened Poisson surface reconstruction of an oriented point cloud (nerfstudio 0.3.2's ``ns-export poisson``, which calls
open3d's ``create_from_point_cloud_poisson`` at depth 9; DESIGN section 4.3m).

The method is fixed here so that host and device can be compared:
- the cube is the points' bounding box with its largest side scaled by ``SCALE`` about the centre; it carries R = 2^d
  cells per axis (h = 1/R in cube units) and a trilinear hat phi_i per node, (R+1)^3 nodes in C order;
- the points are sorted into cells (stable: input order inside a cell); every node sum gathers over the points of the
  node's 8 adjacent cells in cell order, then input order, in fp64, and is rounded to fp32 once;
- density rho_j = sum phi_j(p); normal field v_j = (a / h^3) sum phi_j(p) n_p with a = h^2 (occupied cells) / N, the
  area per sample; colour and fruit sum phi_j(p) c_p / rho_j;
- (K + alpha a S^T S) chi = b with K the Q1 stiffness matrix of the cells inside the cube (Neumann boundaries),
  b_i = sum_j (int grad phi_i phi_j) . v_j and S [N, M] the point samples, alpha = ``POINT_WEIGHT``;
- the surface is the level of chi at the mean of chi over the points (inside below it), its vertices take colour, fruit
  and density from the nearest node, and the vertices below the 0.1 quantile of vertex density are trimmed with every
  face that touches them.

A CUDA ``torch.Tensor`` runs fnr_poisson.cu through ``ops`` (coarse-to-fine Jacobi-preconditioned CG, then the
marching-cubes kernels); anything else runs the numpy / scipy restatement below (sparse assembly from 8x8 Q1 element
matrices and ``spsolve``).  ``restated_splat`` reproduces the device's node sums and right-hand side bit for bit.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import mesh as mesh_mod
from . import ops

SCALE = 1.1  # open3d's default: the cube's side over the bounding box's largest side
POINT_WEIGHT = 2.0  # alpha, open3d's point_weight
TRIM_QUANTILE = 0.1  # nerfstudio removes the vertices below np.quantile(densities, 0.1)
MIN_DEPTH, MAX_DEPTH = 2, 10


def _np(t) -> Optional[np.ndarray]:
    if t is None:
        return None
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def check_depth(depth: int) -> int:
    d = int(depth)
    if not MIN_DEPTH <= d <= MAX_DEPTH:
        raise ValueError(f"Poisson depth must lie in [{MIN_DEPTH}, {MAX_DEPTH}], got {depth}")
    return d


def cube_of(points, scale: float = SCALE) -> Tuple[np.ndarray, float]:
    """(origin [3] fp64, side): the bounding box's largest side times ``scale``, centred on the box."""
    if torch.is_tensor(points):  # the bounds only leave the device
        p = points.detach().reshape(-1, 3)
        if p.shape[0] == 0 or not bool(torch.isfinite(p).all()):
            raise ValueError("the Poisson reconstruction needs at least one point, all finite")
        lo, hi = (b.double().cpu().numpy() for b in torch.aminmax(p, dim=0))
    else:
        p = np.asarray(points, np.float64).reshape(-1, 3)
        if len(p) == 0 or not np.isfinite(p).all():
            raise ValueError("the Poisson reconstruction needs at least one point, all finite")
        lo, hi = p.min(axis=0), p.max(axis=0)
    side = float((hi - lo).max()) * float(scale)
    if not side > 0.0:
        raise ValueError("the points span no extent: the Poisson cube would be empty")
    return (lo + hi) * 0.5 - side * 0.5, side


# ---- the restatement -------------------------------------------------------------------------------------------------
def _cells(points: np.ndarray, depth: int, origin, side: float):
    """Per point: integer cell [n,3], position inside it t [n,3] (fp64, the device's arithmetic)."""
    R = 2 ** depth
    q = (points - np.asarray(origin, np.float64)) / (side / R)
    c = np.floor(q)
    if not np.isfinite(q).all() or (c < 0).any() or (c > R - 1).any():
        raise ValueError("a point is not finite or lies outside the cube")
    return c.astype(np.int64), q - c


def _corner_phi(t: np.ndarray, b: Tuple[int, int, int]) -> np.ndarray:
    w = [t[:, a] if b[a] else 1.0 - t[:, a] for a in range(3)]
    return (w[0] * w[1]) * w[2]


def _corners():
    return [(q & 1, (q >> 1) & 1, (q >> 2) & 1) for q in range(8)]


def _factors(depth: int):
    """1D factors at node I (0..R) per neighbour offset o in (-1, 0, 1): mass, stiffness and gradient-mass."""
    R = 2 ** depth
    h = 1.0 / R
    idx = np.arange(R + 1)
    end = (idx == 0) | (idx == R)
    m, k, g = {}, {}, {}
    for o in (-1, 0, 1):
        valid = (idx + o >= 0) & (idx + o <= R)
        if o:
            m[o] = np.where(valid, h / 6.0, 0.0)
            k[o] = np.where(valid, -1.0 / h, 0.0)
            g[o] = np.where(valid, -0.5 if o > 0 else 0.5, 0.0)
        else:
            m[o] = np.where(end, h / 3.0, (2.0 * h) / 3.0)
            k[o] = np.where(end, 1.0 / h, 2.0 / h)
            g[o] = np.where(idx == 0, -0.5, np.where(idx == R, 0.5, 0.0))
    return m, k, g


def _shifted(v: np.ndarray, Nn: int, dx: int, dy: int, dz: int) -> np.ndarray:
    """v[I+dx, J+dy, K+dz] per node (0 outside the grid); v: [Nn,Nn,Nn,...]."""
    pad = np.zeros((Nn + 2, Nn + 2, Nn + 2) + v.shape[3:], v.dtype)
    pad[1:-1, 1:-1, 1:-1] = v
    return pad[1 + dx:Nn + 1 + dx, 1 + dy:Nn + 1 + dy, 1 + dz:Nn + 1 + dz]


def restated_rhs(normal_field: np.ndarray, depth: int) -> np.ndarray:
    """rhs_kernel restated: b_i = sum over the 27 neighbours (dx, dy, dz in -1..1, x outermost) and the 3 axes of
    (G1 M1 M1 / M1 G1 M1 / M1 M1 G1 coefficient) * v_j, accumulated in fp64 in that order, rounded to fp32."""
    Nn = 2 ** depth + 1
    v = np.asarray(normal_field, np.float32).reshape(Nn, Nn, Nn, 3).astype(np.float64)
    m, _, g = _factors(depth)
    acc = np.zeros((Nn, Nn, Nn))
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                vs = _shifted(v, Nn, dx, dy, dz)
                mx, my, mz = m[dx][:, None, None], m[dy][None, :, None], m[dz][None, None, :]
                gx, gy, gz = g[dx][:, None, None], g[dy][None, :, None], g[dz][None, None, :]
                acc = acc + ((gx * my) * mz) * vs[..., 0]
                acc = acc + ((mx * gy) * mz) * vs[..., 1]
                acc = acc + ((mx * my) * gz) * vs[..., 2]
    return acc.astype(np.float32).reshape(-1)


def restated_splat(points, normals, depth: int, origin, side: float, colors=None, fruit=None) -> Dict[str, np.ndarray]:
    """fnr_poisson_splat restated: {'density', 'normal_field', 'colors', 'fruit', 'rhs'} fp32 as the device writes them,
    plus 'area' (a) and 'occupied' (cells)."""
    depth = check_depth(depth)
    pts = np.asarray(_np(points), np.float64).reshape(-1, 3)
    n = len(pts)
    R, Nn = 2 ** depth, 2 ** depth + 1
    M = Nn ** 3
    c, t = _cells(pts, depth, origin, side)
    lin = (c[:, 0] * R + c[:, 1]) * R + c[:, 2]
    order = np.argsort(lin, kind="stable")  # cell order, then input order
    occupied = int(len(np.unique(lin)))
    h = 1.0 / R
    a = ((h * h) * occupied) / n
    scale = a / ((h * h) * h)
    cs, ts = c[order], t[order]
    nodes, phis = [], []
    for b in _corners():  # contributions in (sorted point, corner) order: per node, cells ascending then input order
        nodes.append(((cs[:, 0] + b[0]) * Nn + cs[:, 1] + b[1]) * Nn + cs[:, 2] + b[2])
        phis.append(_corner_phi(ts, b))
    node = np.stack(nodes, 1).reshape(-1)
    phi = np.stack(phis, 1).reshape(-1)
    src = np.repeat(order, 8)

    def gather(values: np.ndarray) -> np.ndarray:
        return np.bincount(node, weights=phi * values[src], minlength=M)

    rho = np.bincount(node, weights=phi, minlength=M)
    nrm = np.asarray(_np(normals), np.float32).reshape(n, 3).astype(np.float64)
    vfield = np.stack([(scale * gather(nrm[:, k])).astype(np.float32) for k in range(3)], 1)
    out = {"density": rho.astype(np.float32), "normal_field": vfield, "colors": None, "fruit": None, "area": a, "occupied": occupied}
    safe = np.where(rho > 0, rho, 1.0)
    if colors is not None:
        col = np.asarray(_np(colors), np.float32).reshape(n, 3).astype(np.float64)
        out["colors"] = np.stack([np.where(rho > 0, gather(col[:, k]) / safe, 0.0).astype(np.float32) for k in range(3)], 1)
    if fruit is not None:
        fr = np.asarray(_np(fruit), np.float32).reshape(n).astype(np.float64)
        out["fruit"] = np.where(rho > 0, gather(fr) / safe, 0.0).astype(np.float32)
    out["rhs"] = restated_rhs(vfield, depth)
    return out


def sample_matrix(points, depth: int, origin, side: float):
    """S [n, M] (scipy CSR): S[p, i] = phi_i(p)."""
    import scipy.sparse as sp

    pts = np.asarray(_np(points), np.float64).reshape(-1, 3)
    Nn = 2 ** depth + 1
    c, t = _cells(pts, depth, origin, side)
    rows, cols, vals = [], [], []
    for b in _corners():
        rows.append(np.arange(len(pts)))
        cols.append(((c[:, 0] + b[0]) * Nn + c[:, 1] + b[1]) * Nn + c[:, 2] + b[2])
        vals.append(_corner_phi(t, b))
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(len(pts), Nn ** 3))


def element_matrices(depth: int) -> Dict[str, np.ndarray]:
    """The 8x8 Q1 element matrices of a cell of side h = 2^-depth, corners q = bx + 2 by + 4 bz: stiffness 'K' and the
    gradient-mass 'G0', 'G1', 'G2' (int d phi_a / d axis * phi_b)."""
    h = 1.0 / 2 ** depth
    k = np.array([[1.0, -1.0], [-1.0, 1.0]]) / h
    m = np.array([[1.0 / 3.0, 1.0 / 6.0], [1.0 / 6.0, 1.0 / 3.0]]) * h
    g = np.array([[-0.5, -0.5], [0.5, 0.5]])
    out = {"K": np.zeros((8, 8)), "G0": np.zeros((8, 8)), "G1": np.zeros((8, 8)), "G2": np.zeros((8, 8))}
    for qa, a in enumerate(_corners()):
        for qb, b in enumerate(_corners()):
            mm = [m[a[x], b[x]] for x in range(3)]
            out["K"][qa, qb] = (k[a[0], b[0]] * mm[1] * mm[2] + mm[0] * k[a[1], b[1]] * mm[2] + mm[0] * mm[1] * k[a[2], b[2]])
            for x in range(3):
                f = list(mm)
                f[x] = g[a[x], b[x]]
                out[f"G{x}"][qa, qb] = f[0] * f[1] * f[2]
    return out


def assemble(depth: int):
    """{'K', 'G0', 'G1', 'G2'}: the element matrices summed over the R^3 cells inside the cube (scipy CSR, [M, M])."""
    import scipy.sparse as sp

    R, Nn = 2 ** depth, 2 ** depth + 1
    ci = np.stack(np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing="ij"), -1).reshape(-1, 3)
    node = np.stack([((ci[:, 0] + b[0]) * Nn + ci[:, 1] + b[1]) * Nn + ci[:, 2] + b[2] for b in _corners()], 1)  # [cells, 8]
    rows = np.repeat(node, 8, axis=1).reshape(-1)
    cols = np.tile(node, (1, 8)).reshape(-1)
    out = {}
    for name, e in element_matrices(depth).items():
        vals = np.tile(e.reshape(-1), len(ci))
        out[name] = sp.csr_matrix((vals, (rows, cols)), shape=(Nn ** 3, Nn ** 3))
    return out


def operator(points, depth: int, origin, side: float, area: float, alpha: float = POINT_WEIGHT):
    """A = K + alpha a S^T S (scipy CSR, fp64)."""
    S = sample_matrix(points, depth, origin, side)
    return (assemble(depth)["K"] + (alpha * area) * (S.T @ S)).tocsr()


def restated_solve(points, normals, depth: int, origin, side: float, colors=None, fruit=None, alpha: float = POINT_WEIGHT) -> Dict:
    """chi (fp64 [M]) of the screened system by ``spsolve``, with the restated splat."""
    from scipy.sparse.linalg import spsolve

    sp_ = restated_splat(points, normals, depth, origin, side, colors, fruit)
    A = operator(points, depth, origin, side, sp_["area"], alpha)
    sp_["chi"] = spsolve(A.tocsc(), sp_["rhs"].astype(np.float64))
    sp_["operator"] = A
    return sp_


def restated_sample(points, grid, depth: int, origin, side: float) -> np.ndarray:
    """grid_sample_kernel restated (fp64 accumulation in corner order, rounded to fp32)."""
    pts = np.asarray(_np(points), np.float64).reshape(-1, 3)
    R, Nn = 2 ** depth, 2 ** depth + 1
    q = (pts - np.asarray(origin, np.float64)) / (side / R)
    c = np.clip(np.floor(q), 0, R - 1)
    t = q - c
    c = c.astype(np.int64)
    g = np.asarray(grid, np.float64).reshape(-1)
    acc = np.zeros(len(pts))
    for b in _corners():
        acc = acc + _corner_phi(t, b) * g[((c[:, 0] + b[0]) * Nn + c[:, 1] + b[1]) * Nn + c[:, 2] + b[2]]
    return acc.astype(np.float32)


# ---- the mesh --------------------------------------------------------------------------------------------------------
def trim_by_density(mesh: Dict, density: np.ndarray, quantile: float = TRIM_QUANTILE) -> Dict:
    """open3d ``remove_vertices_by_mask(density < np.quantile(density, quantile))``: those vertices go, with every face
    that uses one; the rest keep their order and the faces are renumbered."""
    density = np.asarray(density)
    faces = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    if len(density) == 0:
        return dict(mesh, faces=faces)
    keep = ~(density < np.quantile(density, quantile))
    fkeep = keep[faces].all(axis=1) if len(faces) else np.zeros(0, bool)
    remap = np.cumsum(keep) - 1
    out = {k: (None if v is None else np.asarray(v)[keep]) for k, v in mesh.items() if k != "faces"}
    out["faces"] = remap[faces[fkeep]].astype(np.int64).reshape(-1, 3)
    return out


def reconstruct(points, normals, colors=None, fruit=None, depth: int = 9, alpha: float = POINT_WEIGHT, max_iters: int = 2000,
                tolerance: float = 1e-5, trim_quantile: float = TRIM_QUANTILE) -> Dict:
    """Screened Poisson mesh of an oriented cloud: {'mesh': trimmed {'vertices', 'normals', 'colors', 'fruit', 'density',
    'faces'} (numpy), 'full': the same before trimming, 'chi' [M], 'iso', 'origin', 'side', 'iterations', 'residual'}.
    CUDA tensors run on the device; anything else runs the restatement (spsolve: small depths only)."""
    depth = check_depth(depth)
    origin, side = cube_of(points)
    R = 2 ** depth
    dims = (R + 1,) * 3
    org32 = np.asarray(origin, np.float32)
    vox32 = np.float32(side / R)
    if isinstance(points, torch.Tensor) and points.is_cuda:
        s = ops.poisson_solve(points, normals, depth, origin, side, colors, fruit, alpha, max_iters, tolerance)
        iso = float(ops.poisson_sample(points, s["chi"], depth, origin, side).double().mean())
        values = (s["chi"] - iso).reshape(dims)
        node_col = None if s["colors"] is None else s["colors"].reshape(dims + (3,))
        node_fr = None if s["fruit"] is None else s["fruit"].reshape(dims)
        mc = ops.marching_cubes(values, org32, vox32, node_col, node_fr)
        dens = ops.marching_cubes(values, org32, vox32, None, s["density"].reshape(dims))["fruit"]
        chi, iters, total, res = s["chi"], s["iterations"], s["total_iterations"], s["residual"]
    else:
        s = restated_solve(points, normals, depth, origin, side, colors, fruit, alpha)
        chi32 = s["chi"].astype(np.float32)
        iso = float(restated_sample(points, chi32, depth, origin, side).astype(np.float64).mean())
        values = (chi32 - np.float32(iso)).reshape(dims)
        node_col = None if s["colors"] is None else s["colors"].reshape(dims + (3,))
        node_fr = None if s["fruit"] is None else s["fruit"].reshape(dims)
        mc = mesh_mod.marching_cubes_numpy(values, org32, vox32, node_col, node_fr)
        dens = mesh_mod.marching_cubes_numpy(values, org32, vox32, None, s["density"].reshape(dims))["fruit"]
        chi, iters, total, res = chi32, None, None, None
    full = {k: _np(mc[k]) for k in ("vertices", "normals", "colors", "fruit", "faces")}
    full["density"] = _np(dens)
    return {"mesh": trim_by_density(full, full["density"], trim_quantile), "full": full, "chi": chi, "iso": iso, "origin": origin,
            "side": side, "iterations": iters, "total_iterations": total, "residual": res}
