"""Surface meshes of a trained scene: TSDF fusion of rendered depth maps and marching cubes (nerfstudio 0.3.2's
``ns-export tsdf``; its ``TSDF`` class and scikit-image's ``marching_cubes`` restated, DESIGN section 4.3l).

Where each step runs depends on the input:
- a CUDA ``torch.Tensor`` runs on the GPU (fnr_mesh.cu through ``ops``): the fusion is one thread per grid point looping
  over the frames of a batch; marching cubes is a count pass, a scan of per-chunk totals and an emit pass.
- anything else runs the torch (fusion) / numpy (marching cubes) code below, which is the reference of the GPU path:
  the same fp32 operations in the same order, so the two agree bit for bit.

The triangle table is generated here (``triangle_table``) and committed as ``csrc/fnr_mesh_table.h`` for the kernels
(``python -m fruitnerf_b200.mesh`` rewrites it).  It is crack-free and orientable: every cube face resolves its ambiguous
configuration the same way (the two inside corners are separated), so neighbouring cells draw the same contour on their
shared face, and each closed contour of a cell is triangulated without a diagonal that lies in a cube face.
"""
from __future__ import annotations

from dataclasses import dataclass
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import ops

TRUNCATION_VOXELS = 5.0  # nerfstudio TSDF truncation_margin, in voxel edges of the x axis
MAX_CELL_TRIANGLES = 5  # the most any case of this table has (the classic table has up to 5 as well)
TABLE_HEADER = Path(__file__).resolve().parent / "csrc" / "fnr_mesh_table.h"


# ---- the triangle table ---------------------------------------------------------------------------------------------
def corner_offset(c: int) -> Tuple[int, int, int]:
    """Corner c = dx + 2 dy + 4 dz of a cell."""
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def cell_edges() -> List[Tuple[Tuple[int, int, int], int]]:
    """The 12 edges of a cell as (start corner offset, axis): edge 4 a + 2 hi + lo runs along axis a from the corner whose
    coordinates on the other two axes are lo (the lower axis) and hi (the higher one), 0 on axis a."""
    edges = []
    for a in range(3):
        u, v = [b for b in range(3) if b != a]
        for hi in (0, 1):
            for lo in (0, 1):
                o = [0, 0, 0]
                o[u], o[v] = lo, hi
                edges.append((tuple(o), a))
    return edges


def _edge_index(p: Tuple[int, int, int], q: Tuple[int, int, int]) -> int:
    a = [k for k in range(3) if p[k] != q[k]][0]
    s = min(p, q, key=lambda c: c[a])
    return cell_edges().index((tuple(s), a))


def _faces():
    """(outward normal, the face's 4 corners in cyclic order) for the 6 faces of the unit cell."""
    out = []
    for a in range(3):
        u, v = [b for b in range(3) if b != a]
        for s in (0, 1):
            cyc = []
            for lu, lv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                o = [0, 0, 0]
                o[a], o[u], o[v] = s, lu, lv
                cyc.append(tuple(o))
            n = [0, 0, 0]
            n[a] = 2 * s - 1
            out.append((np.array(n, float), cyc))
    return out


def _mid(e: int) -> np.ndarray:
    o, a = cell_edges()[e]
    m = np.array(o, float)
    m[a] += 0.5
    return m


def _case_segments(case: int) -> Dict[int, int]:
    """Directed contour segments of one case on the cell's faces: next[p] = q for edge vertices p -> q, oriented so that,
    seen from outside the cell, the inside corners lie on the right (which makes the triangles' right-hand normals point
    toward increasing value)."""
    inside = [(case >> c) & 1 for c in range(8)]
    idx = {corner_offset(c): c for c in range(8)}
    nxt = {}
    for n, cyc in _faces():
        flags = [inside[idx[c]] for c in cyc]
        e = [_edge_index(cyc[k], cyc[(k + 1) % 4]) for k in range(4)]  # e[k]: between cyc[k] and cyc[k+1]
        active = [k for k in range(4) if flags[k] != flags[(k + 1) % 4]]
        if not active:
            continue
        if len(active) == 2:
            pairs = [(e[active[0]], e[active[1]], next(cyc[k] for k in range(4) if flags[k]))]
        else:  # ambiguous face: the two inside corners are separated, each cut off by its own segment
            pairs = [(e[(k - 1) % 4], e[k], cyc[k]) for k in range(4) if flags[k]]
        for p, q, corner in pairs:
            pm, qm = _mid(p), _mid(q)
            if np.dot(np.cross(qm - pm, np.array(corner, float) - pm), n) > 0:
                p, q = q, p
            assert p not in nxt
            nxt[p] = q
    return nxt


def _share_face(e1: int, e2: int) -> bool:
    (o1, a1), (o2, a2) = cell_edges()[e1], cell_edges()[e2]
    for a in range(3):  # the face with normal a at side s holds edges not along a whose start has coordinate a = s
        if a != a1 and a != a2 and o1[a] == o2[a]:
            return True
    return False


def _triangulate(loop: Sequence[int]) -> List[Tuple[int, int, int]]:
    """Triangles (L[i], L[k], L[j]), i < k < j, of a closed contour: the triangulation with the fewest diagonals whose
    ends lie in one cube face (such a diagonal could be drawn by the neighbouring cell too), then the shortest diagonals."""
    n = len(loop)
    pos = [_mid(e) for e in loop]

    def cost(i, j):
        if j - i == 1 or (i == 0 and j == n - 1):
            return (0, 0.0)
        return (int(_share_face(loop[i], loop[j])), float(np.linalg.norm(pos[i] - pos[j])))

    best: Dict[Tuple[int, int], Tuple[Tuple[int, float], List]] = {}
    for span in range(1, n):
        for i in range(0, n - span):
            j = i + span
            if span == 1:
                best[(i, j)] = ((0, 0.0), [])
                continue
            cand = None
            for k in range(i + 1, j):
                (b1, l1), t1 = best[(i, k)]
                (b2, l2), t2 = best[(k, j)]
                c1, c2 = cost(i, k), cost(k, j)
                c = (b1 + b2 + c1[0] + c2[0], round(l1 + l2 + c1[1] + c2[1], 9))
                if cand is None or c < cand[0]:
                    cand = (c, t1 + t2 + [(loop[i], loop[k], loop[j])])
            best[(i, j)] = cand
    return best[(0, n - 1)][1]


def triangle_table() -> Tuple[np.ndarray, np.ndarray]:
    """(counts [256] int8, table [256, 5, 3] int8 of edge indices, -1 padded): the triangles of each case, contour by
    contour (contours in order of their smallest edge, each starting at it)."""
    counts = np.zeros(256, np.int8)
    table = np.full((256, MAX_CELL_TRIANGLES, 3), -1, np.int8)
    for case in range(256):
        nxt = _case_segments(case)
        tris, seen = [], set()
        for start in sorted(nxt):
            if start in seen:
                continue
            loop, e = [], start
            while e not in seen:
                seen.add(e)
                loop.append(e)
                e = nxt[e]
            assert e == start
            tris += _triangulate(loop)
        assert len(tris) <= MAX_CELL_TRIANGLES
        counts[case] = len(tris)
        for t, tri in enumerate(tris):
            table[case, t] = tri
    return counts, table


_TABLE = None


def _table():
    global _TABLE
    if _TABLE is None:
        _TABLE = triangle_table()
    return _TABLE


def table_header_text() -> str:
    """The C header the kernels include: the edge definitions and the triangle table of ``triangle_table``."""
    counts, table = _table()
    lines = ["// Generated by `python -m fruitnerf_b200.mesh` from mesh.triangle_table(); do not edit.",
             "// Marching-cubes cases: corner c = dx + 2 dy + 4 dz is inside iff its value is < 0; case = sum of inside bits.",
             "#pragma once", "#include <stdint.h>", "", "namespace fnr {", "",
             "// edge e: (start corner dx, dy, dz, axis)",
             "__device__ const int8_t kMcEdge[12][4] = {"]
    lines.append("    " + ", ".join("{%d, %d, %d, %d}" % (*o, a) for o, a in cell_edges()) + "};")
    lines.append(f"constexpr int kMcMaxTriangles = {MAX_CELL_TRIANGLES};")
    lines.append("__device__ const int8_t kMcTriCount[256] = {")
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(int(c)) for c in counts[r:r + 32]) + ",")
    lines.append("};")
    lines.append(f"// [case][triangle * 3 + corner]: edge indices, -1 padded")
    lines.append(f"__device__ const int8_t kMcTriTable[256][{3 * MAX_CELL_TRIANGLES}] = {{")
    for case in range(256):
        lines.append("    {" + ", ".join(str(int(x)) for x in table[case].reshape(-1)) + "},")
    lines += ["};", "", "}  // namespace fnr", ""]
    return "\n".join(lines)


# ---- marching cubes ---------------------------------------------------------------------------------------------------
def _on_device(x) -> bool:
    return isinstance(x, torch.Tensor) and x.is_cuda


def _f32_3(v) -> np.ndarray:
    v = v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)
    return np.broadcast_to(np.asarray(v, np.float32).reshape(-1), (3,)).copy()


def grid_gradient(values: np.ndarray, voxel_size) -> np.ndarray:
    """[X,Y,Z,3] fp32: central differences (v[i+1] - v[i-1]) * 0.5 inside, one-sided differences on the grid boundary,
    each divided by the voxel edge of its axis."""
    v = np.asarray(values, np.float32)
    vs = _f32_3(voxel_size)
    g = np.empty(v.shape + (3,), np.float32)
    for a in range(3):
        s = np.moveaxis(v, a, 0)
        d = np.empty_like(s)
        d[1:-1] = (s[2:] - s[:-2]) * np.float32(0.5)
        d[0] = s[1] - s[0]
        d[-1] = s[-1] - s[-2]
        g[..., a] = np.moveaxis(d, 0, a) / vs[a]
    return g


def marching_cubes_numpy(values, origin, voxel_size, colors=None, fruit=None) -> Dict[str, np.ndarray]:
    """The level-0 isosurface of ``values`` [X,Y,Z] (numpy): {'vertices' [V,3], 'normals' [V,3], 'colors' [V,3] or None,
    'fruit' [V] or None (fp32), 'faces' [F,3] int64}.  One vertex per grid edge with exactly one inside (< 0) endpoint,
    in (point linear index, axis) order; faces in cell order, then in table order.  Normals are the normalised
    interpolated gradient, or the edge direction toward its outside end where that gradient vanishes."""
    v = np.ascontiguousarray(values, np.float32)
    if v.ndim != 3 or min(v.shape) < 2:
        raise ValueError(f"values must be [X,Y,Z] with every dim >= 2, got {v.shape}")
    X, Y, Z = v.shape
    org, vs = _f32_3(origin), _f32_3(voxel_size)
    inside = v < 0
    act = np.zeros((X, Y, Z, 3), bool)
    act[:-1, :, :, 0] = inside[:-1] != inside[1:]
    act[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    act[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = act.reshape(-1)
    vid = np.cumsum(flat, dtype=np.int64) - 1
    keys = np.flatnonzero(flat)
    p, a = keys // 3, keys % 3
    ia = np.stack(np.unravel_index(p, (X, Y, Z)), axis=1)
    ib = ia.copy()
    ib[np.arange(len(p)), a] += 1
    va, vb = v[tuple(ia.T)], v[tuple(ib.T)]
    s = (np.float32(0.0) - va) / (vb - va)
    coord = ia.astype(np.float32)
    coord[np.arange(len(p)), a] = ia[np.arange(len(p)), a].astype(np.float32) + s
    verts = org + coord * vs
    g = grid_gradient(v, vs)
    ga, gb = g[tuple(ia.T)], g[tuple(ib.T)]
    n = ga + s[:, None] * (gb - ga)
    length = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    along = np.zeros_like(n)  # a vanishing gradient falls back to the edge, toward its outside end
    along[np.arange(len(p)), a] = np.where(vb > va, np.float32(1), np.float32(-1))
    with np.errstate(invalid="ignore", divide="ignore"):
        normals = np.where(length[:, None] > 0, n / length[:, None], along).astype(np.float32)
    near = tuple(np.clip(np.rint(coord).astype(np.int64), 0, np.array([X - 1, Y - 1, Z - 1])).T)  # np.round: half to even
    vcol = None if colors is None else np.asarray(colors, np.float32).reshape(X, Y, Z, 3)[near]
    vfr = None if fruit is None else np.asarray(fruit, np.float32).reshape(X, Y, Z)[near]
    # faces
    counts, table = _table()
    case = np.zeros((X - 1, Y - 1, Z - 1), np.int64)
    for c in range(8):
        dx, dy, dz = corner_offset(c)
        case |= inside[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz].astype(np.int64) << c
    case = case.reshape(-1)
    cells = np.flatnonzero(counts[case] > 0)
    ci, cj, ck = np.unravel_index(cells, (X - 1, Y - 1, Z - 1))
    evid = np.empty((len(cells), 12), np.int64)
    for e, (o, ax) in enumerate(cell_edges()):
        evid[:, e] = vid[(((ci + o[0]) * Y + (cj + o[1])) * Z + (ck + o[2])) * 3 + ax]
    tri = table[case[cells]].astype(np.int64)  # [M,12,3]
    valid = tri[:, :, 0] >= 0
    faces = np.take_along_axis(evid[:, None, :].repeat(MAX_CELL_TRIANGLES, 1), np.where(valid[..., None], tri, 0), axis=2)[valid]
    keep = (faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])  # allow_degenerate=False
    return {"vertices": verts.astype(np.float32), "normals": normals, "colors": vcol, "fruit": vfr,
            "faces": np.ascontiguousarray(faces[keep], dtype=np.int64)}


def marching_cubes(values, origin, voxel_size, colors=None, fruit=None) -> Dict:
    """Level-0 isosurface of a grid (see ``marching_cubes_numpy``).  A CUDA tensor runs fnr_marching_cubes_count/_emit and
    returns CUDA tensors; anything else returns numpy arrays from the restatement."""
    if _on_device(values):
        return ops.marching_cubes(values, origin, voxel_size, colors, fruit)
    cvt = lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else t  # noqa: E731
    return marching_cubes_numpy(cvt(values), origin, voxel_size, cvt(colors), cvt(fruit))


# ---- TSDF fusion --------------------------------------------------------------------------------------------------------
def restated_integrate(values: Tensor, weights: Tensor, colors: Tensor, fruit_state: Optional[Tensor], origin, voxel_size, truncation: float,
                       c2w: Tensor, fx: Tensor, fy: Tensor, cx: Tensor, cy: Tensor, depth: Tensor, rgb: Tensor,
                       fruit: Optional[Tensor] = None) -> None:
    """fnr_tsdf_integrate restated in torch fp32, in place: every grid point is updated by the frames in order, with each
    operation rounded where the kernel rounds it (no fused multiply-adds)."""
    X, Y, Z = values.shape
    dev = values.device
    f32 = dict(dtype=torch.float32, device=dev)
    org, vs = torch.tensor(_f32_3(origin), **f32), torch.tensor(_f32_3(voxel_size), **f32)
    trunc = torch.tensor(truncation, **f32)
    ii, jj, kk = torch.meshgrid(torch.arange(X, device=dev), torch.arange(Y, device=dev), torch.arange(Z, device=dev), indexing="ij")
    x = [org[a] + torch.stack([ii, jj, kk])[a].reshape(-1).to(torch.float32) * vs[a] for a in range(3)]
    val, w, col = values.view(-1), weights.view(-1), colors.view(-1, 3)
    fst = None if fruit_state is None else fruit_state.view(-1)
    B, H, W = depth.shape[0], depth.shape[1], depth.shape[2]
    depth = depth.reshape(B, H, W).to(**f32)
    rgb = rgb.reshape(B, H, W, 3).to(**f32)
    c2w = c2w.reshape(B, 3, 4).to(**f32)
    fx, fy, cx, cy = (torch.as_tensor(t, **f32).reshape(-1).expand(B) for t in (fx, fy, cx, cy))
    one, zero = torch.tensor(1.0, **f32), torch.tensor(0.0, **f32)
    for b in range(B):
        m = c2w[b]
        d = [x[r] - m[r, 3] for r in range(3)]
        p = [(m[0, c] * d[0] + m[1, c] * d[1]) + m[2, c] * d[2] for c in range(3)]
        zc = -p[2]
        u = cx[b] + (fx[b] * p[0]) / zc
        v = cy[b] - (fy[b] * p[1]) / zc
        ok = (zc > 0) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
        col_i = torch.where(ok, torch.floor(u), zero).to(torch.int64)
        row_i = torch.where(ok, torch.floor(v), zero).to(torch.int64)
        t = depth[b][row_i, col_i]
        a_ = ((col_i.to(torch.float32) + 0.5) - cx[b]) / fx[b]
        b_ = ((row_i.to(torch.float32) + 0.5) - cy[b]) / fy[b]
        zpix = t / torch.sqrt(((a_ * a_ + b_ * b_) + one).double()).float()  # correctly rounded, as __fsqrt_rn (torch's fp32 CPU sqrt is not)
        sdf = zpix - zc
        ok &= (t > 0) & (sdf > -trunc)
        tsdf = torch.clamp(sdf / trunc, -1.0, 1.0)
        w1 = w + one
        val.copy_(torch.where(ok, (val * w + tsdf) / w1, val))
        c = rgb[b][row_i, col_i]
        col.copy_(torch.where(ok[:, None], (col * w[:, None] + c) / w1[:, None], col))
        if fruit is not None:
            fr = fruit.reshape(B, H, W).to(**f32)[b][row_i, col_i]
            fst.copy_(torch.where(ok, (fst * w + fr) / w1, fst))
        w.copy_(torch.where(ok, w1, w))


@dataclass
class TSDF:
    """A truncated-signed-distance grid (nerfstudio TSDF): ``values`` [X,Y,Z] (initially -1), count ``weights`` (0),
    ``colors`` [X,Y,Z,3] and the fused fruit probability ``fruit`` [X,Y,Z], all fp32; grid point (i,j,k) lies at
    origin + (i,j,k) * voxel_size."""

    values: Tensor
    weights: Tensor
    colors: Tensor
    fruit: Tensor
    origin: Tensor  # [3] fp32
    voxel_size: Tensor  # [3] fp32
    truncation: float

    @staticmethod
    def from_aabb(aabb, dims, device="cpu") -> "TSDF":
        """A grid spanning ``aabb`` [2,3] with ``dims`` points per axis (an int or three): voxel_size = (max - min) / dims,
        so the max corner itself is not a grid point (nerfstudio TSDF.from_aabb)."""
        box = torch.as_tensor(aabb, dtype=torch.float32).reshape(2, 3).cpu()
        d = [int(v) for v in (dims if isinstance(dims, (list, tuple)) else [dims] * 3)]
        if len(d) != 3 or min(d) < 2:
            raise ValueError(f"TSDF dims must be one or three integers >= 2, got {dims}")
        if not bool((box[1] > box[0]).all()):
            raise ValueError(f"TSDF box min {box[0].tolist()} must be below its max {box[1].tolist()}")
        vs = (box[1] - box[0]) / torch.tensor(d, dtype=torch.float32)
        f32 = dict(dtype=torch.float32, device=device)
        return TSDF(values=-torch.ones(d, **f32), weights=torch.zeros(d, **f32), colors=torch.zeros(d + [3], **f32),
                    fruit=torch.zeros(d, **f32), origin=box[0].clone(), voxel_size=vs,
                    truncation=float(np.float32(TRUNCATION_VOXELS) * np.float32(vs[0])))

    @property
    def dims(self) -> Tuple[int, int, int]:
        return tuple(self.values.shape)

    @property
    def device(self) -> torch.device:
        return self.values.device

    def integrate(self, c2w, fx, fy, cx, cy, depth, rgb, fruit=None) -> None:
        """Fuse B frames: c2w [B,3,4] (OpenGL axes), fx / fy / cx / cy [B], depth [B,H,W] (ray distance), rgb [B,H,W,3],
        fruit [B,H,W] probabilities or None."""
        if _on_device(self.values):
            ops.tsdf_integrate(self.values, self.weights, self.colors, self.fruit if fruit is not None else None, self.origin, self.voxel_size,
                               self.truncation, c2w, fx, fy, cx, cy, depth, rgb, fruit)
            return
        restated_integrate(self.values, self.weights, self.colors, self.fruit, self.origin, self.voxel_size, self.truncation, c2w, fx, fy, cx, cy,
                           depth, rgb, fruit)

    def get_mesh(self) -> Dict:
        """marching_cubes of the grid at level 0 with the fused colours and fruit probabilities."""
        return marching_cubes(self.values, self.origin, self.voxel_size, self.colors, self.fruit)


def fruit_submesh(vertices, normals, colors, fruit, faces, threshold: float = 0.5):
    """The faces whose three vertices all have fruit probability >= ``threshold``, with their vertices compacted in
    order: (vertices, normals, colors, fruit, faces) as numpy arrays."""
    fruit = np.asarray(fruit)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    keep = (fruit[faces] >= threshold).all(axis=1) if len(faces) else np.zeros(0, bool)
    f = faces[keep]
    used = np.zeros(len(fruit), bool)
    used[f.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    pick = lambda a: None if a is None else np.asarray(a)[used]  # noqa: E731
    return pick(vertices), pick(normals), pick(colors), pick(fruit), remap[f].astype(np.int64).reshape(-1, 3)


if __name__ == "__main__":
    TABLE_HEADER.write_text(table_header_text())
    print(f"wrote {TABLE_HEADER}")
