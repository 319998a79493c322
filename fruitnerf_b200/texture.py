"""NeRF textures of the exported meshes (nerfstudio 0.3.2 texture_utils.export_textured_mesh with
``unwrap_method="custom"``; DESIGN section 4.3p), and the project's own ``charts`` unwrap (DESIGN section 4.3r, restated
further down).

Every face gets its own small triangle in a grid atlas, and every texel is coloured by one short ray through the model,
cast from just outside the surface along the inverted normal.  This module owns the atlas layout (the kernel
``fnr_texel_rays`` computes the same texel -> face map in closed form), restates both kernels in numpy (the tests'
reference) and writes the textured OBJ / MTL pair.

The layout, for F faces at p = ``px_per_uv_triangle`` texels per triangle:
* blocks of p rows by p + 3 columns, two faces per block (faces 2k and 2k + 1 in block k), blocks row-major with ``bx``
  per row, the smallest b >= 1 with b^2 (p + 3) >= ceil(F / 2) p, so the atlas is about square;
* texel (a, b) of a block (column, row) belongs to its first slot when a + b <= p, to its second otherwise.  In its
  slot's frame, (a, b) for the first and (p + 2 - a, p - 1 - b) for the second, the face's UV triangle has vertices 0, 1, 2
  at the texel centres (0, 0), (p - 1, 0), (0, p - 1).  The three columns between the two triangles are the gap that
  keeps a bilinear lookup inside one triangle from reading the other's texels;
* an owned texel takes the barycentrics of the closest point of its triangle to its centre, so the gutter texels next to
  the hypotenuse carry the colour of the nearest edge point;
* slots >= F (after the last face) are owned by no face; their texels take the rays of face F - 1 and are never sampled;
* ``vt`` is OBJ's: v points up, v = 1 - (row + 0.5) / H at a texel centre.
"""
from __future__ import annotations

import math
import pathlib
from typing import Dict, Tuple

import numpy as np

MAX_SIDE = 16384  # FNR_TEXTURE_MAX_SIDE

# nerfstudio texture_utils.export_textured_mesh's material, with this mesh's material and image names
MTL_LINES = ("# Generated with nerfstudio", "newmtl {name}", "Ka 1.00000000 1.00000000 1.00000000", "Kd 1.00000000 1.00000000 1.00000000",
             "Ks 0.00000000 0.00000000 0.00000000", "Tr 1.00000000", "illum 1", "Ns 1.00000000", "map_Kd {png}")


class AtlasTooLargeError(RuntimeError):
    """The atlas of a mesh would have a side over MAX_SIDE texels, or its charts do not fit into the chosen atlas."""


def check_px_per_uv_triangle(px_per_uv_triangle: int) -> int:
    p = int(px_per_uv_triangle)
    if p < 2 or p > MAX_SIDE:
        raise ValueError(f"px_per_uv_triangle must be an integer in [2, {MAX_SIDE}], got {px_per_uv_triangle}")
    return p


def atlas_layout(num_faces: int, px_per_uv_triangle: int) -> Tuple[int, int, int]:
    """(blocks per row, width, height) of the atlas, whatever its size."""
    F, p = int(num_faces), check_px_per_uv_triangle(px_per_uv_triangle)
    if F < 1:
        raise ValueError(f"a texture atlas needs at least one face, got {F}")
    nb, bw = (F + 1) // 2, p + 3
    q = -(-nb * p // bw)  # b^2 bw >= nb p  <=>  b^2 >= ceil(nb p / bw)
    bx = math.isqrt(q - 1) + 1
    return bx, bx * bw, -(-nb // bx) * p


def atlas_size(num_faces: int, px_per_uv_triangle: int) -> Tuple[int, int]:
    """(width, height) of the atlas; AtlasTooLargeError when a side exceeds MAX_SIDE."""
    _, W, H = atlas_layout(num_faces, px_per_uv_triangle)
    if max(W, H) > MAX_SIDE:
        raise AtlasTooLargeError(f"the texture atlas of {num_faces} faces at --px-per-uv-triangle {px_per_uv_triangle} would be {W}x{H} "
                                 f"texels, more than {MAX_SIDE} a side: lower --px-per-uv-triangle or export a coarser mesh")
    return W, H


def uv_coordinates(num_faces: int, px_per_uv_triangle: int) -> np.ndarray:
    """[F,3,2] float64 (u, v) of each face's three vertices, face vertex k at UV vertex k."""
    F, p = int(num_faces), int(px_per_uv_triangle)
    bx, W, H = atlas_layout(F, p)
    f = np.arange(F, dtype=np.int64)
    k, half = f // 2, f % 2
    col0 = (k % bx) * (p + 3)
    row0 = (k // bx) * p
    lx = np.array([0, p - 1, 0], np.int64)
    ly = np.array([0, 0, p - 1], np.int64)
    col = col0[:, None] + np.where(half[:, None] == 1, p + 2 - lx[None], lx[None])
    row = row0[:, None] + np.where(half[:, None] == 1, p - 1 - ly[None], ly[None])
    return np.stack([(col + 0.5) / W, 1.0 - (row + 0.5) / H], axis=-1)


def texel_slots(num_faces: int, px_per_uv_triangle: int, texel_start: int = 0, num_texels=None):
    """Per texel of [texel_start, texel_start + n) (row-major): (slot, la, lb), the slot and the texel centre in the slot's
    frame, int64.  Slot s >= F is owned by no face."""
    p = int(px_per_uv_triangle)
    bx, W, H = atlas_layout(num_faces, p)
    n = W * H - texel_start if num_texels is None else int(num_texels)
    t = np.arange(texel_start, texel_start + n, dtype=np.int64)
    row, col = t // W, t % W
    a, b = col % (p + 3), row % p
    half = (a + b >= p + 1).astype(np.int64)
    slot = 2 * ((row // p) * bx + col // (p + 3)) + half
    return slot, np.where(half == 1, p + 2 - a, a), np.where(half == 1, p - 1 - b, b)


def texel_owners(num_faces: int, px_per_uv_triangle: int) -> np.ndarray:
    """[H,W] int64: the face owning each texel, -1 for the texels after the last face."""
    _, W, H = atlas_layout(num_faces, px_per_uv_triangle)
    slot, _, _ = texel_slots(num_faces, px_per_uv_triangle)
    return np.where(slot < num_faces, slot, -1).reshape(H, W)


def texel_barycentrics(num_faces: int, px_per_uv_triangle: int, texel_start: int = 0, num_texels=None):
    """(face [n] int64, barycentrics [n,3] fp32) of each texel as fnr_texel_rays computes them."""
    p = int(px_per_uv_triangle)
    slot, la, lb = texel_slots(num_faces, p, texel_start, num_texels)
    f32 = np.float32
    pm1 = f32(p - 1)
    xs, ys = la.astype(f32), lb.astype(f32)
    g = la + lb > p - 1
    xs[g] = np.minimum(np.maximum(xs[g] - f32(0.5), f32(0)), pm1)
    ys[g] = pm1 - xs[g]
    s, t = xs / pm1, ys / pm1
    w0 = (f32(1) - s) - t
    return np.minimum(slot, num_faces - 1), np.stack([w0, s, t], axis=1)


def restated_texel_rays(vertices, normals, faces, px_per_uv_triangle: int, width: int, height: int, raylen: float, texel_start: int = 0,
                        num_texels=None) -> Tuple[np.ndarray, np.ndarray]:
    """fnr_texel_rays in numpy fp32, bit for bit: (origins, directions) [n,3]."""
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    if atlas_layout(len(fc), px_per_uv_triangle)[1:] != (width, height):
        raise ValueError(f"{width}x{height} is not the atlas of {len(fc)} faces at {px_per_uv_triangle} px per uv triangle")
    face, w = texel_barycentrics(len(fc), px_per_uv_triangle, texel_start, num_texels)
    return _texel_rays(vertices, normals, fc, face, w, raylen)


def _texel_rays(vertices, normals, faces, face, w, raylen: float) -> Tuple[np.ndarray, np.ndarray]:
    """The ray of each (face, fp32 barycentrics w [n,3]) in fp32 (the kernels' texel_ray): origins, directions [n,3]."""
    f32 = np.float32
    v = np.asarray(vertices, f32).reshape(-1, 3)
    nv = np.asarray(normals, f32).reshape(-1, 3)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    w = np.asarray(w, f32).reshape(-1, 3)
    idx = fc[np.asarray(face, np.int64)]
    w0, w1, w2 = (w[:, k:k + 1] for k in range(3))

    def interp(a):
        return (w0 * a[idx[:, 0]] + w1 * a[idx[:, 1]]) + w2 * a[idx[:, 2]]

    def norm(a):
        return np.sqrt((a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2])

    x, n = interp(v), interp(nv)
    length = norm(n)
    bad = ~(length > f32(1e-12))
    if bad.any():
        e1 = v[idx[bad, 1]] - v[idx[bad, 0]]
        e2 = v[idx[bad, 2]] - v[idx[bad, 0]]
        c = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], axis=1)
        cl = norm(c)
        flat = ~(cl > f32(1e-12))
        c[flat] = f32([0, 0, 1])
        cl[flat] = f32(1)
        n[bad], length[bad] = c, cl
    n = n / length[:, None]
    half = f32(0.5) * f32(raylen)
    return x + half * n, -n


def restated_mean_edge(vertices, faces) -> float:
    """The mean first-edge length |v1 - v0| in fp64 (fnr_mesh_mean_edge up to the order of the sum)."""
    v = np.asarray(vertices, np.float32).reshape(-1, 3).astype(np.float64)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    d = v[fc[:, 1]] - v[fc[:, 0]]
    return float(np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).sum() / len(fc))


# ---- the `charts` unwrap (fnr_chart_unwrap; DESIGN section 4.3r) --------------------------------------------------------
# Faces are grouped into connected charts of one dominant signed normal axis, every chart is projected onto its axis plane
# at one scale s of texels per unit length (so texel density follows surface area), and the charts are packed by
# next-fit shelves into one N x N atlas.  include/fruitnerf_b200.h writes out every step; this is its numpy restatement,
# bit for bit, used on test-sized meshes.
UNWRAP_MIN_SIDE = 16  # FNR_UNWRAP_MIN_SIDE
UNWRAP_MARGIN = 3  # FNR_UNWRAP_MARGIN: texels around a chart's rectangle
UNWRAP_GUTTER = 2  # FNR_UNWRAP_GUTTER: texels around a triangle that take its closest point
UNWRAP_BISECTIONS = 40  # FNR_UNWRAP_BISECTIONS
# (texel x, texel y) axes per label +x, -x, +y, -y, +z, -z: negative area in texel space, positive in vt space
_CHART_AXES = np.array([[2, 1], [1, 2], [0, 2], [2, 0], [1, 0], [0, 1]], np.int64)
_NO_OWNER = np.uint64(0xFFFFFFFFFFFFFFFF)
_WORK_PER_PASS = 1 << 22


def check_num_pixels_per_side(num_pixels_per_side: int) -> int:
    n = int(num_pixels_per_side)
    if n < UNWRAP_MIN_SIDE or n > MAX_SIDE:
        raise ValueError(f"num_pixels_per_side must be an integer in [{UNWRAP_MIN_SIDE}, {MAX_SIDE}], got {num_pixels_per_side}")
    return n


def charts_too_many(num_charts: int, num_pixels_per_side: int) -> AtlasTooLargeError:
    return AtlasTooLargeError(f"{num_charts} charts do not fit into a {num_pixels_per_side}x{num_pixels_per_side} atlas even at 7x7 texels each: "
                              f"raise --num-pixels-per-side or decimate the mesh first with --target-num-faces")


def chart_labels(vertices, faces) -> Tuple[np.ndarray, np.ndarray]:
    """(labels [F] int32, projected corners [F,3,2] fp64): the dominant signed axis 2k + (n_k < 0) of each right-hand
    normal, ties to the lower axis, and the two kept coordinates in the label's order."""
    P = np.asarray(vertices, np.float32).reshape(-1, 3).astype(np.float64)[np.asarray(faces, np.int64).reshape(-1, 3)] + 0.0
    e1, e2 = P[:, 1] - P[:, 0], P[:, 2] - P[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], axis=1)
    a = np.abs(n)
    k = np.zeros(len(n), np.int64)
    best = a[:, 0].copy()
    for j in (1, 2):
        m = a[:, j] > best
        k[m], best[m] = j, a[m, j]
    label = 2 * k + (n[np.arange(len(n)), k] < 0)
    proj = np.take_along_axis(P, _CHART_AXES[label][:, None, :], axis=2)
    return label.astype(np.int32), proj


def _interior_edges(faces, num_vertices: int) -> Tuple[np.ndarray, np.ndarray]:
    """The two faces of every edge held by exactly two half-edges (fnr_mesh_edges.cuh's keys, stably sorted)."""
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b = fc, np.roll(fc, -1, axis=1)
    key = (np.minimum(a, b) * int(num_vertices) + np.maximum(a, b)).reshape(-1)
    order = np.argsort(key, kind="stable")
    _, first, count = np.unique(key[order], return_index=True, return_counts=True)
    i = first[count == 2]
    return order[i] // 3, order[i + 1] // 3


def chart_ids(labels, fa, fb, cut) -> Tuple[np.ndarray, int]:
    """Chart of every face: components of the interior edges whose faces share a label and are not cut, numbered in
    order of their smallest face."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    F = len(labels)
    join = (labels[fa] == labels[fb]) & ~cut[fa] & ~cut[fb]
    g = coo_matrix((np.ones(int(join.sum()), np.int8), (fa[join], fb[join])), shape=(F, F))
    C, comp = connected_components(g, directed=False)
    _, first = np.unique(comp, return_index=True)  # component c's smallest face
    rank = np.empty(C, np.int64)
    rank[np.argsort(first)] = np.arange(C)
    return rank[comp].astype(np.int32), int(C)


def chart_extents(proj, charts, num_charts: int) -> Tuple[np.ndarray, np.ndarray]:
    """(ext [C,2] = max - min, p_min [C,2]) of every chart's projected corners."""
    o = np.argsort(charts, kind="stable")
    starts = np.searchsorted(charts[o], np.arange(num_charts))
    lo = np.minimum.reduceat(proj.min(axis=1)[o], starts, axis=0)
    hi = np.maximum.reduceat(proj.max(axis=1)[o], starts, axis=0)
    return hi - lo, lo


def chart_order(ext) -> np.ndarray:
    """The packing order: (ext_y desc, ext_x desc, id asc)."""
    return np.lexsort((np.arange(len(ext)), -ext[:, 0], -ext[:, 1]))


def pack_charts(ext, order, scale: float, num_pixels_per_side: int):
    """Next-fit shelves of the charts' rectangles (floor(s ext) + 1 + 2 margin texels a side), taken in ``order``, into
    N x N: offsets [C,2] int32 (top-left texel), or None when a rectangle does not fit."""
    N, m2 = int(num_pixels_per_side), 2 * UNWRAP_MARGIN
    s = float(scale)
    ex, ey = ext[order, 0].tolist(), ext[order, 1].tolist()
    out = np.empty((len(ext), 2), np.int32)
    x = y = shelf = 0
    for c, a, b in zip(order.tolist(), ex, ey):
        w, h = math.floor(s * a) + 1 + m2, math.floor(s * b) + 1 + m2
        if w > N:
            return None
        if x + w > N:
            y, x, shelf = y + shelf, 0, 0
        if y + h > N:
            return None
        out[c] = (x, y)
        x += w
        shelf = max(shelf, h)
    return out


def chart_scale(ext, num_pixels_per_side: int):
    """(s, hi, offsets): the largest scale that packs after UNWRAP_BISECTIONS halvings of [0, N / largest extent], the
    final upper bracket (which does not pack) and the offsets at s.  AtlasTooLargeError when s = 0 does not pack."""
    N = int(num_pixels_per_side)
    order = chart_order(ext)
    if pack_charts(ext, order, 0.0, N) is None:
        raise charts_too_many(len(ext), N)
    emax = float(ext.max()) if ext.size else 0.0
    if not emax > 0.0:
        return 0.0, 0.0, pack_charts(ext, order, 0.0, N)
    lo, hi = 0.0, N / emax
    for _ in range(UNWRAP_BISECTIONS):
        mid = (lo + hi) * 0.5
        if pack_charts(ext, order, mid, N) is not None:
            lo = mid
        else:
            hi = mid
    return lo, hi, pack_charts(ext, order, lo, N)


def chart_uv(proj, charts, offsets, pmin, scale: float) -> np.ndarray:
    """[F,3,2] fp64 texel coordinates offset + margin + s (p - p_min) of every corner."""
    c = np.asarray(charts, np.int64)
    o = (offsets[c] + UNWRAP_MARGIN).astype(np.float64)[:, None, :]
    return o + float(scale) * (proj - pmin[c][:, None, :])


def chart_vt(uv, num_pixels_per_side: int) -> np.ndarray:
    """OBJ vt of texel coordinates: (x / N, 1 - y / N)."""
    uv = np.asarray(uv, np.float64)
    N = float(num_pixels_per_side)
    return np.stack([uv[..., 0] / N, 1.0 - uv[..., 1] / N], axis=-1)


def _texel_boxes(uv, N: int):
    """Per face: the first column and row and the size of its texel box grown by the gutter, clamped to the atlas."""
    mn, mx = uv.min(axis=1), uv.max(axis=1)
    lo = np.maximum(np.ceil(mn - (UNWRAP_GUTTER + 0.5)), 0).astype(np.int64)
    hi = np.minimum(np.floor(mx + (UNWRAP_GUTTER - 0.5)), N - 1).astype(np.int64)
    return lo, np.maximum(hi - lo + 1, 0)


def _work_items(uv, N: int):
    """(face, col, row) of every texel of every face's box, in face order, in passes of about _WORK_PER_PASS."""
    lo, size = _texel_boxes(uv, N)
    n = size[:, 0] * size[:, 1]
    end = np.cumsum(n)
    f0 = 0
    while f0 < len(n):
        base = end[f0] - n[f0]
        f1 = max(int(np.searchsorted(end, base + _WORK_PER_PASS, side="right")), f0 + 1)
        face = np.repeat(np.arange(f0, f1), n[f0:f1])
        q = np.arange(base, end[f1 - 1]) - np.repeat(end[f0:f1] - n[f0:f1], n[f0:f1])
        w = size[face, 0]
        yield face, lo[face, 0] + q % w, lo[face, 1] + q // w
        f0 = f1


def _edge_fn(ax, ay, bx, by, cx, cy):
    return (cx - ax) * (by - ay) - (cy - ay) * (bx - ax)


def _edge_fns(uv, face, col, row):
    t = uv[face]
    x, y = t[:, :, 0], t[:, :, 1]
    cx, cy = col + 0.5, row + 0.5
    return (x, y, cx, cy, _edge_fn(x[:, 1], y[:, 1], x[:, 2], y[:, 2], cx, cy), _edge_fn(x[:, 2], y[:, 2], x[:, 0], y[:, 0], cx, cy),
            _edge_fn(x[:, 0], y[:, 0], x[:, 1], y[:, 1], cx, cy))


def chart_closest(uv, face, col, row) -> Tuple[np.ndarray, np.ndarray]:
    """(d2 [n] fp64, barycentrics [n,3] fp32) of the closest point of face's UV triangle to each texel centre."""
    f32 = np.float32
    x, y, cx, cy, e0, e1, e2 = _edge_fns(uv, face, col, row)
    total = (e0 + e1) + e2
    inside = (e0 >= 0) & (e1 >= 0) & (e2 >= 0) & (total > 0)
    best = bt = bk = None
    for k in range(3):
        k1 = (k + 1) % 3
        dx, dy = x[:, k1] - x[:, k], y[:, k1] - y[:, k]
        l2 = dx * dx + dy * dy
        num = (cx - x[:, k]) * dx + (cy - y[:, k]) * dy
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(l2 > 0, np.minimum(np.maximum(num / np.where(l2 > 0, l2, 1.0), 0.0), 1.0), 0.0)
        qx, qy = cx - (x[:, k] + t * dx), cy - (y[:, k] + t * dy)
        d2 = qx * qx + qy * qy
        if k == 0:
            best, bt, bk = d2, t, np.zeros(len(d2), np.int64)
        else:
            m = d2 < best
            best, bt, bk = np.where(m, d2, best), np.where(m, t, bt), np.where(m, k, bk)
    w = np.zeros((len(best), 3), f32)
    wt = bt.astype(f32)
    r = np.arange(len(best))
    w[r, bk] = f32(1) - wt
    w[r, (bk + 1) % 3] = wt
    with np.errstate(divide="ignore", invalid="ignore"):
        w1, w2 = (e1 / total).astype(f32), (e2 / total).astype(f32)
    w[inside] = np.stack([np.maximum((f32(1) - w1[inside]) - w2[inside], f32(0)), w1[inside], w2[inside]], axis=1)
    w[~inside & ~(total > 0)] = f32([1, 0, 0])
    return np.where(inside, 0.0, best), w


def _conflict_faces(uv, N: int) -> np.ndarray:
    """Faces strictly inside at a texel centre that another, smaller face is strictly inside too."""
    texel, face = [], []
    for f, col, row in _work_items(uv, N):
        _, _, _, _, e0, e1, e2 = _edge_fns(uv, f, col, row)
        m = (e0 > 0) & (e1 > 0) & (e2 > 0)
        texel.append(row[m] * N + col[m])
        face.append(f[m])
    texel, face = np.concatenate(texel), np.concatenate(face)
    hit = np.bincount(texel, minlength=N * N) >= 2
    m = hit[texel]
    texel, face = texel[m], face[m]
    _, first, inv = np.unique(texel, return_index=True, return_inverse=True)  # items come in face order: the first is the smallest face
    return np.unique(face[face != face[first][inv]])


def restated_chart_unwrap(vertices, faces, num_pixels_per_side: int) -> Dict:
    """fnr_chart_unwrap in numpy, bit for bit: {'labels', 'charts' [F] int32, 'offsets' [C,2] int32, 'uv' [F,3,2] fp64
    texel coordinates, 'owner' [N*N] int32 (-1: none), 'texels', 'texel_faces' [n] int32 and 'barycentrics' [n,3] fp32
    of the owned texels in texel order, 'rounds', 'num_charts', 'scale', 'scale_fails' (the last bisection bracket above
    the scale, which does not pack)}.  AtlasTooLargeError when the charts do not fit at 7 x 7 texels each."""
    N = check_num_pixels_per_side(num_pixels_per_side)
    v = np.asarray(vertices, np.float32).reshape(-1, 3)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(fc) < 1:
        raise ValueError("the mesh has no faces")
    labels, proj = chart_labels(v, fc)
    fa, fb = _interior_edges(fc, len(v))
    cut = np.zeros(len(fc), bool)
    rounds = 0
    while True:
        charts, C = chart_ids(labels, fa, fb, cut)
        ext, pmin = chart_extents(proj, charts, C)
        s, hi, offsets = chart_scale(ext, N)
        uv = chart_uv(proj, charts, offsets, pmin, s)
        split = _conflict_faces(uv, N)
        split = split[~cut[split]]
        if len(split) == 0:
            break
        cut[split] = True
        rounds += 1
    keys = np.full(N * N, _NO_OWNER, np.uint64)
    for f, col, row in _work_items(uv, N):
        d2, _ = chart_closest(uv, f, col, row)
        m = d2 <= UNWRAP_GUTTER * UNWRAP_GUTTER
        key = (d2[m].astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | f[m].astype(np.uint64)
        np.minimum.at(keys, row[m] * N + col[m], key)
    texels = np.flatnonzero(keys != _NO_OWNER)
    tf = (keys[texels] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    _, w = chart_closest(uv, tf, texels % N, texels // N)
    owner = np.full(N * N, -1, np.int32)
    owner[texels] = tf
    return {"labels": labels, "charts": charts, "offsets": offsets, "uv": uv, "owner": owner, "texels": texels.astype(np.int32),
            "texel_faces": tf.astype(np.int32), "barycentrics": w, "rounds": rounds, "num_charts": C, "scale": s, "scale_fails": hi}


def restated_chart_texel_rays(vertices, normals, faces, texel_faces, barycentrics, raylen: float) -> Tuple[np.ndarray, np.ndarray]:
    """fnr_chart_texel_rays in numpy fp32, bit for bit: (origins, directions) [n,3] of the owned texels."""
    return _texel_rays(vertices, normals, faces, texel_faces, barycentrics, raylen)


# ---- OBJ / MTL ---------------------------------------------------------------------------------------------------------
_ROWS_PER_PASS = 1 << 20
_P10 = 10 ** np.arange(18, -1, -1, dtype=np.int64)


def _chars(s: bytes, n: int):
    a = np.frombuffer(s, np.uint8)
    return np.broadcast_to(a, (n, len(a))), np.ones((n, len(a)), bool)


def _ints(x: np.ndarray):
    """Decimal digits of non-negative integers [n], right-aligned, with the mask of the significant ones."""
    x = np.asarray(x, np.int64)
    width = max(1, len(str(int(x.max())))) if x.size else 1
    digits = (x[:, None] // _P10[None, -width:]) % 10
    ndig = np.ones_like(x)
    for k in range(1, width):
        ndig += x >= 10 ** k
    keep = np.arange(width)[None, :] >= width - ndig[:, None]
    return (digits + ord("0")).astype(np.uint8), keep


def _floats(x: np.ndarray):
    """Nine significant digits in scientific notation (-d.dddddddde-XX), enough for an fp32 value to round-trip."""
    x = np.asarray(x, np.float64)
    if not np.isfinite(x).all():
        raise ValueError("an OBJ value is not finite")
    a = np.abs(x)
    e = np.where(a > 0, np.floor(np.log10(np.where(a > 0, a, 1.0))), 0).astype(np.int64)
    for _ in range(2):  # log10 may be one off next to a power of ten
        m = np.rint(a * 10.0 ** (8 - e))
        e = e + (m >= 1e9) - ((m < 1e8) & (a > 0))
    m = np.rint(a * 10.0 ** (8 - e)).astype(np.int64)
    if np.abs(e).max(initial=0) > 99:
        raise ValueError("an OBJ value's exponent has more than two digits")
    n = len(x)
    out = np.empty((n, 15), np.uint8)
    out[:, 0] = ord("-")
    out[:, 1] = m // 10 ** 8 + ord("0")
    out[:, 2] = ord(".")
    out[:, 3:11] = (m[:, None] // _P10[None, -8:]) % 10 + ord("0")
    out[:, 11] = ord("e")
    out[:, 12] = np.where(e < 0, ord("-"), ord("+"))
    out[:, 13] = np.abs(e) // 10 + ord("0")
    out[:, 14] = np.abs(e) % 10 + ord("0")
    keep = np.ones((n, 15), bool)
    keep[:, 0] = np.signbit(x) & (x != 0)
    return out, keep


def _join(pieces) -> bytes:
    mat = np.concatenate([p[0] for p in pieces], axis=1)
    keep = np.concatenate([p[1] for p in pieces], axis=1)
    return mat[keep].tobytes()


def _float_lines(fh, tag: bytes, values: np.ndarray) -> None:
    values = np.asarray(values, np.float64)
    for r0 in range(0, len(values), _ROWS_PER_PASS):
        blk = values[r0:r0 + _ROWS_PER_PASS]
        n = len(blk)
        pieces = [_chars(tag, n)]
        for j in range(blk.shape[1]):
            pieces += [_chars(b" ", n), _floats(blk[:, j])]
        fh.write(_join(pieces + [_chars(b"\n", n)]))


def write_textured_obj(obj_path, mtl_name: str, png_name: str, vertices, normals, faces, uv) -> None:
    """Write ``obj_path`` (``mtllib`` / ``usemtl``, then ``v``, ``vt`` (three per face, in face order), ``vn`` and
    ``f v/vt/vn`` lines, 1-based) and the material ``mtl_name`` next to it, whose ``map_Kd`` is ``png_name``.  vertices,
    normals [V,3]; faces [F,3]; uv [F,3,2].  Floats have nine significant digits, so fp32 values round-trip."""
    obj_path = pathlib.Path(obj_path)
    v = np.asarray(vertices).reshape(-1, 3)
    nrm = np.asarray(normals).reshape(-1, 3)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    uv = np.asarray(uv, np.float64).reshape(-1, 3, 2)
    if len(nrm) != len(v) or len(uv) != len(fc):
        raise ValueError(f"{len(v)} vertices with {len(nrm)} normals, {len(fc)} faces with {len(uv)} uv triangles")
    if fc.size and (fc.min() < 0 or fc.max() >= len(v)):
        raise ValueError(f"face indices must lie in [0, {len(v)})")
    material = pathlib.Path(mtl_name).stem
    obj_path.parent.mkdir(parents=True, exist_ok=True)
    (obj_path.parent / mtl_name).write_text("\n".join(MTL_LINES).format(name=material, png=png_name) + "\n")
    with open(obj_path, "wb") as fh:
        fh.write(f"mtllib {mtl_name}\nusemtl {material}\n".encode("ascii"))
        _float_lines(fh, b"v", v)
        _float_lines(fh, b"vt", uv.reshape(-1, 2))
        _float_lines(fh, b"vn", nrm)
        for r0 in range(0, len(fc), _ROWS_PER_PASS):
            blk = fc[r0:r0 + _ROWS_PER_PASS] + 1
            n = len(blk)
            t = 3 * np.arange(r0, r0 + n, dtype=np.int64)[:, None] + np.arange(1, 4)[None]
            pieces = [_chars(b"f", n)]
            for k in range(3):
                vi = _ints(blk[:, k])
                pieces += [_chars(b" ", n), vi, _chars(b"/", n), _ints(t[:, k]), _chars(b"/", n), vi]
            fh.write(_join(pieces + [_chars(b"\n", n)]))


def read_textured_obj(path) -> Dict:
    """A triangle OBJ as ``write_textured_obj`` writes it -> {'v' [V,3], 'vt' [T,2], 'vn' [N,3] float64, 'f' [F,3,3] int64
    (v / vt / vn per corner, 1-based as in the file), 'mtllib', 'usemtl'}."""
    rows = {"v": [], "vt": [], "vn": [], "f": []}
    out = {"mtllib": None, "usemtl": None}
    with open(path) as fh:
        for line in fh:
            tok = line.split()
            if not tok or tok[0].startswith("#"):
                continue
            if tok[0] in ("mtllib", "usemtl"):
                out[tok[0]] = tok[1]
            elif tok[0] == "f":
                if len(tok) != 4:
                    raise ValueError(f"{path}: only triangles are read, got {line.strip()!r}")
                rows["f"].append([[int(c) for c in corner.split("/")] for corner in tok[1:]])
            elif tok[0] in rows:
                rows[tok[0]].append([float(c) for c in tok[1:]])
    out["v"] = np.array(rows["v"], np.float64).reshape(-1, 3)
    out["vt"] = np.array(rows["vt"], np.float64).reshape(-1, 2)
    out["vn"] = np.array(rows["vn"], np.float64).reshape(-1, 3)
    out["f"] = np.array(rows["f"], np.int64).reshape(-1, 3, 3)
    return out
