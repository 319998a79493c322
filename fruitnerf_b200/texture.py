"""NeRF textures of the exported meshes (nerfstudio 0.3.2 texture_utils.export_textured_mesh with
``unwrap_method="custom"``; DESIGN section 4.3p).

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
    """The atlas of a mesh would have a side over MAX_SIDE texels."""


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
    f32 = np.float32
    v = np.asarray(vertices, f32).reshape(-1, 3)
    nv = np.asarray(normals, f32).reshape(-1, 3)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    if atlas_layout(len(fc), px_per_uv_triangle)[1:] != (width, height):
        raise ValueError(f"{width}x{height} is not the atlas of {len(fc)} faces at {px_per_uv_triangle} px per uv triangle")
    face, w = texel_barycentrics(len(fc), px_per_uv_triangle, texel_start, num_texels)
    idx = fc[face]
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
