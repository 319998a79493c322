"""Mesh decimation before NeRF texturing (``--target-num-faces`` of the ``tsdf`` / ``poisson`` exports; DESIGN section
4.3q): Garland-Heckbert quadric error metrics with parallel edge collapse in rounds.

``decimate`` runs fnr_mesh_decimate (fnr_decimate.cu) on the device; ``restated_decimate`` is the numpy restatement the
tests hold it to, bit for bit.  The method, in the order both sides compute it:

- Quadrics.  Each face gives the plane quadric of its unit normal weighted by its area; each boundary edge (an edge in
  one face) adds, to both its vertices, the plane through the edge perpendicular to its face, weighted by
  BOUNDARY_WEIGHT * |e|^2.  A vertex's quadric sums its corners in face order.  A collapse keeps Q_a + Q_b.
- Each round, on the mesh as it stands: the 3F half-edges keyed ``min * V + max`` and stably sorted; an edge is a run
  of equal keys, a boundary edge in one face and an interior edge in two.  An edge (a, b) is valid when it is in one or
  two faces, a != b, |N(a) & N(b)| equals its face count (the link condition), it is not an interior edge with both
  ends on the boundary, for an interior edge the two opposite vertices are distinct and not adjacent, and no face
  around a or b that survives the collapse has dot(n_old, n_new) <= 0 (unnormalised normals) at the new position.
- The new position minimises v^T (Q_a + Q_b) v by Gaussian elimination with partial pivoting; a pivot at or below
  PIVOT_REL times the largest diagonal entry takes the best of a, b and the midpoint instead (ties in that order).
  The cost is clamped at 0.
- Valid edges are ranked by (cost bits, edge order).  m1[v] is the least rank at v, m2[v] the least m1 over v and its
  neighbours, and an edge is selected when its rank equals m2 at both ends.  Selected edges are kept in rank order
  while the face count before them exceeds target + 1.  b goes to a, faces with a repeated index are dropped and the
  rest compacted in order.
- The loop ends at target + 1 faces or fewer, or when a round finds no valid edge.  Unused vertices are dropped in
  input order, and the vertex normals are the normalised sums of the right-hand face normals (0 where they vanish).

Every fp64 operation below is an elementwise numpy operation in the kernels' order (no dot, matmul or pairwise sum;
per-vertex sums through ``np.add.at`` in corner order), so the two sides agree bit for bit.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from . import ops

BOUNDARY_WEIGHT = 100.0  # fnr_decimate.cu kBoundaryWeight
PIVOT_REL = 1e-8         # fnr_decimate.cu kPivotRel
NO_RANK = np.iinfo(np.int32).max
NO_COST = np.uint64(0x7FF0000000000000)  # the bits of +inf: after every clamped, finite cost
# the 10 entries of a symmetric 4x4 quadric, in storage order
QUADRIC_IJ = ((0, 0), (0, 1), (0, 2), (0, 3), (1, 1), (1, 2), (1, 3), (2, 2), (2, 3), (3, 3))
_SLOT = np.array([[0, 1, 2, 3], [1, 4, 5, 6], [2, 5, 7, 8], [3, 6, 8, 9]])  # (i, j) -> storage slot


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def plane_quadric(u: np.ndarray, d: np.ndarray, w: np.ndarray) -> np.ndarray:
    """[n,10]: w * p p^T of the planes p = (u, d), entry by entry as w * (p_i * p_j)."""
    p = np.concatenate([u, d[:, None]], axis=1)
    return np.stack([w * (p[:, i] * p[:, j]) for i, j in QUADRIC_IJ], axis=1)


def _unit_plane(m: np.ndarray, point: np.ndarray, w: np.ndarray) -> np.ndarray:
    """The quadric of the plane with normal m through point, weight w; 0 where |m| = 0."""
    ln = np.sqrt(_dot(m, m))
    ok = ln > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        u = m / ln[:, None]
        q = plane_quadric(u, -_dot(u, point), w)
    return np.where(ok[:, None], q, 0.0)


def corner_quadrics(P: np.ndarray, f: np.ndarray, boundary: np.ndarray) -> np.ndarray:
    """[F,3,10]: what each corner adds to its vertex: the face's area-weighted plane, then the constraint planes of the
    boundary half-edges (``boundary`` [F,3]; half-edge k runs from corner k to corner k + 1) that leave and enter it."""
    p = P[f]
    n = _cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    qf = _unit_plane(n, p[:, 0], np.sqrt(_dot(n, n)) * 0.5)
    qb = []
    for k in range(3):
        e = p[:, (k + 1) % 3] - p[:, k]
        qb.append(_unit_plane(_cross(e, n), p[:, k], BOUNDARY_WEIGHT * _dot(e, e)))
    out = np.empty((len(f), 3, 10))
    for k in range(3):
        c = qf
        c = np.where(boundary[:, k, None], c + qb[k], c)
        k2 = (k + 2) % 3
        c = np.where(boundary[:, k2, None], c + qb[k2], c)
        out[:, k] = c
    return out


def quadric_cost(q: np.ndarray, x: np.ndarray) -> np.ndarray:
    """v^T Q v for v = (x, 1), as r_i = ((q_i0 x + q_i1 y) + q_i2 z) + q_i3 and ((x r_0 + y r_1) + z r_2) + r_3,
    clamped at 0.  q [n,10], x [n,3]."""
    r = [((q[:, _SLOT[i, 0]] * x[:, 0] + q[:, _SLOT[i, 1]] * x[:, 1]) + q[:, _SLOT[i, 2]] * x[:, 2]) + q[:, _SLOT[i, 3]] for i in range(4)]
    c = ((x[:, 0] * r[0] + x[:, 1] * r[1]) + x[:, 2] * r[2]) + r[3]
    return np.where(c > 0, c, 0.0)


def placement(q: np.ndarray, pa: np.ndarray, pb: np.ndarray):
    """(position [n,3], cost [n]) of collapsing edges with quadric q = Q_a + Q_b and ends pa, pb."""
    n = len(q)
    M = np.empty((n, 3, 4))
    for i in range(3):
        for j in range(3):
            M[:, i, j] = q[:, _SLOT[i, j]]
        M[:, i, 3] = -q[:, _SLOT[i, 3]]
    s = np.maximum(np.maximum(np.abs(M[:, 0, 0]), np.abs(M[:, 1, 1])), np.abs(M[:, 2, 2]))
    tol = PIVOT_REL * s
    singular = np.zeros(n, bool)
    rows = np.arange(n)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for k in range(3):
            p = k + np.argmax(np.abs(M[:, k:, k]), axis=1)
            singular |= ~(np.abs(M[rows, p, k]) > tol)
            rk, rp = M[rows, k].copy(), M[rows, p].copy()
            M[rows, k], M[rows, p] = rp, rk
            for i in range(k + 1, 3):
                fac = M[:, i, k] / M[:, k, k]
                for j in range(k, 4):
                    M[:, i, j] = M[:, i, j] - fac * M[:, k, j]
        u = np.empty((n, 3))
        for k in (2, 1, 0):
            acc = M[:, k, 3]
            for j in range(k + 1, 3):
                acc = acc - M[:, k, j] * u[:, j]
            u[:, k] = acc / M[:, k, k]
    solved = quadric_cost(q, np.where(singular[:, None], 0.0, u))
    mid = (pa + pb) * 0.5
    ca, cb, cm = quadric_cost(q, pa), quadric_cost(q, pb), quadric_cost(q, mid)
    best, cost = pa.copy(), ca.copy()
    tb = cb < cost
    best[tb], cost[tb] = pb[tb], cb[tb]
    tm = cm < cost
    best[tm], cost[tm] = mid[tm], cm[tm]
    return np.where(singular[:, None], best, u), np.where(singular, cost, solved)


def _ranges(starts: np.ndarray, counts: np.ndarray):
    """(owner, index): owner i repeated counts[i] times, with starts[i] + 0 .. counts[i] - 1."""
    owner = np.repeat(np.arange(len(starts)), counts)
    first = np.cumsum(counts) - counts
    return owner, starts[owner] + (np.arange(int(counts.sum())) - first[owner])


def _face_normals(P, f):
    p = P[f]
    return _cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])


def edges_of(f: np.ndarray, V: int) -> Dict[str, np.ndarray]:
    """The edge structure of faces f: half-edge h = 3 face + k runs from corner k to corner k + 1.  'key' / 'he' the
    stably sorted keys min * V + max and their half-edges; per edge (run of equal keys, in key order) its first slot
    'slot', ends 'a' < 'b' (or equal), face count 'count' and the first two half-edges 'h0', 'h1' (h1 = -1 for one)."""
    a = f.reshape(-1)
    b = f[:, [1, 2, 0]].reshape(-1)
    key = np.minimum(a, b).astype(np.uint64) * np.uint64(V) + np.maximum(a, b).astype(np.uint64)
    he = np.argsort(key, kind="stable")
    skey = key[he]
    start = np.ones(len(skey), bool)
    start[1:] = skey[1:] != skey[:-1]
    slot = np.flatnonzero(start)
    count = np.diff(np.append(slot, len(skey)))
    h1 = np.where(count >= 2, he[np.minimum(slot + 1, len(he) - 1)], -1)
    ek = skey[slot]
    return {"key": skey, "he": he, "slot": slot, "a": (ek // np.uint64(V)).astype(np.int64), "b": (ek % np.uint64(V)).astype(np.int64),
            "count": count, "h0": he[slot], "h1": h1}


def _adjacency(E: Dict, V: int):
    from scipy.sparse import coo_matrix

    m = E["a"] != E["b"]
    a, b = E["a"][m], E["b"][m]
    return coo_matrix((np.ones(2 * len(a), np.int32), (np.concatenate([a, b]), np.concatenate([b, a]))), shape=(V, V)).tocsr()


def _adjacent(A, x: np.ndarray, y: np.ndarray) -> np.ndarray:
    if len(x) == 0:
        return np.zeros(0, bool)
    return np.asarray(A[x, y]).reshape(-1) > 0


def decimation_round(P: np.ndarray, Q: np.ndarray, f: np.ndarray, target: int) -> Dict:
    """One round on the mesh (P [V,3], Q [V,10], faces f [F,3]) as it stands.  Returns the edges (``edges_of``) with
    per-edge 'valid', 'cost', 'position', 'rank' (-1 where invalid), 'selected' and 'kept', the vertices' 'm1' and
    'm2', and the mesh after the kept collapses: 'P', 'Q', 'faces'.  P and Q are not modified."""
    V, F = len(P), len(f)
    E = edges_of(f, V)
    a, b, c = E["a"], E["b"], E["count"]
    ne = len(a)
    A = _adjacency(E, V)
    onb = np.zeros(V, bool)
    onb[a[c == 1]] = True
    onb[b[c == 1]] = True
    cand = ((c == 1) | (c == 2)) & (a != b)
    idx = np.flatnonzero(cand)
    ca, cb = a[idx], b[idx]
    common = np.asarray(A[ca].multiply(A[cb]).sum(axis=1)).reshape(-1) if len(idx) else np.zeros(0, np.int64)
    ok = common == c[idx]
    inner = c[idx] == 2
    ok &= ~(inner & onb[ca] & onb[cb])
    h0, h1 = E["h0"][idx], E["h1"][idx]
    o1 = f[h0 // 3, (h0 % 3 + 2) % 3]
    o2 = np.where(inner, f[np.maximum(h1, 0) // 3, (np.maximum(h1, 0) % 3 + 2) % 3], o1)
    ok &= ~(inner & ((o1 == o2) | _adjacent(A, o1, np.where(inner, o2, o1))))
    pos, cost = placement(Q[ca] + Q[cb], P[ca], P[cb])
    # flips: every corner of a and of b whose face does not hold both
    corner = np.argsort(f.reshape(-1), kind="stable")
    vstart = np.searchsorted(f.reshape(-1)[corner], np.arange(V + 1))
    ends = np.concatenate([ca, cb])
    owner, at = _ranges(vstart[ends], vstart[ends + 1] - vstart[ends])
    e_of = np.concatenate([np.arange(len(idx)), np.arange(len(idx))])[owner]
    g = corner[at] // 3
    fg = f[g]
    ea, eb = ca[e_of], cb[e_of]
    both = ((fg == ea[:, None]).any(1)) & ((fg == eb[:, None]).any(1))
    moved = (fg == ea[:, None]) | (fg == eb[:, None])
    pold = P[fg]
    pnew = np.where(moved[:, :, None], pos[e_of][:, None, :], pold)
    n_old = _cross(pold[:, 1] - pold[:, 0], pold[:, 2] - pold[:, 0])
    n_new = _cross(pnew[:, 1] - pnew[:, 0], pnew[:, 2] - pnew[:, 0])
    flip = ~both & ~(_dot(n_old, n_new) > 0)
    ok &= np.bincount(e_of[flip], minlength=len(idx)) == 0
    valid = np.zeros(ne, bool)
    valid[idx] = ok
    ecost = np.zeros(ne)
    ecost[idx] = cost
    epos = np.zeros((ne, 3))
    epos[idx] = pos
    # ranks over every slot of the sorted half-edges, as the device sorts them
    ckey = np.full(3 * F, NO_COST, np.uint64)
    ckey[E["slot"][valid]] = ecost[valid].view(np.uint64)
    order = np.argsort(ckey, kind="stable")
    nv = int(valid.sum())
    slot_rank = np.full(3 * F, -1, np.int64)
    slot_rank[order[:nv]] = np.arange(nv)
    rank = slot_rank[E["slot"]]
    m1 = np.full(V, NO_RANK, np.int64)
    np.minimum.at(m1, a[valid], rank[valid])
    np.minimum.at(m1, b[valid], rank[valid])
    m2 = m1.copy()
    np.minimum.at(m2, a, m1[b])
    np.minimum.at(m2, b, m1[a])
    selected = valid & (rank == m2[a]) & (rank == m2[b])
    removed = np.zeros(nv, np.int64)
    removed[rank[selected]] = c[selected]
    before = np.cumsum(removed) - removed
    kept = selected.copy()
    kept[selected] = F - before[rank[selected]] > target + 1
    P2, Q2 = P.copy(), Q.copy()
    ka, kb = a[kept], b[kept]
    P2[ka] = epos[kept]
    Q2[ka] = Q[ka] + Q[kb]
    remap = np.arange(V)
    remap[kb] = ka
    g2 = remap[f]
    keep = (g2[:, 0] != g2[:, 1]) & (g2[:, 1] != g2[:, 2]) & (g2[:, 0] != g2[:, 2])
    return {**E, "valid": valid, "cost": ecost, "position": epos, "rank": rank, "selected": selected, "kept": kept, "m1": m1, "m2": m2,
            "P": P2, "Q": Q2, "faces": g2[keep]}


def _check(vertices, faces, target):
    P = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
    f = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)
    if int(target) < 1:
        raise ValueError(f"target_num_faces must be >= 1, got {target}")
    if f.size and (f.min() < 0 or f.max() >= len(P)):
        raise ValueError(f"face indices must lie in [0, {len(P)})")
    return P, f, int(target)


def initial_quadrics(P: np.ndarray, f: np.ndarray) -> np.ndarray:
    """[V,10]: each vertex's quadric, its corners summed in face order."""
    E = edges_of(f, len(P))
    boundary = np.zeros(3 * len(f), bool)
    boundary[E["h0"][E["count"] == 1]] = True
    Q = np.zeros((len(P), 10))
    np.add.at(Q, f.reshape(-1), corner_quadrics(P, f, boundary.reshape(-1, 3)).reshape(-1, 10))
    return Q


def vertex_normals(P: np.ndarray, f: np.ndarray) -> np.ndarray:
    """[V,3]: the normalised sum, in face order, of the right-hand face normals (area-weighted); 0 where it vanishes."""
    s = np.zeros((len(P), 3))
    np.add.at(s, f.reshape(-1), np.repeat(_face_normals(P, f), 3, axis=0))
    ln = np.sqrt(_dot(s, s))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where((ln > 0)[:, None], s / ln[:, None], 0.0)


def restated_decimate(vertices, faces, target_num_faces: int, max_rounds: Optional[int] = None) -> Dict:
    """The numpy restatement of fnr_mesh_decimate: {'vertices' [V',3] fp64, 'normals' [V',3] fp64, 'faces' [F',3]
    int64, 'rounds'}.  F' is target or target + 1, or more when a round found no valid edge."""
    P, f, N = _check(vertices, faces, target_num_faces)
    Q = initial_quadrics(P, f)
    rounds = 0
    while len(f) > N + 1 and (max_rounds is None or rounds < max_rounds):
        r = decimation_round(P, Q, f, N)
        if not r["valid"].any():
            break
        P, Q, f = r["P"], r["Q"], r["faces"]
        rounds += 1
    used = np.zeros(len(P), bool)
    used[f.reshape(-1)] = True
    new = np.cumsum(used) - 1
    n = vertex_normals(P, f)
    return {"vertices": P[used], "normals": n[used], "faces": new[f].reshape(-1, 3).astype(np.int64), "rounds": rounds}


def decimate(vertices, faces, target_num_faces: int) -> Dict:
    """Decimate to target_num_faces faces (or target + 1; more when no edge can collapse).  CUDA tensors run
    fnr_mesh_decimate and return CUDA tensors; anything else runs ``restated_decimate``."""
    if isinstance(vertices, torch.Tensor) and vertices.is_cuda:
        return ops.mesh_decimate(vertices, faces, int(target_num_faces))
    cvt = lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else t  # noqa: E731
    return restated_decimate(cvt(vertices), cvt(faces), target_num_faces)
