"""Count the hash-table gradient reds of fruit_nerf's level-major scatter kernel (`level_scatter_kernel`) on the CPU, per
level, for the bench.py batch or any other: what the device should issue, to judge its measured time against.

    python tools/scatter_reds.py [--variant small|big] [--rays 4096] [--samples 192] [--salt 0] [--aabb] [--json FILE]

A warp of the kernel holds 32 consecutive points of the flat [rays x samples] batch at one level.  Columns:
  reds_now          one float2 red per corner of nonzero weight (the per-point scatter, `level_scatter`)
  merged            one red per run of equal rows in adjacent lanes, per corner (`warp_level_scatter` without pairing)
  merged_paired     the same, with an x-neighbour pair of runs that end at the same lane on rows r, r ^ 1 as one float4 red
  distinct_per_warp distinct rows a warp touches: the least number of float2 reds any per-warp merge could issue
Every encoding gradient is taken as nonzero.  Rows and weights are the oracle's (`oracle.ns_torch.hash_corner_indices`).
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import fruit_ref as fr  # noqa: E402
from oracle import ns_torch as ns  # noqa: E402

NULL = -1
X_PAIRS = ((0, 3), (1, 2), (4, 7), (5, 6))  # corners that differ in x only, ceil x first (oracle corner order)
CORNER_SEL = (7, 5, 4, 6, 3, 1, 0, 2)  # x | y << 1 | z << 2, 1 = ceil


def level_keys(pos: torch.Tensor, scale: torch.Tensor, level: int, log2T: int) -> np.ndarray:
    """[N, 8] table rows of one level, NULL where the corner's trilinear weight is zero (the kernel adds nothing there)."""
    idx, off = ns.hash_corner_indices(pos, scale.reshape(1), log2T)
    rows = idx[:, 0, :].numpy() + (level << log2T)
    o = off[:, 0, :]
    w = torch.ones(pos.shape[0], 8)
    for k, s in enumerate(CORNER_SEL):
        wx = o[:, 0] if s & 1 else 1.0 - o[:, 0]
        wy = o[:, 1] if s & 2 else 1.0 - o[:, 1]
        wz = o[:, 2] if s & 4 else 1.0 - o[:, 2]
        w[:, k] = wx * wy * wz
    return np.where(w.numpy() != 0.0, rows, NULL)


def count_reds(keys: np.ndarray) -> dict:
    """Red counts of one level from its [N, 8] keys, N in warp order (NULL = nothing to add)."""
    n = keys.shape[0]
    pad = (-n) % 32
    k = np.concatenate([keys, np.full((pad, 8), NULL, keys.dtype)]).reshape(-1, 32, 8)
    nxt = np.concatenate([k[:, 1:], np.full((k.shape[0], 1, 8), NULL - 1, k.dtype)], axis=1)  # lane 31 ends every run
    tail = (k != nxt) & (k != NULL)
    paired = sum(int((tail[..., a] & tail[..., b] & ((k[..., a] ^ k[..., b]) == 1)).sum()) for a, b in X_PAIRS)
    flat = np.sort(k.reshape(k.shape[0], -1), axis=1)
    distinct = (flat != NULL) & np.concatenate([np.ones((flat.shape[0], 1), bool), flat[:, 1:] != flat[:, :-1]], axis=1)
    merged = int(tail.sum())
    return {"reds_now": int((k != NULL).sum()), "merged": merged, "merged_paired": merged - paired,
            "distinct_per_warp": int(distinct.sum())}


def batch_counts(origins, directions, starts, ends, scalings, log2T: int, contraction: bool = True) -> list:
    """Per-level counts for a ray batch (origins/directions [R,3], starts/ends [R,S]) in the kernel's point order."""
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    pos, _ = fr.sample_positions(origins[:, None, :], directions[:, None, :], starts[..., None], ends[..., None], aabb, contraction)
    pos = pos.reshape(-1, 3)
    return [count_reds(level_keys(pos, scalings[l], l, log2T)) for l in range(scalings.numel())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="small", choices=["small", "big"])
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--samples", type=int, default=192)
    ap.add_argument("--salt", type=int, default=0)
    ap.add_argument("--aabb", action="store_true", help="AABB positions instead of the scene contraction")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    from fruitnerf_b200 import synthetic as syn

    max_res, log2T = (2048, 19) if args.variant == "small" else (4096, 21)  # bench.build_field
    scalings = ns.hash_scalings(16, 16, max_res)
    o, d, s, e, _ = syn.ray_batch(args.rays, args.samples, salt=args.salt)
    per_level = batch_counts(o, d, s, e, scalings, log2T, contraction=not args.aabb)
    cols = ("reds_now", "merged", "merged_paired", "distinct_per_warp")
    print(f"{'level':>5} {'scale':>6} " + " ".join(f"{c:>17}" for c in cols))
    for l, c in enumerate(per_level):
        print(f"{l:>5} {int(scalings[l]):>6} " + " ".join(f"{c[k] / 1e6:>16.2f}M" for k in cols))
    total = {k: sum(c[k] for c in per_level) for k in cols}
    print(f"{'all':>12} " + " ".join(f"{total[k] / 1e6:>16.2f}M" for k in cols))
    if args.json:
        Path(args.json).write_text(json.dumps({"args": vars(args), "per_level": per_level, "total": total}) + "\n")


if __name__ == "__main__":
    main()
