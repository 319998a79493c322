"""tools/scatter_reds.py: the vectorised red counts of the scatter kernel's warp merge against a lane-by-lane count."""
import sys
from pathlib import Path

import numpy as np
import torch

from fruitnerf_b200 import synthetic as syn
from oracle import fruit_ref as fr
from oracle import ns_torch as ns

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import scatter_reds as sr  # noqa: E402


def _brute_force(keys):
    """Walk each warp lane by lane: a run ends where the next lane's row differs (or at lane 31); an x-neighbour pair of
    run ends at one lane on rows r, r ^ 1 is one red."""
    now = merged = paired = distinct = 0
    for c0 in range(0, keys.shape[0], 32):
        warp = [list(keys[i]) if i < keys.shape[0] else [sr.NULL] * 8 for i in range(c0, c0 + 32)]
        distinct += len({r for lane in warp for r in lane if r != sr.NULL})
        for lane in range(32):
            ends = []
            for k in range(8):
                r = warp[lane][k]
                if r == sr.NULL:
                    ends.append(False)
                    continue
                now += 1
                ends.append(lane == 31 or warp[lane + 1][k] != r)
            merged += sum(ends)
            paired += sum(1 for a, b in sr.X_PAIRS if ends[a] and ends[b] and warp[lane][a] ^ warp[lane][b] == 1)
    return {"reds_now": now, "merged": merged, "merged_paired": merged - paired, "distinct_per_warp": distinct}


def test_counts_match_a_lane_by_lane_count():
    """5 x 45 points (a ragged last warp), levels 0, 7 and 15 of a 2^5-row table (collisions) and of the bench table."""
    o, d, s, e, _ = syn.ray_batch(5, 45, salt=3)
    scalings = ns.hash_scalings(16, 16, 2048)
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    pos, _ = fr.sample_positions(o[:, None, :], d[:, None, :], s[..., None], e[..., None], aabb, True)
    for log2T in (5, 19):
        per_level = sr.batch_counts(o, d, s, e, scalings, log2T)
        for l in (0, 7, 15):
            keys = sr.level_keys(pos.reshape(-1, 3), scalings[l], l, log2T)
            assert per_level[l] == _brute_force(keys), (log2T, l)
    assert per_level[0]["merged_paired"] < per_level[0]["merged"] < per_level[0]["reds_now"]


def test_zero_weight_corners_and_odd_x_do_not_pair():
    # one warp: lanes 0-9 share a cell with even floor x (pairs), lanes 10-19 one with odd floor x (no pairs), lanes 20-31
    # hold a point on the x face of a cell (ceil-x corners weigh 0 and are NULL)
    keys = np.full((32, 8), sr.NULL, np.int64)
    keys[:10] = [1, 3, 5, 7, 9, 11, 13, 15]
    keys[:10, [3, 2, 7, 6]] = keys[:10, [0, 1, 4, 5]] ^ 1
    keys[10:20] = [20, 30, 40, 50, 60, 70, 80, 90]
    keys[10:20, [3, 2, 7, 6]] = [23, 33, 43, 53]
    keys[20:, [3, 2, 7, 6]] = [100, 101, 102, 103]
    want = {"reds_now": 10 * 8 + 10 * 8 + 12 * 4, "merged": 8 + 8 + 4, "merged_paired": 4 + 8 + 4, "distinct_per_warp": 20}
    assert sr.count_reds(keys) == want == _brute_force(keys)
