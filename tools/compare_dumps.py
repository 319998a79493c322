"""Compare two `bench.py --dump-outputs` directories: max deviation per array, absolute and relative to the array's scale
(max |a| of the first directory).

    python tools/compare_dumps.py OLD_DIR NEW_DIR [--tol 2e-3]

Exits non-zero if an array is missing on one side or deviates by more than --tol of its scale.
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--tol", type=float, default=2e-3)
    args = ap.parse_args()
    old, new = Path(args.old), Path(args.new)
    names = sorted({p.name for p in old.glob("*.npy")} | {p.name for p in new.glob("*.npy")})
    bad = 0
    for name in names:
        if not (old / name).exists() or not (new / name).exists():
            print(f"{name[:-4]:<48} missing in {'old' if not (old / name).exists() else 'new'}")
            bad += 1
            continue
        a, b = np.load(old / name).astype(np.float64), np.load(new / name).astype(np.float64)
        if a.shape != b.shape:
            print(f"{name[:-4]:<48} shape {a.shape} vs {b.shape}")
            bad += 1
            continue
        dev = float(np.abs(a - b).max()) if a.size else 0.0
        scale = float(np.abs(a).max()) if a.size else 0.0
        rel = dev / scale if scale > 0 else (0.0 if dev == 0 else float("inf"))
        ok = rel <= args.tol
        bad += not ok
        print(f"{name[:-4]:<48} max|d| {dev:.3e}  scale {scale:.3e}  rel {rel:.3e}  {'identical' if dev == 0 else ''}"
              f"{'' if ok else '  OVER TOLERANCE'}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
