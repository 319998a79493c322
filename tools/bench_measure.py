"""Time of the per-fruit measurement's three phases (fnr_measure.cu): grouping by connected components, assignment to
centres, and measurement of the groups, each timed on its own.  Inputs: the fruit mesh of the synthetic apple scene fused
at 512^3 (40 views traced at 512x512, as tools/bench_tsdf.py fuses them) with the scene's fruit centres, and a lattice of
1300 spheres marched on the device (about 18 M faces) with its lattice centres.

    python tools/bench_measure.py --json out/bench_measure.json

Each phase runs once as warm-up and then --repeats times between CUDA events; the median is reported.  Every phase
includes its host reads (the index check, the group count, the centres' finiteness).  Next to each time is the DRAM floor
of its compulsory bytes at 3.35 TB/s (the H100 SXM data sheet): components read the faces and write the labels;
assignment reads the faces, the vertices and the centres and writes the labels; measurement reads the faces, vertices
and labels and writes the per-group outputs.  The sorts, the union-find and the three passes over each group's faces
move more than that, so the ratio is what the implementation spends over the least any implementation must.  The
assignment is a brute-force search, so its floor is also bounded by 8 fp64 operations per face and centre at 34 TFLOP/s
(the data sheet's fp64 rate without tensor cores); the larger of the two bounds is used.  The card's
name and power limit are written next to the numbers.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_tsdf import card, frames, fuse  # noqa: E402

from fruitnerf_b200 import mesh as M  # noqa: E402
from fruitnerf_b200 import ops  # noqa: E402
from fruitnerf_b200.data.synthetic_scene import make_geometry  # noqa: E402
from fruitnerf_b200.synthetic import sphere_lattice  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP64_FLOP_PER_S = 34e12
GROUP_OUT_BYTES = 8 * 3 + 8 * (1 + 3 + 5 + 2) + 4  # int64 counts, fp64 area / centroid / sphere / volume / coverage, fit_ok


def timed(fn, repeats: int):
    fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        ev[0].record()
        out = fn()
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return statistics.median(ms), out


def run(name: str, v: torch.Tensor, f: torch.Tensor, centres: torch.Tensor, repeats: int) -> dict:
    V, F, K = int(v.shape[0]), int(f.shape[0]), int(centres.shape[0])
    comp_ms, (labels, G) = timed(lambda: ops.mesh_components(f, V), repeats)
    asg_ms, alab = timed(lambda: ops.mesh_assign_centers(v, f, centres), repeats)
    meas_ms, _ = timed(lambda: ops.mesh_measure_groups(v, f, labels, G), repeats)
    meas_c_ms, _ = timed(lambda: ops.mesh_measure_groups(v, f, alab, K), repeats)
    floor = lambda b: 1e3 * b / HBM_BYTES_PER_S  # noqa: E731
    b_comp = 24 * F + 4 * F
    b_asg = 24 * F + 24 * V + 24 * K + 4 * F
    b_meas = lambda g: 24 * F + 24 * V + 4 * F + GROUP_OUT_BYTES * g  # noqa: E731
    res = {"mesh": name, "vertices": V, "faces": F, "components": G, "centres": K,
           "components_ms": comp_ms, "components_floor_ms": floor(b_comp),
           "assign_ms": asg_ms, "assign_floor_ms": max(floor(b_asg), 1e3 * 8 * F * K / FP64_FLOP_PER_S),
           "measure_components_ms": meas_ms, "measure_components_floor_ms": floor(b_meas(G)),
           "measure_centres_ms": meas_c_ms, "measure_centres_floor_ms": floor(b_meas(K))}
    for k in ("components", "assign", "measure_components", "measure_centres"):
        res[k + "_over_floor"] = res[k + "_ms"] / res[k + "_floor_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=512)
    ap.add_argument("--views", type=int, default=40)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--json", type=Path, default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "runs": []}
    fr = frames(a.views, a.size, dev)
    tsdf = M.TSDF.from_aabb([[-1, -1, -1], [1, 1, 1]], a.grid, device=dev)
    fuse(tsdf, fr, 10)
    del fr
    m = {k: (None if t is None else t.cpu().numpy()) for k, t in tsdf.get_mesh().items()}
    del tsdf
    torch.cuda.empty_cache()
    fv, _, _, _, ff = M.fruit_submesh(m["vertices"], m["normals"], m["colors"], m["fruit"], m["faces"])
    centres = make_geometry(12, 0).fruit_centers.double().to(dev)
    out["runs"].append(run(f"apple scene fruit mesh, TSDF {a.grid}^3", torch.from_numpy(fv).double().to(dev), torch.from_numpy(ff).to(dev),
                           centres, a.repeats))
    print(json.dumps(out["runs"][-1]), flush=True)
    v, f, cen, _ = sphere_lattice(dev)
    out["runs"].append(run("lattice of 1300 spheres", v, f, cen.to(dev), a.repeats))
    print(json.dumps(out["runs"][-1]), flush=True)
    if a.json:
        a.json.parent.mkdir(parents=True, exist_ok=True)
        a.json.write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
