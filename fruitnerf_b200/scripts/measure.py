"""Measure each fruit of a fruit mesh (``fruit_mesh.ply`` of ``ns-export-semantics tsdf`` or ``fruit_poisson_mesh.ply`` of
``poisson``): per group of faces its area, centroid, fitted sphere, volume, solid-angle coverage and edge counts
(measure.measure_fruits; DESIGN section 4.3n).  The groups are the mesh's connected components, or with
``--count-json`` the faces nearest each of ``count``'s centres, so that row k belongs to centre k of that file.

    python -m fruitnerf_b200.scripts.measure --mesh OUT/fruit_mesh.ply --json OUT/measure.json
    python -m fruitnerf_b200.scripts.measure --mesh OUT/fruit_mesh.ply --count-json OUT/count.json \\
        --transform-json RUN/dataparser_transforms.json --csv OUT/measure.csv

The meshes are in the dataparser frame.  ``count``'s centres are in the frame of the semantic point cloud, 2 / scale times
the dataparser frame, so ``--count-json`` needs the run's ``--transform-json``.  With ``--transform-json`` positions are
mapped back to the capture frame and sizes are in the capture's units.
"""
from __future__ import annotations

import argparse
import csv
import json
import math
import os

import numpy as np
import torch

from .. import measure as ME
from ..export.exporter_utils import read_mesh_ply

COLUMNS = ("id", "faces", "area", "centroid_x", "centroid_y", "centroid_z", "center_x", "center_y", "center_z", "radius", "rms", "fit_ok",
           "volume", "coverage", "volume_extrapolated", "equivalent_diameter", "boundary_edges", "nonmanifold_edges", "closed")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--mesh", required=True, help="binary little-endian PLY triangle mesh (the exporter's fruit_mesh.ply)")
    ap.add_argument("--count-json", default=None, help="count's JSON: one group per entry of its 'centers' (centre mode)")
    ap.add_argument("--transform-json", default=None, help="the run's dataparser_transforms.json: report in the capture frame and units")
    ap.add_argument("--max-distance", type=float, default=None, help="centre mode: faces farther than this from every centre stay "
                    "unassigned, in count-frame units (default: no limit)")
    ap.add_argument("--device", default="cuda:0", help="CUDA device to measure on (cuda or cuda:N), or cpu for the numpy restatement")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    ap.add_argument("--csv", default=None, help="also write one row per group to this CSV file")
    a = ap.parse_args(argv)
    for name in ("mesh", "count_json", "transform_json"):
        path = getattr(a, name)
        if path is not None and not os.path.isfile(path):
            ap.error(f"--{name.replace('_', '-')} {path}: no such file")
    if a.count_json is not None and a.transform_json is None:
        ap.error("--count-json needs --transform-json: count's centres are in the point cloud's frame, 2 / scale times the mesh's")
    if a.max_distance is not None and a.count_json is None:
        ap.error("--max-distance applies to centre mode: give --count-json")
    if a.max_distance is not None and not a.max_distance > 0:
        ap.error(f"--max-distance must be > 0, got {a.max_distance}")
    return ap, a


def rows(res) -> list:
    out = []
    for k in range(res["num_groups"]):
        c, p = res["centroid"][k], res["center"][k]
        vals = (k, res["faces"][k], res["area"][k], *c, *p, res["radius"][k], res["rms"][k], res["fit_ok"][k], res["volume"][k],
                res["coverage"][k], res["volume_extrapolated"][k], res["equivalent_diameter"][k], res["boundary_edges"][k],
                res["nonmanifold_edges"][k], res["closed"][k])
        out.append({name: _plain(v) for name, v in zip(COLUMNS, vals)})
    return out


def _plain(v):
    """A JSON value: Python int / bool / float, NaN as None."""
    if isinstance(v, (bool, np.bool_)):
        return bool(v)
    if isinstance(v, (int, np.integer)):
        return int(v)
    v = float(v)
    return None if math.isnan(v) else v


def measure_mesh(ap, a) -> dict:
    dev = torch.device(a.device)
    if dev.type == "cuda" and not torch.cuda.is_available():
        ap.error(f"--device {a.device}: no CUDA device is available (use --device cpu for the numpy restatement)")
    vertices, _, _, faces = read_mesh_ply(a.mesh)
    if len(faces) == 0:
        ap.error(f"--mesh {a.mesh}: the mesh has no faces")
    transform = ME.load_transform(a.transform_json) if a.transform_json else None
    centers, md = None, None
    if a.count_json:
        with open(a.count_json) as fh:
            centers = np.asarray(json.load(fh)["centers"], np.float64).reshape(-1, 3) * ME.count_to_mesh_scale(transform)
        md = None if a.max_distance is None else a.max_distance * ME.count_to_mesh_scale(transform)
    if dev.type == "cuda":
        res = ME.measure_fruits(torch.from_numpy(vertices).to(dev), torch.from_numpy(faces).to(dev),
                                None if centers is None else torch.from_numpy(centers).to(dev), md)
    else:
        res = ME.measure_fruits(vertices, faces, centers, md)
    if transform is not None:
        res = ME.to_capture_frame(res, transform)
    units = "capture (dataparser / scale)" if transform is not None else "dataparser"
    return {"mesh": str(a.mesh), "mode": "centers" if centers is not None else "components", "frame": units,
            "scale": None if transform is None else transform["scale"], "num_groups": int(res["num_groups"]),
            "unassigned_faces": int(res["unassigned_faces"]), "unassigned_area": _plain(res["unassigned_area"]), "groups": rows(res)}


def main(argv=None) -> dict:
    ap, a = parse_args(argv)
    out = measure_mesh(ap, a)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)
    if a.csv:
        os.makedirs(os.path.dirname(a.csv) or ".", exist_ok=True)
        with open(a.csv, "w", newline="") as fh:
            w = csv.DictWriter(fh, fieldnames=COLUMNS)
            w.writeheader()
            w.writerows(out["groups"])
    return out


if __name__ == "__main__":
    main()
