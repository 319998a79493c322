"""Uniform-volume point-cloud export (fruit_nerf/export/exporter_utils.py:47-258).

The reference loops ``model(ray_bundle)`` -> dense [B,S,*] outputs -> three boolean-mask gathers ->
``.cpu()`` per batch.  Here each batch is ONE kernel that evaluates the field and compacts the three
point sets on the device (ops.export_batch); a single device->host copy happens at the end.  PLY
files are written directly (open3d is not needed for a binary point-cloud PLY).
"""
from __future__ import annotations

import pathlib
from typing import Dict, Optional

import numpy as np
import torch

from .. import ops

SET_NAMES = ("semantic_colormap", "semantic", "density")  # exporter_utils.py:193-256


def export_slab(num_rays: int, world_size: int, rank: int):
    """Contiguous slab [lo, hi) of the export rays owned by ``rank``: the rays of the face grid are independent
    (components/ray_generators.py:52-64), so the volume shards with no data-path collective."""
    per = (num_rays + world_size - 1) // world_size
    lo = min(rank * per, num_rays)
    return lo, min(lo + per, num_rays)


def merge_export_shards(local: Dict[str, tuple], world_size: int) -> Dict[str, tuple]:
    """All ranks contribute (rows [n,7], keys [n]) per set; everyone receives the concatenation (the surviving point
    lists are small next to the volume).  Keys are global point indices, so sorting by key restores the reference order."""
    if world_size <= 1:
        return local
    import torch.distributed as dist

    gathered = [None] * world_size
    dist.all_gather_object(gathered, {k: (r.cpu().numpy(), q.cpu().numpy()) for k, (r, q) in local.items()})
    out = {}
    for name in local:
        rows = np.concatenate([g[name][0] for g in gathered], axis=0)
        keys = np.concatenate([g[name][1] for g in gathered], axis=0)
        out[name] = (torch.from_numpy(rows), torch.from_numpy(keys))
    return out


def sample_volume(pipeline, num_points: int, output_dir: Optional[pathlib.Path] = None, config=None, transform_json: dict = None,
                  capacity: Optional[int] = None, world_size: int = 1, rank: int = 0) -> Dict[str, Dict]:
    """Returns {name: {'points' [N,3] float64, 'colors' [N,3] float64, 'alpha' [N], 'path'}} for the
    three clouds.  ``num_points`` is the number of export rays (datamanager.setup_inference).  With ``world_size`` > 1
    each rank evaluates its slab of rays and the (small) selected point lists are gathered at the end."""
    model = pipeline.model
    dm = pipeline.datamanager
    dev = next(model.parameters()).device
    S = model.num_inference_samples
    lo, hi = export_slab(num_points, world_size, rank)
    total = (hi - lo) * S
    capacity = capacity or max(1, min(total, 1 << 24))
    buffers = ops.ExportBuffers(capacity=capacity, device=dev)
    gen = dm.orthographic_ray_generator
    B = gen.ray_batch_size
    with torch.no_grad():
        if world_size <= 1:
            done = 0
            while done < num_points:
                ray_bundle, _ = dm.next_sample_volume(0)
                n = ray_bundle.origins.shape[0]
                if n == 0:
                    break
                model.get_export_outputs(ray_bundle.to(dev) if hasattr(ray_bundle, "to") else ray_bundle, buffers=buffers,
                                         point_base=done * S, dense=False)
                done += n
        else:  # this rank's slab, same batch size; point keys stay global
            for start in range(lo, hi, B):
                full = gen(count=start // B + 1) if start % B == 0 and start + B <= hi else None
                if full is None:
                    from ..compat import RayBundle

                    pts = gen.surface_points[start:min(start + B, hi)]
                    n = pts.shape[0]
                    full = RayBundle(origins=pts, directions=gen.surface_normal.repeat(n, 1).to(dev), pixel_area=torch.zeros(n, 1, device=dev),
                                     nears=torch.zeros(n, 1, device=dev), fars=torch.ones(n, 1, device=dev) * gen.surface_vector_norm)
                model.get_export_outputs(full.to(dev), buffers=buffers, point_base=start * S, dense=False)
    counts = buffers.counts.cpu().tolist()  # the single D2H sync
    if max(counts) > capacity:
        raise RuntimeError(f"export capacity {capacity} too small for {max(counts)} selected points; pass capacity=")
    scale = 1.0
    if transform_json is not None:
        scale = 2.0 / float(transform_json["scale"])  # pcd.scale(1/scale) then pcd.scale(2) (exporter_utils.py:190-191)
    local = {name: (buffers.rows[k][: counts[k]], buffers.keys[k][: counts[k]]) for k, name in enumerate(SET_NAMES)}
    merged = merge_export_shards(local, world_size)
    out = {}
    for k, name in enumerate(SET_NAMES):
        rows, keys = merged[name]
        order = torch.argsort(keys)  # reference order = batch-major point order
        rows = rows[order].double().cpu().numpy()
        colors = rows[:, 3:6].copy()
        if name != "semantic_colormap" and colors.shape[0] != 0:
            full = rows[:, 3:7]
            colors = (full / full.max())[:, :3]  # exporter_utils.py:203, 228: normalise by the max over rgb+alpha
        path = None
        if output_dir is not None and config is not None and getattr(config, "load_dir", None) is not None:
            parts = pathlib.Path(config.load_dir).parts  # upstream: outputs/<experiment>/<method>/<timestamp>/nerfstudio_models
            sub = parts[-3] if len(parts) >= 3 else ""
            path = str(pathlib.Path(output_dir) / sub / f"{name}.ply")
        out[name] = {"points": rows[:, :3] * scale, "colors": colors, "alpha": rows[:, 6], "path": path}
    return out


MAX_EMPTY_BATCHES = 100  # consecutive batches without a kept ray after which generate_point_cloud gives up


def generate_point_cloud(pipeline, num_points: int = 1000000, remove_outliers: bool = True, reorient_normals: bool = True,
                         estimate_normals: bool = False, rgb_output_name: str = "rgb", depth_output_name: str = "depth",
                         normal_output_name: Optional[str] = None, use_bounding_box: bool = True,
                         bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.0), std_ratio: float = 10.0) -> Dict:
    """nerfstudio exporter_utils.generate_point_cloud (0.3.2) on the GPU.  Renders training-ray batches until at least
    ``num_points`` rays are kept (the last batch whole), back-projects each ray's median depth, keeps rays with
    accumulation > 0.5 (and, with the box, points strictly inside it), then optionally removes statistical outliers
    (20 neighbours, ``std_ratio``), estimates normals (30 neighbours) and flips them against the view direction.
    Returns {'points' [N,3], 'colors' [N,3], 'normals' [N,3] or None}, float64 numpy, in the dataparser frame.

    Unlike the reference, which loops forever when no ray survives, this raises RuntimeError after
    ``MAX_EMPTY_BATCHES`` consecutive batches that keep nothing."""
    from .. import pointcloud

    if normal_output_name is not None:
        raise ValueError(f"normal output '{normal_output_name}': FruitModel renders no normals; estimate them from the cloud")
    if use_bounding_box and not all(lo < hi for lo, hi in zip(bounding_box_min, bounding_box_max)):
        raise ValueError("Bounding box min must be smaller than max")
    model, dm = pipeline.model, pipeline.datamanager
    dev = next(model.parameters()).device
    buffers = ops.PointBuffers(max(0, num_points) + dm.config.train_num_rays_per_batch, dev)
    box = (bounding_box_min, bounding_box_max) if use_bounding_box else None
    count = empty = 0
    with torch.no_grad():
        while count < num_points:
            ray_bundle, _ = dm.next_train(0)
            outputs = model(ray_bundle)
            rgba = model.get_rgba_image(outputs, rgb_output_name)
            ops.backproject_select(ray_bundle.origins, ray_bundle.directions, outputs[depth_output_name], rgba[..., :3], rgba[..., 3],
                                   buffers, box)
            kept = int(buffers.count.item())  # the one host read per batch
            if kept > buffers.capacity:
                raise RuntimeError(f"point buffer of {buffers.capacity} rows overflowed ({kept}): the ray batch size changed")
            empty = empty + 1 if kept == count else 0
            if empty >= MAX_EMPTY_BATCHES:
                raise RuntimeError(f"no ray was kept in {MAX_EMPTY_BATCHES} consecutive batches ({count} points so far): "
                                   "check the bounding box and the trained model")
            count = kept
        points = buffers.points[:count].double()
        colors = buffers.colors[:count]
        view_dirs = buffers.view_dirs[:count]
        if remove_outliers:
            points, ind = pointcloud.remove_statistical_outliers(points, 20, std_ratio, return_index=True)
            colors, view_dirs = colors[ind], view_dirs[ind]
        normals = None
        if estimate_normals:
            normals = pointcloud.estimate_normals(points, 30, view_dirs if reorient_normals else None)
            if reorient_normals:
                normals = normals.float().double()  # the reference reorients fp32 normals and stores them back
    return {"points": points.cpu().numpy(), "colors": colors.double().cpu().numpy(),
            "normals": None if normals is None else normals.cpu().numpy()}


def write_ply(path,points: np.ndarray, colors: np.ndarray, normals: Optional[np.ndarray] = None) -> None:
    """Binary little-endian PLY with double xyz, double nx/ny/nz when ``normals`` is given, and uchar rgb -- what
    open3d's write_point_cloud produces for a coloured cloud (fruit_nerf/scripts/exporter.py:116-119)."""
    pts = np.asarray(points, dtype="<f8")
    col = np.clip(np.asarray(colors, dtype=np.float64) * 255.0, 0, 255).astype(np.uint8)
    n = pts.shape[0]
    normal_props = "property double nx\nproperty double ny\nproperty double nz\n" if normals is not None else ""
    header = (
        "ply\nformat binary_little_endian 1.0\ncomment fruitnerf_b200 export\n"
        f"element vertex {n}\nproperty double x\nproperty double y\nproperty double z\n{normal_props}"
        "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n"
    )
    fields = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    if normals is not None:
        fields += [("nx", "<f8"), ("ny", "<f8"), ("nz", "<f8")]
    rec = np.empty(n, dtype=fields + [("r", "u1"), ("g", "u1"), ("b", "u1")])
    rec["x"], rec["y"], rec["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    if normals is not None:
        nrm = np.asarray(normals, dtype="<f8")
        rec["nx"], rec["ny"], rec["nz"] = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    rec["r"], rec["g"], rec["b"] = col[:, 0], col[:, 1], col[:, 2]
    pathlib.Path(path).parent.mkdir(parents=True, exist_ok=True)
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rec.tobytes())


_PLY_TYPES = {
    "char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2",
    "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4", "float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8",
}


def read_ply(path):
    """Binary little-endian PLY point cloud -> (points [N,3] float64, colors [N,3] float64 in [0,1] or None).

    Reads what ``write_ply`` and open3d's write_point_cloud produce: float or double x/y/z, optional uchar
    red/green/blue; any other vertex property is skipped by its declared type.  Elements other than ``vertex`` must have
    no rows (a point cloud has no faces)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, elements = None, []
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: PLY header has no end_header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "end_header":
                break
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == "property":
                if not elements:
                    raise ValueError(f"{path}: property before any element")
                if tok[1] == "list":
                    raise ValueError(f"{path}: list property '{tok[-1]}' is not supported in a point cloud")
                if tok[1] not in _PLY_TYPES:
                    raise ValueError(f"{path}: unknown PLY type '{tok[1]}'")
                elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: only binary_little_endian PLY is supported, got {fmt}")
        vertex = None
        for name, count, props in elements:
            if name == "vertex":
                vertex = np.frombuffer(f.read(count * np.dtype(props).itemsize), dtype=np.dtype(props), count=count)
            elif count:
                raise ValueError(f"{path}: element '{name}' with {count} rows is not a point cloud")
    if vertex is None or not {"x", "y", "z"} <= set(vertex.dtype.names):
        raise ValueError(f"{path}: no vertex x/y/z")
    points = np.stack([vertex["x"], vertex["y"], vertex["z"]], axis=1).astype(np.float64)
    colors = None
    if {"red", "green", "blue"} <= set(vertex.dtype.names):
        colors = np.stack([vertex["red"], vertex["green"], vertex["blue"]], axis=1).astype(np.float64) / 255.0
    return points, colors
