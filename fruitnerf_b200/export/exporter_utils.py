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
                         bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.0), std_ratio: float = 10.0,
                         fruit: bool = False) -> Dict:
    """nerfstudio exporter_utils.generate_point_cloud (0.3.2) on the GPU.  Renders training-ray batches until at least
    ``num_points`` rays are kept (the last batch whole), back-projects each ray's median depth, keeps rays with
    accumulation > 0.5 (and, with the box, points strictly inside it), then optionally removes statistical outliers
    (20 neighbours, ``std_ratio``), estimates normals (30 neighbours) and flips them against the view direction.
    Returns {'points' [N,3], 'colors' [N,3], 'normals' [N,3] or None}, float64 numpy, in the dataparser frame.  With
    ``fruit``, also 'fruit' [N] fp32: each kept ray's sigmoid(semantics), in the same order (the Poisson export's per-point
    fruit probability).

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
    fbuf = ops.PointBuffers(buffers.capacity, dev) if fruit else None  # same selection, sigmoid(semantics) as its colour
    box = (bounding_box_min, bounding_box_max) if use_bounding_box else None
    count = empty = 0
    with torch.no_grad():
        while count < num_points:
            ray_bundle, _ = dm.next_train(0)
            outputs = model(ray_bundle)
            rgba = model.get_rgba_image(outputs, rgb_output_name)
            ops.backproject_select(ray_bundle.origins, ray_bundle.directions, outputs[depth_output_name], rgba[..., :3], rgba[..., 3],
                                   buffers, box)
            if fbuf is not None:
                prob = torch.sigmoid(outputs["semantics"].detach().float().reshape(-1, 1)).expand(-1, 3)
                ops.backproject_select(ray_bundle.origins, ray_bundle.directions, outputs[depth_output_name], prob, rgba[..., 3], fbuf, box)
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
        fruit_prob = fbuf.colors[:count, 0] if fbuf is not None else None
        if remove_outliers:
            points, ind = pointcloud.remove_statistical_outliers(points, 20, std_ratio, return_index=True)
            colors, view_dirs = colors[ind], view_dirs[ind]
            fruit_prob = fruit_prob[ind] if fruit_prob is not None else None
        normals = None
        if estimate_normals:
            normals = pointcloud.estimate_normals(points, 30, view_dirs if reorient_normals else None)
            if reorient_normals:
                normals = normals.float().double()  # the reference reorients fp32 normals and stores them back
    out = {"points": points.cpu().numpy(), "colors": colors.double().cpu().numpy(),
           "normals": None if normals is None else normals.cpu().numpy()}
    if fruit_prob is not None:
        out["fruit"] = fruit_prob.cpu().numpy()
    return out


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


def read_line_set_points(path) -> np.ndarray:
    """The vertices of a PLY line set as open3d's write_line_set produces it -> [N,3] float64.

    A ``vertex`` element with float or double x/y/z (other scalar vertex properties are skipped by their declared type)
    and any further elements (open3d's ``edge`` element, list properties included), which are not read.  Both ``ascii``
    and ``binary_little_endian`` files are read.  ``read_ply`` keeps refusing such files: they are no point cloud."""
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
                kind = "list" if tok[1] == "list" else _PLY_TYPES.get(tok[1])
                if kind is None:
                    raise ValueError(f"{path}: unknown PLY type '{tok[1]}'")
                elements[-1][2].append((tok[-1], kind))
        if fmt not in ("ascii", "binary_little_endian"):
            raise ValueError(f"{path}: only ascii and binary_little_endian PLY are supported, got {fmt}")
        vertex = None
        for name, count, props in elements:  # the elements before the vertices are skipped row by row
            if name == "vertex" or count:
                if any(kind == "list" for _, kind in props):
                    if name == "vertex":
                        raise ValueError(f"{path}: list property in the vertex element")
                    raise ValueError(f"{path}: element '{name}' with list properties before the vertices")
            if fmt == "ascii":
                rows = [f.readline().split() for _ in range(count)]
                if name != "vertex":
                    continue
                if any(len(r) != len(props) for r in rows):
                    raise ValueError(f"{path}: vertex rows do not have {len(props)} values")
                table = np.array(rows, dtype=np.float64).reshape(count, len(props))
                vertex = {p: table[:, i] for i, (p, _) in enumerate(props)}
            else:
                dt = np.dtype(props)
                data = f.read(count * dt.itemsize)
                if name != "vertex":
                    continue
                if len(data) != count * dt.itemsize:
                    raise ValueError(f"{path}: file ends inside the vertex element")
                rec = np.frombuffer(data, dtype=dt, count=count)
                vertex = {p: rec[p] for p in dt.names}
            break
    if vertex is None or not {"x", "y", "z"} <= set(vertex):
        raise ValueError(f"{path}: no vertex x/y/z")
    return np.stack([vertex["x"], vertex["y"], vertex["z"]], axis=1).astype(np.float64)


# ---- the `tsdf` mesh export (nerfstudio 0.3.2 exporter_utils / tsdf_utils.export_tsdf_mesh) ------------------------------
def tsdf_cameras(cameras, downscale_factor: float = 2):
    """The training cameras as distortion-free perspective render cameras (``render.CameraSet``), rescaled by
    1 / ``downscale_factor``: upstream renders them with ``disable_distortion=True``.  Fisheye and equirectangular cameras
    are refused: a TSDF projects grid points through a pinhole."""
    from ..render import CameraSet

    if cameras.camera_type != "perspective":
        raise ValueError(f"the tsdf export needs perspective cameras; these are {cameras.camera_type!r}")
    if downscale_factor < 1:
        raise ValueError(f"downscale_factor must be >= 1, got {downscale_factor}")
    return CameraSet.from_cameras(cameras).rescale_output_resolution(1.0 / downscale_factor)


@torch.no_grad()
def _fuse(model, cams, tsdf, batch_size: int, depth_output_name: str, rgb_output_name: str) -> None:
    """Render every camera (rays from fnr_camera_rays, the model's forward chunk by chunk into device frame buffers) and fuse
    ``batch_size`` frames at a time.  Nothing goes to the host."""
    from ..compat import RayBundle

    dev = tsdf.device
    cams = cams.to(dev)
    H, W = cams.height, cams.width
    P = H * W
    chunk = min(int(model.config.eval_num_rays_per_chunk), P)
    o_buf = torch.empty((chunk, 3), dtype=torch.float32, device=dev)
    d_buf = torch.empty((chunk, 3), dtype=torch.float32, device=dev)
    F = len(cams)
    for f0 in range(0, F, batch_size):
        n = min(batch_size, F - f0)
        depth = torch.empty((n, P), dtype=torch.float32, device=dev)
        rgb = torch.empty((n, P, 3), dtype=torch.float32, device=dev)
        fruit = torch.empty((n, P), dtype=torch.float32, device=dev)
        for b in range(n):
            cam_idx = torch.full((chunk, 1), f0 + b, dtype=torch.long, device=dev)
            for p0 in range(0, P, chunk):
                m = min(chunk, P - p0)
                o, d = ops.camera_rays(cams.camera_to_worlds, cams.fx, cams.fy, cams.cx, cams.cy, "perspective", H, W, f0 + b, p0, m,
                                       out=(o_buf, d_buf))
                out = model(RayBundle(origins=o, directions=d, camera_indices=cam_idx[:m]))
                for name in (depth_output_name, rgb_output_name, "semantics"):
                    if name not in out:
                        raise KeyError(f"the model has no output {name!r}")
                depth[b, p0:p0 + m] = out[depth_output_name].reshape(m)
                rgb[b, p0:p0 + m] = out[rgb_output_name].reshape(m, 3)
                fruit[b, p0:p0 + m] = torch.sigmoid(out["semantics"].reshape(m))
        sl = slice(f0, f0 + n)
        tsdf.integrate(cams.camera_to_worlds[sl], cams.fx[sl].float(), cams.fy[sl].float(), cams.cx[sl].float(), cams.cy[sl].float(),
                       depth.view(n, H, W), rgb.view(n, H, W, 3), fruit.view(n, H, W))


def export_tsdf_mesh(pipeline, output_dir, downscale_factor: int = 2, depth_output_name: str = "depth", rgb_output_name: str = "rgb",
                     resolution=128, batch_size: int = 10, use_bounding_box: bool = True, bounding_box_min=(-1.0, -1.0, -1.0),
                     bounding_box_max=(1.0, 1.0, 1.0), refine_mesh_using_initial_aabb_estimate: bool = False,
                     refinement_epsilon: float = 1e-2) -> Dict:
    """nerfstudio export_tsdf_mesh on the GPU: render the training cameras at 1 / ``downscale_factor`` resolution, fuse
    them ``batch_size`` frames at a time into a ``resolution``^3 TSDF (one value or three) spanning the bounding box (or
    the scene box), and extract the level-0 mesh.  With ``refine_mesh_using_initial_aabb_estimate`` the fusion runs again
    in the first mesh's vertex box widened by ``refinement_epsilon``.  The projection uses the rescaled intrinsics, those
    of the rendered images.

    Writes ``tsdf_mesh.ply`` (every face, vertex colours) and ``fruit_mesh.ply`` (the faces whose three vertices have a
    fused fruit probability >= 0.5, vertices compacted in order; possibly empty) in the dataparser frame.  An empty mesh
    raises RuntimeError and writes nothing.  Returns {'mesh', 'fruit_mesh': dicts of numpy arrays, 'aabb' [2,3] of the
    final grid, 'paths'}."""
    from .. import mesh as M

    model = pipeline.model
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("export_tsdf_mesh needs the model on a CUDA device: the fusion and marching cubes are CUDA kernels")
    res = [int(r) for r in (resolution if isinstance(resolution, (list, tuple)) else [resolution])]
    if len(res) not in (1, 3) or min(res) < 2:
        raise ValueError(f"resolution must be one or three integers >= 2, got {resolution}")
    res = res * 3 if len(res) == 1 else res
    if batch_size < 1:
        raise ValueError(f"batch_size must be >= 1, got {batch_size}")
    if use_bounding_box:
        if not all(lo < hi for lo, hi in zip(bounding_box_min, bounding_box_max)):
            raise ValueError("Bounding box min must be smaller than max")
        aabb = torch.tensor([list(bounding_box_min), list(bounding_box_max)], dtype=torch.float32)
    else:
        aabb = pipeline.datamanager.train_dataset.scene_box.aabb.detach().float().cpu()
    cams = tsdf_cameras(pipeline.datamanager.train_dataset.cameras, downscale_factor)

    def run(box):
        tsdf = M.TSDF.from_aabb(box, res, device=dev)
        _fuse(model, cams, tsdf, batch_size, depth_output_name, rgb_output_name)
        out = {k: (None if v is None else v.cpu().numpy()) for k, v in tsdf.get_mesh().items()}
        if out["faces"].shape[0] == 0:
            raise RuntimeError(f"the TSDF in the box {box.tolist()} gave an empty mesh: check the bounding box and the trained model")
        return out

    mesh = run(aabb)
    if refine_mesh_using_initial_aabb_estimate:
        v = torch.from_numpy(mesh["vertices"])
        aabb = torch.stack([v.min(dim=0).values - refinement_epsilon, v.max(dim=0).values + refinement_epsilon]).float()
        mesh = run(aabb)
    fv, fn, fc, ff, fidx = M.fruit_submesh(mesh["vertices"], mesh["normals"], mesh["colors"], mesh["fruit"], mesh["faces"])
    fruit_mesh = {"vertices": fv, "normals": fn, "colors": fc, "fruit": ff, "faces": fidx}
    out_dir = pathlib.Path(output_dir)
    paths = {"mesh": str(out_dir / "tsdf_mesh.ply"), "fruit_mesh": str(out_dir / "fruit_mesh.ply")}
    write_mesh_ply(paths["mesh"], mesh["vertices"], mesh["normals"], mesh["colors"], mesh["faces"])
    write_mesh_ply(paths["fruit_mesh"], fv, fn, fc, fidx)
    return {"mesh": mesh, "fruit_mesh": fruit_mesh, "aabb": aabb.numpy(), "paths": paths}


def export_poisson_mesh(pipeline, output_dir, num_points: int = 1000000, remove_outliers: bool = True, reorient_normals: bool = True,
                        depth_output_name: str = "depth", rgb_output_name: str = "rgb", save_point_cloud: bool = False,
                        use_bounding_box: bool = True, bounding_box_min=(-1.0, -1.0, -1.0), bounding_box_max=(1.0, 1.0, 1.0),
                        std_ratio: float = 10.0, depth: int = 9) -> Dict:
    """nerfstudio ExportPoissonMesh on the GPU: the surface cloud of ``generate_point_cloud`` with estimated normals and
    per-point fruit probabilities, a screened Poisson reconstruction at ``depth`` (poisson.reconstruct: dense grid, open3d's
    scale 1.1 and point weight 2), and the trim of the vertices below the 0.1 quantile of density.

    Writes ``poisson_mesh.ply`` (vertex colours) and ``fruit_poisson_mesh.ply`` (the faces whose three vertices have a fruit
    probability >= 0.5; possibly empty) in the dataparser frame, and with ``save_point_cloud`` also ``point_cloud.ply``.
    An empty mesh raises RuntimeError and writes nothing.  Returns {'mesh', 'fruit_mesh': dicts of numpy arrays,
    'point_cloud', 'iterations', 'residual', 'paths'}."""
    from .. import mesh as M
    from .. import poisson

    poisson.check_depth(depth)
    dev = next(pipeline.model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("export_poisson_mesh needs the model on a CUDA device: the reconstruction runs as CUDA kernels")
    pcd = generate_point_cloud(pipeline, num_points=num_points, remove_outliers=remove_outliers, reorient_normals=reorient_normals,
                               estimate_normals=True, rgb_output_name=rgb_output_name, depth_output_name=depth_output_name,
                               use_bounding_box=use_bounding_box, bounding_box_min=bounding_box_min, bounding_box_max=bounding_box_max,
                               std_ratio=std_ratio, fruit=True)
    if len(pcd["points"]) == 0:
        raise RuntimeError("the surface cloud is empty: the Poisson reconstruction gave an empty mesh")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    r = poisson.reconstruct(t(pcd["points"]), t(pcd["normals"]).float(), t(pcd["colors"]).float(), t(pcd["fruit"]).float(), depth=depth)
    mesh = r["mesh"]
    if mesh["faces"].shape[0] == 0:
        raise RuntimeError(f"the Poisson reconstruction of {len(pcd['points'])} points gave an empty mesh")
    fv, fn, fc, ff, fidx = M.fruit_submesh(mesh["vertices"], mesh["normals"], mesh["colors"], mesh["fruit"], mesh["faces"])
    fruit_mesh = {"vertices": fv, "normals": fn, "colors": fc, "fruit": ff, "faces": fidx}
    out_dir = pathlib.Path(output_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    paths = {"mesh": str(out_dir / "poisson_mesh.ply"), "fruit_mesh": str(out_dir / "fruit_poisson_mesh.ply")}
    if save_point_cloud:
        paths["point_cloud"] = str(out_dir / "point_cloud.ply")
        write_ply(paths["point_cloud"], pcd["points"], pcd["colors"], normals=pcd["normals"])
    write_mesh_ply(paths["mesh"], mesh["vertices"], mesh["normals"], mesh["colors"], mesh["faces"])
    write_mesh_ply(paths["fruit_mesh"], fv, fn, fc, fidx)
    return {"mesh": mesh, "fruit_mesh": fruit_mesh, "point_cloud": pcd, "iterations": r["iterations"], "residual": r["residual"],
            "paths": paths}


@torch.no_grad()
def export_textured_mesh(pipeline, mesh: Dict, output_dir, prefix: str = "", px_per_uv_triangle: int = 4, unwrap_method: str = "custom",
                         num_pixels_per_side: int = 1024, unwrap: Optional[Dict] = None) -> Dict:
    """nerfstudio texture_utils.export_textured_mesh on the GPU, for one mesh dict of ``export_tsdf_mesh`` /
    ``export_poisson_mesh`` ('vertices', 'normals', 'faces').  The rays are cast from 0.5 raylen outside the surface along
    the inverted normal, near 0, far raylen, camera 0, with raylen = 2 * the mean first-edge length (fnr_mesh_mean_edge);
    they go through the model chunk by chunk on the device, the ``rgb`` output is quantised by fnr_compose_frame, and one
    device-to-host copy gives the colours.

    * ``unwrap_method="custom"`` (nerfstudio's): every face gets its own triangle of the atlas (texture.py), and every
      texel a ray (fnr_texel_rays).
    * ``unwrap_method="charts"`` (DESIGN section 4.3r): the ``num_pixels_per_side``-square chart atlas of
      ``chart_unwrap_mesh`` (pass ``unwrap`` to reuse one); only the owned texels get a ray (fnr_chart_texel_rays), the
      others stay black.

    Writes ``{prefix}mesh.obj``, ``{prefix}material_0.mtl`` and ``{prefix}material_0.png`` under ``output_dir``.  Returns
    {'obj', 'mtl', 'png': paths, 'width', 'height', 'raylen'}.  An atlas that cannot be made raises
    texture.AtlasTooLargeError before anything is rendered or written."""
    from PIL import Image

    from .. import texture
    from ..compat import RayBundle
    from ..render import _turbo_table, render_into_buffers

    model = pipeline.model
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("export_textured_mesh needs the model on a CUDA device: the texel rays are a CUDA kernel")
    if unwrap_method not in ("custom", "charts"):
        raise ValueError(f"unwrap_method must be 'custom' or 'charts', got {unwrap_method!r}")
    faces = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    if unwrap_method == "charts":
        if unwrap is None:
            unwrap = chart_unwrap_mesh(mesh, num_pixels_per_side, dev)
        W = H = texture.check_num_pixels_per_side(num_pixels_per_side)
        P = int(unwrap["num_owned"])
    else:
        p = texture.check_px_per_uv_triangle(px_per_uv_triangle)
        W, H = texture.atlas_size(len(faces), p)
        P = W * H
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)  # noqa: E731
    verts, nrms, fdev = t(mesh["vertices"], np.float32).reshape(-1, 3), t(mesh["normals"], np.float32).reshape(-1, 3), t(faces, np.int64)
    raylen = float(np.float32(2.0 * float(ops.mesh_mean_edge(verts, fdev))))
    chunk = max(1, min(int(model.config.eval_num_rays_per_chunk), P))
    o_buf = torch.empty((chunk, 3), dtype=torch.float32, device=dev)
    d_buf = torch.empty((chunk, 3), dtype=torch.float32, device=dev)
    cam_idx = torch.zeros((chunk, 1), dtype=torch.long, device=dev)
    nears = torch.zeros((chunk, 1), dtype=torch.float32, device=dev)
    fars = torch.full((chunk, 1), raylen, dtype=torch.float32, device=dev)

    def chunk_rays(t0: int, n: int) -> RayBundle:
        if unwrap_method == "charts":
            o, d = ops.chart_texel_rays(verts, nrms, fdev, unwrap["texel_faces"], unwrap["barycentrics"], raylen, t0, n, out=(o_buf, d_buf))
        else:
            o, d = ops.texel_rays(verts, nrms, fdev, p, W, H, raylen, t0, n, out=(o_buf, d_buf))
        return RayBundle(origins=o, directions=d, camera_indices=cam_idx[:n], nears=nears[:n], fars=fars[:n])

    bufs = render_into_buffers(model, chunk_rays, P, chunk, ["rgb"], {}, lambda _stage: None)
    if unwrap_method == "charts":  # the owned texels' colours, scattered into a black image
        colours = ops.compose_frame([ops.FrameImage(bufs["rgb"], "color")], None, 1, P, _turbo_table(dev)).cpu().numpy().reshape(P, 3)
        image = np.zeros((H * W, 3), np.uint8)
        image[unwrap["texels"].cpu().numpy()] = colours
        image = image.reshape(H, W, 3)
        uv = texture.chart_vt(unwrap["uv"].cpu().numpy(), W)
    else:
        image = ops.compose_frame([ops.FrameImage(bufs["rgb"], "color")], None, H, W, _turbo_table(dev)).cpu().numpy()
        uv = texture.uv_coordinates(len(faces), p)
    out_dir = pathlib.Path(output_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    mtl, png = f"{prefix}material_0.mtl", f"{prefix}material_0.png"
    paths = {"obj": str(out_dir / f"{prefix}mesh.obj"), "mtl": str(out_dir / mtl), "png": str(out_dir / png)}
    Image.fromarray(image).save(paths["png"])
    texture.write_textured_obj(paths["obj"], mtl, png, mesh["vertices"], mesh["normals"], faces, uv)
    return {**paths, "width": W, "height": H, "raylen": raylen}


def chart_unwrap_mesh(mesh: Dict, num_pixels_per_side: int, device) -> Dict:
    """The `charts` atlas of ``mesh`` (ops.chart_unwrap, DESIGN section 4.3r) on ``device``; texture.AtlasTooLargeError when
    its charts do not fit into num_pixels_per_side^2 texels."""
    from .. import texture

    N = texture.check_num_pixels_per_side(num_pixels_per_side)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(device)  # noqa: E731
    return ops.chart_unwrap(t(mesh["vertices"], np.float32).reshape(-1, 3), t(np.asarray(mesh["faces"]).reshape(-1, 3), np.int64), N)


def decimate_for_texture(mesh: Dict, target_num_faces: int, device) -> Dict:
    """``mesh`` decimated on the device (fnr_mesh_decimate, DESIGN section 4.3q) to target_num_faces faces or one more,
    as {'vertices', 'normals' [V',3] fp32, 'faces' [F',3] int64, 'rounds'}; a mesh with at most target_num_faces faces
    comes back as it is.  A mesh on which no edge can collapse before the target stops early, with a one-line note."""
    from .. import ops

    faces = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    if len(faces) <= target_num_faces:
        return mesh
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(device)  # noqa: E731
    r = ops.mesh_decimate(t(mesh["vertices"], np.float64).reshape(-1, 3), t(faces, np.int64), int(target_num_faces))
    out = {"vertices": r["vertices"].to(torch.float32).cpu().numpy(), "normals": r["normals"].to(torch.float32).cpu().numpy(),
           "faces": r["faces"].cpu().numpy(), "rounds": r["rounds"]}
    if len(out["faces"]) > target_num_faces + 1:
        print(f"note: decimation stopped at {len(out['faces'])} faces (target {target_num_faces}): no edge left that can collapse")
    return out


def export_textured_meshes(pipeline, result: Dict, output_dir, px_per_uv_triangle: int = 4,
                           target_num_faces: Optional[int] = None, unwrap_method: str = "custom",
                           num_pixels_per_side: int = 1024) -> Dict[str, str]:
    """Texture the scene mesh (``mesh.obj`` / ``material_0.{mtl,png}``) and, unless it is empty, the fruit mesh
    (``fruit_mesh.obj`` / ``fruit_material_0.{mtl,png}``) of an ``export_tsdf_mesh`` / ``export_poisson_mesh`` result.
    With ``target_num_faces`` each mesh is first decimated to that many faces on its own (``decimate_for_texture``); the
    PLYs are never decimated.  Both atlases are then sized (``custom``) or unwrapped (``charts``), so an atlas that cannot
    be made for either mesh (texture.AtlasTooLargeError) writes nothing, and only then rendered.  Returns the paths, keyed
    'mesh_obj', 'mesh_mtl', 'mesh_png' and 'fruit_mesh_obj', ...."""
    from .. import texture

    jobs = [(key, prefix) for key, prefix in (("mesh", ""), ("fruit_mesh", "fruit_")) if len(result[key]["faces"]) > 0]
    meshes = {key: result[key] for key, _ in jobs}
    dev = next(pipeline.model.parameters()).device
    if target_num_faces is not None:
        if dev.type != "cuda":
            raise RuntimeError("decimation before texturing needs the model on a CUDA device: fnr_mesh_decimate is a CUDA kernel")
        meshes = {key: decimate_for_texture(m, int(target_num_faces), dev) for key, m in meshes.items()}
    unwraps = {}
    for key, _ in jobs:
        if unwrap_method == "charts":
            if dev.type != "cuda":
                raise RuntimeError("the charts unwrap needs the model on a CUDA device: fnr_chart_unwrap is a CUDA kernel")
            unwraps[key] = chart_unwrap_mesh(meshes[key], num_pixels_per_side, dev)
        else:
            texture.atlas_size(len(meshes[key]["faces"]), px_per_uv_triangle)
    paths = {}
    for key, prefix in jobs:
        r = export_textured_mesh(pipeline, meshes[key], output_dir, prefix, px_per_uv_triangle, unwrap_method, num_pixels_per_side,
                                 unwraps.get(key))
        paths.update({f"{key}_{kind}": r[kind] for kind in ("obj", "mtl", "png")})
    return paths


_FACE_DTYPE = np.dtype([("n", "u1"), ("v", "<i4", (3,))])  # packed: 13 bytes per face


def write_mesh_ply(path, vertices: np.ndarray, normals: np.ndarray, colors: Optional[np.ndarray], faces: np.ndarray) -> None:
    """Binary little-endian triangle mesh: vertex double x/y/z, double nx/ny/nz, uchar red/green/blue (``write_ply``'s
    colour conversion; black without ``colors``), then ``face`` rows of ``list uchar int vertex_indices``."""
    v = np.asarray(vertices, dtype="<f8").reshape(-1, 3)
    n = v.shape[0]
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= n or n > 0x7FFFFFFF):
        raise ValueError(f"face indices must lie in [0, {n}) and fit an int")
    col = np.zeros((n, 3), np.uint8) if colors is None else np.clip(np.asarray(colors, dtype=np.float64).reshape(-1, 3) * 255.0, 0, 255).astype(np.uint8)
    nrm = np.asarray(normals, dtype="<f8").reshape(-1, 3)
    header = (
        "ply\nformat binary_little_endian 1.0\ncomment fruitnerf_b200 export\n"
        f"element vertex {n}\nproperty double x\nproperty double y\nproperty double z\n"
        "property double nx\nproperty double ny\nproperty double nz\n"
        "property uchar red\nproperty uchar green\nproperty uchar blue\n"
        f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n"
    )
    rec = np.empty(n, dtype=[("p", "<f8", (3,)), ("n", "<f8", (3,)), ("c", "u1", (3,))])
    rec["p"], rec["n"], rec["c"] = v, nrm, col
    frec = np.empty(f.shape[0], dtype=_FACE_DTYPE)
    frec["n"], frec["v"] = 3, f
    pathlib.Path(path).parent.mkdir(parents=True, exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(rec.tobytes())
        fh.write(frec.tobytes())


def read_mesh_ply(path):
    """A binary little-endian triangle mesh as ``write_mesh_ply`` writes it -> (vertices [N,3], normals [N,3] or None,
    colors [N,3] in [0,1] or None, faces [F,3] int64).  Scalar vertex properties of any type are read by name; the face
    element must hold one ``list uchar int`` (or ``uint``) property of triangles."""
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
                    if tok[2] not in ("uchar", "uint8") or tok[3] not in ("int", "int32", "uint", "uint32"):
                        raise ValueError(f"{path}: unsupported list property {' '.join(tok[1:])}")
                    elements[-1][2].append((tok[4], "list", _PLY_TYPES[tok[3]]))
                elif tok[1] in _PLY_TYPES:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]], None))
                else:
                    raise ValueError(f"{path}: unknown PLY type '{tok[1]}'")
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: only binary_little_endian PLY is supported, got {fmt}")
        vertex, faces = None, np.zeros((0, 3), np.int64)
        for name, count, props in elements:
            lists = [p for p in props if p[1] == "list"]
            if lists:
                if name != "face" or len(props) != 1:
                    raise ValueError(f"{path}: list properties are only read as the face element's single vertex list")
                dt = np.dtype([("n", "u1"), ("v", lists[0][2], (3,))])
                rec = np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)
                if count and (rec["n"] != 3).any():
                    raise ValueError(f"{path}: only triangle faces are supported")
                faces = rec["v"].astype(np.int64)
                continue
            dt = np.dtype([(p[0], p[1]) for p in props])
            rec = np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)
            if name == "vertex":
                vertex = rec
            elif count:
                raise ValueError(f"{path}: unexpected element '{name}' with {count} rows")
    if vertex is None or not {"x", "y", "z"} <= set(vertex.dtype.names):
        raise ValueError(f"{path}: no vertex x/y/z")
    names = set(vertex.dtype.names)
    stack = lambda keys: np.stack([vertex[k] for k in keys], axis=1).astype(np.float64)  # noqa: E731
    normals = stack(("nx", "ny", "nz")) if {"nx", "ny", "nz"} <= names else None
    colors = stack(("red", "green", "blue")) / 255.0 if {"red", "green", "blue"} <= names else None
    return stack(("x", "y", "z")), normals, colors, faces
