"""Novel-view renders of a trained model: the camera paths of nerfstudio 0.3.2's ``ns-render`` (what the reference's
``debug/render.py`` launches) and the frame loop that turns them into uint8 images on the device.

nerfstudio is not installed here, so its path semantics are restated from memory (DESIGN section 4.3i):

* ``get_path_from_json``          -- a viewer camera-path file: per-keyframe ``camera_to_world`` (flattened 4x4) and
  ``fov``; focal length (H/2) / tan(fov / 2), equirectangular fx = W/2, fy = H; cx = W/2, cy = H/2.
* ``get_interpolated_poses_many`` -- slerp of the rotations and linear translations / intrinsics between consecutive
  cameras, ``steps`` poses per pair with both ends included.
* ``get_spiral_path``             -- a spiral of local camera centres around one camera, each looking at a point on its
  optical axis.

``render_frames`` keeps a frame on the device from ray generation (``ops.camera_rays``) through the model to the uint8
image (``ops.compose_frame``); the host receives one buffer per frame and encodes it on a writer thread.
"""
from __future__ import annotations

import math
import queue
import shutil
import subprocess
import threading
from dataclasses import dataclass, replace
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import ops
from .compat import RayBundle
from .data.synthetic_scene import camera_rays as pinhole_rays
from .image_metrics import _turbo_table

REFUSED_CAMERA_TYPES = ("omnidirectional", "vr180")
_DISTORTION_KEYS = ("distortion_params", "k1", "k2", "k3", "k4", "p1", "p2")


@dataclass
class CameraSet:
    """F render cameras of one size and camera model: c2w [F,3,4] (OpenGL axes, fp32) and per-frame fx / fy / cx / cy [F]
    (fp64, so that python-float intrinsics of a data set's cameras keep every bit)."""

    camera_to_worlds: Tensor
    fx: Tensor
    fy: Tensor
    cx: Tensor
    cy: Tensor
    height: int
    width: int
    camera_type: str = "perspective"

    def __post_init__(self):
        F = self.camera_to_worlds.shape[0]
        self.camera_to_worlds = self.camera_to_worlds.to(torch.float32).reshape(F, 3, 4).contiguous()
        for name in ("fx", "fy", "cx", "cy"):
            v = getattr(self, name)  # a python float stays fp64: torch.as_tensor would round it to fp32 first
            v = (v if torch.is_tensor(v) else torch.tensor(v, dtype=torch.float64)).to(self.camera_to_worlds.device, torch.float64).reshape(-1)
            setattr(self, name, (v.expand(F) if v.numel() == 1 else v).contiguous())
        if self.camera_type not in ops.CAMERA_TYPES:
            raise ValueError(f"camera_type must be one of {sorted(ops.CAMERA_TYPES)}, got {self.camera_type!r}")

    def __len__(self) -> int:
        return int(self.camera_to_worlds.shape[0])

    def to(self, device) -> "CameraSet":
        return replace(self, camera_to_worlds=self.camera_to_worlds.to(device), fx=self.fx.to(device), fy=self.fy.to(device),
                       cx=self.cx.to(device), cy=self.cy.to(device))

    @staticmethod
    def from_cameras(cams, indices: Optional[Sequence[int]] = None) -> "CameraSet":
        """Perspective, distortion-free cameras with the poses and intrinsics of a data set's cameras (``SyntheticCameras``,
        shared or per-image intrinsics), all of them or ``indices``, as nerfstudio's camera paths build them."""
        pick = (lambda v: v) if indices is None else (lambda v: v[list(indices)] if torch.is_tensor(v) else v)
        return CameraSet(pick(cams.camera_to_worlds), pick(cams.fx), pick(cams.fy), pick(cams.cx), pick(cams.cy), cams.height, cams.width)

    def rescale_output_resolution(self, scale: float) -> "CameraSet":
        """nerfstudio Cameras.rescale_output_resolution: intrinsics times ``scale`` (fp32), sizes truncated."""
        if scale == 1.0:
            return self
        fx, fy, cx, cy = (t.float() * scale for t in (self.fx, self.fy, self.cx, self.cy))
        return replace(self, fx=fx, fy=fy, cx=cx, cy=cy,
                       height=int(self.height * scale), width=int(self.width * scale))


# ---- camera models, restated in torch (the tests' reference for fnr_camera_rays) ------------------------------------
def restated_camera_rays(cams: CameraSet, frame: int, pixel_start: int, num_pixels: int) -> Tuple[Tensor, Tensor]:
    """Rays of pixels [pixel_start, pixel_start + n) of one frame.  Perspective: ``synthetic_scene.camera_rays`` itself
    (fp32, on the cameras' device).  Fisheye and equirectangular: the closed forms in fp64 on the host."""
    p = torch.arange(pixel_start, pixel_start + num_pixels, device=cams.camera_to_worlds.device)
    ys, xs = p // cams.width, p % cams.width
    c2w = cams.camera_to_worlds[frame]
    fx, fy, cx, cy = (float(t[frame]) for t in (cams.fx, cams.fy, cams.cx, cams.cy))
    if cams.camera_type == "perspective":
        return pinhole_rays(c2w, fx, fy, cx, cy, ys, xs)
    u = (xs.cpu().double() + 0.5 - cx) / fx
    v = -(ys.cpu().double() + 0.5 - cy) / fy
    if cams.camera_type == "fisheye":
        theta = torch.sqrt(u * u + v * v).clamp(0.0, math.pi)
        k = torch.where(theta > 0, torch.sin(theta) / torch.where(theta > 0, theta, torch.ones_like(theta)), torch.zeros_like(theta))
        d = torch.stack([u * k, v * k, -torch.cos(theta)], dim=-1)  # theta = 0: the optical axis (0, 0, -1)
    else:
        theta, phi = -math.pi * u, math.pi * (0.5 - v)
        d = torch.stack([-torch.sin(theta) * torch.sin(phi), torch.cos(phi), -torch.cos(theta) * torch.sin(phi)], dim=-1)
    m = c2w.cpu().double()
    d = d @ m[:3, :3].T
    d = d / d.norm(dim=-1, keepdim=True)
    return m[:3, 3].expand_as(d), d


# ---- camera paths (nerfstudio 0.3.2 camera_utils / camera_paths, restated) -----------------------------------------
def get_path_from_json(camera_path: Dict) -> CameraSet:
    """A viewer camera-path file -> CameraSet.  What the renderer cannot honour is refused: crop boxes (they need a
    background override), the stereo camera types, time-conditioned keyframes and lens distortion."""
    if camera_path.get("crop") is not None:
        raise NotImplementedError("camera path has 'crop' data: crop boxes need a background-colour override the renderer does not have")
    camera_type = camera_path.get("camera_type", "perspective")
    if camera_type in REFUSED_CAMERA_TYPES:
        raise NotImplementedError(f"camera_type {camera_type!r} is not supported (perspective, fisheye, equirectangular)")
    if camera_type not in ops.CAMERA_TYPES:
        raise ValueError(f"unknown camera_type {camera_type!r}")
    H, W = int(camera_path["render_height"]), int(camera_path["render_width"])
    keyframes = camera_path["camera_path"]
    if not keyframes:
        raise ValueError("camera path has no cameras")
    for where in (camera_path, *keyframes):
        bad = [k for k in _DISTORTION_KEYS if k in where]
        if bad:
            raise NotImplementedError(f"camera path carries distortion parameters {bad}: the render cameras are distortion-free")
        if "render_time" in where or "time" in where:
            raise NotImplementedError("camera path has time entries: time-conditioned models are not supported")
    c2w = torch.stack([torch.tensor(c["camera_to_world"], dtype=torch.float32).view(4, 4)[:3] for c in keyframes])
    if camera_type == "equirectangular":
        fx = torch.full((len(keyframes),), W / 2.0)
        fy = torch.full((len(keyframes),), float(H))
    else:
        fov = torch.tensor([float(c["fov"]) for c in keyframes], dtype=torch.float32)
        fx = fy = (H / 2.0) / torch.tan(fov * (math.pi / 180.0) / 2.0)  # three_js_perspective_camera_focal_length
    return CameraSet(c2w, fx, fy, torch.full_like(fx, W / 2.0), torch.full_like(fx, H / 2.0), H, W, camera_type)


def path_fps(camera_path: Dict, num_frames: int) -> float:
    """Video frame rate of a camera-path file: frames / ``seconds`` (ns-render), else its ``fps``."""
    if camera_path.get("seconds"):
        return num_frames / float(camera_path["seconds"])
    if camera_path.get("fps"):
        return float(camera_path["fps"])
    raise ValueError("camera path has neither 'seconds' nor 'fps'")


_EPS = np.finfo(float).eps * 4.0


def quaternion_from_matrix(R: np.ndarray) -> np.ndarray:
    """(w, x, y, z), w >= 0: the eigenvector of the largest eigenvalue of the symmetric 4x4 K of the rotation."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = np.asarray(R, dtype=np.float64)[:3, :3].ravel()
    K = np.array([[m00 - m11 - m22, 0.0, 0.0, 0.0], [m01 + m10, m11 - m00 - m22, 0.0, 0.0], [m02 + m20, m12 + m21, m22 - m00 - m11, 0.0],
                  [m21 - m12, m02 - m20, m10 - m01, m00 + m11 + m22]]) / 3.0
    w, V = np.linalg.eigh(K)
    q = V[[3, 0, 1, 2], np.argmax(w)]
    return -q if q[0] < 0.0 else q


def quaternion_slerp(q0: np.ndarray, q1: np.ndarray, fraction: float) -> np.ndarray:
    q0, q1 = q0 / np.linalg.norm(q0), q1 / np.linalg.norm(q1)
    if fraction == 0.0:
        return q0
    if fraction == 1.0:
        return q1
    d = float(np.dot(q0, q1))
    if abs(abs(d) - 1.0) < _EPS:
        return q0
    if d < 0.0:  # shortest path
        d, q1 = -d, -q1
    angle = math.acos(d)
    if abs(angle) < _EPS:
        return q0
    isin = 1.0 / math.sin(angle)
    return q0 * (math.sin((1.0 - fraction) * angle) * isin) + q1 * (math.sin(fraction * angle) * isin)


def quaternion_matrix(q: np.ndarray) -> np.ndarray:
    q = np.array(q, dtype=np.float64)
    n = np.dot(q, q)
    if n < _EPS:
        return np.identity(3)
    q = np.outer(q * math.sqrt(2.0 / n), q * math.sqrt(2.0 / n))
    return np.array([[1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0]],
                     [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0]],
                     [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2]]])


def get_ordered_poses_and_k(poses: Tensor, Ks: Tensor) -> Tuple[Tensor, Tensor]:
    """Greedy nearest-translation order starting at camera 0."""
    order, rest = [0], list(range(1, poses.shape[0]))
    while rest:
        dist = torch.norm(poses[order[-1]][:, 3] - poses[rest][:, :, 3], dim=1)
        order.append(rest.pop(int(torch.argmin(dist))))
    return poses[order], Ks[order]


def get_interpolated_poses_many(poses: Tensor, Ks: Tensor, steps_per_transition: int = 10, order_poses: bool = False) -> Tuple[Tensor, Tensor]:
    """poses [N,3,4], Ks [N,3,3] -> steps * (N - 1) poses and intrinsics: for each consecutive pair, t = linspace(0, 1,
    steps) with both ends (interior cameras appear twice), rotations slerped, translations and K linear."""
    if order_poses:
        poses, Ks = get_ordered_poses_and_k(poses, Ks)
    traj, k_interp = [], []
    ts = np.linspace(0, 1, steps_per_transition)
    for i in range(poses.shape[0] - 1):
        a, b = poses[i].cpu().numpy().astype(np.float64), poses[i + 1].cpu().numpy().astype(np.float64)
        qa, qb = quaternion_from_matrix(a[:3, :3]), quaternion_from_matrix(b[:3, :3])
        for t in ts:
            pose = np.zeros((3, 4))
            pose[:, :3] = quaternion_matrix(quaternion_slerp(qa, qb, float(t)))
            pose[:, 3] = (1 - t) * a[:3, 3] + t * b[:3, 3]
            traj.append(pose)
            k_interp.append(Ks[i] * (1.0 - t) + Ks[i + 1] * t)
    return torch.tensor(np.stack(traj), dtype=torch.float32), torch.stack(k_interp).to(torch.float32)


def get_interpolated_camera_path(cams: CameraSet, steps: int, order_poses: bool) -> CameraSet:
    Ks = torch.zeros((len(cams), 3, 3))  # fp32, as nerfstudio's Cameras.get_intrinsics_matrices
    Ks[:, 0, 0], Ks[:, 1, 1], Ks[:, 0, 2], Ks[:, 1, 2], Ks[:, 2, 2] = cams.fx.cpu(), cams.fy.cpu(), cams.cx.cpu(), cams.cy.cpu(), 1.0
    poses, Ks = get_interpolated_poses_many(cams.camera_to_worlds.cpu(), Ks, steps, order_poses)
    cx, cy = Ks[0, 0, 2], Ks[0, 1, 2]  # the first interpolated K's principal point for every frame; size 2 cx x 2 cy
    return CameraSet(poses, Ks[:, 0, 0], Ks[:, 1, 1], cx, cy, int(cy * 2), int(cx * 2))


def _normalize(x: Tensor) -> Tensor:
    return x / torch.linalg.norm(x)


def viewmatrix(lookat: Tensor, up: Tensor, pos: Tensor) -> Tensor:
    """[3,4] camera-to-world whose +z is ``lookat`` (the camera looks along -lookat)."""
    vec2 = _normalize(lookat)
    vec0 = _normalize(torch.linalg.cross(_normalize(up), vec2))
    vec1 = _normalize(torch.linalg.cross(vec2, vec0))
    return torch.stack([vec0, vec1, vec2, pos], 1)


def spiral_centres(steps: int, radius: float, rots: int = 1, zrate: float = 0.5) -> Tensor:
    """Local camera centres radius * (cos t, -sin t, -sin(t zrate)), t in linspace(0, 2 pi rots, steps rots + 1)[:-1]."""
    ts = torch.linspace(0.0, 2.0 * math.pi * rots, steps * rots + 1)[:-1]
    return torch.stack([torch.cos(ts), -torch.sin(ts), -torch.sin(ts * zrate)], dim=-1) * radius


def get_spiral_path(cams: CameraSet, index: int = 0, steps: int = 30, radius: float = 0.1, rots: int = 1, zrate: float = 0.5) -> CameraSet:
    """Spiral around camera ``index``: each local pose looks from its centre at (0, 0, -min(fx, fy)) with up = the
    camera's z axis, then is left-multiplied by the camera's pose."""
    c2w = cams.camera_to_worlds[index].cpu()
    fx, fy, cx, cy = (t[index].cpu() for t in (cams.fx, cams.fy, cams.cx, cams.cy))
    c2w = c2w.float()
    up = c2w[:3, 2]
    target = torch.stack([torch.zeros(()), torch.zeros(()), -torch.minimum(fx, fy).float()])
    g = torch.eye(4)
    g[:3] = c2w
    poses = []
    for centre in spiral_centres(steps, radius, rots, zrate):
        local = torch.eye(4)
        local[:3] = viewmatrix(centre - target, up, centre)
        poses.append((g @ local)[:3])
    return CameraSet(torch.stack(poses), fx, fy, cx, cy, int(cy * 2), int(cx * 2))


# ---- frame composition ------------------------------------------------------------------------------------------
def frame_kind(name: str, channels: int) -> str:
    """ns-render's choice per output: a name containing 'depth' -> apply_depth_colormap; otherwise apply_colormap, i.e. a
    3-channel image as is and a 1-channel float image through turbo."""
    if "depth" in name:
        if channels != 1:
            raise NotImplementedError(f"depth output {name!r} has {channels} channels")
        return "depth"
    if channels == 3:
        return "color"
    if channels == 1:
        return "turbo"
    raise NotImplementedError(f"output {name!r} has {channels} channels: only 1- and 3-channel outputs are colour-mapped")


def plane_or_auto(plane: Optional[float]) -> Optional[float]:
    """nerfstudio's ``near_plane or min(depth)``: None and 0 both mean the frame's own extreme."""
    return float(plane) if plane else None


def tensor_output_names(outputs: Dict) -> List[str]:
    return [k for k, v in outputs.items() if torch.is_tensor(v)]


@torch.no_grad()
def probe_outputs(model) -> List[str]:
    """Names of the tensor outputs the model renders (one ray through ``model.forward``)."""
    dev = model.device
    o = torch.zeros((1, 3), device=dev)
    d = torch.tensor([[0.0, 0.0, -1.0]], device=dev)
    bundle = RayBundle(origins=o, directions=d, camera_indices=torch.zeros((1, 1), dtype=torch.long, device=dev))
    return tensor_output_names(model(bundle))


@torch.no_grad()
def render_into_buffers(model, chunk_rays: Callable[[int, int], RayBundle], num_rays: int, chunk: int, names: Sequence[str],
                        bufs: Dict[str, Tensor], stage: Callable[[str], None]) -> Dict[str, Tensor]:
    """One image through the model, chunk by chunk, with nothing leaving the device: ``chunk_rays(p0, n)`` gives the rays
    of pixels [p0, p0 + n) and the outputs ``names`` land in rows p0 .. p0 + n of ``bufs[name]`` ([num_rays, C] fp32,
    allocated on first use and reused for the next image).  ``stage`` is told "rays" and "field" as each chunk's ray
    generation and forward start.  Shared by ``render_frames`` and ``evaluate.evaluate_split``."""
    dev = model.device
    for p0 in range(0, num_rays, chunk):
        n = min(chunk, num_rays - p0)
        stage("rays")
        bundle = chunk_rays(p0, n)
        stage("field")
        out = model(bundle)
        for name in names:
            if name not in out or not torch.is_tensor(out[name]):
                raise KeyError(f"the model has no output {name!r}; available: {tensor_output_names(out)}")
            t = out[name].reshape(n, -1)
            if name not in bufs:
                bufs[name] = torch.empty((num_rays, t.shape[1]), dtype=torch.float32, device=dev)
            bufs[name][p0:p0 + n] = t
    return bufs


@torch.no_grad()
def render_frames(pipeline, cameras: CameraSet, output_names: Sequence[str], num_rays_per_chunk: Optional[int] = None,
                  depth_near_plane: Optional[float] = None, depth_far_plane: Optional[float] = None,
                  sink: Optional[Callable[[np.ndarray], None]] = None, on_stage: Optional[Callable[[str], None]] = None) -> List[np.ndarray]:
    """Render every camera of ``cameras`` into a uint8 [H, W * len(output_names), 3] image (ns-render's
    _render_trajectory_video frame).  Each frame stays on the device: rays per chunk from fnr_camera_rays, the model's
    forward per chunk written into preallocated frame buffers, one fnr_compose_frame and one device-to-host copy.
    Frames go to ``sink`` when given (returning []), else are returned.  ``on_stage(name)`` is called as each stage
    ("rays", "field", "compose") starts and with "done" after a frame's copy (benchmark timing hooks)."""
    model = pipeline.model
    dev = model.device
    if dev.type != "cuda":
        raise RuntimeError("render_frames needs the model on a CUDA device: ray generation and composition are CUDA kernels")
    names = list(output_names)
    if not names:
        raise ValueError("no output names to render")
    cams = cameras.to(dev)
    H, W = cams.height, cams.width
    P = H * W
    chunk = int(num_rays_per_chunk or model.config.eval_num_rays_per_chunk)
    n_max = min(chunk, P)
    turbo = _turbo_table(dev)
    o_buf = torch.empty((n_max, 3), dtype=torch.float32, device=dev)
    d_buf = torch.empty((n_max, 3), dtype=torch.float32, device=dev)
    scratch = torch.empty(ops.L.FNR_COMPOSE_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
    needed = list(dict.fromkeys(names + (["accumulation"] if any("depth" in n for n in names) else [])))
    near, far = plane_or_auto(depth_near_plane), plane_or_auto(depth_far_plane)
    stage = on_stage or (lambda _name: None)
    frames, bufs = [], {}
    for f in range(len(cams)):
        cam_idx = torch.full((n_max, 1), f, dtype=torch.long, device=dev)

        def chunk_rays(p0: int, n: int, f=f, cam_idx=cam_idx) -> RayBundle:
            o, d = ops.camera_rays(cams.camera_to_worlds, cams.fx, cams.fy, cams.cx, cams.cy, cams.camera_type, H, W, f, p0, n,
                                   out=(o_buf, d_buf))
            return RayBundle(origins=o, directions=d, camera_indices=cam_idx[:n])

        render_into_buffers(model, chunk_rays, P, chunk, needed, bufs, stage)
        stage("compose")
        images = []
        for name in names:
            kind = frame_kind(name, bufs[name].shape[1])
            images.append(ops.FrameImage(bufs[name], kind, near, far) if kind == "depth" else ops.FrameImage(bufs[name], kind))
        acc = bufs.get("accumulation") if "accumulation" in needed else None
        frame = ops.compose_frame(images, acc, H, W, turbo, scratch).cpu().numpy()
        stage("done")
        if sink is not None:
            sink(frame)
        else:
            frames.append(frame)
    return frames


# ---- writers ----------------------------------------------------------------------------------------------------
def ffmpeg_command(ffmpeg: str, path: Path, width: int, height: int, fps: float) -> List[str]:
    """Raw RGB frames on stdin -> H.264 (yuv420p, padded to even sizes)."""
    return [ffmpeg, "-y", "-loglevel", "error", "-f", "rawvideo", "-pix_fmt", "rgb24", "-s", f"{width}x{height}", "-r", f"{fps:g}", "-i", "-",
            "-vf", "pad=ceil(iw/2)*2:ceil(ih/2)*2", "-c:v", "libx264", "-pix_fmt", "yuv420p", "-qp", "20", str(path)]


def require_ffmpeg() -> str:
    exe = shutil.which("ffmpeg")
    if exe is None:
        raise SystemExit("error: --output-format video needs an `ffmpeg` binary on PATH; none was found.  "
                         "Use --output-format images to write the frames as image files instead.")
    return exe


class FrameWriter:
    """Writes frames on a background thread so that encoding overlaps the next frame's GPU work.
    ``images``: ``<output_path without suffix>/{frame:05d}.{png,jpg}``; ``video``: raw RGB into an ffmpeg subprocess."""

    def __init__(self, output_path, output_format: str = "video", image_format: str = "jpeg", jpeg_quality: int = 100, fps: float = 24.0,
                 max_pending: int = 4):
        if output_format not in ("images", "video"):
            raise ValueError(f"output_format must be 'images' or 'video', got {output_format!r}")
        if image_format not in ("jpeg", "png"):
            raise ValueError(f"image_format must be 'jpeg' or 'png', got {image_format!r}")
        self.output_path = Path(output_path)
        self.output_format, self.image_format, self.jpeg_quality, self.fps = output_format, image_format, int(jpeg_quality), float(fps)
        self.ffmpeg = require_ffmpeg() if output_format == "video" else None
        self.image_dir = self.output_path.parent / self.output_path.stem
        self.count = 0
        self._proc: Optional[subprocess.Popen] = None
        self._size: Optional[Tuple[int, int]] = None
        self._error: Optional[BaseException] = None
        self._queue: "queue.Queue" = queue.Queue(maxsize=max_pending)
        self._thread = threading.Thread(target=self._run, name="render-writer", daemon=True)
        self._thread.start()

    def _write(self, index: int, frame: np.ndarray) -> None:
        if self.output_format == "images":
            from PIL import Image

            self.image_dir.mkdir(parents=True, exist_ok=True)
            if self.image_format == "png":
                Image.fromarray(frame).save(self.image_dir / f"{index:05d}.png")
            else:
                Image.fromarray(frame).save(self.image_dir / f"{index:05d}.jpg", quality=self.jpeg_quality)
            return
        H, W = frame.shape[:2]
        if self._proc is None:
            self.output_path.parent.mkdir(parents=True, exist_ok=True)
            self._size = (H, W)
            self._proc = subprocess.Popen(ffmpeg_command(self.ffmpeg, self.output_path, W, H, self.fps), stdin=subprocess.PIPE)
        if (H, W) != self._size:
            raise ValueError(f"frame {index} is {W}x{H}, the video is {self._size[1]}x{self._size[0]}")
        self._proc.stdin.write(np.ascontiguousarray(frame).tobytes())

    def _run(self) -> None:
        while True:
            item = self._queue.get()
            if item is None:
                return
            if self._error is None:
                try:
                    self._write(*item)
                except BaseException as e:  # re-raised in the rendering thread
                    self._error = e

    def _raise(self) -> None:
        if self._error is not None:
            raise RuntimeError(f"writing frames to {self.output_path} failed: {self._error}") from self._error

    def __call__(self, frame: np.ndarray) -> None:
        self._raise()
        if frame.dtype != np.uint8 or frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError(f"frames must be uint8 [H,W,3], got {frame.dtype} {frame.shape}")
        self._queue.put((self.count, frame))
        self.count += 1

    def close(self) -> None:
        self._queue.put(None)
        self._thread.join()
        if self._proc is not None:
            self._proc.stdin.close()
            rc = self._proc.wait()
            if rc != 0 and self._error is None:
                self._error = RuntimeError(f"ffmpeg exited with status {rc}")
        self._raise()
