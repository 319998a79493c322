"""The camera model of captured data sets (nerfstudio 0.3.2 ``Cameras`` / ``camera_utils``), restated in torch.

This is the host statement of the lens that ``fnr_pixel_batch_lens`` / ``fnr_camera_rays_lens`` evaluate on the device
(DESIGN.md section 4.3j): the CPU branch of the datamanager, the ray model of the synthetic lens data sets and the
tests' reference.  It is not a fall-back for CUDA tensors, which go to the kernels.

Pixel (x, y) of a camera with intrinsics fx, fy, cx, cy has the normalised coordinates u = (x + 0.5 - cx) / fx and
v = -(y + 0.5 - cy) / fy (fp32).  Unless the camera is equirectangular, (u, v) is undistorted by Newton's method on
the OpenCV radial / tangential model with coefficients [k1, k2, k3, k4, p1, p2] (``radial_and_tangential_undistort``,
in fp64), then mapped to a camera-space direction by the camera type, rotated into the world and normalised (fp32).
Because v is flipped before the undistortion, this is OpenCV's model in y-down pixel coordinates with p1 negated.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
from torch import Tensor

# nerfstudio CAMERA_MODEL_TO_TYPE for the types the ray generator models
CAMERA_MODEL_TO_TYPE = {
    "SIMPLE_PINHOLE": "perspective",
    "PINHOLE": "perspective",
    "SIMPLE_RADIAL": "perspective",
    "RADIAL": "perspective",
    "OPENCV": "perspective",
    "OPENCV_FISHEYE": "fisheye",
    "EQUIRECTANGULAR": "equirectangular",
}
# what write_dataset names each type
TYPE_TO_CAMERA_MODEL = {"perspective": "OPENCV", "fisheye": "OPENCV_FISHEYE", "equirectangular": "EQUIRECTANGULAR"}


def get_distortion_params(k1: float = 0.0, k2: float = 0.0, k3: float = 0.0, k4: float = 0.0, p1: float = 0.0, p2: float = 0.0) -> Tensor:
    """camera_utils.get_distortion_params: the [6] fp32 vector [k1, k2, k3, k4, p1, p2]."""
    return torch.tensor([k1, k2, k3, k4, p1, p2], dtype=torch.float32)


def _split(params: Tensor):
    return tuple(params[..., i] for i in range(6))


def _residual_and_jacobian(x: Tensor, y: Tensor, xd: Tensor, yd: Tensor, params: Tensor):
    """camera_utils._compute_residual_and_jacobian.  The expressions keep the op order of the device (fnr_common.cuh
    undistort_rt), so in fp64 the two agree bit for bit."""
    k1, k2, k3, k4, p1, p2 = _split(params)
    r = x * x + y * y
    d = 1.0 + r * (k1 + r * (k2 + r * (k3 + r * k4)))
    fx = d * x + 2.0 * p1 * x * y + p2 * (r + 2.0 * x * x) - xd
    fy = d * y + 2.0 * p2 * x * y + p1 * (r + 2.0 * y * y) - yd
    d_r = k1 + r * (2.0 * k2 + r * (3.0 * k3 + r * 4.0 * k4))
    d_x = 2.0 * x * d_r
    d_y = 2.0 * y * d_r
    fx_x = d + d_x * x + 2.0 * p1 * y + 6.0 * p2 * x
    fx_y = d_y * x + 2.0 * p1 * x + 2.0 * p2 * y
    fy_x = d_x * y + 2.0 * p2 * y + 2.0 * p1 * x
    fy_y = d + d_y * y + 2.0 * p2 * x + 6.0 * p1 * y
    return fx, fy, fx_x, fx_y, fy_x, fy_y


def radial_and_tangential_undistort(coords: Tensor, distortion_params: Tensor, eps: float = 1e-3, max_iterations: int = 10) -> Tensor:
    """camera_utils.radial_and_tangential_undistort: [..., 2] distorted -> undistorted normalised coordinates, in the dtype
    of ``coords``.  Exactly ``max_iterations`` Newton steps, no convergence test; a zero step wherever |det| <= eps."""
    params = distortion_params.to(coords.dtype)
    xd, yd = coords[..., 0], coords[..., 1]
    x, y = xd, yd
    for _ in range(max_iterations):
        fx, fy, fx_x, fx_y, fy_x, fy_y = _residual_and_jacobian(x, y, xd, yd, params)
        den = fy_x * fx_y - fx_x * fy_y
        ok = torch.abs(den) > eps
        safe = torch.where(ok, den, torch.ones_like(den))
        x = torch.where(ok, x + (fx * fy_y - fy * fx_y) / safe, x)
        y = torch.where(ok, y + (fy * fx_x - fx * fy_x) / safe, y)
    return torch.stack([x, y], dim=-1)


def distort(coords: Tensor, distortion_params: Tensor) -> Tensor:
    """The forward model that ``radial_and_tangential_undistort`` inverts: [..., 2] undistorted -> distorted."""
    k1, k2, k3, k4, p1, p2 = _split(distortion_params.to(coords.dtype))
    x, y = coords[..., 0], coords[..., 1]
    r = x * x + y * y
    d = 1.0 + r * (k1 + r * (k2 + r * (k3 + r * k4)))
    return torch.stack([d * x + 2.0 * p1 * x * y + p2 * (r + 2.0 * x * x), d * y + 2.0 * p2 * x * y + p1 * (r + 2.0 * y * y)], dim=-1)


def pixel_coords(xs: Tensor, ys: Tensor, fx: Tensor, fy: Tensor, cx: Tensor, cy: Tensor) -> Tensor:
    """[..., 2] normalised coordinates (u, v) of pixel centres, fp32 with fp32 intrinsics (correctly rounded divisions)."""
    f32 = lambda t: torch.as_tensor(t, dtype=torch.float32, device=xs.device)  # noqa: E731
    u = (xs.to(torch.float32) + 0.5 - f32(cx)) / f32(fx)
    v = -((ys.to(torch.float32) + 0.5 - f32(cy)) / f32(fy))
    return torch.stack([u, v], dim=-1)


def _sqrt(x: Tensor) -> Tensor:
    """Correctly rounded fp32 square root, as the device's sqrtf: torch's vectorised CPU sqrt can be 1 ulp off, while the
    fp64 root of an fp32 value rounds to the exact fp32 result."""
    return torch.sqrt(x.double()).to(x.dtype)


def camera_directions(camera_type: str, uv: Tensor) -> Tensor:
    """Cameras._generate_rays_from_coords: camera-space directions [..., 3] (OpenGL axes) of coordinates [..., 2]."""
    u, v = uv[..., 0], uv[..., 1]
    if camera_type == "perspective":
        return torch.stack([u, v, -torch.ones_like(u)], dim=-1)
    if camera_type == "fisheye":
        theta = _sqrt(u * u + v * v).clamp(max=math.pi)
        k = torch.where(theta > 0, torch.sin(theta) / torch.where(theta > 0, theta, torch.ones_like(theta)), torch.zeros_like(theta))
        return torch.stack([u * k, v * k, -torch.cos(theta)], dim=-1)  # theta = 0: the optical axis (0, 0, -1)
    if camera_type == "equirectangular":
        theta, phi = -math.pi * u, math.pi * (0.5 - v)
        return torch.stack([-torch.sin(theta) * torch.sin(phi), torch.cos(phi), -torch.cos(theta) * torch.sin(phi)], dim=-1)
    raise ValueError(f"unknown camera_type {camera_type!r}")


def lens_rays(c2w: Tensor, fx, fy, cx, cy, distortion: Optional[Tensor], camera_type: str, ys: Tensor, xs: Tensor) -> Tuple[Tensor, Tensor]:
    """Origins and unit directions [R,3] of pixels (ys, xs) [R]: c2w [R,3,4] (or [3,4]), intrinsics [R] or scalars,
    distortion [R,6], [6] or None.  The arithmetic of the device's lens branch: fp32 pixel step, fp64 undistortion,
    fp32 direction, rotation with rounded products and 3-term sums left to right."""
    uv = pixel_coords(xs, ys, fx, fy, cx, cy)
    if distortion is not None and camera_type != "equirectangular":
        uv = radial_and_tangential_undistort(uv.double(), distortion.to(uv.device).double()).float()
    d = camera_directions(camera_type, uv)
    m = c2w.to(torch.float32)
    w = [(m[..., k, 0] * d[..., 0] + m[..., k, 1] * d[..., 1]) + m[..., k, 2] * d[..., 2] for k in range(3)]
    n = _sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]).clamp_min(1e-12)
    dirs = torch.stack([wk / n for wk in w], dim=-1)
    return m[..., :3, 3].expand_as(dirs), dirs
