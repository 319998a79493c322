"""Time of the lens ray kernels: ``fnr_pixel_batch_lens`` at 4096 and 65 536 rays for a pinhole (per-image intrinsics, no
distortion), an OPENCV camera (COLMAP-sized k1 k2 p1 p2) and a fisheye, next to the shared-pinhole ``fnr_pixel_batch``;
and ``fnr_camera_rays_lens`` for one 1920x1080 frame.  CUDA events over many launches; the card's name, power limit and
max SM clock are read in the same run.

    python tools/bench_lens_rays.py [--iters 200] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from fruitnerf_b200 import ops  # noqa: E402
from tools.bench_render import gpu_info  # noqa: E402

OPENCV = [-0.12, 0.045, 0.0, 0.0, 0.0012, -0.0009]


def _time_us(fn, iters: int) -> float:
    for _ in range(10):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return 1e3 * start.elapsed_time(end) / iters


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_lens_rays needs a CUDA device")
    dev = torch.device("cuda:0")
    ops.L.load()
    N, H, W = 36, 1080, 1920  # a captured data set at full resolution: the gathers read from a 36 x 1080p image stack
    g = torch.Generator(device=dev).manual_seed(0)
    imgs = torch.rand(N, H, W, 3, device=dev, generator=g)
    masks = torch.rand(N, H, W, 1, device=dev, generator=g)
    c2w = torch.eye(4, device=dev)[:3].expand(N, 3, 4).contiguous()
    fx, fy, cx, cy = (torch.full((N,), v, device=dev) for v in (1500.0, 1500.0, W / 2.0, H / 2.0))
    dist = torch.tensor(OPENCV, device=dev).expand(N, 6).contiguous()
    res = {**gpu_info(), "images": [N, H, W], "iters": a.iters, "pixel_batch_us": {}}
    for R in (4096, 65536):
        r = torch.rand(R, 3, device=dev, generator=g)
        row = {"shared_pinhole (fnr_pixel_batch)": _time_us(lambda: ops.pixel_batch(r, c2w, imgs, masks, 1500.0, 1500.0, W / 2.0, H / 2.0), a.iters),
               "pinhole": _time_us(lambda: ops.pixel_batch_lens(r, c2w, imgs, masks, fx, fy, cx, cy, None, "perspective"), a.iters),
               "opencv": _time_us(lambda: ops.pixel_batch_lens(r, c2w, imgs, masks, fx, fy, cx, cy, dist, "perspective"), a.iters),
               "fisheye": _time_us(lambda: ops.pixel_batch_lens(r, c2w, imgs, masks, fx, fy, cx, cy, dist, "fisheye"), a.iters)}
        res["pixel_batch_us"][str(R)] = row
    f64 = [t.double() for t in (fx, fy, cx, cy)]
    res["camera_rays_1080p_us"] = {
        "fnr_camera_rays (perspective)": _time_us(lambda: ops.camera_rays(c2w, *f64, "perspective", H, W, 0, 0, H * W), a.iters // 4),
        "opencv": _time_us(lambda: ops.camera_rays_lens(c2w, fx, fy, cx, cy, dist, "perspective", H, W, 0, 0, H * W), a.iters // 4),
        "fisheye": _time_us(lambda: ops.camera_rays_lens(c2w, fx, fy, cx, cy, dist, "fisheye", H, W, 0, 0, H * W), a.iters // 4)}
    print(json.dumps(res, indent=1))
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
