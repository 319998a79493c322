"""Cost of the `eval` command against the pipeline's host evaluation, in one call:

* the synthetic apple scene's held-out views through ``FruitPipeline.get_average_eval_image_metrics`` (every chunk's
  outputs copied to the host, PSNR / SSIM on CPU tensors) and through ``evaluate.evaluate_split`` (device buffers,
  fnr_image_stats + fnr_ssim), the two alternating, wall clock around a device synchronise; and evaluate_split's
  stages (rays / field / metrics) by CUDA events;
* on a synthetic 1080x1920 view: the two kernels alone by CUDA events over many launches, with the bytes they must read
  (stats: rgb, image, logit, accumulation, mask = 36 B per pixel; SSIM: the two images = 24 B per pixel, each read once)
  over their time as a share of the H100 SXM data sheet's 3.35 TB/s of HBM3, next to the same scores computed by
  image_metrics on host tensors as the pipeline method does.

The model is freshly initialised: the sample counts per ray are fixed, so the cost does not depend on training.

    python tools/bench_eval.py [--image-size 256] [--num-images 20] [--repeats 3] [--launches 50]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from bench_render import gpu_info  # noqa: E402
from fruitnerf_b200 import evaluate as E  # noqa: E402
from fruitnerf_b200 import image_metrics as M  # noqa: E402
from fruitnerf_b200 import ops  # noqa: E402
from fruitnerf_b200.scripts.train import synthetic_spec  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
STATS_BYTES_PER_PIXEL, SSIM_BYTES_PER_PIXEL = 36, 24


def wall(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def bench_scene(a, dev) -> dict:
    torch.manual_seed(0)
    spec = synthetic_spec("fruit_nerf", num_images=a.num_images, image_size=a.image_size, num_fruits=5)
    pipeline = spec.pipeline.setup(device=dev, test_mode="test")
    pipeline.eval()
    n = len(pipeline.datamanager.eval_dataset)
    host = lambda: pipeline.get_average_eval_image_metrics()  # noqa: E731
    device = lambda: E.evaluate_split(pipeline)  # noqa: E731
    host(), device()  # warm-up: module loads, allocator, every chunk shape
    times = {"host": [], "device": []}
    for _ in range(a.repeats):
        times["host"].append(wall(host))
        times["device"].append(wall(device))
    events = []

    def on_stage(name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append((name, e))

    E.evaluate_split(pipeline, on_stage=on_stage)
    torch.cuda.synchronize()
    ms = defaultdict(float)
    for (name, e0), (_, e1) in zip(events, events[1:]):
        if name != "done":
            ms[name] += e0.elapsed_time(e1)
    best = {k: min(v) for k, v in times.items()}
    return {"images": n, "size": f"{a.image_size}x{a.image_size}", "repeats": a.repeats,
            "seconds_per_image": {k: [round(t / n, 5) for t in v] for k, v in times.items()},
            "best_seconds_per_image": {k: round(t / n, 5) for k, t in best.items()},
            "host_over_device": round(best["host"] / best["device"], 3),
            "evaluate_split_ms_per_image": {k: round(v / n, 3) for k, v in ms.items()}}


def time_launches(fn, launches: int) -> float:
    """Mean milliseconds per call by CUDA events around ``launches`` back-to-back calls."""
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def bench_kernels(a, dev) -> dict:
    H, W = a.height, a.width
    P = H * W
    g = torch.Generator().manual_seed(0)
    image = torch.rand(H, W, 3, generator=g)
    rgb = (image + 0.1 * torch.randn(H, W, 3, generator=g)).reshape(-1, 3).contiguous()
    sem, acc = torch.randn(P, 1, generator=g) * 4, torch.rand(P, 1, generator=g)
    mask = (torch.rand(H, W, 1, generator=g) > 0.6).float()
    d = [t.to(dev) for t in (rgb, sem, acc, image, mask)]
    record = torch.zeros(ops.L.FNR_IMAGE_RECORD_DOUBLES, dtype=torch.float64, device=dev)
    scratch = ops.image_metrics_scratch(H, W, dev)
    stats_ms = time_launches(lambda: ops.image_stats(*d, record, scratch), a.launches)
    ssim_ms = time_launches(lambda: ops.image_ssim(d[0], d[3], record, scratch), a.launches)

    def host_scores():  # what image_metrics_and_images computes per image, on host tensors as the pipeline method holds them
        im, pr = torch.moveaxis(image, -1, 0)[None], torch.moveaxis(rgb.reshape(H, W, 3).clamp(0, 1), -1, 0)[None]
        return float(M.psnr(im, pr)), float(M.ssim(im, pr)), float(M.binary_jaccard((torch.sigmoid(sem) > 0.9).reshape(H, W), mask[..., 0]))

    host_scores()
    t0 = time.perf_counter()
    for _ in range(3):
        psnr, ssim, _ = host_scores()
    host_ms = (time.perf_counter() - t0) / 3 * 1e3
    got = dict(zip(ops.L.IMAGE_RECORD_FIELDS, record.cpu().tolist()))
    share = lambda nbytes, ms: round(nbytes * P / (ms * 1e-3) / HBM_BYTES_PER_S, 4)  # noqa: E731
    return {"size": f"{W}x{H}", "launches": a.launches,
            "image_stats": {"ms": round(stats_ms, 4), "bytes": STATS_BYTES_PER_PIXEL * P, "share_of_3.35TB/s": share(STATS_BYTES_PER_PIXEL, stats_ms)},
            "ssim": {"ms": round(ssim_ms, 4), "bytes": SSIM_BYTES_PER_PIXEL * P, "share_of_3.35TB/s": share(SSIM_BYTES_PER_PIXEL, ssim_ms)},
            "host_scores_ms": round(host_ms, 2), "ssim_device_minus_host": got["ssim"] - ssim}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--image-size", type=int, default=256)
    ap.add_argument("--num-images", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval needs a CUDA device: nothing here can be timed without one")
    dev = torch.device("cuda:0")
    res = {"metric": "eval_seconds_per_image", **gpu_info(), "scene": bench_scene(a, dev), "kernels": bench_kernels(a, dev)}
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
