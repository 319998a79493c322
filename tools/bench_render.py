"""Frames per second of the `render` command: a 1920x1080 `interpolate` path of fruit_nerf at the eval sample counts
(proposal 256 / 96, field 48 per ray), with ray generation (fnr_camera_rays), the model forward (proposal sampler +
fnr_render_forward) and composition (fnr_compose_frame + the one device-to-host copy) timed with CUDA events.

The model is freshly initialised on the synthetic scene: the sample counts per ray are fixed, so the rate does not depend
on training.  Frames go to a null sink (encoding runs on a writer thread in the CLI and is not part of this figure).

    python tools/bench_render.py [--frames 4] [--warmup 1] [--chunk 32768] [--outputs rgb depth semantics_colormap]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from fruitnerf_b200 import render as R  # noqa: E402
from fruitnerf_b200.scripts.train import synthetic_spec  # noqa: E402


def gpu_info() -> dict:
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable ({e})"
    return info


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chunk", type=int, default=32768)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--outputs", nargs="+", default=["rgb", "depth", "semantics_colormap"])
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_render needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    spec = synthetic_spec("fruit_nerf", num_images=20, image_size=64, num_fruits=5)
    pipeline = spec.pipeline.setup(device=dev, test_mode="inference")
    pipeline.eval()
    src = R.CameraSet.from_cameras(pipeline.datamanager.train_dataset.cameras, [0, 1])
    s = a.width / src.width
    src = R.CameraSet(src.camera_to_worlds, src.fx * s, src.fy * s, a.width / 2.0, a.height / 2.0, a.height, a.width)
    steps = a.frames + a.warmup
    path = R.get_interpolated_camera_path(src, steps, False)
    path = R.CameraSet(path.camera_to_worlds, path.fx, path.fy, path.cx, path.cy, a.height, a.width)
    warm = R.CameraSet(path.camera_to_worlds[:a.warmup], path.fx[:a.warmup], path.fy[:a.warmup], path.cx[:a.warmup], path.cy[:a.warmup],
                       a.height, a.width)
    timed = R.CameraSet(path.camera_to_worlds[a.warmup:], path.fx[a.warmup:], path.fy[a.warmup:], path.cx[a.warmup:], path.cy[a.warmup:],
                        a.height, a.width)
    sink = lambda frame: None  # noqa: E731
    R.render_frames(pipeline, warm, a.outputs, a.chunk, sink=sink)
    torch.cuda.synchronize()

    events = []  # (stage, event) in launch order

    def on_stage(name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append((name, e))

    t0 = time.perf_counter()
    R.render_frames(pipeline, timed, a.outputs, a.chunk, sink=sink, on_stage=on_stage)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ms = defaultdict(float)
    for (name, e0), (_, e1) in zip(events, events[1:]):
        if name != "done":
            ms[name] += e0.elapsed_time(e1)
    n = len(timed)
    rays = n * a.width * a.height
    res = {
        "metric": "render_frames_per_s", "value": round(n / wall, 4), "frames": n, "size": f"{a.width}x{a.height}", "outputs": a.outputs,
        "chunk": a.chunk, "rays_per_s": round(rays / wall, 1),
        "ms_per_frame": {"total_wall": round(1000 * wall / n, 2), **{k: round(v / n, 3) for k, v in ms.items()}},
        **gpu_info(),
    }
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
