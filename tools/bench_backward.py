"""Device time of the render backward (`fnr_render_backward`: compositing backward + field backward) alone, at the
bench.py shape (4096 rays x 192 samples, the bench.py field and batch), and optionally its split into phases.

    python tools/bench_backward.py [--variant small|big] [--steps 20] [--phases] [--build-dir DIR] [--json FILE]

Each timed call is the autograd backward of `ops.render` (zeroing of the flat gradient buffer + the library call), CUDA
events around it, the L2 flushed before every call as bench.py does.  `--phases` builds the library with
-DFNR_BWD_PHASE_TIMERS into --build-dir (a temporary directory by default, never the package's own library), and
prints the clock64() cycles per 128-point tile of every phase of the field backward kernel: stash / upstream loads,
forward recompute, dx, dW, the dW flush to the global gradient, and the hash-table scatter.  The phase marks
synchronise the CTA, so the timer build is a little slower than the normal one; its split is what it is for.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

PHASES = ("load", "recompute", "dx", "dw", "dw_flush", "scatter")  # enum BwdPhase of fnr_wgmma.cuh


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_max_sm_clock_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["power_limit_max_sm_clock_sm_clock"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="small", choices=["small", "big"])
    ap.add_argument("--kernel", default="auto", choices=["auto", "simt", "tcgen05"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--phases", action="store_true", help="per-phase cycles from a -DFNR_BWD_PHASE_TIMERS build")
    ap.add_argument("--build-dir", default=None, help="where --phases builds its library (default: a temporary directory)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    from fruitnerf_b200 import _lib as L

    tmp = None
    if args.phases:
        from fruitnerf_b200 import _build

        out = args.build_dir or (tmp := tempfile.TemporaryDirectory(prefix="fnr_phases_")).name
        L.LIB_PATH = _build.build(defines=["FNR_BWD_PHASE_TIMERS"], out_dir=out)
    lib = L.load()

    import bench
    from fruitnerf_b200 import ops
    from fruitnerf_b200 import synthetic as syn

    impl = {"auto": L.FNR_IMPL_AUTO, "simt": L.FNR_IMPL_SIMT, "tcgen05": L.FNR_IMPL_TCGEN05}[args.kernel]
    dev = torch.device("cuda", 0)
    field = bench.build_field(args.variant, dev)
    o, d, s, e, cam = (t.to(dev) for t in syn.ray_batch(bench.R_RAYS, bench.S_SAMPLES, salt=0, num_images=bench.NUM_IMAGES))
    params = field.kernel_params()
    out = ops.render(field.kernel_shape(), params, o, d, s, e, cam.to(torch.int32), field.position_mode(),
                     field.appearance_mode(), impl=impl)
    node = out["rgb"].grad_fn  # the _Render node: its backward is one fnr_render_backward call
    gen = torch.Generator(device=dev).manual_seed(0)
    g_rgb = torch.randn(out["rgb"].shape, device=dev, generator=gen) * 1e-3
    g_sem = torch.randn(out["semantics"].shape, device=dev, generator=gen) * 1e-3
    grads = (g_rgb, None, None, None, g_sem, None, None, None, None)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)

    def backward():
        ops._Render.backward(node, *grads)

    for _ in range(args.warmup):
        backward()
    torch.cuda.synchronize()
    if args.phases:
        lib.fnr_bwd_phase_cycles(ctypes.cast(ctypes.create_string_buffer(8 * len(PHASES)), ctypes.POINTER(ctypes.c_uint64)))
    ms = []
    for i in range(args.steps):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        backward()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    res = {"variant": args.variant, "kernel": args.kernel, "rays": bench.R_RAYS, "samples": bench.S_SAMPLES,
           "render_backward_ms_median": statistics.median(ms), "render_backward_ms_min": min(ms),
           "render_backward_ms_max": max(ms), "steps": args.steps, "card": card()}
    if args.phases:
        buf = (ctypes.c_uint64 * len(PHASES))()
        if lib.fnr_bwd_phase_cycles(buf) != 0:
            raise RuntimeError("fnr_bwd_phase_cycles failed")
        tiles = args.steps * ((bench.R_RAYS * bench.S_SAMPLES + 127) // 128)
        per_tile = {p: buf[i] / tiles for i, p in enumerate(PHASES)}
        res["phase_cycles_per_tile"] = {p: round(v) for p, v in per_tile.items()}
        res["phase_cycles_per_tile_total"] = round(sum(per_tile.values()))
        res["note"] = ("phase timer build (CTA barrier at every mark): cycles of thread 0 of each CTA per 128-point tile, "
                       "CTAs sharing an SM overlap")
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
