"""Device time of the render forward (`fnr_render_forward`: field forward + compositing) alone, at the bench.py shape
(4096 rays x 192 samples, the bench.py field and batch), in training mode (the encoding stash written for the backward)
and in inference mode.

    python tools/bench_forward.py [--variant small|big] [--kernel auto|simt|tcgen05] [--steps 20] [--kernels] [--lib FILE]
                                  [--no-gather [--build-dir DIR]] [--json FILE]

Each timed call is one `ops.render` (output allocation + the library call), CUDA events around it, the L2 flushed before
every call as bench.py does.  `--kernels` then runs the same calls again under torch.profiler, in a run of their own after
the timed one, and adds the device time of each kernel of the forward per call (field forward and compositing).  `--lib`
times another build of the library (the C ABI is the same).  `--no-gather` builds the library with -DFNR_FWD_NO_GATHER into
--build-dir (a temporary directory by default, never the package's own library) and times that: fruit_nerf's
tensor-core forward and export then make up their encodings instead of gathering them from the hash table, so the
difference to the normal build is the most that hiding the gather could save.  Its outputs are meaningless.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from tools.bench_backward import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="small", choices=["small", "big"])
    ap.add_argument("--kernel", default="auto", choices=["auto", "simt", "tcgen05"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true", help="device time per kernel from a torch.profiler run after the timed one")
    ap.add_argument("--lib", default=None, help="library to time (default: the package's)")
    ap.add_argument("--no-gather", action="store_true", help="time a -DFNR_FWD_NO_GATHER build (diagnostic)")
    ap.add_argument("--build-dir", default=None, help="where --no-gather builds its library (default: a temporary directory)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    from fruitnerf_b200 import _lib as L

    tmp = None
    if args.no_gather:
        from fruitnerf_b200 import _build

        out = args.build_dir or (tmp := tempfile.TemporaryDirectory(prefix="fnr_no_gather_")).name
        L.LIB_PATH = _build.build(defines=["FNR_FWD_NO_GATHER"], out_dir=out)
    elif args.lib:
        L.LIB_PATH = Path(args.lib).resolve()
    L.load()

    import bench
    from fruitnerf_b200 import ops
    from fruitnerf_b200 import synthetic as syn

    impl = {"auto": L.FNR_IMPL_AUTO, "simt": L.FNR_IMPL_SIMT, "tcgen05": L.FNR_IMPL_TCGEN05}[args.kernel]
    dev = torch.device("cuda", 0)
    field = bench.build_field(args.variant, dev)
    o, d, s, e, cam = (t.to(dev) for t in syn.ray_batch(bench.R_RAYS, bench.S_SAMPLES, salt=0, num_images=bench.NUM_IMAGES))
    cam = cam.to(torch.int32)
    params = field.kernel_params()
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)

    def forward(train: bool):
        # training mode: parameters that need gradients, so the forward writes the encoding stash
        with torch.set_grad_enabled(train):
            return ops.render(field.kernel_shape(), params, o, d, s, e, cam, field.position_mode(), field.appearance_mode(), impl=impl)

    res = {"variant": args.variant, "kernel": args.kernel, "lib": str(L.LIB_PATH), "rays": bench.R_RAYS, "samples": bench.S_SAMPLES,
           "steps": args.steps}
    for mode, train in (("train", True), ("inference", False)):
        for _ in range(args.warmup):
            forward(train)
        torch.cuda.synchronize()
        ms = []
        for i in range(args.steps):
            flush.fill_(float(i))
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = forward(train)
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
            del out
        res[f"{mode}_ms_median"], res[f"{mode}_ms_min"], res[f"{mode}_ms_max"] = statistics.median(ms), min(ms), max(ms)
    if args.kernels:
        from torch.profiler import ProfilerActivity, profile

        for mode, train in (("train", True), ("inference", False)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(args.steps):
                    flush.fill_(float(i))
                    forward(train)
                torch.cuda.synchronize()
            per_kernel = {ka.key: ka.self_device_time_total / 1e3 for ka in prof.key_averages() if "fnr::" in ka.key}  # the library's kernels
            res[f"{mode}_kernel_ms_per_call"] = {k: round(v / args.steps, 4) for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1])}
    res["card"] = card()
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
