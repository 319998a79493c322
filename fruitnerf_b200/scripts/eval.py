"""``ns-eval`` for this package's run folders: ``python -m fruitnerf_b200.scripts.eval --load-config RUN/config.yml
--output-path eval.json``.

nerfstudio 0.3.2's ``ns-eval`` (``ComputePSNR``) loads a run, averages the image metrics over its held-out views and
writes ``{"experiment_name", "method_name", "checkpoint", "results"}``.  Same option names, parsed with argparse (tyro is
not available offline).  The views are rendered and scored on the GPU (``evaluate.evaluate_split``; fnr_image_stats,
fnr_ssim).  Beyond ns-eval: ``--split train`` scores the training views, ``--per-image`` adds the per-image rows under
``"per_image"``, ``--num-rays-per-chunk`` overrides the model's chunk size.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="ns-eval")
    ap.add_argument("--load-config", type=Path, required=True, help="a run folder's config.yml")
    ap.add_argument("--output-path", type=Path, default=Path("output.json"), help="the JSON file to write")
    ap.add_argument("--render-output-path", type=Path, default=None, help="also write every evaluation image into this folder")
    ap.add_argument("--split", choices=("eval", "train"), default="eval")
    ap.add_argument("--per-image", action="store_true", help="add the per-image rows to the JSON")
    ap.add_argument("--num-rays-per-chunk", type=int, default=None)
    return ap


def experiment_name(config, config_path: Path) -> str:
    """nerfstudio lays runs out as outputs/<experiment_name>/<method_name>/<timestamp>/config.yml; a run folder that is
    not under a folder named after its method goes by its own name."""
    name = getattr(config, "experiment_name", None)
    if name:
        return str(name)
    run = Path(config_path).resolve().parent
    return run.parent.parent.name if run.parent.name == config.method_name and run.parent.parent.name else run.name


def refuse(message: str) -> None:
    print(f"error: {message}", file=sys.stderr)
    sys.exit(1)


def main(args: argparse.Namespace, pipeline=None, config=None, checkpoint_path=None) -> dict:
    """Evaluate and write the JSON; returns what was written.  ``pipeline``, ``config``, ``checkpoint_path``: an already
    loaded run (else ``eval_setup(load_config)``)."""
    if Path(args.output_path).suffix != ".json":  # ns-eval asserts this before it renders anything
        refuse(f"--output-path must end in .json, got {args.output_path}")
    if pipeline is None:
        if not Path(args.load_config).is_file():
            refuse(f"no config at {args.load_config}: pass a run folder's config.yml")
        import torch

        if not torch.cuda.is_available():
            refuse("ns-eval needs a CUDA device: the views are rendered and scored by CUDA kernels, and there is no CPU path")
        from .exporter import eval_setup

        config, pipeline, checkpoint_path, _ = eval_setup(args.load_config, eval_num_rays_per_chunk=args.num_rays_per_chunk)
    if pipeline.device.type != "cuda":
        refuse("ns-eval needs the pipeline on a CUDA device: the views are rendered and scored by CUDA kernels, and there is no CPU path")
    ds = pipeline.datamanager.eval_dataset if args.split == "eval" else pipeline.datamanager.train_dataset
    if ds is None or len(ds) == 0:
        refuse(f"the run has no {args.split} split to evaluate" + ("; --split train scores the training views" if args.split == "eval" else ""))
    from ..evaluate import evaluate_split

    scores = evaluate_split(pipeline, split=args.split, num_rays_per_chunk=args.num_rays_per_chunk, render_output_path=args.render_output_path)
    out = {
        "experiment_name": experiment_name(config, args.load_config),
        "method_name": config.method_name,
        "checkpoint": str(checkpoint_path),
        "results": scores["results"],
    }
    if args.per_image:
        out["per_image"] = scores["per_image"]
    Path(args.output_path).parent.mkdir(parents=True, exist_ok=True)
    Path(args.output_path).write_text(json.dumps(out, indent=2))
    print(f"evaluated {len(scores['per_image'])} {args.split} images -> {args.output_path}")
    return out


def entrypoint(argv=None, pipeline=None, config=None, checkpoint_path=None) -> dict:
    return main(build_parser().parse_args(argv), pipeline, config, checkpoint_path)


if __name__ == "__main__":
    entrypoint()
