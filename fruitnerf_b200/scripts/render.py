"""``ns-render`` for this package's run folders: ``python -m fruitnerf_b200.scripts.render {camera-path,interpolate,spiral}``.

The reference ships a launcher for nerfstudio 0.3.2's ``ns-render`` (debug/render.py).  Same subcommands, option names and
defaults, parsed with argparse (tyro is not available offline); the semantics are restated in ``fruitnerf_b200.render``
and DESIGN section 4.3i.  Frames are rendered and colour-mapped on the GPU (fnr_camera_rays, fnr_compose_frame) and
written as images or piped into ``ffmpeg``.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path
from typing import Optional

from .. import render as R


def add_common(p: argparse.ArgumentParser) -> None:
    """BaseRender's fields."""
    p.add_argument("--load-config", type=Path, required=True, help="a run folder's config.yml")
    p.add_argument("--output-path", type=Path, default=Path("renders/output.mp4"))
    p.add_argument("--image-format", choices=("jpeg", "png"), default="jpeg")
    p.add_argument("--jpeg-quality", type=int, default=100)
    p.add_argument("--downscale-factor", type=float, default=1.0)
    p.add_argument("--eval-num-rays-per-chunk", type=int, default=None)
    p.add_argument("--rendered-output-names", nargs="+", default=["rgb"])
    p.add_argument("--depth-near-plane", type=float, default=None)
    p.add_argument("--depth-far-plane", type=float, default=None)
    p.add_argument("--output-format", choices=("images", "video"), default="video")


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="ns-render")
    sub = ap.add_subparsers(dest="command", required=True)
    p = sub.add_parser("camera-path", help="render a viewer camera-path file")
    add_common(p)
    p.add_argument("--camera-path-filename", type=Path, default=Path("camera_path.json"))
    p = sub.add_parser("interpolate", help="render a path interpolated between the data set's cameras")
    add_common(p)
    p.add_argument("--pose-source", choices=("eval", "train"), default="eval")
    p.add_argument("--interpolation-steps", type=int, default=10)
    p.add_argument("--order-poses", action=argparse.BooleanOptionalAction, default=False)
    p.add_argument("--frame-rate", type=int, default=24)
    p = sub.add_parser("spiral", help="render a spiral around the first eval camera")
    add_common(p)
    p.add_argument("--seconds", type=float, default=3.0)
    p.add_argument("--frame-rate", type=int, default=24)
    p.add_argument("--radius", type=float, default=0.1)
    return ap


def check_output_names(names, available) -> None:
    """ns-render's check: a requested name the model does not output prints the available keys and exits with 1."""
    for name in names:
        if name not in available:
            print(f"Error: could not find {name} in the model outputs", file=sys.stderr)
            print(f"Please set --rendered-output-names to one of: {list(available)}", file=sys.stderr)
            sys.exit(1)


def main(args: argparse.Namespace, pipeline=None) -> R.FrameWriter:
    """Run one subcommand.  ``pipeline``: an already loaded pipeline (else ``eval_setup(load_config, test_mode="inference")``)."""
    if args.output_format == "video":
        R.require_ffmpeg()  # before anything is loaded or rendered
    path_json = None
    if args.command == "camera-path":
        path_json = json.loads(Path(args.camera_path_filename).read_text())
        R.get_path_from_json(path_json)  # refusals before the model is loaded
    if pipeline is None:
        from .exporter import eval_setup

        _, pipeline, _, _ = eval_setup(args.load_config, eval_num_rays_per_chunk=args.eval_num_rays_per_chunk, test_mode="inference")
    dm = pipeline.datamanager
    if args.command == "camera-path":
        cameras = R.get_path_from_json(path_json)
        fps = R.path_fps(path_json, len(cameras))
    elif args.command == "interpolate":
        ds = dm.eval_dataset if args.pose_source == "eval" else dm.train_dataset
        source = R.CameraSet.from_cameras(ds.cameras)
        cameras = R.get_interpolated_camera_path(source, args.interpolation_steps, args.order_poses)
        fps = len(cameras) / (args.interpolation_steps * len(source) / args.frame_rate)  # ns-render: seconds = steps * N / rate
    else:
        steps = int(args.frame_rate * args.seconds)
        cameras = R.get_spiral_path(R.CameraSet.from_cameras(dm.eval_dataset.cameras, [0]), 0, steps=steps, radius=args.radius)
        fps = len(cameras) / args.seconds
    cameras = cameras.rescale_output_resolution(1.0 / args.downscale_factor)
    check_output_names(args.rendered_output_names, R.probe_outputs(pipeline.model))
    writer = R.FrameWriter(args.output_path, args.output_format, args.image_format, args.jpeg_quality, fps)
    try:
        R.render_frames(pipeline, cameras, args.rendered_output_names, args.eval_num_rays_per_chunk, args.depth_near_plane, args.depth_far_plane,
                        sink=writer)
    finally:
        writer.close()
    where = writer.image_dir if args.output_format == "images" else args.output_path
    print(f"rendered {writer.count} frames of {cameras.width}x{cameras.height} -> {where}")
    return writer


def entrypoint(argv=None, pipeline=None) -> R.FrameWriter:
    return main(build_parser().parse_args(argv), pipeline)


if __name__ == "__main__":
    entrypoint()
