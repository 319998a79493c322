"""Held-out evaluation of a trained model with nothing leaving the device until the end (the `eval` command, nerfstudio
``ns-eval``; DESIGN section 4.3o).

``FruitPipeline.get_average_eval_image_metrics`` copies every output of every chunk to the host and scores the image
there, as upstream does.  ``evaluate_split`` renders each image of a split into device buffers (the chunk loop of
``render.render_frames``), scores it with two kernels (``ops.image_stats``, ``ops.image_ssim``) into one row of an
[N, 12] record tensor, times it with a pair of CUDA events, and copies the records and the times once.  Same keys and
meaning as the pipeline method, plus per-image rows, precision / recall beside ``fruit_iou`` and the pooled IoU.
"""
from __future__ import annotations

import math
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence

import torch
from torch import Tensor

from . import ops
from ._lib import IMAGE_RECORD_FIELDS
from .image_metrics import _turbo_table, binary_jaccard
from .render import probe_outputs, render_into_buffers

# per-image keys whose mean over the split is reported (the others are integers)
MEAN_KEYS = ("psnr", "ssim", "iou", "fruit_iou", "fruit_precision", "fruit_recall", "mean_accumulation", "num_rays_per_sec", "fps")


def _ratio(num: float, den: float, empty: float) -> float:
    return num / den if den > 0 else empty


def image_row(image_idx: int, num_rays: int, record: Sequence[float], iou: float, seconds: float) -> Dict:
    """One image's scores from its record (slots ``_lib.IMAGE_RECORD_FIELDS``), the reference's ``iou`` and its time."""
    r = dict(zip(IMAGE_RECORD_FIELDS, (float(v) for v in record)))
    mse = r["sse"] / (3 * num_rays)
    tp, fp, fn = int(r["fruit_tp"]), int(r["fruit_fp"]), int(r["fruit_fn"])
    rate = num_rays / max(seconds, 1e-9)
    return {
        "image_idx": int(image_idx),
        "num_rays": int(num_rays),
        "psnr": math.inf if mse == 0 else (10.0 * math.log10(1.0 / mse) if mse > 0 else math.nan),  # torch: 10 log10(1 / 0) = inf
        "ssim": r["ssim"],
        "iou": float(iou),
        "fruit_iou": _ratio(tp, tp + fp + fn, 1.0),  # an empty prediction of an empty mask agrees
        "fruit_precision": _ratio(tp, tp + fp, 0.0),
        "fruit_recall": _ratio(tp, tp + fn, 0.0),
        "fruit_tp": tp,
        "fruit_fp": fp,
        "fruit_fn": fn,
        "mean_accumulation": r["accumulation_sum"] / num_rays,
        "num_rays_per_sec": rate,
        "fps": rate / num_rays,
    }


def aggregate(rows: List[Dict]) -> Dict[str, float]:
    """The mean of every float key over the images (``get_average_eval_image_metrics``'s keys among them) and
    ``fruit_iou_pooled``, the IoU of the confusion counts summed over the split."""
    if not rows:
        raise ValueError("no images to aggregate")
    out = {k: float(sum(r[k] for r in rows) / len(rows)) for k in MEAN_KEYS}
    tp, fp, fn = (sum(r[k] for r in rows) for k in ("fruit_tp", "fruit_fp", "fruit_fn"))
    out["fruit_iou_pooled"] = _ratio(tp, tp + fp + fn, 1.0)
    return out


def _eval_image_arrays(bufs: Dict[str, Tensor], image: Tensor, mask: Tensor, num_proposal_iterations: int, H: int, W: int, turbo: Tensor,
                       scratch: Tensor) -> Dict[str, Tensor]:
    """uint8 device images under the keys of ``image_metrics.image_metrics_and_images``: ``img`` is the photograph and
    the render side by side."""
    acc = bufs["accumulation"]
    depth_keys = ["depth"] + [f"prop_depth_{i}" for i in range(num_proposal_iterations) if f"prop_depth_{i}" in bufs]
    frames = {"img": [ops.FrameImage(image.reshape(-1, 3), "color"), ops.FrameImage(bufs["rgb"], "color")],
              "accumulation": [ops.FrameImage(acc, "turbo")]}
    for key in depth_keys:
        frames[key] = [ops.FrameImage(bufs[key], "depth")]
    frames["semantics_colormap"] = [ops.FrameImage(torch.sigmoid(bufs["semantics"]).expand(-1, 3).contiguous(), "color")]
    frames["fruit_mask"] = [ops.FrameImage(mask.reshape(-1, 1).expand(-1, 3).contiguous(), "color")]
    return {key: ops.compose_frame(images, acc, H, W, turbo, scratch) for key, images in frames.items()}


@torch.no_grad()
def evaluate_split(pipeline, split: str = "eval", num_rays_per_chunk: Optional[int] = None, render_output_path=None,
                   on_stage: Optional[Callable[[str], None]] = None) -> Dict:
    """Render and score every image of ``split`` ("eval", or "train": the training images with their own camera indices;
    as everywhere in eval mode the field takes the mean or zero appearance embedding, not a per-image one).  Returns
    ``{"results": means, "per_image": rows}`` (``aggregate``, ``image_row``).  Rays come from the data set's own cameras
    as ``next_eval_image`` makes them; the images are visited in index order and the datamanager's ``eval_count`` is
    left alone.  ``render_output_path``: also write ``<idx:06d>-<key>.jpg`` for the images ``_save_eval_images`` writes
    (one device-to-host copy per file, outside the image's timed span).  ``on_stage(name)`` is called as each stage
    ("rays", "field", "metrics") of an image starts and with "done" at its end (benchmark timing hooks).  The pipeline's
    and the model's training flags are restored on exit."""
    if split not in ("eval", "train"):
        raise ValueError(f"split must be 'eval' or 'train', got {split!r}")
    model = pipeline.model
    dev = model.device
    if dev.type != "cuda":
        raise RuntimeError("evaluate_split needs the model on a CUDA device: the image scores are CUDA kernels")
    ds = pipeline.datamanager.eval_dataset if split == "eval" else pipeline.datamanager.train_dataset
    if ds is None or len(ds) == 0:
        raise ValueError(f"the pipeline has no {split} images")
    cams = ds.cameras
    H, W = cams.height, cams.width
    P, N = H * W, len(ds)
    chunk = int(num_rays_per_chunk or model.config.eval_num_rays_per_chunk)
    nprop = model.config.num_proposal_iterations
    stage = on_stage or (lambda _name: None)
    needed = ["rgb", "semantics", "accumulation"]
    if render_output_path is not None:
        out_dir = Path(render_output_path)
        out_dir.mkdir(parents=True, exist_ok=True)
        turbo = _turbo_table(dev)
        compose_scratch = torch.empty(ops.L.FNR_COMPOSE_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
    records = torch.zeros((N, ops.L.FNR_IMAGE_RECORD_DOUBLES), dtype=torch.float64, device=dev)
    ious = torch.zeros(N, dtype=torch.float32, device=dev)
    scratch = ops.image_metrics_scratch(H, W, dev)
    events = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(N)]
    bufs: Dict[str, Tensor] = {}
    was_pipeline, was_model = pipeline.training, model.training
    pipeline.eval()
    try:
        if render_output_path is not None:
            available = probe_outputs(model)
            needed += ["depth"] + [f"prop_depth_{k}" for k in range(nprop) if f"prop_depth_{k}" in available]
        for i in range(N):
            events[i][0].record()
            stage("rays")
            bundle = cams.generate_rays(i)
            image = ds.images[i].to(dev, torch.float32).contiguous()
            mask = ds.fruit_masks[i].to(dev, torch.float32).contiguous()
            render_into_buffers(model, lambda p0, n: bundle.get_row_major_sliced_ray_bundle(p0, p0 + n), P, chunk, needed, bufs, stage)
            stage("metrics")
            ops.image_stats(bufs["rgb"], bufs["semantics"], bufs["accumulation"], image, mask, records[i], scratch)
            ops.image_ssim(bufs["rgb"], image, records[i], scratch)
            # the reference's `iou` (softmax over the image rows, image_metrics.py) for parity of the keys
            ious[i] = binary_jaccard(torch.softmax(bufs["semantics"].view(H, W, 1), dim=0)[..., 0], mask.view(H, W))
            events[i][1].record()
            if render_output_path is not None:
                from PIL import Image

                arrays = _eval_image_arrays(bufs, image, mask, nprop, H, W, turbo, compose_scratch)
                for key, arr in arrays.items():
                    Image.fromarray(arr.cpu().numpy()).save(out_dir / f"{i:06d}-{key}.jpg")
            stage("done")
        torch.cuda.synchronize(dev)
    finally:
        pipeline.train(was_pipeline)
        model.train(was_model)
    rec, iou = records.cpu().tolist(), ious.cpu().tolist()
    rows = [image_row(i, P, rec[i], iou[i], events[i][0].elapsed_time(events[i][1]) / 1e3) for i in range(N)]
    return {"results": aggregate(rows), "per_image": rows}
