"""``ns-train fruit_nerf`` on the synthetic apple scene, end to end (BASELINE.json configs[1]; SURVEY.md 8f ranks 3-4):
train -> held-out PSNR / fruit IoU -> uniform-volume export -> fruit count.  (The cross-check of a trained model
against the CPU oracle lives in tests/test_gpu_training.py: the product never imports the oracle.)

    python -m fruitnerf_b200.scripts.train --steps 3000 --json gpurun_out/train_synthetic.json
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import time
from typing import Dict, Optional

import numpy as np
import torch

from ..clustering import count_fruits
from ..export.exporter_utils import sample_volume
from ..fruit_nerf_config import METHODS
from ..trainer import Trainer


def synthetic_spec(method: str = "fruit_nerf", num_images: int = 40, image_size: int = 160, num_fruits: int = 12, seed: int = 0,
                   rays_per_batch: Optional[int] = None, schedule_steps: Optional[int] = None):
    """The method's TrainerSpec pointed at the synthetic scene.  ``schedule_steps``: let the exponential learning-rate decay
    (1e-2 -> 1e-4) complete within a short run instead of the 200 000 steps of the stock schedule -- with a constant 1e-2,
    Adam(eps=1e-15) destabilises on this nearly noise-free scene after ~2-3 k iterations (DESIGN.md section 7)."""
    spec = copy.deepcopy(METHODS[method])
    if schedule_steps:
        for o in spec.optimizers.values():
            o["scheduler"] = {"type": "ExponentialDecay", "lr_final": 1e-4, "max_steps": int(schedule_steps)}
    dm = spec.pipeline.datamanager
    dm.synthetic_scene = dict(num_images=num_images, height=image_size, width=image_size, num_fruits=num_fruits, seed=seed)
    dm.seed = seed
    if rays_per_batch:
        dm.train_num_rays_per_batch = rays_per_batch
    return spec


def export_and_count(trainer: Trainer, points_per_side: int = 256, half_extent: float = 0.3) -> Dict:
    """Uniform-volume export of the semantic cloud (exporter_utils.sample_volume) and stages 1-2 of the clustering."""
    pipeline = trainer.pipeline
    model, dm = pipeline.model, pipeline.datamanager
    was_training = pipeline.training
    saved = (model.proposal_sampler, model.field.spatial_distortion, model.test_mode, dm.config.eval_num_rays_per_batch, dm.train_count)
    pipeline.eval()
    model.test_mode = "export"
    dm.config.eval_num_rays_per_batch = 32768
    dm.train_count = 0
    model.setup_inference(render_rgb=True, num_inference_samples=points_per_side)
    lo, hi = (-half_extent,) * 3, (half_extent,) * 3
    num_rays = dm.setup_inference(aabb=(lo, hi), num_points=points_per_side)
    torch.cuda.synchronize()
    t0 = time.time()
    clouds = sample_volume(pipeline, num_rays, transform_json={"scale": trainer.pipeline.datamanager.train_dataset.dataparser_scale})
    torch.cuda.synchronize()
    export_s = time.time() - t0
    model.proposal_sampler, model.field.spatial_distortion, model.test_mode, dm.config.eval_num_rays_per_batch, dm.train_count = saved
    pipeline.train(was_training)
    pts = clouds["semantic_colormap"]["points"]
    h = 2.0 * (2 * half_extent) / (points_per_side - 1)  # grid spacing after the exporter's scale(2)
    geom = dm.train_dataset.geometry
    res = count_fruits(torch.from_numpy(pts).to(trainer.device), eps=2.5 * h, min_samples=8,
                       cluster_merge_distance=geom.fruit_radius if geom is not None else 0.04)
    out = {"export_seconds": export_s, "export_points": int(num_rays * points_per_side),
           "cloud_sizes": {k: int(v["points"].shape[0]) for k, v in clouds.items()}, "fruit_count": res["count"],
           "fruit_count_before_merge": res["count_before_merge"]}
    if geom is not None:
        gt = geom.fruit_centers.numpy()
        out["fruit_count_gt"] = int(gt.shape[0])
        if res["count"]:
            d = np.linalg.norm(res["centers"][:, None, :] - gt[None], axis=-1)
            out["matched_within_radius"] = int((d.min(axis=0) < 1.5 * geom.fruit_radius).sum())
            out["mean_center_error"] = float(d.min(axis=0).mean())
    return out


def phase_timing_ms(trainer: Trainer, iters: int = 20) -> Dict:
    """CUDA-event time of the pieces of a training iteration at the CURRENT state of the model (sample distribution
    matters: trained proposal networks concentrate samples on surfaces)."""
    pipe = trainer.pipeline
    names = ("batch", "forward", "loss", "backward", "optimizer")
    acc = {n: 0.0 for n in names}
    host0 = time.time()
    for _ in range(iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
        for params in trainer.param_groups.values():
            for p in params:
                p.grad = None
        ev[0].record()
        ray_bundle, batch = pipe.datamanager.next_train(trainer.step)
        ev[1].record()
        out = pipe.model(ray_bundle)
        ev[2].record()
        loss = sum(pipe.model.get_loss_dict(out, batch).values())
        ev[3].record()
        loss.backward()
        ev[4].record()
        for name, opt in trainer.optimizers.items():
            if all(p.grad is not None for p in trainer.param_groups[name]):
                opt.step()
        ev[5].record()
        torch.cuda.synchronize()
        for i, n in enumerate(names):
            acc[n] += ev[i].elapsed_time(ev[i + 1])
    out = {n: v / iters for n, v in acc.items()}
    out["wall_ms_per_iteration"] = 1e3 * (time.time() - host0) / iters
    return out


def train_synthetic(steps: int = 3000, method: str = "fruit_nerf", device: str = "cuda:0", log_every: int = 250, seed: int = 0,
                    image_size: int = 160, num_images: int = 40, num_fruits: int = 12, points_per_side: int = 256,
                    output_dir: Optional[str] = None, return_trainer: bool = False, eval_every: int = 500, phase_timing: bool = False, use_cuda_graph: bool = True,
                    short_schedule: bool = True):
    torch.manual_seed(seed)
    spec = synthetic_spec(method, num_images, image_size, num_fruits, seed, schedule_steps=steps if short_schedule else None)
    trainer = Trainer(spec, device=device, output_dir=output_dir, use_cuda_graph=use_cuda_graph)
    torch.cuda.synchronize()
    t0 = time.time()
    history = trainer.train(steps, log_every=log_every, eval_every=eval_every)
    torch.cuda.synchronize()
    train_s = time.time() - t0
    rays = spec.pipeline.datamanager.train_num_rays_per_batch
    res = {"method": method, "steps": steps, "lr_schedule": "1e-2 -> 1e-4 over the run" if short_schedule else "stock (200k steps)", "cuda_graph": bool(trainer.use_cuda_graph), "rays_per_batch": rays, "train_seconds": train_s, "train_rays_per_s": steps * rays / train_s,
           "ms_per_iteration": 1e3 * train_s / steps, "history": history,
           "scene": {"images": num_images, "size": image_size, "fruits": num_fruits}}
    if phase_timing:
        res["phase_ms"] = phase_timing_ms(trainer)
    res["eval"] = trainer.pipeline.get_average_eval_image_metrics(trainer.step)
    res["export"] = export_and_count(trainer, points_per_side)
    if output_dir:
        res["checkpoint"] = str(trainer.save_checkpoint())
    return (res, trainer) if return_trainer else res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--method", default="fruit_nerf", choices=sorted(METHODS))
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--image-size", type=int, default=160)
    ap.add_argument("--num-images", type=int, default=40)
    ap.add_argument("--num-fruits", type=int, default=12)
    ap.add_argument("--points-per-side", type=int, default=256)
    ap.add_argument("--output-dir", default=None)
    ap.add_argument("--stock-schedule", action="store_true", help="keep the 200k-step learning-rate decay of the method config")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-graph", action="store_true", help="enqueue every iteration op by op instead of replaying CUDA graphs")
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    res = train_synthetic(a.steps, a.method, image_size=a.image_size, num_images=a.num_images, num_fruits=a.num_fruits,
                          points_per_side=a.points_per_side, output_dir=a.output_dir, use_cuda_graph=not a.no_graph,
                          short_schedule=not a.stock_schedule, seed=a.seed)
    print(json.dumps({k: v for k, v in res.items() if k != "history"}))
    if a.json:
        os.makedirs(os.path.dirname(a.json) or ".", exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
