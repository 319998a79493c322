"""The `eval` command on the device: fnr_image_stats / fnr_ssim against their fp64 restatement and against image_metrics'
torch functions, evaluate_split against the pipeline's host evaluation on a briefly trained model, and the CLI on its run
folder."""
import json
import math

import numpy as np
import pytest
import torch

from fruitnerf_b200 import _lib, ops
from fruitnerf_b200 import evaluate as E
from fruitnerf_b200 import image_metrics as M

from .test_eval_host import make_view, torch_scores

pytestmark = pytest.mark.gpu

F = _lib.IMAGE_RECORD_FIELDS
EXACT = ("rgb_min", "rgb_max", "image_min", "image_max", "fruit_tp", "fruit_fp", "fruit_fn", "fruit_tn", "data_range")


def kernel_record(view, dev):
    rgb, sem, acc, image, mask = (t.to(dev) for t in view)
    rec = ops.image_stats(rgb, sem, acc, image, mask)
    ops.image_ssim(rgb, image, rec)
    return rec


def check_against_restatement(view, dev, ssim_vs_torch=1e-5):
    rec = kernel_record(view, dev)
    got = dict(zip(F, rec.cpu().tolist()))
    want = M.restated_image_scores(*view)
    for k in EXACT:
        assert got[k] == want[k], (k, got[k], want[k])
    for k in ("sse", "accumulation_sum", "ssim"):
        assert abs(got[k] - want[k]) <= 1e-6 * abs(want[k]), (k, got[k], want[k])
    rgb, sem, _, image, mask = view
    _, ssim, _ = torch_scores(rgb, sem, image, mask)
    assert abs(got["ssim"] - ssim) < ssim_vs_torch
    again = kernel_record(view, dev)
    assert torch.equal(rec.view(torch.int64), again.view(torch.int64))  # bit for bit
    return got


@pytest.mark.parametrize("H,W", [(11, 11), (37, 53), (480, 640), (1080, 1920)])
def test_kernels_match_the_restatement(native_lib, cuda_device, H, W):
    got = check_against_restatement(make_view(H, W, seed=H + W), cuda_device)
    assert got["fruit_tp"] + got["fruit_fp"] + got["fruit_fn"] + got["fruit_tn"] == H * W
    assert 0.5 < got["ssim"] < 1.0


def test_rgb_outside_the_unit_range_is_clamped(native_lib, cuda_device):
    got = check_against_restatement(make_view(64, 80, seed=3, noise=0.6, offset=0.3), cuda_device)
    assert got["rgb_min"] == 0.0 and got["rgb_max"] == 1.0


def test_constant_and_identical_images(native_lib, cuda_device):
    rgb, sem, acc, image, mask = make_view(48, 40, seed=4)
    # a constant render of a textured photograph
    check_against_restatement((torch.full_like(rgb, 0.25), sem, acc, image, mask), cuda_device)
    # the photograph itself: SSIM 1 in every window, zero squared error
    got = check_against_restatement((image.reshape(-1, 3).clone(), sem, acc, image, mask), cuda_device)
    assert abs(got["ssim"] - 1.0) < 1e-12 and got["sse"] == 0.0
    assert E.image_row(0, 48 * 40, [got[k] for k in F], 0.0, 1.0)["psnr"] == math.inf


@pytest.mark.parametrize("fill", [0.0, 1.0])
def test_all_fruit_and_no_fruit(native_lib, cuda_device, fill):
    rgb, sem, acc, image, mask = make_view(32, 45, seed=7)
    P = 32 * 45
    full_mask = torch.full_like(mask, fill)
    got = check_against_restatement((rgb, sem, acc, image, full_mask), cuda_device)
    assert (got["fruit_tp"] + got["fruit_fn"] == P) if fill else (got["fruit_tp"] + got["fruit_fn"] == 0)
    # the prediction empty (or full) as well
    logits = torch.full_like(sem, 8.0 if fill else -8.0)
    got = check_against_restatement((rgb, logits, acc, image, full_mask), cuda_device)
    row = E.image_row(0, P, [got[k] for k in F], 0.0, 1.0)
    assert row["fruit_iou"] == 1.0
    assert (got["fruit_tp"] == P) if fill else (got["fruit_tn"] == P)


def test_wrappers_refuse_bad_inputs(native_lib, cuda_device):
    view = make_view(16, 20)
    rgb, sem, acc, image, mask = (t.to(cuda_device) for t in view)
    with pytest.raises(_lib.FruitNerfNativeError, match="CUDA"):
        ops.image_stats(rgb.cpu(), sem, acc, image, mask)
    with pytest.raises(_lib.FruitNerfNativeError, match="CUDA"):
        ops.image_ssim(rgb, image.cpu(), torch.zeros(12, dtype=torch.float64, device=cuda_device))
    with pytest.raises(ValueError, match="rgb"):
        ops.image_stats(rgb[:-1], sem, acc, image, mask)
    with pytest.raises(ValueError, match="semantics"):
        ops.image_stats(rgb, sem.double(), acc, image, mask)
    with pytest.raises(ValueError, match="contiguous"):
        ops.image_stats(rgb, sem, acc, image.transpose(0, 1).contiguous().transpose(0, 1), mask)
    with pytest.raises(ValueError, match=r"\[H,W,3\]"):
        ops.image_stats(rgb, sem, acc, image.reshape(-1, 3), mask)
    with pytest.raises(ValueError, match="record"):
        ops.image_ssim(rgb, image, torch.zeros(12, device=cuda_device))
    small = make_view(11, 11)
    s_rgb, s_sem, s_acc, s_image, s_mask = (t.to(cuda_device) for t in small)
    rec = ops.image_stats(s_rgb[:110], s_sem[:110], s_acc[:110], s_image[:10].contiguous(), s_mask[:10].contiguous())  # stats have no size floor
    assert float(rec[6:10].sum()) == 110
    with pytest.raises(_lib.FruitNerfNativeError, match="smaller than the 11x11 window"):
        ops.image_ssim(s_rgb[:110], s_image[:10].contiguous(), rec)
    with pytest.raises(_lib.FruitNerfNativeError, match="scratch"):
        ops.image_ssim(rgb, image, ops.image_stats(rgb, sem, acc, image, mask), scratch=torch.empty(64, dtype=torch.uint8, device=cuda_device))


# ---- end to end -------------------------------------------------------------------------------------------------
def _tiny_spec(seed=0):  # as test_gpu_training.py
    from fruitnerf_b200.scripts.train import synthetic_spec

    spec = synthetic_spec("fruit_nerf", num_images=20, image_size=64, num_fruits=5, seed=seed, rays_per_batch=2048)
    m = spec.pipeline.model
    m.log2_hashmap_size = 17
    m.proposal_weights_anneal_max_num_iters = 100
    return spec


@pytest.fixture(scope="module")
def trained_run(native_lib, cuda_device, tmp_path_factory):
    from fruitnerf_b200.trainer import Trainer

    torch.manual_seed(0)
    run = tmp_path_factory.mktemp("eval") / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    return run


def test_evaluate_split_agrees_with_the_pipeline_evaluation(trained_run, cuda_device):
    from fruitnerf_b200.scripts.exporter import eval_setup

    _, pipeline, _, _ = eval_setup(trained_run / "config.yml")
    dm = pipeline.datamanager
    n = len(dm.eval_dataset)
    dm.eval_count = 0
    want_rows = [pipeline.get_eval_image_metrics_and_images(0)[0] for _ in range(n)]
    dm.eval_count = 0
    want = pipeline.get_average_eval_image_metrics()

    pipeline.train()
    pipeline.model.eval()  # flags that differ, to see each restored
    count = dm.eval_count
    stages = []
    got = E.evaluate_split(pipeline, num_rays_per_chunk=1000, on_stage=stages.append)
    assert pipeline.training and not pipeline.model.training
    assert dm.eval_count == count  # the images are visited by index; the datamanager's cursor is left alone
    pipeline.eval()
    assert stages[0] == "rays" and stages[-1] == "done" and stages.count("metrics") == stages.count("done") == n

    assert len(got["per_image"]) == n
    for row, ref in zip(got["per_image"], want_rows):
        assert row["image_idx"] == ref["image_idx"] and row["num_rays"] == ref["num_rays"]
        for k in ("psnr", "ssim", "iou", "fruit_iou"):
            assert abs(row[k] - ref[k]) < 1e-4, (row["image_idx"], k, row[k], ref[k])
        assert row["num_rays_per_sec"] > 0 and row["fps"] > 0 and 0 <= row["mean_accumulation"] <= 1.0 + 1e-6
    for k in ("psnr", "ssim", "iou", "fruit_iou"):
        assert abs(got["results"][k] - want[k]) < 1e-4, (k, got["results"][k], want[k])
    assert got["results"]["psnr"] > 10 and got["results"]["ssim"] > 0.1  # a model that learnt something

    # the chunk size does not change a score, and the training views are scored with --split train's path
    again = E.evaluate_split(pipeline)
    for a, b in zip(got["per_image"], again["per_image"]):
        assert all(abs(a[k] - b[k]) < 1e-5 for k in ("ssim", "psnr", "fruit_iou")), (a, b)
    train = E.evaluate_split(pipeline, split="train")
    assert len(train["per_image"]) == len(dm.train_dataset) and train["results"]["psnr"] > 10
    with pytest.raises(ValueError, match="split"):
        E.evaluate_split(pipeline, split="test")


def test_command_on_a_run_folder(trained_run, cuda_device, tmp_path):
    from PIL import Image

    from fruitnerf_b200.scripts.eval import entrypoint
    from fruitnerf_b200.scripts.exporter import eval_setup

    out = tmp_path / "eval.json"
    entrypoint(["--load-config", str(trained_run / "config.yml"), "--output-path", str(out)])
    got = json.loads(out.read_text())
    assert list(got) == ["experiment_name", "method_name", "checkpoint", "results"]
    assert got["experiment_name"] == "apple" and got["method_name"] == "fruit_nerf" and got["checkpoint"].endswith("step-000000300.ckpt")
    assert set(got["results"]) == set(E.MEAN_KEYS) | {"fruit_iou_pooled"}

    _, pipeline, _, _ = eval_setup(trained_run / "config.yml")
    n = len(pipeline.datamanager.eval_dataset)
    cams = pipeline.datamanager.eval_dataset.cameras
    H, W = cams.height, cams.width
    images = tmp_path / "images"
    entrypoint(["--load-config", str(trained_run / "config.yml"), "--output-path", str(out), "--per-image", "--render-output-path", str(images),
                "--num-rays-per-chunk", "2048"])
    both = json.loads(out.read_text())
    assert [r["image_idx"] for r in both["per_image"]] == list(range(n))
    for k in ("psnr", "ssim", "fruit_iou"):
        assert abs(both["results"][k] - got["results"][k]) < 1e-6

    # the files _save_eval_images writes for the same images, of the same sizes and nearly the same pixels
    reference = tmp_path / "reference"
    pipeline.datamanager.eval_count = 0
    pipeline.get_average_eval_image_metrics(output_path=reference)
    names = sorted(p.name for p in reference.iterdir())
    assert sorted(p.name for p in images.iterdir()) == names and len(names) % n == 0 and len(names) // n >= 6
    for name in names:
        a, b = np.asarray(Image.open(images / name)).astype(np.int16), np.asarray(Image.open(reference / name)).astype(np.int16)
        assert a.shape == b.shape == ((H, 2 * W, 3) if name.endswith("-img.jpg") else (H, W, 3)), name
        assert float(np.abs(a - b).mean()) < 3.0, name
