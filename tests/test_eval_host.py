"""Host side of the `eval` command: the fp64 restatement of the score kernels against image_metrics' torch functions, the
claim that the SSIM crop makes the padding irrelevant, aggregation of the per-image rows, and the CLI (parsing, JSON
schema, refusals).  No GPU."""
import json
import math
from types import SimpleNamespace

import pytest
import torch

from fruitnerf_b200 import _lib
from fruitnerf_b200 import evaluate as E
from fruitnerf_b200 import image_metrics as M
from fruitnerf_b200.scripts import eval as cli


def make_view(H, W, seed=0, noise=0.2, offset=0.0):
    """A rendered view that resembles its photograph (rgb strays outside [0,1]), logits clear of the 0.9 threshold."""
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(H, W, 3, generator=g)
    rgb = (image + noise * torch.randn(H, W, 3, generator=g) + offset).reshape(-1, 3).contiguous()
    sem = torch.randn(H * W, 1, generator=g) * 4
    thr = math.log(9.0)
    sem = torch.where((sem - thr).abs() < 1e-3, sem + 0.01, sem)
    acc = torch.rand(H * W, 1, generator=g)
    mask = (torch.rand(H, W, 1, generator=g) > 0.6).float()
    return rgb, sem, acc, image, mask


def torch_scores(rgb, sem, image, mask):
    H, W = image.shape[:2]
    c = rgb.reshape(H, W, 3).clamp(0, 1)
    im, pr = torch.moveaxis(image, -1, 0)[None], torch.moveaxis(c, -1, 0)[None]
    return float(M.psnr(im, pr)), float(M.ssim(im, pr)), float(M.binary_jaccard((torch.sigmoid(sem) > 0.9).reshape(H, W), mask[..., 0]))


@pytest.mark.parametrize("H,W", [(11, 11), (37, 53), (53, 37), (12, 90), (128, 96)])
def test_restatement_matches_the_torch_metrics(H, W):
    rgb, sem, acc, image, mask = make_view(H, W, seed=H * 1000 + W)
    r = M.restated_image_scores(rgb, sem, acc, image, mask)
    assert set(r) == set(_lib.IMAGE_RECORD_FIELDS)
    row = E.image_row(0, H * W, [r[k] for k in _lib.IMAGE_RECORD_FIELDS], 0.0, 1.0)
    psnr, ssim, iou = torch_scores(rgb, sem, image, mask)
    assert abs(row["psnr"] - psnr) < 1e-6 * abs(psnr) + 1e-5  # fp32 log10 of an fp32 mean on the torch side
    assert abs(row["ssim"] - ssim) < 1e-6
    assert abs(row["fruit_iou"] - iou) < 1e-6
    assert abs(row["mean_accumulation"] - float(acc.double().mean())) < 1e-12
    assert r["fruit_tp"] + r["fruit_fp"] + r["fruit_fn"] + r["fruit_tn"] == H * W
    assert r["rgb_min"] == 0.0 and r["rgb_max"] == 1.0  # clamped before the range is taken


def test_the_crop_makes_the_padding_irrelevant():
    """image_metrics.ssim reflect-pads, filters and crops; the restatement never pads.  Equal interiors mean no kept
    pixel's window reached the padding: replacing the reflect padding by anything else changes nothing either."""
    rgb, sem, acc, image, mask = make_view(40, 31, seed=5)
    r = M.restated_image_scores(rgb, sem, acc, image, mask)
    _, ssim, _ = torch_scores(rgb, sem, image, mask)
    assert abs(r["ssim"] - ssim) < 1e-6
    # a one-pixel interior is the single window that covers the whole 11x11 image
    rgb, sem, acc, image, mask = make_view(11, 11, seed=6)
    r = M.restated_image_scores(rgb, sem, acc, image, mask)
    g = M._gaussian_window(11, 1.5, torch.float64, "cpu")
    w2 = (g.t() @ g)[..., None]
    x, y = rgb.reshape(11, 11, 3).clamp(0, 1).double(), image.double()
    mx, my = (w2 * x).sum((0, 1)), (w2 * y).sum((0, 1))
    vx, vy, vxy = (w2 * x * x).sum((0, 1)) - mx * mx, (w2 * y * y).sum((0, 1)) - my * my, (w2 * x * y).sum((0, 1)) - mx * my
    c1, c2 = (0.01 * r["data_range"]) ** 2, (0.03 * r["data_range"]) ** 2
    want = (((2 * mx * my + c1) * (2 * vxy + c2)) / ((mx * mx + my * my + c1) * (vx + vy + c2))).mean()
    assert abs(r["ssim"] - float(want)) < 1e-12


def test_restatement_refuses_images_smaller_than_the_window():
    rgb, sem, acc, image, mask = make_view(10, 40)
    with pytest.raises(ValueError, match="11x11"):
        M.restated_image_scores(rgb, sem, acc, image, mask)


def test_identical_images_score_one_and_infinite_psnr():
    rgb, sem, acc, image, mask = make_view(24, 30, seed=1)
    r = M.restated_image_scores(image.reshape(-1, 3), sem, acc, image, mask)
    row = E.image_row(3, 24 * 30, [r[k] for k in _lib.IMAGE_RECORD_FIELDS], 0.0, 0.5)
    assert row["psnr"] == math.inf and row["ssim"] == 1.0 and row["image_idx"] == 3 and row["fps"] == 2.0
    assert "Infinity" in json.dumps(row)


def record(sse=3.0, tp=0, fp=0, fn=0, tn=0, acc=0.0, ssim=0.5):
    return [sse, 0.0, 1.0, 0.0, 1.0, acc, tp, fp, fn, tn, ssim, 1.0]


def test_rows_and_aggregation():
    P = 100
    a = E.image_row(0, P, record(sse=3.0, tp=10, fp=10, fn=20, tn=60, acc=50.0, ssim=0.4), 0.0, 0.1)
    assert a["psnr"] == pytest.approx(20.0) and a["fruit_iou"] == 0.25 and a["fruit_precision"] == 0.5
    assert a["fruit_recall"] == pytest.approx(1 / 3) and a["mean_accumulation"] == 0.5 and a["num_rays_per_sec"] == pytest.approx(1000.0)
    both_empty = E.image_row(1, P, record(tn=100, ssim=0.8), 0.0, 0.1)
    assert both_empty["fruit_iou"] == 1.0 and both_empty["fruit_precision"] == 0.0 and both_empty["fruit_recall"] == 0.0
    no_prediction = E.image_row(2, P, record(fn=30, tn=70), 0.0, 0.1)
    assert no_prediction["fruit_iou"] == 0.0 and no_prediction["fruit_precision"] == 0.0 and no_prediction["fruit_recall"] == 0.0
    no_truth = E.image_row(3, P, record(fp=5, tn=95), 0.0, 0.1)
    assert no_truth["fruit_iou"] == 0.0 and no_truth["fruit_recall"] == 0.0
    rows = [a, both_empty, no_prediction, no_truth]
    res = E.aggregate(rows)
    assert set(res) == set(E.MEAN_KEYS) | {"fruit_iou_pooled"}
    assert {"psnr", "ssim", "iou", "fruit_iou", "num_rays_per_sec", "fps"} <= set(res)  # get_average_eval_image_metrics' keys
    assert res["fruit_iou"] == pytest.approx((0.25 + 1.0 + 0.0 + 0.0) / 4)
    assert res["fruit_iou_pooled"] == pytest.approx(10 / (10 + 15 + 50))
    assert res["ssim"] == pytest.approx((0.4 + 0.8 + 0.5 + 0.5) / 4)
    assert E.aggregate([both_empty])["fruit_iou_pooled"] == 1.0
    with pytest.raises(ValueError):
        E.aggregate([])


def test_exported_symbols_and_record_fields():
    for name in ("fnr_image_metrics_scratch_bytes", "fnr_image_stats", "fnr_ssim"):
        assert name in _lib.EXPORTED_SYMBOLS
    assert len(_lib.IMAGE_RECORD_FIELDS) == _lib.FNR_IMAGE_RECORD_DOUBLES


# ---- the command ------------------------------------------------------------------------------------------------
def test_cli_parsing():
    a = cli.build_parser().parse_args(["--load-config", "run/config.yml", "--output-path", "e.json"])
    assert str(a.load_config) == "run/config.yml" and a.split == "eval" and not a.per_image and a.render_output_path is None
    assert a.num_rays_per_chunk is None
    a = cli.build_parser().parse_args(["--load-config", "c.yml", "--output-path", "e.json", "--render-output-path", "imgs", "--split", "train",
                                       "--per-image", "--num-rays-per-chunk", "4096"])
    assert str(a.render_output_path) == "imgs" and a.split == "train" and a.per_image and a.num_rays_per_chunk == 4096
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--output-path", "e.json"])
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--load-config", "c.yml", "--split", "test"])


def fake_pipeline(device="cuda", num_eval=2):
    ds = None if num_eval is None else [0] * num_eval
    return SimpleNamespace(device=torch.device(device), datamanager=SimpleNamespace(eval_dataset=ds, train_dataset=[0] * 5))


def test_cli_writes_the_ns_eval_json(tmp_path, monkeypatch):
    rows = [E.image_row(i, 100, record(tp=i + 1, fn=1, tn=98 - i), 0.0, 0.1) for i in range(2)]
    calls = []

    def fake_evaluate_split(pipeline, **kw):
        calls.append(kw)
        return {"results": E.aggregate(rows), "per_image": rows}

    monkeypatch.setattr(E, "evaluate_split", fake_evaluate_split)
    config = SimpleNamespace(method_name="fruit_nerf")
    run = tmp_path / "outputs" / "apple" / "fruit_nerf" / "run0"
    out = tmp_path / "deep" / "eval.json"
    argv = ["--load-config", str(run / "config.yml"), "--output-path", str(out)]
    cli.entrypoint(argv, fake_pipeline(), config, run / "nerfstudio_models" / "step-000000300.ckpt")
    got = json.loads(out.read_text())
    assert list(got) == ["experiment_name", "method_name", "checkpoint", "results"]
    assert got["experiment_name"] == "apple" and got["method_name"] == "fruit_nerf" and got["checkpoint"].endswith("step-000000300.ckpt")
    assert set(got["results"]) == set(E.MEAN_KEYS) | {"fruit_iou_pooled"}
    assert calls[-1] == {"split": "eval", "num_rays_per_chunk": None, "render_output_path": None}
    cli.entrypoint(argv + ["--per-image", "--split", "train", "--num-rays-per-chunk", "512", "--render-output-path", str(tmp_path / "im")],
                   fake_pipeline(), config, "ckpt")
    got = json.loads(out.read_text())
    assert len(got["per_image"]) == 2 and got["per_image"][1]["image_idx"] == 1 and got["per_image"][0]["fruit_tp"] == 1
    assert calls[-1]["split"] == "train" and calls[-1]["num_rays_per_chunk"] == 512 and calls[-1]["render_output_path"] == tmp_path / "im"
    # a run folder outside nerfstudio's layout goes by its own name
    assert cli.experiment_name(config, tmp_path / "myrun" / "config.yml") == "myrun"
    assert cli.experiment_name(SimpleNamespace(method_name="fruit_nerf", experiment_name="pears"), run / "config.yml") == "pears"


def test_cli_refusals(tmp_path, capsys):
    config = SimpleNamespace(method_name="fruit_nerf")
    good = ["--load-config", str(tmp_path / "config.yml"), "--output-path", str(tmp_path / "eval.json")]

    def refused(argv, pipeline, match):
        with pytest.raises(SystemExit) as e:
            cli.entrypoint(argv, pipeline, config, "ckpt")
        assert e.value.code == 1
        assert match in capsys.readouterr().err
        assert not (tmp_path / "eval.json").exists()

    refused(["--load-config", str(tmp_path / "config.yml"), "--output-path", str(tmp_path / "eval.txt")], fake_pipeline(), ".json")
    refused(good, None, "no config at")  # nothing at that path, and no pipeline handed in
    refused(good, fake_pipeline("cpu"), "CUDA device")
    refused(good, fake_pipeline(num_eval=None), "no eval split")
    refused(good, fake_pipeline(num_eval=0), "no eval split")
