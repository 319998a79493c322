"""CPU tests of the lens model of captured data sets (DESIGN.md section 4.3j): the torch restatement against OpenCV, its
edge cases, the dataparser's ``lens_distortion`` mode, lens data sets on disk and the ``train --data`` command line."""
import json
import math

import numpy as np
import pytest
import torch
import yaml

from fruitnerf_b200 import render as R
from fruitnerf_b200.data import camera_model as cm
from fruitnerf_b200.data.fruit_datamanager import FruitDataManagerConfig
from fruitnerf_b200.data.fruitnerf_dataparser import FruitNerf, FruitNerfDataParserConfig
from fruitnerf_b200.data.synthetic_scene import SyntheticCameras, camera_rays, make_apple_scene, trace, write_dataset

# COLMAP-sized OPENCV coefficients of a phone / action camera
COLMAP = dict(k1=-0.12, k2=0.045, k3=-0.008, p1=0.0012, p2=-0.0009)
STRONG = [-0.45, 0.25, -0.05, 0.0, 0.01, -0.01]


@pytest.mark.parametrize("coeffs", [{"k1": COLMAP["k1"]}, {"k2": COLMAP["k2"]}, {"k3": COLMAP["k3"]}, {"p1": COLMAP["p1"]}, {"p2": COLMAP["p2"]},
                                    COLMAP], ids=["k1", "k2", "k3", "p1", "p2", "all"])
def test_undistortion_inverts_opencv_projection(coeffs):
    """Every pixel centre of a 640x480 camera: OpenCV's projection of the undistorted direction lands on the pixel.  The
    restatement flips y before undistorting, so OpenCV sees y-down coordinates and -p1."""
    cv2 = pytest.importorskip("cv2")
    fx, fy, cx, cy = 512.0, 498.0, 321.7, 238.4
    ys, xs = torch.meshgrid(torch.arange(480), torch.arange(640), indexing="ij")
    ys, xs = ys.reshape(-1), xs.reshape(-1)
    uv = cm.pixel_coords(xs, ys, fx, fy, cx, cy).double()
    und = cm.radial_and_tangential_undistort(uv, cm.get_distortion_params(**coeffs).double())
    pts = np.stack([und[:, 0].numpy(), -und[:, 1].numpy(), np.ones(len(und))], 1)
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    c = {k: coeffs.get(k, 0.0) for k in ("k1", "k2", "k3", "p1", "p2")}
    proj, _ = cv2.projectPoints(pts, np.zeros(3), np.zeros(3), K, np.array([c["k1"], c["k2"], -c["p1"], c["p2"], c["k3"]]))
    err = np.abs(proj[:, 0, :] - np.stack([xs.numpy() + 0.5, ys.numpy() + 0.5], 1)).max()
    assert err < 1e-4, err
    # and the forward model used for test data is OpenCV's too
    assert torch.allclose(cm.distort(und, cm.get_distortion_params(**coeffs).double()), uv, atol=1e-9)


def test_zero_coefficients_leave_coordinates_bit_identical():
    uv = cm.pixel_coords(torch.arange(0, 640, 3), torch.arange(0, 640, 3) % 480, 500.0, 500.0, 320.0, 240.0)
    out = cm.radial_and_tangential_undistort(uv.double(), torch.zeros(6, dtype=torch.float64)).float()
    assert torch.equal(out, uv)
    o, d = cm.lens_rays(torch.eye(4)[:3], 500.0, 500.0, 320.0, 240.0, torch.zeros(6), "perspective", torch.tensor([3, 77]), torch.tensor([5, 600]))
    o2, d2 = cm.lens_rays(torch.eye(4)[:3], 500.0, 500.0, 320.0, 240.0, None, "perspective", torch.tensor([3, 77]), torch.tensor([5, 600]))
    assert torch.equal(d, d2)


def test_singular_jacobian_takes_a_zero_step():
    # k1 = -1 at (1, 0): d = 1 + k1 r = 0, so fy_y = 0 and det = 0 -> the guard keeps the point where it is
    dist = torch.tensor([-1.0, 0, 0, 0, 0, 0], dtype=torch.float64)
    pt = torch.tensor([[1.0, 0.0]], dtype=torch.float64)
    assert torch.equal(cm.radial_and_tangential_undistort(pt, dist), pt)
    _, _, fx_x, fx_y, fy_x, fy_y = cm._residual_and_jacobian(pt[:, 0], pt[:, 1], pt[:, 0], pt[:, 1], dist)
    assert float(fy_x * fx_y - fx_x * fy_y) == 0.0
    # a regular point of the same model does step (det = -0.25)
    pt2 = torch.tensor([[0.7, 0.1]], dtype=torch.float64)
    assert not torch.equal(cm.radial_and_tangential_undistort(pt2, dist, max_iterations=1), pt2)


def test_strong_coefficients_take_exactly_ten_newton_steps():
    """At the corners of a wide image the iteration does not converge; the result is the tenth iterate, no more, no less."""
    ys, xs = torch.tensor([0, 0, 479, 479]), torch.tensor([0, 639, 0, 639])
    uv = cm.pixel_coords(xs, ys, 300.0, 300.0, 320.0, 240.0).double()
    dist = torch.tensor(STRONG, dtype=torch.float64)
    ten = cm.radial_and_tangential_undistort(uv, dist)
    assert torch.equal(ten, cm.radial_and_tangential_undistort(uv, dist, max_iterations=10))
    nine, eleven = cm.radial_and_tangential_undistort(uv, dist, max_iterations=9), cm.radial_and_tangential_undistort(uv, dist, max_iterations=11)
    assert not torch.equal(ten, nine) and not torch.equal(ten, eleven)
    resid = (cm.distort(ten, dist) - uv).abs().max()
    assert float(resid) > 1e-3  # not converged: the corners lie outside the region the model inverts


def test_fisheye_without_coefficients_is_the_render_camera():
    cams = R.CameraSet(torch.eye(4)[:3][None], 60.0, 62.0, 40.0, 30.0, 60, 80, camera_type="fisheye")
    o_ref, d_ref = R.restated_camera_rays(cams, 0, 0, 60 * 80)
    p = torch.arange(60 * 80)
    o, d = cm.lens_rays(cams.camera_to_worlds[0], 60.0, 62.0, 40.0, 30.0, None, "fisheye", p // 80, p % 80)
    assert torch.allclose(d.double(), d_ref, atol=1e-6) and torch.equal(o.double(), o_ref)


# ---- dataparser -------------------------------------------------------------------------------------------------------
def _lens_scene(tmp_path, name="lens", **kw):
    kw = {"num_images": 10, "height": 16, "width": 20, "num_fruits": 12, "noise_std": 0.0, **kw}
    train, ev = make_apple_scene(**kw)
    path = write_dataset(train, tmp_path / name)
    return train, path


def _edit(path, fn):
    meta = json.loads(path.read_text())
    fn(meta)
    path.write_text(json.dumps(meta))
    return path


def _parse(path, split="train", lens=True, downscale=1):
    return FruitNerf(FruitNerfDataParserConfig(data=path.parent, downscale_factor=downscale, lens_distortion=lens)).get_dataparser_outputs(split)


def test_dataparser_reads_shared_and_per_frame_distortion(tmp_path):
    train, path = _lens_scene(tmp_path, distortion=[-0.1, 0.02, 0.0, 0.0, 0.001, -0.002], intrinsics_jitter=0.03)
    cams = _parse(path).cameras
    n = len(cams)  # the parser's own 90 % split of the 9 written frames
    split = np.linspace(0, len(train) - 1, math.ceil(len(train) * 0.9), dtype=int)
    assert cams.camera_type == "perspective" and cams.distortion_params.shape == (n, 6)
    assert torch.equal(cams.distortion_params, train.cameras.distortion_params[split])
    assert torch.equal(cams.fx, train.cameras.fx[split]) and torch.equal(cams.cy, train.cameras.cy[split])

    def shared(meta):
        for f in meta["frames"]:
            for k in ("k1", "k2", "k3", "k4", "p1", "p2"):
                f.pop(k)
        meta.update(k1=-0.2, k2=0.03, p2=0.004)
    cams = _parse(_edit(path, shared)).cameras
    want = torch.tensor([-0.2, 0.03, 0.0, 0.0, 0.0, 0.004], dtype=torch.float32)
    assert torch.equal(cams.distortion_params, want.expand(n, 6))


def test_dataparser_distort_fixed_quirk(tmp_path):
    """Only k1, k2, k3, p1, p2 at the top level make the coefficients shared: k4 alone there is ignored in favour of the
    frames', and once they are shared the frames' are ignored."""
    _, path = _lens_scene(tmp_path, distortion=[-0.1, 0.0, 0.0, 0.0, 0.0, 0.0])
    cams = _parse(_edit(path, lambda m: m.update(k4=0.5))).cameras
    assert torch.all(cams.distortion_params[:, 0] == torch.tensor(-0.1)) and torch.all(cams.distortion_params[:, 3] == 0)
    cams = _parse(_edit(path, lambda m: m.update(p1=0.003))).cameras
    want = torch.tensor([0.0, 0.0, 0.0, 0.5, 0.003, 0.0], dtype=torch.float32)
    assert torch.equal(cams.distortion_params, want.expand(len(cams), 6))


def test_dataparser_per_frame_intrinsics_follow_split_and_downscale(tmp_path):
    from PIL import Image

    train, path = _lens_scene(tmp_path, intrinsics_jitter=0.05)
    for folder in ("images", "semantics"):
        (path.parent / f"{folder}_2").mkdir()
        for f in sorted((path.parent / folder).iterdir()):
            Image.open(f).resize((10, 8), Image.NEAREST).save(path.parent / f"{folder}_2" / f.name)
    ev = np.setdiff1d(np.arange(len(train)), np.linspace(0, len(train) - 1, math.ceil(len(train) * 0.9), dtype=int))
    cams = _parse(path, "val", downscale=2).cameras
    assert (cams.height, cams.width) == (8, 10) and cams.distortion_params is None
    for k in ("fx", "fy", "cx", "cy"):
        assert torch.equal(getattr(cams, k), getattr(train.cameras, k)[ev] * 0.5), k
    assert cams.has_lens


@pytest.mark.parametrize("model,kind", [("OPENCV", "perspective"), ("PINHOLE", "perspective"), ("SIMPLE_RADIAL", "perspective"),
                                        ("RADIAL", "perspective"), ("SIMPLE_PINHOLE", "perspective"), ("OPENCV_FISHEYE", "fisheye"),
                                        ("EQUIRECTANGULAR", "equirectangular")])
def test_dataparser_camera_model_mapping(tmp_path, model, kind):
    _, path = _lens_scene(tmp_path, camera_type="fisheye")
    cams = _parse(_edit(path, lambda m: m.update(camera_model=model))).cameras
    assert cams.camera_type == kind
    # flag off: camera_model ignored, exactly as before
    off = _parse(path, lens=False).cameras
    assert off.camera_type == "perspective" and not off.has_lens


def test_dataparser_refusals(tmp_path):
    _, path = _lens_scene(tmp_path)
    for model in ("OMNIDIRECTIONALSTEREO_L", "VR180_R"):
        with pytest.raises(NotImplementedError, match="stereo"):
            _parse(_edit(path, lambda m: m.update(camera_model=model)))
    with pytest.raises(ValueError, match="unknown camera_model"):
        _parse(_edit(path, lambda m: m.update(camera_model="KANNALA")))

    def sizes(m):
        m["camera_model"] = "OPENCV"
        m.pop("h")
        for i, f in enumerate(m["frames"]):
            f["h"] = 16 if i % 2 else 18
    with pytest.raises(NotImplementedError, match="one \\[N,H,W\\] image stack"):
        _parse(_edit(path, sizes))


def test_all_zero_opencv_folder_is_the_shared_pinhole(tmp_path):
    train, _ = make_apple_scene(num_images=10, height=16, width=20, num_fruits=3, noise_std=0.0)
    path = write_dataset(train, tmp_path / "pinhole")
    assert json.loads(path.read_text())["camera_model"] == "OPENCV"
    on, off = _parse(path).cameras, _parse(path, lens=False).cameras
    assert not on.has_lens and on.distortion_params is None and on.camera_type == "perspective"
    assert (on.fx, on.fy, on.cx, on.cy, on.height, on.width) == (off.fx, off.fy, off.cx, off.cy, off.height, off.width)
    assert all(isinstance(v, float) for v in (on.fx, on.fy, on.cx, on.cy))
    assert torch.equal(on.camera_to_worlds, off.camera_to_worlds)


@pytest.mark.parametrize("camera_type", ["perspective", "fisheye", "equirectangular"])
def test_lens_data_set_round_trips_through_disk(tmp_path, camera_type):
    train, path = _lens_scene(tmp_path, camera_type=camera_type, distortion=[[-0.1, 0.01, 0.0, 0.0, 0.001, 0.0]], intrinsics_jitter=0.02, height=40,
                              width=64)
    meta = json.loads(path.read_text())
    assert meta["camera_model"] == cm.TYPE_TO_CAMERA_MODEL[camera_type] and "fl_x" not in meta and "k1" in meta["frames"][0]
    cfg = FruitNerfDataParserConfig(data=path.parent, downscale_factor=1, lens_distortion=True, train_split_fraction=1.0)
    cams = FruitNerf(cfg).get_dataparser_outputs("train").cameras
    assert cams.camera_type == camera_type
    for k in ("fx", "fy", "cx", "cy", "distortion_params"):
        assert torch.equal(getattr(cams, k), getattr(train.cameras, k)), k


def test_old_config_without_the_flag_loads(tmp_path):
    text = yaml.dump(FruitNerfDataParserConfig(data=tmp_path))
    assert "lens_distortion" in text
    old = "\n".join(line for line in text.splitlines() if "lens_distortion" not in line)
    cfg = yaml.load(old, Loader=yaml.Loader)
    assert cfg.lens_distortion is False and cfg.data == tmp_path


def test_lens_cameras_refuse_non_finite_values_when_moved():
    cams = SyntheticCameras(torch.eye(4)[:3][None].repeat(2, 1, 1), torch.tensor([100.0, float("nan")]), 100.0, 8.0, 8.0, 16, 16)
    with pytest.raises(ValueError, match="finite"):
        cams.to("cpu")
    cams = SyntheticCameras(torch.eye(4)[:3][None].repeat(2, 1, 1), 100.0, 100.0, 8.0, 8.0, 16, 16, "fisheye", torch.full((2, 6), float("inf")))
    with pytest.raises(ValueError, match="finite"):
        cams.to("cpu")


# ---- rays and targets end to end ------------------------------------------------------------------------------------
def _pixel_mismatch(dm, outs, geom, ignore_lens: bool) -> float:
    """Share of a batch's target pixels that the analytic scene, traced along the batch rays, does not reproduce."""
    rb, batch = dm.next_train(0)
    o, d = rb.origins, rb.directions
    if ignore_lens:  # the same pixels through a shared pinhole with the mean intrinsics
        cams, idx = dm.train_dataset.cameras, batch["indices"]
        f = [float(t.mean()) for t in cams.intrinsics()]
        o, d = camera_rays(cams.camera_to_worlds[idx[:, 0]], *f, idx[:, 1], idx[:, 2])
    # parser frame -> the scene's frame: p = R^T (p' / s - t)
    T, s = outs.dataparser_transform, outs.dataparser_scale
    Rm, t = T[:, :3], T[:, 3]
    o_w = (o / s - t) @ Rm
    d_w = d @ Rm
    rgb, mask, _ = trace(geom, o_w, d_w / d_w.norm(dim=-1, keepdim=True))
    bad = ((rgb - batch["image"]).abs().max(dim=-1).values > 3.0 / 255) | (mask != batch["fruit_mask"])[:, 0]
    return float(bad.float().mean())


def test_batch_rays_reproduce_their_target_pixels(tmp_path):
    """A noise-free distorted, per-frame-jittered data set written to disk and read back through the datamanager: the
    scene traced along each drawn ray gives the drawn pixel, except near silhouette edges (where the 8-bit, 0.5-px
    rounding of the written image meets a colour step).  With the lens ignored a large share fails."""
    train, path = _lens_scene(tmp_path, num_images=10, height=48, width=64, distortion=[-0.25, 0.06, 0.0, 0.0, 0.002, -0.003],
                              intrinsics_jitter=0.04)
    dp = FruitNerfDataParserConfig(data=path.parent, downscale_factor=1, lens_distortion=True)
    dm = FruitDataManagerConfig(train_num_rays_per_batch=4000, dataparser=dp).setup(device="cpu")
    assert dm.train_dataset.cameras.has_lens
    aware = _pixel_mismatch(dm, dm.train_dataparser_outputs, train.geometry, ignore_lens=False)
    ignored = _pixel_mismatch(dm, dm.train_dataparser_outputs, train.geometry, ignore_lens=True)
    # measured on CPU: 0 of the 4000 pixels with the lens, 34 % without
    assert aware < 0.01, aware
    assert ignored > 0.15, ignored


def test_cpu_lens_batches_and_eval_images_share_rays():
    train, _ = make_apple_scene(num_images=10, height=12, width=14, num_fruits=2, noise_std=0.0, camera_type="fisheye",
                                distortion=[-0.1, 0, 0, 0, 0, 0], intrinsics_jitter=0.05)
    dm = FruitDataManagerConfig(train_num_rays_per_batch=500).setup(device="cpu", train_dataset=train, eval_dataset=train)
    rb, batch = dm.next_train(0)
    idx = batch["indices"]
    assert torch.equal(batch["image"], train.images[idx[:, 0], idx[:, 1], idx[:, 2]])
    fx, fy = train.cameras.intrinsics()[:2]
    assert torch.equal(rb.pixel_area[:, 0], (1.0 / (fx.double() * fy.double())).float()[idx[:, 0]])
    for i in idx[:5, 0].tolist():
        full = train.cameras.generate_rays(i)
        sel = idx[:, 0] == i
        assert torch.equal(full.directions[idx[sel, 1], idx[sel, 2]], rb.directions[sel])


# ---- command line ----------------------------------------------------------------------------------------------------
def test_train_data_command_line(monkeypatch, tmp_path):
    from fruitnerf_b200.scripts import train as T

    with pytest.raises(SystemExit):
        T.main(["--data", str(tmp_path)])
    seen = {}
    monkeypatch.setattr(T, "train_data", lambda data, out, steps, method, **kw: seen.update(data=data, out=out, steps=steps, **kw) or {"ok": 1})
    T.main(["--data", str(tmp_path), "--output-dir", str(tmp_path / "run"), "--steps", "7", "--downscale-factor", "2"])
    assert seen["data"] == str(tmp_path) and seen["out"] == str(tmp_path / "run") and seen["steps"] == 7 and seen["downscale_factor"] == 2
    spec = T.data_spec(tmp_path, downscale_factor=2)
    dm = spec.pipeline.datamanager
    assert dm.synthetic_scene is None and dm.dataparser.lens_distortion and dm.dataparser.downscale_factor == 2
