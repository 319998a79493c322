"""The `render` command on the device: fnr_camera_rays against the torch restatement of the camera models,
fnr_compose_frame byte for byte against the torch composition (image_metrics.apply_colormap / apply_depth_colormap), and
render_frames / the CLI end to end on a briefly trained model."""
import json
import math

import numpy as np
import pytest
import torch

from fruitnerf_b200 import ops
from fruitnerf_b200 import render as R
from fruitnerf_b200.data.synthetic_scene import look_at_c2w, make_apple_scene
from fruitnerf_b200.image_metrics import _turbo_table, apply_colormap, apply_depth_colormap

pytestmark = pytest.mark.gpu


def _camera_set(kind, dev, F=3, H=37, W=53, seed=0):
    g = torch.Generator().manual_seed(seed)
    poses = torch.stack([look_at_c2w(torch.randn(3, generator=g) * 2, torch.randn(3, generator=g) * 0.1) for _ in range(F)]).float()
    fx = 20 + 40 * torch.rand(F, generator=g)
    fy = fx * (0.9 + 0.2 * torch.rand(F, generator=g))
    cx, cy = W / 2 + torch.rand(F, generator=g) - 0.5, H / 2 + torch.rand(F, generator=g) - 0.5
    if kind == "equirectangular":
        fx, fy, cx, cy = torch.full((F,), W / 2), torch.full((F,), float(H)), torch.full((F,), W / 2), torch.full((F,), H / 2)
    return R.CameraSet(poses, fx, fy, cx, cy, H, W, kind).to(dev)


RANGES = [(0, 37 * 53), (0, 1), (52, 2), (53 * 7 - 5, 300), (100, 53), (37 * 53 - 17, 17), (1000, 961)]


def test_perspective_rays_are_bitwise_generate_rays(native_lib, cuda_device):
    cams = _camera_set("perspective", cuda_device)
    for f in range(len(cams)):
        for p0, n in RANGES:
            o, d = ops.camera_rays(cams.camera_to_worlds, cams.fx, cams.fy, cams.cx, cams.cy, "perspective", cams.height, cams.width, f, p0, n)
            ro, rd = R.restated_camera_rays(cams, f, p0, n)
            assert torch.equal(o, ro), (f, p0, n)
            bad = (d != rd).any(-1)
            assert not bool(bad.any()), (f, p0, n, int(bad.sum()), float((d - rd).abs().max()))
    # the synthetic scene's own cameras, through SyntheticCameras.generate_rays on the device
    train, _ = make_apple_scene(num_images=10, height=48, width=64, num_fruits=2, noise_std=0.0)
    cams = train.cameras.to(cuda_device)
    cs = R.CameraSet.from_cameras(cams)
    for i in (0, 7):
        ref = cams.generate_rays(i)
        o, d = ops.camera_rays(cs.camera_to_worlds, cs.fx, cs.fy, cs.cx, cs.cy, "perspective", 48, 64, i, 0, 48 * 64)
        assert torch.equal(d, ref.directions.reshape(-1, 3)) and torch.equal(o, ref.origins.reshape(-1, 3))


@pytest.mark.parametrize("kind", ["fisheye", "equirectangular"])
def test_fisheye_and_equirectangular_rays_match_fp64(native_lib, cuda_device, kind):
    cams = _camera_set(kind, cuda_device)
    buf = (torch.empty((4000, 3), device=cuda_device), torch.empty((4000, 3), device=cuda_device))
    for f in range(len(cams)):
        for p0, n in RANGES:
            o, d = ops.camera_rays(cams.camera_to_worlds, cams.fx, cams.fy, cams.cx, cams.cy, kind, cams.height, cams.width, f, p0, n, out=buf)
            ro, rd = R.restated_camera_rays(cams, f, p0, n)
            assert torch.equal(o.cpu().double(), ro)
            err = float((d.cpu().double() - rd).abs().max())
            assert err < 1e-6, (kind, f, p0, n, err)
    # the fisheye axis pixel: (0, 0, -1) rotated, not 0 / 0
    if kind == "fisheye":
        c = R.CameraSet(cams.camera_to_worlds[:1], 10.0, 10.0, 2.5, 1.5, 3, 5, "fisheye").to(cuda_device)
        _, d = ops.camera_rays(c.camera_to_worlds, c.fx, c.fy, c.cx, c.cy, "fisheye", 3, 5, 0, 7, 1)
        assert bool(torch.isfinite(d).all())
        assert torch.allclose(d[0], -c.camera_to_worlds[0, :, 2], atol=1e-6)


def test_bad_ranges_are_refused(native_lib, cuda_device):
    cams = _camera_set("perspective", cuda_device, F=2, H=4, W=5)
    args = (cams.camera_to_worlds, cams.fx, cams.fy, cams.cx, cams.cy, "perspective", 4, 5)
    with pytest.raises(ops.L.FruitNerfNativeError, match="invalid arguments"):
        ops.camera_rays(*args, 0, 15, 6)
    with pytest.raises(ops.L.FruitNerfNativeError, match="invalid arguments"):
        ops.camera_rays(*args, 2, 0, 1)
    with pytest.raises(ValueError):
        ops.camera_rays(*args[:5], "vr180", 4, 5, 0, 0, 1)
    with pytest.raises(ops.L.FruitNerfNativeError, match="CUDA"):
        ops.camera_rays(cams.camera_to_worlds.cpu(), *args[1:], 0, 0, 1)


# ---- composition --------------------------------------------------------------------------------------------------
def torch_frame(outputs, names, H, W, near=None, far=None):
    """ns-render's per-frame image with image_metrics' colour maps, quantised as mediapy's to_uint8."""
    acc = outputs["accumulation"].reshape(H, W, 1)
    imgs = []
    for n in names:
        x = outputs[n].reshape(H, W, -1)
        imgs.append(apply_depth_colormap(x, accumulation=acc, near_plane=near, far_plane=far) if "depth" in n else apply_colormap(x))
    img = torch.cat(imgs, dim=1).cpu().numpy()
    return (np.clip(img, 0.0, 1.0) * 255 + 0.5).astype(np.uint8)


def kernel_frame(outputs, names, H, W, dev, near=None, far=None):
    images = []
    for n in names:
        t = outputs[n].reshape(H * W, -1)
        kind = R.frame_kind(n, t.shape[1])
        images.append(ops.FrameImage(t, kind, R.plane_or_auto(near), R.plane_or_auto(far)) if kind == "depth" else ops.FrameImage(t, kind))
    return ops.compose_frame(images, outputs["accumulation"], H, W, _turbo_table(dev)).cpu().numpy()


def _fake_outputs(H, W, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    P = H * W
    colors = torch.tensor([[1.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    sem = torch.randn(P, 1, generator=g) * 4
    out = {
        "rgb": torch.rand(P, 3, generator=g),
        "accumulation": torch.rand(P, 1, generator=g).clamp_max(1.0),
        "depth": 0.2 + 3 * torch.rand(P, 1, generator=g),
        "semantics": sem,
        "semantics_colormap": colors[(torch.sigmoid(sem) > 0.9).long()[:, 0]],
        "prop_depth_0": 0.1 + 5 * torch.rand(P, 1, generator=g),
    }
    if P >= 7:
        out["accumulation"][:7] = torch.tensor([0.0, 1.0, 0.5, 1e-7, 1 - 1e-7, 0.25, 0.75])[:, None]
        out["rgb"][:4] = torch.tensor([[0.0, 1.0, 0.5], [1 / 255, 0.5 / 255, 254.5 / 255], [1.0, 1.0, 1.0], [0.0, 0.0, 0.0]])
    return {k: v.to(dev) for k, v in out.items()}


NAMES = ["rgb", "depth", "accumulation", "semantics", "semantics_colormap", "prop_depth_0"]


@pytest.mark.parametrize("H, W", [(33, 47), (120, 200), (1, 1)])
def test_compose_frame_is_bytewise_the_torch_composition(native_lib, cuda_device, H, W):
    out = _fake_outputs(H, W, cuda_device)
    for names in (NAMES, ["rgb"], ["depth"], ["semantics_colormap", "accumulation"], NAMES[::-1]):
        for near, far in ((None, None), (0.5, 2.5), (0.0, 2.0), (1.0, None), (None, 1.5)):
            got = kernel_frame(out, names, H, W, cuda_device, near, far)
            want = torch_frame(out, names, H, W, near, far)
            assert got.shape == (H, W * len(names), 3)
            diff = got != want
            assert not diff.any(), (names, near, far, int(diff.sum()), np.argwhere(diff)[:5].tolist())


def test_compose_frame_nan_and_constant_depth(native_lib, cuda_device):
    H, W = 40, 64
    out = _fake_outputs(H, W, cuda_device, seed=1)
    nan = dict(out, depth=out["depth"].clone())
    nan["depth"][123] = float("nan")
    const = dict(out, depth=torch.full_like(out["depth"], 1.7), prop_depth_0=torch.zeros_like(out["depth"]))
    for o in (nan, const):
        for near, far in ((None, None), (0.5, 2.5)):
            got = kernel_frame(o, NAMES, H, W, cuda_device, near, far)
            assert np.array_equal(got, torch_frame(o, NAMES, H, W, near, far)), (near, far)


def test_compose_frame_repeats_bit_for_bit_at_1080p(native_lib, cuda_device):
    H, W = 1080, 1920
    out = _fake_outputs(H, W, cuda_device, seed=2)
    a = kernel_frame(out, ["rgb", "depth", "semantics"], H, W, cuda_device)
    b = kernel_frame(out, ["rgb", "depth", "semantics"], H, W, cuda_device)
    assert np.array_equal(a, b)
    assert np.array_equal(a, torch_frame(out, ["rgb", "depth", "semantics"], H, W))


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
    run = tmp_path_factory.mktemp("render") / "outputs" / "apple" / "fruit_nerf" / "run0"
    trainer = Trainer(_tiny_spec(), device=cuda_device, output_dir=str(run), use_cuda_graph=True)
    trainer.train(300, log_every=10**9, eval_every=10**9)
    trainer.save_checkpoint()
    del trainer
    return run


def test_render_frames_equals_the_camera_ray_bundle_path(trained_run, cuda_device, tmp_path):
    from PIL import Image

    from fruitnerf_b200.scripts.exporter import eval_setup
    from fruitnerf_b200.scripts.render import entrypoint

    _, pipeline, _, _ = eval_setup(trained_run / "config.yml", test_mode="inference")
    cams = pipeline.datamanager.eval_dataset.cameras
    H, W = cams.height, cams.width
    ref = pipeline.model.get_outputs_for_camera_ray_bundle(cams.generate_rays(0))
    ref = {k: v.to(cuda_device) for k, v in ref.items()}
    want = torch_frame(ref, NAMES, H, W)
    assert float(ref["accumulation"].mean()) > 0.5
    one = R.CameraSet.from_cameras(cams, [0])
    for chunk in (4096, 1000):
        got = R.render_frames(pipeline, one, NAMES, num_rays_per_chunk=chunk)
        assert len(got) == 1 and got[0].shape == (H, W * len(NAMES), 3)
        diff = got[0] != want
        assert not diff.any(), (chunk, int(diff.sum()))

    # the same camera as a viewer camera-path file (fov from the focal length), through the CLI
    c2w = torch.eye(4)
    c2w[:3] = cams.camera_to_worlds[0].cpu()
    fov = math.degrees(2 * math.atan((H / 2) / cams.fy))
    path = {"render_height": H, "render_width": W, "seconds": 1.0, "camera_path": [{"camera_to_world": c2w.flatten().tolist(), "fov": fov}]}
    pf = tmp_path / "path.json"
    pf.write_text(json.dumps(path))
    out = tmp_path / "renders" / "cp.mp4"
    names = ["rgb", "depth", "semantics_colormap"]
    w = entrypoint(["camera-path", "--load-config", str(trained_run / "config.yml"), "--camera-path-filename", str(pf), "--output-path", str(out),
                    "--output-format", "images", "--image-format", "png", "--rendered-output-names", *names])
    assert w.count == 1
    # The file gives the data set's camera back up to the fp32 rounding of the focal length through its fov.  A ray moved by
    # that rounding can move a pixel's median depth to the neighbouring sample or its semantic label across 0.9, so the
    # frame is not compared with the data-set camera's: the file's camera is checked against that camera, and the CLI's
    # frame against the in-process render of the file's camera, byte for byte.
    cp = R.get_path_from_json(path)
    assert torch.equal(cp.camera_to_worlds, one.camera_to_worlds.cpu()) and (cp.height, cp.width) == (H, W)
    assert torch.equal(cp.cx, one.cx.cpu()) and torch.equal(cp.cy, one.cy.cpu())
    assert torch.allclose(cp.fx, one.fx.cpu(), rtol=1e-6, atol=0) and torch.allclose(cp.fy, one.fy.cpu(), rtol=1e-6, atol=0)
    img = np.asarray(Image.open(tmp_path / "renders" / "cp" / "00000.png"))
    want3 = R.render_frames(pipeline, cp, names)[0]
    assert img.shape == want3.shape and np.array_equal(img, want3), int(np.abs(img.astype(np.int16) - want3).max())
    # and that render is the data-set camera's frame, except where a pixel sits on such a discontinuity
    near = np.abs(want3.astype(np.int16) - torch_frame(ref, names, H, W).astype(np.int16)).max(axis=-1) <= 1
    assert near.mean() >= 0.99, float(near.mean())

    # interpolate and spiral write the expected number of frames of the expected size
    out = tmp_path / "renders" / "interp.mp4"
    w = entrypoint(["interpolate", "--load-config", str(trained_run / "config.yml"), "--output-path", str(out), "--output-format", "images",
                    "--interpolation-steps", "3", "--rendered-output-names", "rgb", "depth", "semantics_colormap", "--downscale-factor", "2"])
    n_eval = len(cams)
    files = sorted((tmp_path / "renders" / "interp").iterdir())
    assert w.count == len(files) == 3 * (n_eval - 1) and files[0].name == "00000.jpg"
    assert np.asarray(Image.open(files[-1])).shape == (H // 2, 3 * (W // 2), 3)
    out = tmp_path / "renders" / "spiral.mp4"
    w = entrypoint(["spiral", "--load-config", str(trained_run / "config.yml"), "--output-path", str(out), "--output-format", "images",
                    "--seconds", "0.5", "--frame-rate", "8", "--image-format", "png"])
    files = sorted((tmp_path / "renders" / "spiral").iterdir())
    assert w.count == len(files) == 4 and np.asarray(Image.open(files[0])).shape == (H, W, 3)
