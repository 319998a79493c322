"""The lens kernels (fnr_pixel_batch_lens, fnr_camera_rays_lens) against the torch restatement of data/camera_model.py,
against the pinhole kernels, and end to end: training, export and rendering of a distorted data set on disk."""
import json
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from fruitnerf_b200 import _lib as L
from fruitnerf_b200 import ops
from fruitnerf_b200.data import camera_model as cm
from fruitnerf_b200.data.synthetic_scene import look_at_c2w, make_apple_scene, write_dataset

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
COEFFS = {"none": None, "k1": [-0.12, 0, 0, 0, 0, 0], "k2": [0, 0.05, 0, 0, 0, 0], "k3": [0, 0, -0.01, 0, 0, 0], "k4": [0, 0, 0, 0.004, 0, 0],
          "p1": [0, 0, 0, 0, 0.0015, 0], "p2": [0, 0, 0, 0, 0, -0.001], "all": [-0.12, 0.05, -0.01, 0.004, 0.0015, -0.001],
          "strong": [-0.45, 0.25, -0.05, 0.0, 0.01, -0.01]}  # strong: the corners do not converge in 10 steps


def _cameras(F, per_frame, H=48, W=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    c2w = torch.stack([look_at_c2w(torch.randn(3, generator=g), torch.zeros(3)) for _ in range(F)]).float()
    base = torch.tensor([0.55 * W, 0.6 * W, W / 2 + 0.3, H / 2 - 0.2])
    intr = base * (1 + (0.05 * (2 * torch.rand(F, 4, generator=g) - 1) if per_frame else torch.zeros(F, 4)))
    return c2w, [intr[:, k].contiguous() for k in range(4)]


@pytest.mark.parametrize("camera_type", ["perspective", "fisheye", "equirectangular"])
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("coeffs", list(COEFFS))
def test_lens_kernels_match_the_restatement(native_lib, cuda_device, camera_type, per_frame, coeffs):
    F, H, W = 3, 48, 64
    c2w, intr = _cameras(F, per_frame, H, W)
    dist = None if COEFFS[coeffs] is None else torch.tensor(COEFFS[coeffs], dtype=torch.float32).expand(F, 6).contiguous()
    dev = [t.to(cuda_device) for t in intr]
    dd = None if dist is None else dist.to(cuda_device)
    p = torch.arange(H * W)
    for f in range(F):
        o, d = ops.camera_rays_lens(c2w.to(cuda_device), *dev, dd, camera_type, H, W, f, 0, H * W)
        o_ref, d_ref = cm.lens_rays(c2w[f], *(t[f] for t in intr), None if dist is None else dist[f], camera_type, p // W, p % W)
        assert torch.equal(o.cpu(), o_ref)
        err = float((d.cpu() - d_ref).abs().max())
        if camera_type == "perspective":
            # the fp64 Newton steps are op for op the restatement's and the rest is correctly rounded fp32: bit-identical
            assert err == 0.0, err
        assert err <= 2e-7, err  # fisheye / equirectangular: sincosf against the host's sin / cos
    # the training sampler draws the same rays
    N = F
    imgs, masks = torch.rand(N, H, W, 3, device=cuda_device), torch.rand(N, H, W, 1, device=cuda_device)
    r = torch.rand(4096, 3, device=cuda_device)
    o, d, cam, idx, img, m = ops.pixel_batch_lens(r, c2w.to(cuda_device), imgs, masks, *dev, dd, camera_type)
    i = idx.cpu()
    o_ref, d_ref = cm.lens_rays(c2w[i[:, 0]], *(t[i[:, 0]] for t in intr), None if dist is None else dist[i[:, 0]], camera_type, i[:, 1], i[:, 2])
    assert torch.equal(o.cpu(), o_ref) and float((d.cpu() - d_ref).abs().max()) <= 2e-7
    assert torch.equal(img, imgs[idx[:, 0], idx[:, 1], idx[:, 2]]) and torch.equal(m, masks[idx[:, 0], idx[:, 1], idx[:, 2]])


def test_pixel_batch_lens_without_a_lens_is_the_pinhole_kernel(native_lib, cuda_device):
    F, H, W = 7, 96, 128
    c2w, _ = _cameras(F, False, H, W)
    c2w = c2w.to(cuda_device)
    fx, fy, cx, cy = 1.1 * W, 1.05 * W, W / 2.0, H / 2.0
    imgs, masks = torch.rand(F, H, W, 3, device=cuda_device), torch.rand(F, H, W, 1, device=cuda_device)
    r = torch.rand(65536, 3, device=cuda_device)
    a = ops.pixel_batch(r, c2w, imgs, masks, fx, fy, cx, cy)
    arrays = [torch.full((F,), v, dtype=torch.float32, device=cuda_device) for v in (fx, fy, cx, cy)]
    b = ops.pixel_batch_lens(r, c2w, imgs, masks, *arrays, None, "perspective")
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("camera_type", ["perspective", "fisheye"])
def test_training_and_evaluation_rays_are_bit_identical(native_lib, cuda_device, camera_type):
    F, H, W = 4, 60, 80
    c2w, intr = _cameras(F, True, H, W, seed=3)
    c2w, intr = c2w.to(cuda_device), [t.to(cuda_device) for t in intr]
    dist = torch.tensor(COEFFS["all"], device=cuda_device).expand(F, 6).contiguous()
    imgs, masks = torch.rand(F, H, W, 3, device=cuda_device), torch.rand(F, H, W, 1, device=cuda_device)
    o, d, cam, idx, _, _ = ops.pixel_batch_lens(torch.rand(20000, 3, device=cuda_device), c2w, imgs, masks, *intr, dist, camera_type)
    for f in range(F):
        fo, fd = ops.camera_rays_lens(c2w, *intr, dist, camera_type, H, W, f, 0, H * W)
        sel = idx[:, 0] == f
        p = idx[sel, 1] * W + idx[sel, 2]
        assert torch.equal(fd[p], d[sel]) and torch.equal(fo[p], o[sel])


def test_lens_entries_refuse_bad_arguments(native_lib, cuda_device):
    lib = L.load()
    buf = torch.zeros(64, device=cuda_device)
    p = buf.data_ptr()

    def batch(fx=p, camera_type=L.FNR_CAMERA_PERSPECTIVE, num_rays=1):
        return lib.fnr_pixel_batch_lens(p, p, p, p, 1, 2, 2, fx, p, p, p, None, camera_type, num_rays, p, p, p, p, p, p, None)

    def rays(fx=p, camera_type=L.FNR_CAMERA_PERSPECTIVE, num_pixels=1):
        return lib.fnr_camera_rays_lens(p, fx, p, p, p, None, 1, camera_type, 2, 2, 0, 0, num_pixels, p, p, None)

    for call in (batch, rays):
        assert call() == 0
        assert call(fx=None) != 0 and "NULL" in lib.fnr_last_error().decode()
        assert call(camera_type=7) != 0 and "camera_type 7" in lib.fnr_last_error().decode()
    assert batch(num_rays=-1) != 0 and "fnr_pixel_batch_lens" in lib.fnr_last_error().decode()
    assert rays(num_pixels=-1) != 0 and "fnr_camera_rays_lens" in lib.fnr_last_error().decode()
    torch.cuda.synchronize()


def test_cuda_graph_training_on_a_distorted_data_set(native_lib, cuda_device):
    from fruitnerf_b200.scripts.train import synthetic_spec
    from fruitnerf_b200.trainer import Trainer

    torch.manual_seed(0)
    spec = synthetic_spec("fruit_nerf", rays_per_batch=2048)
    spec.pipeline.datamanager.synthetic_scene = dict(num_images=20, height=64, width=64, num_fruits=5, camera_type="fisheye",
                                                     distortion=COEFFS["all"], intrinsics_jitter=0.03)
    spec.pipeline.model.log2_hashmap_size = 17
    trainer = Trainer(spec, device=cuda_device, use_cuda_graph=True)
    assert trainer.pipeline.datamanager.train_dataset.cameras.has_lens
    trainer.train(5, log_every=10**9, eval_every=10**9)  # warm-up and capture
    torch.cuda.synchronize()
    # replays enqueue without waiting on the device: a host read of a device tensor would fail under this mode
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = [trainer.train_iteration(trainer.step + k)[0].clone() for k in range(100)]  # the graph reuses its output
    finally:
        torch.cuda.set_sync_debug_mode("default")
    trainer.step += 100
    assert len(trainer._graphs) >= 1
    first, last = float(torch.stack(losses[:10]).mean()), float(torch.stack(losses[-10:]).mean())
    assert last < 0.8 * first, (first, last)


@pytest.fixture(scope="module")
def lens_run(native_lib, cuda_device, tmp_path_factory):
    """A distorted, per-frame-jittered data set on disk, trained for 300 steps with `train --data`, and the same images
    trained as if the cameras were a shared pinhole."""
    root = tmp_path_factory.mktemp("lens")
    dist = [-0.22, 0.05, 0.0, 0.0, 0.0015, -0.001]
    full, _ = make_apple_scene(num_images=50, height=96, width=96, num_fruits=8, noise_std=0.01, distortion=dist, intrinsics_jitter=0.04,
                               elevations=(12.0, 30.0, 50.0))
    data = root / "data"
    write_dataset(full, data)
    meta = json.loads((data / "transforms.json").read_text())
    fx, fy, cx, cy = (float(t.mean()) for t in full.cameras.intrinsics())
    for f in meta["frames"]:
        for k in ("fl_x", "fl_y", "cx", "cy", "k1", "k2", "k3", "k4", "p1", "p2"):
            f.pop(k)
    meta.update(fl_x=fx, fl_y=fy, cx=cx, cy=cy, camera_model="PINHOLE")
    pinhole = root / "pinhole"
    pinhole.mkdir()
    for sub in ("images", "semantics"):
        (pinhole / sub).symlink_to(data / sub)
    (pinhole / "transforms.json").write_text(json.dumps(meta))
    out = {}
    for name, folder in (("lens", data), ("pinhole", pinhole)):
        run = root / f"run_{name}"
        r = subprocess.run([sys.executable, "-m", "fruitnerf_b200.scripts.train", "--data", str(folder), "--steps", "300", "--output-dir", str(run),
                            "--downscale-factor", "1"], cwd=ROOT, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        out[name] = (run, json.loads(r.stdout.strip().splitlines()[-1]))
    return out


def test_train_data_export_and_render_on_a_distorted_data_set(lens_run, tmp_path):
    run, res = lens_run["lens"]
    _, res_pin = lens_run["pinhole"]
    print(f"held-out PSNR after 300 steps: lens-aware {res['eval']['psnr']:.2f} dB, lens-ignored {res_pin['eval']['psnr']:.2f} dB")
    assert res["lens_distortion"] and res["camera_type"] == "perspective"
    # first H100 run: 15.83 dB (lens-ignored 15.69 dB; after 300 steps the model is still too blurred for the lens to matter much)
    assert res["eval"]["psnr"] > 14.0, res["eval"]
    assert (run / "config.yml").exists() and (run / "dataparser_transforms.json").exists()
    r = subprocess.run([sys.executable, "-m", "fruitnerf_b200.scripts.exporter", "pointcloud", "--load-config", str(run / "config.yml"),
                        "--output-dir", str(tmp_path / "pcd"), "--num-points", "20000", "--normal-method", "open3d"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert list((tmp_path / "pcd").rglob("*.ply"))
    r = subprocess.run([sys.executable, "-m", "fruitnerf_b200.scripts.render", "interpolate", "--load-config", str(run / "config.yml"),
                        "--output-path", str(tmp_path / "renders" / "interp.mp4"), "--output-format", "images", "--interpolation-steps", "2",
                        "--rendered-output-names", "rgb", "depth"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert len(list((tmp_path / "renders" / "interp").iterdir())) >= 2
