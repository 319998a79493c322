"""Host side of the `render` command: the camera models restated in torch, the camera paths (interpolation, pose order,
spiral, camera-path files), the CLI surface and its refusals, and the frame writers."""
import json
import math
import os
import stat

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation, Slerp

from fruitnerf_b200 import render as R
from fruitnerf_b200.data.synthetic_scene import look_at_c2w, make_apple_scene
from fruitnerf_b200.scripts import render as cli


def _cams(kind, H=9, W=14, fx=6.0, fy=5.0, cx=None, cy=None, c2w=None):
    c2w = torch.eye(4)[:3] if c2w is None else c2w
    return R.CameraSet(c2w[None], fx, fy, W / 2.0 if cx is None else cx, H / 2.0 if cy is None else cy, H, W, kind)


def _rand_pose(seed):
    g = torch.Generator().manual_seed(seed)
    return look_at_c2w(torch.randn(3, generator=g) * 2, torch.randn(3, generator=g) * 0.2).float()


@pytest.mark.parametrize("kind", ["perspective", "fisheye", "equirectangular"])
def test_principal_point_ray_is_the_camera_minus_z_axis(kind):
    c2w = _rand_pose(1)
    cams = _cams(kind, H=3, W=5, cx=2.5, cy=1.5, c2w=c2w)  # pixel (row 1, col 2) has its centre on the principal point
    o, d = R.restated_camera_rays(cams, 0, 7, 1)
    np.testing.assert_allclose(d[0].double().numpy(), -c2w[:3, 2].double().numpy(), atol=1e-6)
    np.testing.assert_allclose(o[0].double().numpy(), c2w[:3, 3].double().numpy(), atol=0)


@pytest.mark.parametrize("kind", ["perspective", "fisheye", "equirectangular"])
def test_directions_have_unit_norm(kind):
    cams = _cams(kind, H=31, W=47, fx=9.0, fy=7.5, c2w=_rand_pose(2))
    _, d = R.restated_camera_rays(cams, 0, 0, 31 * 47)
    np.testing.assert_allclose(d.double().norm(dim=-1).numpy(), 1.0, atol=1e-6)


def test_fisheye_angle_to_the_axis_is_radius_over_focal():
    f = 20.0
    cams = _cams("fisheye", H=1, W=101, fx=f, fy=f, cx=0.5, cy=0.5)  # column x sits x pixels right of the axis
    _, d = R.restated_camera_rays(cams, 0, 0, 101)
    ang = torch.acos((-d[:, 2]).clamp(-1, 1)).numpy()
    r = np.arange(101, dtype=np.float64)
    np.testing.assert_allclose(ang, np.minimum(r / f, np.pi), atol=1e-7)


def test_equirectangular_columns_are_azimuth_and_rows_elevation():
    H, W = 18, 36
    cams = _cams("equirectangular", H=H, W=W, fx=W / 2, fy=H)
    _, d = R.restated_camera_rays(cams, 0, 0, H * W)
    d = d.reshape(H, W, 3).numpy()
    u = (np.arange(W) + 0.5 - W / 2) / (W / 2)
    v = -(np.arange(H) + 0.5 - H / 2) / H
    az = np.arctan2(d[..., 0], -d[..., 2])  # 0 on the -z axis, positive to +x
    np.testing.assert_allclose(az[H // 2], np.pi * u, atol=1e-9)
    np.testing.assert_allclose(np.arcsin(d[:, 0, 1]), np.pi * v, atol=1e-9)  # elevation above the xz plane


def test_perspective_restatement_is_generate_rays_bit_for_bit():
    train, _ = make_apple_scene(num_images=10, height=23, width=37, num_fruits=2, noise_std=0.0)
    cams = train.cameras
    cs = R.CameraSet.from_cameras(cams)
    for i in (0, 4):
        ref = cams.generate_rays(i)
        for p0, n in ((0, 23 * 37), (36, 2), (37 * 5 - 3, 200), (23 * 37 - 1, 1)):
            o, d = R.restated_camera_rays(cs, i, p0, n)
            assert torch.equal(d, ref.directions.reshape(-1, 3)[p0:p0 + n])
            assert torch.equal(o, ref.origins.reshape(-1, 3)[p0:p0 + n])


def _ring(n, radius=2.0):
    poses = []
    for i in range(n):
        a = 2 * math.pi * i / n
        eye = torch.tensor([radius * math.cos(a), radius * math.sin(a), 0.5 + 0.1 * math.sin(3 * a)])
        poses.append(look_at_c2w(eye, torch.zeros(3)))
    return torch.stack(poses).float()


def _Ks(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    K = torch.zeros(n, 3, 3)
    K[:, 0, 0], K[:, 1, 1] = 50 + 10 * torch.rand(n, generator=g), 55 + 10 * torch.rand(n, generator=g)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 32.0, 24.0, 1.0
    return K


def test_interpolation_matches_scipy_slerp():
    poses, Ks, steps = _ring(6), _Ks(6), 7
    traj, k = R.get_interpolated_poses_many(poses, Ks, steps)
    assert traj.shape == (steps * 5, 3, 4) and k.shape == (steps * 5, 3, 3)
    ts = np.linspace(0, 1, steps)
    for i in range(5):
        rots = Rotation.from_matrix(poses[i:i + 2, :, :3].double().numpy())
        want = Slerp([0, 1], rots)(ts).as_matrix()
        got = traj[i * steps:(i + 1) * steps, :, :3].double().numpy()
        np.testing.assert_allclose(got, want, atol=1e-6)
        tr = (1 - ts)[:, None] * poses[i, :, 3].double().numpy() + ts[:, None] * poses[i + 1, :, 3].double().numpy()
        np.testing.assert_allclose(traj[i * steps:(i + 1) * steps, :, 3].double().numpy(), tr, atol=1e-6)
        np.testing.assert_allclose(k[i * steps:(i + 1) * steps].double().numpy(),
                                   (1 - ts)[:, None, None] * Ks[i].double().numpy() + ts[:, None, None] * Ks[i + 1].double().numpy(), atol=1e-5)
        # both endpoints reproduce the input cameras (interior cameras appear twice)
        np.testing.assert_allclose(traj[i * steps].numpy(), poses[i].numpy(), atol=1e-6)
        np.testing.assert_allclose(traj[(i + 1) * steps - 1].numpy(), poses[i + 1].numpy(), atol=1e-6)


def test_order_poses_restores_a_shuffled_ring():
    n = 9
    ring = _ring(n)
    perm = [0, *np.random.default_rng(3).permutation(np.arange(1, n)).tolist()]
    shuffled, Ks = ring[perm], _Ks(n)[perm]
    ordered, ok = R.get_ordered_poses_and_k(shuffled, Ks)
    order = [perm.index(i) for i in range(n)]
    if not torch.equal(ordered[1], ring[1]):  # the greedy walk may go round either way
        order = [perm.index(i) for i in [0, *range(n - 1, 0, -1)]]
    assert torch.equal(ordered, shuffled[order]) and torch.equal(ok, Ks[order])
    traj, _ = R.get_interpolated_poses_many(shuffled, Ks, 3, order_poses=True)
    assert torch.allclose(traj[3], shuffled[order[1]], atol=1e-6)


def test_spiral_positions_and_orthonormal_rotations():
    c2w = _rand_pose(5)
    cams = R.CameraSet(c2w[None], 80.0, 90.0, 40.0, 30.0, 60, 80)
    steps, radius = 24, 0.3
    path = R.get_spiral_path(cams, 0, steps=steps, radius=radius)
    assert len(path) == steps and (path.height, path.width) == (60, 80)
    t = np.linspace(0, 2 * np.pi, steps + 1)[:-1]
    centres = radius * np.stack([np.cos(t), -np.sin(t), -np.sin(0.5 * t)], axis=1)
    Rs, ts = c2w[:3, :3].double().numpy(), c2w[:3, 3].double().numpy()
    np.testing.assert_allclose(path.camera_to_worlds[:, :, 3].double().numpy(), centres @ Rs.T + ts, atol=1e-6)
    rot = path.camera_to_worlds[:, :, :3].double()
    np.testing.assert_allclose((rot.transpose(1, 2) @ rot).numpy(), np.broadcast_to(np.eye(3), (steps, 3, 3)), atol=1e-6)
    np.testing.assert_allclose(torch.linalg.det(rot).numpy(), 1.0, atol=1e-6)
    # every camera looks at (0, 0, -min(fx, fy)) of the start camera's frame
    target = Rs @ np.array([0, 0, -80.0]) + ts
    look = -rot[:, :, 2].numpy()
    to_target = target - path.camera_to_worlds[:, :, 3].double().numpy()
    np.testing.assert_allclose(look, to_target / np.linalg.norm(to_target, axis=1, keepdims=True), atol=1e-6)


def _path_json(camera_type=None, fovs=(50.0, 70.0), H=60, W=100, **extra):
    d = {"render_height": H, "render_width": W, "seconds": 2.0,
         "camera_path": [{"camera_to_world": torch.eye(4).flatten().tolist(), "fov": f} for f in fovs]}
    if camera_type is not None:
        d["camera_type"] = camera_type
    d.update(extra)
    return d


def test_path_from_json_known_answers():
    cams = R.get_path_from_json(_path_json())
    assert cams.camera_type == "perspective" and (cams.height, cams.width) == (60, 100) and len(cams) == 2
    want = 30.0 / np.tan(np.radians([50.0, 70.0]) / 2)
    np.testing.assert_allclose(cams.fx.numpy(), want, rtol=1e-6)
    assert torch.equal(cams.fx, cams.fy)
    assert cams.cx.tolist() == [50.0, 50.0] and cams.cy.tolist() == [30.0, 30.0]
    assert R.path_fps(_path_json(), 2) == 1.0
    eq = R.get_path_from_json(_path_json("equirectangular"))
    assert eq.fx.tolist() == [50.0, 50.0] and eq.fy.tolist() == [60.0, 60.0] and eq.camera_type == "equirectangular"
    assert R.get_path_from_json(_path_json("fisheye")).camera_type == "fisheye"
    t = torch.eye(4)
    t[:3, 3] = torch.tensor([1.0, 2.0, 3.0])
    one = R.get_path_from_json({"render_height": 4, "render_width": 6, "camera_path": [{"camera_to_world": t.flatten().tolist(), "fov": 90}]})
    assert torch.equal(one.camera_to_worlds[0], t[:3])


def test_cli_defaults_and_option_names():
    ap = cli.build_parser()
    a = ap.parse_args(["camera-path", "--load-config", "run/config.yml"])
    assert (a.output_path.as_posix(), a.image_format, a.jpeg_quality, a.downscale_factor, a.eval_num_rays_per_chunk) == \
        ("renders/output.mp4", "jpeg", 100, 1.0, None)
    assert (a.rendered_output_names, a.depth_near_plane, a.depth_far_plane, a.output_format) == (["rgb"], None, None, "video")
    assert a.camera_path_filename.as_posix() == "camera_path.json"
    a = ap.parse_args(["interpolate", "--load-config", "c.yml"])
    assert (a.pose_source, a.interpolation_steps, a.order_poses, a.frame_rate) == ("eval", 10, False, 24)
    a = ap.parse_args(["interpolate", "--load-config", "c.yml", "--order-poses", "--pose-source", "train", "--rendered-output-names", "rgb",
                       "depth", "--output-format", "images", "--image-format", "png"])
    assert a.order_poses and a.pose_source == "train" and a.rendered_output_names == ["rgb", "depth"] and a.image_format == "png"
    a = ap.parse_args(["spiral", "--load-config", "c.yml"])
    assert (a.seconds, a.frame_rate, a.radius) == (3.0, 24, 0.1)
    with pytest.raises(SystemExit):
        ap.parse_args(["spiral", "--load-config", "c.yml", "--output-format", "gif"])


class _StubModel:
    device = torch.device("cpu")

    def __call__(self, bundle):
        n = bundle.origins.shape[0]
        return {"rgb": torch.zeros(n, 3), "depth": torch.zeros(n, 1), "weights_list": []}


class _StubPipeline:
    model = _StubModel()
    datamanager = None


def test_unknown_output_name_exits_with_1_and_lists_the_keys(tmp_path, capsys):
    f = tmp_path / "path.json"
    f.write_text(json.dumps(_path_json()))
    args = ["camera-path", "--load-config", str(tmp_path / "none.yml"), "--camera-path-filename", str(f), "--output-format", "images",
            "--output-path", str(tmp_path / "out.mp4"), "--rendered-output-names", "rgb", "normals"]
    with pytest.raises(SystemExit) as e:
        cli.entrypoint(args, pipeline=_StubPipeline())
    assert e.value.code == 1
    err = capsys.readouterr().err
    assert "normals" in err and "'rgb'" in err and "'depth'" in err and "weights_list" not in err
    assert not (tmp_path / "out").exists()


@pytest.mark.parametrize("change, match", [
    (dict(crop={"crop_bg_color": {"r": 0, "g": 0, "b": 0}, "crop_center": [0, 0, 0], "crop_scale": [1, 1, 1]}), "crop"),
    (dict(camera_type="omnidirectional"), "omnidirectional"),
    (dict(camera_type="vr180"), "vr180"),
    ("time", "time"),
    ("distortion", "distortion"),
])
def test_refused_camera_paths(tmp_path, change, match):
    d = _path_json()
    if change == "time":
        for i, c in enumerate(d["camera_path"]):
            c["render_time"] = i / 2
    elif change == "distortion":
        d["camera_path"][0]["distortion_params"] = [0.1, 0, 0, 0, 0, 0]
    else:
        d.update(change)
    with pytest.raises(NotImplementedError, match=match):
        R.get_path_from_json(d)
    f = tmp_path / "path.json"
    f.write_text(json.dumps(d))
    # refused before the (missing) run folder is read
    with pytest.raises(NotImplementedError, match=match):
        cli.entrypoint(["camera-path", "--load-config", str(tmp_path / "missing" / "config.yml"), "--camera-path-filename", str(f),
                        "--output-format", "images"])


def test_camera_path_with_crop_null_is_accepted():
    assert len(R.get_path_from_json(_path_json(crop=None))) == 2


def _stub_ffmpeg(bin_dir, log):
    exe = bin_dir / "ffmpeg"
    exe.write_text(f'#!/bin/sh\nprintf "%s\\n" "$@" > "{log}.args"\ncat > "{log}.raw"\n')
    exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    return exe


def test_video_frames_are_piped_to_ffmpeg(tmp_path, monkeypatch):
    bin_dir = tmp_path / "bin"
    bin_dir.mkdir()
    log = tmp_path / "ffmpeg"
    _stub_ffmpeg(bin_dir, log)
    monkeypatch.setenv("PATH", str(bin_dir) + os.pathsep + os.environ.get("PATH", ""))
    H, W, n, fps = 6, 10, 5, 12.5
    frames = [np.full((H, W, 3), i * 40, dtype=np.uint8) for i in range(n)]
    frames[2][1, 3] = (1, 2, 3)
    w = R.FrameWriter(tmp_path / "out" / "video.mp4", "video", fps=fps)
    for fr in frames:
        w(fr)
    w.close()
    raw = (tmp_path / "ffmpeg.raw").read_bytes()
    assert len(raw) == n * H * W * 3 and raw == b"".join(f.tobytes() for f in frames)
    args = (tmp_path / "ffmpeg.args").read_text().split("\n")
    assert args[args.index("-s") + 1] == f"{W}x{H}" and args[args.index("-r") + 1] == "12.5"
    assert args[args.index("-pix_fmt") + 1] == "rgb24" and str(tmp_path / "out" / "video.mp4") in args


def test_video_without_ffmpeg_fails_before_rendering(tmp_path, monkeypatch):
    monkeypatch.setenv("PATH", str(tmp_path))
    with pytest.raises(SystemExit) as e:
        cli.entrypoint(["spiral", "--load-config", str(tmp_path / "missing.yml")])
    assert "--output-format images" in str(e.value.code)
    with pytest.raises(SystemExit):
        R.FrameWriter(tmp_path / "v.mp4", "video")


@pytest.mark.parametrize("fmt, ext", [("png", "png"), ("jpeg", "jpg")])
def test_image_frames_are_written_under_the_output_stem(tmp_path, fmt, ext):
    from PIL import Image

    frames = [np.random.default_rng(i).integers(0, 256, (5, 7, 3), dtype=np.uint8) for i in range(3)]
    w = R.FrameWriter(tmp_path / "r" / "interp.mp4", "images", fmt, jpeg_quality=100)
    for fr in frames:
        w(fr)
    w.close()
    files = sorted(os.listdir(tmp_path / "r" / "interp"))
    assert files == [f"{i:05d}.{ext}" for i in range(3)]
    img = np.asarray(Image.open(tmp_path / "r" / "interp" / files[1]))
    assert img.shape == (5, 7, 3)
    if fmt == "png":
        assert np.array_equal(img, frames[1])


def test_frame_kinds_follow_ns_render():
    assert R.frame_kind("rgb", 3) == "color" and R.frame_kind("semantics_colormap", 3) == "color"
    assert R.frame_kind("accumulation", 1) == "turbo" and R.frame_kind("semantics", 1) == "turbo"
    assert R.frame_kind("depth", 1) == "depth" and R.frame_kind("prop_depth_0", 1) == "depth"
    with pytest.raises(NotImplementedError):
        R.frame_kind("features", 8)
    assert R.plane_or_auto(0.0) is None and R.plane_or_auto(None) is None and R.plane_or_auto(0.5) == 0.5
