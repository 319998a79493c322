"""The `tsdf` mesh export on the host: the triangle table (closed, orientable meshes on analytic and random fields), the
numpy marching cubes, the torch TSDF fusion against a per-voxel loop, the mesh PLY format, the CLI options and the C-ABI
refusals of fnr_mesh.cu (these return before any launch, so they run without a GPU)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from fruitnerf_b200 import mesh as M


def grid(n, lo=-0.5, hi=0.5):
    """Grid points in [lo, hi]^3 with n points per axis: (X, Y, Z fp64, origin, voxel size)."""
    vs = (hi - lo) / (n - 1)
    g = lo + np.arange(n) * vs
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    return X, Y, Z, lo, vs


def edge_counts(faces):
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    _, directed = np.unique(d, axis=0, return_counts=True)
    _, undirected = np.unique(np.sort(d, axis=1), axis=0, return_counts=True)
    return directed, undirected


def assert_closed_orientable(faces):
    directed, undirected = edge_counts(faces)
    assert (undirected == 2).all(), np.bincount(undirected)
    assert (directed == 1).all(), np.bincount(directed)


def euler(m):
    _, undirected = edge_counts(m["faces"])
    return len(m["vertices"]) - len(undirected) + len(m["faces"])


def test_header_is_the_generated_table():
    assert M.TABLE_HEADER.read_text() == M.table_header_text()
    counts, table = M.triangle_table()
    assert counts[0] == counts[255] == 0 and counts.max() <= M.MAX_CELL_TRIANGLES
    for case in range(256):  # no triangle repeats an edge, so allow_degenerate=False never drops one
        t = table[case, : counts[case]]
        assert (t >= 0).all() and all(len(set(row)) == 3 for row in t.tolist())


def test_every_case_alone_is_a_closed_surface():
    """Each case in a 4^3 grid whose other points are outside: the cell's surface must close."""
    for case in range(1, 255):
        v = np.ones((4, 4, 4), np.float32)
        for c in range(8):
            dx, dy, dz = M.corner_offset(c)
            v[1 + dx, 1 + dy, 1 + dz] = -1.0 if case >> c & 1 else 1.0
        assert_closed_orientable(M.marching_cubes_numpy(v, 0.0, 1.0)["faces"])


def test_sphere():
    n, r = 48, 0.37
    X, Y, Z, lo, vs = grid(n)
    rad = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    m = M.marching_cubes_numpy((rad - r).astype(np.float32), lo, vs)
    V, F = m["vertices"].astype(np.float64), m["faces"]
    assert len(F) > 1000
    assert_closed_orientable(F)
    assert euler(m) == 2
    rr = np.linalg.norm(V, axis=1)
    assert np.abs(rr / r - 1).max() < 0.01
    a, b, c = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6
    assert abs(vol / (4 / 3 * math.pi * r ** 3) - 1) < 0.02
    assert (np.einsum("ij,ij->i", m["normals"], V / rr[:, None]) > 0.9).all()
    face_n = np.cross(b - a, c - a)
    vert_n = m["normals"][F].sum(axis=1)
    assert (np.einsum("ij,ij->i", face_n, vert_n) > 0).all()  # winding agrees with the gradient normal


def test_torus():
    X, Y, Z, lo, vs = grid(64)
    R, r = 0.3, 0.1
    q = np.sqrt(X ** 2 + Y ** 2) - R
    m = M.marching_cubes_numpy((np.sqrt(q ** 2 + Z ** 2) - r).astype(np.float32), lo, vs)
    assert_closed_orientable(m["faces"])
    assert euler(m) == 0


def test_plane_vertices_are_exact():
    n = 17
    vs = np.float32(1 / 16)
    k = np.arange(n, dtype=np.float32)
    z = np.float32(-0.5) + k * vs
    level = np.float32(0.3)
    v = np.broadcast_to((z - level)[None, None, :], (n, n, n)).astype(np.float32)
    m = M.marching_cubes_numpy(v, -0.5, vs)
    assert len(m["vertices"]) == n * n and len(m["faces"]) == 2 * (n - 1) ** 2
    # exactly the fp32 arithmetic of the kernel: s = -v_a / (v_b - v_a), coord = k_a + s, world = origin + coord * vs
    ka = int(np.flatnonzero(z - level < 0).max())
    s = (np.float32(0) - v[0, 0, ka]) / (v[0, 0, ka + 1] - v[0, 0, ka])
    want = np.float32(-0.5) + (np.float32(ka) + s) * vs
    assert (m["vertices"][:, 2] == want).all()
    assert abs(float(want) - 0.3) < 4 * np.finfo(np.float32).eps
    np.testing.assert_array_equal(m["normals"], np.tile(np.float32([0, 0, 1]), (n * n, 1)))


def test_constant_grids_are_empty():
    for val in (1.0, -1.0, 0.0):
        m = M.marching_cubes_numpy(np.full((5, 6, 7), val, np.float32), 0.0, 1.0)
        assert m["vertices"].shape == (0, 3) and m["faces"].shape == (0, 3)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_field_is_closed_and_orientable(seed):
    """Ambiguous faces and cells galore: a table that resolves a face differently in the two cells sharing it leaves holes."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((24, 25, 26)).astype(np.float32)
    v[[0, -1]] = 1
    v[:, [0, -1]] = 1
    v[:, :, [0, -1]] = 1
    m = M.marching_cubes_numpy(v, 0.0, 1.0)
    assert len(m["faces"]) > 10000
    assert_closed_orientable(m["faces"])


def test_attributes_come_from_the_nearest_grid_point():
    rng = np.random.default_rng(3)
    v = rng.standard_normal((6, 7, 8)).astype(np.float32)
    col = rng.uniform(size=(6, 7, 8, 3)).astype(np.float32)
    fr = rng.uniform(size=(6, 7, 8)).astype(np.float32)
    m = M.marching_cubes_numpy(v, (1.0, 2.0, 3.0), (0.5, 0.25, 0.125), col, fr)
    coord = (m["vertices"] - np.float32([1, 2, 3])) / np.float32([0.5, 0.25, 0.125])
    near = tuple(np.round(coord).astype(np.int64).T)
    np.testing.assert_array_equal(m["colors"], col[near])
    np.testing.assert_array_equal(m["fruit"], fr[near])
    assert m["faces"].max() < len(m["vertices"])


# ---- TSDF fusion ------------------------------------------------------------------------------------------------------
def camera(eye=(0.0, 0.0, 2.0)):
    """c2w [1,3,4] looking down -z from ``eye`` (OpenGL axes)."""
    c2w = torch.zeros(1, 3, 4)
    c2w[0, :, :3] = torch.eye(3)
    c2w[0, :, 3] = torch.tensor(eye)
    return c2w


def naive_integrate(state, origin, vs, trunc, c2w, fx, fy, cx, cy, depth, rgb, fruit):
    """Per voxel, per frame, with numpy fp32 scalars: the sequential update as the issue states it."""
    f = np.float32
    values, weights, colors, fst = (s.numpy() for s in state)
    X, Y, Z = values.shape
    B, H, W = depth.shape
    for i, j, k in np.ndindex(X, Y, Z):
        x = [f(origin[a]) + f(idx) * f(vs[a]) for a, idx in enumerate((i, j, k))]
        for b in range(B):
            m = c2w[b].numpy().astype(np.float32)
            d = [f(x[r]) - m[r, 3] for r in range(3)]
            p = [(m[0, c] * d[0] + m[1, c] * d[1]) + m[2, c] * d[2] for c in range(3)]
            zc = -p[2]
            if not zc > 0:
                continue
            u = f(cx[b]) + (f(fx[b]) * p[0]) / zc
            v = f(cy[b]) - (f(fy[b]) * p[1]) / zc
            if not (0 <= u < W and 0 <= v < H):
                continue
            col, row = int(np.floor(u)), int(np.floor(v))
            t = f(depth[b, row, col])
            if not t > 0:
                continue
            a_ = (f(col) + f(0.5) - f(cx[b])) / f(fx[b])
            b_ = (f(row) + f(0.5) - f(cy[b])) / f(fy[b])
            zpix = t / np.sqrt((a_ * a_ + b_ * b_) + f(1))
            sdf = zpix - zc
            if not sdf > -f(trunc):
                continue
            tsdf = min(max(sdf / f(trunc), f(-1)), f(1))
            w = weights[i, j, k]
            w1 = w + f(1)
            values[i, j, k] = (values[i, j, k] * w + tsdf) / w1
            colors[i, j, k] = (colors[i, j, k] * w + rgb[b, row, col].numpy()) / w1
            fst[i, j, k] = (fst[i, j, k] * w + f(fruit[b, row, col])) / w1
            weights[i, j, k] = w1


def test_restated_fusion_equals_the_per_voxel_loop():
    g = torch.Generator().manual_seed(0)
    tsdf = M.TSDF.from_aabb([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5]], 8)
    ref = M.TSDF.from_aabb([[-0.5, -0.5, -0.5], [0.5, 0.5, 0.5]], 8)
    c2w = torch.cat([camera((0.05, -0.02, 1.2)), camera((-0.1, 0.07, 1.1))])
    c2w[1, :, :3] = torch.tensor([[0.9950042, 0.0, 0.0998334], [0.0, 1.0, 0.0], [-0.0998334, 0.0, 0.9950042]])
    H, W = 12, 10
    fx, fy, cx, cy = torch.tensor([9.0, 8.5]), torch.tensor([9.5, 9.0]), torch.tensor([5.0, 4.7]), torch.tensor([6.0, 6.2])
    depth = 1.0 + 0.5 * torch.rand(2, H, W, generator=g)
    depth[0, 0, 0] = 0.0
    rgb, fruit = torch.rand(2, H, W, 3, generator=g), torch.rand(2, H, W, generator=g)
    tsdf.integrate(c2w, fx, fy, cx, cy, depth, rgb, fruit)
    naive_integrate((ref.values, ref.weights, ref.colors, ref.fruit), ref.origin.numpy(), ref.voxel_size.numpy(), ref.truncation, c2w,
                    fx.numpy(), fy.numpy(), cx.numpy(), cy.numpy(), depth.numpy(), rgb, fruit.numpy())
    assert int((tsdf.weights > 0).sum()) > 100 and int((tsdf.weights == 2).sum()) > 50
    for name in ("values", "weights", "colors", "fruit"):
        assert torch.equal(getattr(tsdf, name), getattr(ref, name)), name


def plane_frame(D, H=16, W=16, f=12.0):
    """Depth map of a plane at depth D along the optical axis, as ray distances of the pixel-centre rays."""
    cx, cy = W / 2, H / 2
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    a, b = (xs + 0.5 - cx) / f, (ys + 0.5 - cy) / f
    return torch.tensor(D * np.sqrt(a * a + b * b + 1), dtype=torch.float32)[None], (f, f, cx, cy)


def test_plane_gives_the_clamped_signed_distance():
    tsdf = M.TSDF.from_aabb([[-0.2, -0.2, -0.5], [0.2, 0.2, 0.5]], 16)
    depth, (fx, fy, cx, cy) = plane_frame(2.0)  # the plane z = 0 seen from z = 2
    tsdf.integrate(camera(), [fx], [fy], [cx], [cy], depth, torch.rand(1, 16, 16, 3))
    z = tsdf.origin[2] + torch.arange(16, dtype=torch.float32) * tsdf.voxel_size[2]
    zc = 2.0 - z
    want = torch.clamp((2.0 - zc) / tsdf.truncation, -1, 1)
    seen = tsdf.weights > 0
    behind = (2.0 - zc) <= -tsdf.truncation
    for k in range(16):
        sl = seen[:, :, k]
        if bool(behind[k]):
            assert not bool(sl.any())  # behind the truncation band: untouched
            assert bool((tsdf.values[:, :, k] == -1).all())
        else:
            assert bool(sl.all())
            torch.testing.assert_close(tsdf.values[:, :, k][sl], want[k].expand(int(sl.sum())), atol=1e-5, rtol=0)
    assert tsdf.truncation == pytest.approx(5 * 0.4 / 16)


def test_off_image_voxels_are_untouched_and_frames_average_with_count_weights():
    tsdf = M.TSDF.from_aabb([[-3.0, -3.0, -0.1], [3.0, 3.0, 0.1]], [32, 32, 4])
    depth, (fx, fy, cx, cy) = plane_frame(2.0)
    rgb_a, rgb_b = torch.full((1, 16, 16, 3), 0.2), torch.full((1, 16, 16, 3), 0.8)
    fr_a, fr_b = torch.zeros(1, 16, 16), torch.ones(1, 16, 16)
    tsdf.integrate(camera(), [fx], [fy], [cx], [cy], depth, rgb_a, fr_a)
    tsdf.integrate(camera(), [fx], [fy], [cx], [cy], depth, rgb_b, fr_b)
    tsdf.integrate(camera(), [fx], [fy], [cx], [cy], depth, rgb_b, fr_b)
    seen = tsdf.weights > 0
    assert 0 < int(seen.sum()) < seen.numel()
    assert bool((tsdf.weights[seen] == 3).all())
    assert bool((tsdf.values[~seen] == -1).all()) and bool((tsdf.colors[~seen] == 0).all())
    torch.testing.assert_close(tsdf.colors[seen], torch.full_like(tsdf.colors[seen], (0.2 + 0.8 + 0.8) / 3))
    torch.testing.assert_close(tsdf.fruit[seen], torch.full_like(tsdf.fruit[seen], 2 / 3))
    # the corner voxels project off the 16x16 image
    x = tsdf.origin[0] + 31 * tsdf.voxel_size[0]
    assert abs(float(cx + fx * x / 2.0)) > 16 and not bool(seen[31, 31].any())


def test_pixel_boundary_picks_floor():
    """A voxel projecting exactly onto the boundary between pixel columns 7 and 8 reads column 8 (floor u = 8)."""
    tsdf = M.TSDF.from_aabb([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]], 2)
    depth = torch.full((1, 16, 16), 2.0)
    depth[:, :, 8] = 2.25  # only column 8 has the plane 0.25 further away
    c2w = camera((0.0, 0.0, 2.0))
    tsdf.integrate(c2w, [10.0], [10.0], [8.0], [8.0], depth, torch.rand(1, 16, 16, 3))
    # grid point (0, 0, 0) projects to u = 8 exactly, v = 8 exactly
    assert float(tsdf.weights[0, 0, 0]) == 1
    a = np.float32(0.5) / np.float32(10.0)
    zpix = np.float32(2.25) / np.sqrt(np.float32(a * a + a * a) + np.float32(1))
    assert float(tsdf.values[0, 0, 0]) == pytest.approx(min(max((float(zpix) - 2.0) / tsdf.truncation, -1), 1), abs=1e-6)


def test_tsdf_refuses_bad_grids():
    with pytest.raises(ValueError):
        M.TSDF.from_aabb([[0, 0, 0], [1, 1, 1]], 1)
    with pytest.raises(ValueError):
        M.TSDF.from_aabb([[0, 0, 0], [1, 0, 1]], 8)
    with pytest.raises(ValueError):
        M.marching_cubes_numpy(np.zeros((1, 4, 4), np.float32), 0, 1)


def test_fruit_submesh_keeps_order_and_compacts():
    v = np.arange(15, dtype=np.float32).reshape(5, 3)
    fr = np.array([0.9, 0.1, 0.6, 0.5, 0.7], np.float32)
    faces = np.array([[0, 2, 3], [0, 1, 2], [3, 4, 2]])
    fv, fn, fc, ff, fidx = M.fruit_submesh(v, v, None, fr, faces)
    np.testing.assert_array_equal(fv, v[[0, 2, 3, 4]])
    np.testing.assert_array_equal(fidx, [[0, 1, 2], [2, 3, 1]])
    assert fc is None and ff.tolist() == fr[[0, 2, 3, 4]].tolist()
    assert M.fruit_submesh(v, v, None, np.zeros(5), faces)[4].shape == (0, 3)


# ---- PLY ----------------------------------------------------------------------------------------------------------------
def test_mesh_ply_round_trip(tmp_path):
    from fruitnerf_b200.export.exporter_utils import read_mesh_ply, write_mesh_ply

    rng = np.random.default_rng(0)
    v, n, c = rng.standard_normal((50, 3)), rng.standard_normal((50, 3)), rng.uniform(size=(50, 3))
    f = rng.integers(0, 50, (70, 3))
    write_mesh_ply(tmp_path / "m.ply", v, n, c, f)
    v2, n2, c2, f2 = read_mesh_ply(tmp_path / "m.ply")
    np.testing.assert_array_equal(v2, v)
    np.testing.assert_array_equal(n2, n)
    np.testing.assert_array_equal(c2, np.clip(c * 255, 0, 255).astype(np.uint8) / 255.0)
    np.testing.assert_array_equal(f2, f)
    write_mesh_ply(tmp_path / "e.ply", np.zeros((0, 3)), np.zeros((0, 3)), None, np.zeros((0, 3)))
    v3, _, _, f3 = read_mesh_ply(tmp_path / "e.ply")
    assert v3.shape == (0, 3) and f3.shape == (0, 3)
    with pytest.raises(ValueError):
        write_mesh_ply(tmp_path / "b.ply", v, n, c, [[0, 1, 50]])


def test_mesh_ply_bytes_of_one_triangle(tmp_path):
    from fruitnerf_b200.export.exporter_utils import write_mesh_ply

    write_mesh_ply(tmp_path / "t.ply", [[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 0, 1]] * 3, [[1, 0, 0], [0, 1, 0], [0, 0, 0.5]], [[0, 1, 2]])
    data = (tmp_path / "t.ply").read_bytes()
    header = (b"ply\nformat binary_little_endian 1.0\ncomment fruitnerf_b200 export\nelement vertex 3\n"
              b"property double x\nproperty double y\nproperty double z\nproperty double nx\nproperty double ny\nproperty double nz\n"
              b"property uchar red\nproperty uchar green\nproperty uchar blue\nelement face 1\n"
              b"property list uchar int vertex_indices\nend_header\n")
    assert data.startswith(header)
    body = data[len(header):]
    assert len(body) == 3 * (6 * 8 + 3) + 13
    assert body[48:51] == bytes([255, 0, 0]) and body[2 * 51 + 48:3 * 51] == bytes([0, 0, 127])
    assert body[-13:] == bytes([3]) + np.array([0, 1, 2], "<i4").tobytes()


# ---- CLI ----------------------------------------------------------------------------------------------------------------
def test_cli_defaults():
    import argparse

    from fruitnerf_b200.scripts.exporter import add_tsdf_parser, tsdf_exporter_from_args

    sub = argparse.ArgumentParser().add_subparsers(dest="command")
    p = add_tsdf_parser(sub)
    exp = tsdf_exporter_from_args(p.parse_args(["--load-config", "c.yml", "--output-dir", "o"]))
    assert exp.downscale_factor == 2 and exp.depth_output_name == "depth" and exp.rgb_output_name == "rgb"
    assert list(exp.resolution) == [128] and exp.batch_size == 10 and exp.use_bounding_box is True
    assert tuple(exp.bounding_box_min) == (-1, -1, -1) and tuple(exp.bounding_box_max) == (1, 1, 1)
    assert exp.refine_mesh_using_initial_aabb_estimate is False and exp.refinement_epsilon == 1e-2
    assert exp.texture_method == "tsdf"
    exp.validate()
    a = p.parse_args(["--load-config", "c", "--output-dir", "o", "--resolution", "64", "32", "16", "--refine-mesh-using-initial-aabb-estimate",
                      "true", "--use-bounding-box", "false"])
    exp = tsdf_exporter_from_args(a)
    exp.validate()
    assert list(exp.resolution) == [64, 32, 16] and exp.refine_mesh_using_initial_aabb_estimate and not exp.use_bounding_box


@pytest.mark.parametrize("args, match", [
    (["--texture-method", "nerf"], "xatlas"),
    (["--resolution", "1"], "resolution"),
    (["--resolution", "64", "64"], "resolution"),
    (["--downscale-factor", "0"], "downscale"),
    (["--bounding-box-min", "0", "0", "0", "--bounding-box-max", "1", "0", "1"], "Bounding box"),
])
def test_cli_refusals(args, match, capsys, tmp_path):
    from fruitnerf_b200.scripts.exporter import entrypoint

    with pytest.raises(SystemExit) as e:
        entrypoint(["tsdf", "--load-config", str(tmp_path / "missing.yml"), "--output-dir", str(tmp_path / "out"), *args])
    assert e.value.code == 2
    assert match in capsys.readouterr().err
    assert not (tmp_path / "out").exists()


def test_fisheye_cameras_are_refused():
    from fruitnerf_b200.data.synthetic_scene import SyntheticCameras
    from fruitnerf_b200.export.exporter_utils import tsdf_cameras

    c2w = camera()
    for kind in ("fisheye", "equirectangular"):
        cams = SyntheticCameras(c2w, torch.tensor([10.0]), torch.tensor([10.0]), torch.tensor([8.0]), torch.tensor([8.0]), 16, 16, kind)
        with pytest.raises(ValueError, match="perspective"):
            tsdf_cameras(cams)
    cams = SyntheticCameras(c2w, 10.0, 12.0, 8.0, 6.0, 16, 20)
    rc = tsdf_cameras(cams, 2)
    assert (rc.height, rc.width) == (8, 10) and float(rc.fx[0]) == 5.0 and float(rc.cy[0]) == 3.0


# ---- C ABI --------------------------------------------------------------------------------------------------------------
def test_cabi_refusals(native_lib):
    lib = native_lib
    o3 = (C.c_float * 3)(0, 0, 0)
    v3 = (C.c_float * 3)(0.1, 0.1, 0.1)
    bad_v = (C.c_float * 3)(0.1, 0.0, 0.1)
    nan_v = (C.c_float * 3)(0.1, float("nan"), 0.1)
    P = 16  # any non-NULL address: nothing is dereferenced on a refusal

    def tsdf(**kw):
        a = dict(values=P, weights=P, colors=P, fruit=None, nx=4, ny=4, nz=4, origin=o3, vs=v3, trunc=0.5, c2w=P, fx=P, fy=P, cx=P, cy=P,
                 depth=P, rgb=P, frame_fruit=None, B=0, H=8, W=8)
        a.update(kw)
        return lib.fnr_tsdf_integrate(a["values"], a["weights"], a["colors"], a["fruit"], a["nx"], a["ny"], a["nz"], a["origin"], a["vs"],
                                      a["trunc"], a["c2w"], a["fx"], a["fy"], a["cx"], a["cy"], a["depth"], a["rgb"], a["frame_fruit"], a["B"],
                                      a["H"], a["W"], None)

    assert tsdf() == 0  # B = 0: nothing to do
    for kw in (dict(values=None), dict(weights=None), dict(colors=None), dict(c2w=None), dict(fx=None), dict(depth=None), dict(rgb=None),
               dict(frame_fruit=P), dict(nx=1), dict(nz=0), dict(vs=bad_v), dict(vs=nan_v), dict(vs=None), dict(origin=None),
               dict(trunc=0.0), dict(trunc=float("inf")), dict(trunc=float("nan")), dict(H=0), dict(W=-1), dict(B=-1)):
        assert tsdf(**kw) == -1, kw
        assert b"fnr_tsdf_integrate" in lib.fnr_last_error()
    nbytes = C.c_size_t(0)
    assert lib.fnr_marching_cubes_scratch_bytes(4, 5, 6, C.byref(nbytes)) == 0 and nbytes.value == 16 + 4 * 120
    assert lib.fnr_marching_cubes_scratch_bytes(1, 5, 6, C.byref(nbytes)) == -1
    assert lib.fnr_marching_cubes_scratch_bytes(4, 5, 6, None) == -1
    assert lib.fnr_marching_cubes_count(None, 4, 5, 6, P, 1000, P, None) == -1
    assert lib.fnr_marching_cubes_count(P, 4, 5, 6, P, 100, P, None) == -1  # scratch too small
    assert lib.fnr_marching_cubes_count(P, 4, 5, 6, P, 1000, None, None) == -1

    def emit(V, F, **kw):
        a = dict(values=P, colors=None, fruit=None, origin=o3, vs=v3, scratch=P, nbytes=1000, vertices=P, normals=P, vcol=None, vfr=None, faces=P)
        a.update(kw)
        return lib.fnr_marching_cubes_emit(a["values"], a["colors"], a["fruit"], 4, 5, 6, a["origin"], a["vs"], a["scratch"], a["nbytes"], V, F,
                                           a["vertices"], a["normals"], a["vcol"], a["vfr"], a["faces"], None)

    assert emit(0, 0) == 0
    assert emit(1 << 31, 10) == -2
    assert b"2^31 - 1" in lib.fnr_last_error()
    for V, F, kw in ((5, 2, dict(vertices=None)), (5, 2, dict(faces=None)), (5, 2, dict(colors=P)), (5, 2, dict(vfr=P)), (-1, 0, {}),
                     (5, 2, dict(vs=bad_v)), (5, 2, dict(scratch=None)), (5, 2, dict(nbytes=10))):
        assert emit(V, F, **kw) == -1, kw


def test_vanishing_gradient_gives_the_edge_direction():
    """Values alternating -1, 1, -1, ... along x: every interior central difference is zero, so the interior vertices take
    the direction of their edge, toward its outside (positive) end."""
    x = np.arange(8)
    v = np.broadcast_to(np.where(x % 2, 1.0, -1.0)[:, None, None], (8, 3, 3)).astype(np.float32)
    m = M.marching_cubes_numpy(v, 0.0, 1.0)
    np.testing.assert_allclose(np.linalg.norm(m["normals"], axis=1), 1.0, rtol=1e-6)
    coord = m["vertices"][:, 0]
    interior = (coord > 1) & (coord < 6)
    assert interior.sum() == 5 * 9
    want = np.where(np.floor(coord[interior]) % 2 == 0, 1.0, -1.0)  # from an even (inside) point: +x
    np.testing.assert_array_equal(m["normals"][interior], np.stack([want, 0 * want, 0 * want], 1).astype(np.float32))
