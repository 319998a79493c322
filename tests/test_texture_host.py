"""NeRF textures of exported meshes on the host: the per-face atlas (sizes, ownership, the no-bleed property, vt
orientation) checked by brute force, the numpy restatement of fnr_texel_rays against a per-texel closest-point search, the
ray length, the OBJ / MTL writer, the CLI options and the C-ABI refusals of fnr_texture.cu (these return before any
launch, so they run without a GPU)."""
import ctypes as C

import numpy as np
import pytest

from fruitnerf_b200 import texture as T

FACE_COUNTS = [1, 2, 3, 7, 1000, 2 ** 20 + 1]
PX = [2, 4, 7]


def footprint_ok(uv, owners, face_ids, W, H):
    """Bilinear lookups at ``uv`` [n,2] read only texels owned by ``face_ids`` [n] (weights below 1e-6 count as not read)."""
    x = uv[:, 0] * W - 0.5
    y = (1.0 - uv[:, 1]) * H - 0.5
    ok = np.ones(len(uv), bool)
    for c, w in ((np.floor(x), 1 - (x - np.floor(x))), (np.floor(x) + 1, x - np.floor(x))):
        for r, wy in ((np.floor(y), 1 - (y - np.floor(y))), (np.floor(y) + 1, y - np.floor(y))):
            read = w * wy > 1e-6
            ci, ri = c.astype(np.int64), r.astype(np.int64)
            inside = (ci >= 0) & (ci < W) & (ri >= 0) & (ri < H)
            ok &= ~read | (inside & (owners[np.clip(ri, 0, H - 1), np.clip(ci, 0, W - 1)] == face_ids))
    return ok


@pytest.mark.parametrize("p", PX)
@pytest.mark.parametrize("F", FACE_COUNTS)
def test_atlas_layout(F, p):
    bx, W, H = T.atlas_layout(F, p)
    nb = (F + 1) // 2
    assert W == bx * (p + 3) and H == -(-nb // bx) * p
    assert bx * bx * (p + 3) >= nb * p and (bx == 1 or (bx - 1) ** 2 * (p + 3) < nb * p)  # the smallest such bx
    assert T.atlas_size(F, p) == (W, H) and T.atlas_layout(F, p) == (bx, W, H)
    owners = T.texel_owners(F, p)
    counts = np.bincount(owners[owners >= 0], minlength=F)
    assert len(counts) == F and (counts > 0).all()
    # blocks are disjoint: face 2k and 2k+1 share block k, and each face owns texels of its block only
    rows, cols = np.nonzero(owners >= 0)
    f = owners[rows, cols]
    assert ((rows // p) * bx + cols // (p + 3) == f // 2).all()
    # the first slot of a block owns a + b <= p, the second the rest of the block
    per_block = p * (p + 3)
    first = sum(p - b + 1 for b in range(p))
    assert (counts[0::2] == first).all() and (counts[1::2] == per_block - first).all()
    # unowned texels belong to slots after the last face
    slot, _, _ = T.texel_slots(F, p)
    assert (slot.reshape(H, W)[owners < 0] >= F).all() and (slot.reshape(H, W)[owners >= 0] < F).all()
    assert int((slot >= F).sum()) == int((owners < 0).sum())
    # every UV triangle is non-degenerate and has its vertices at texel centres
    uv = T.uv_coordinates(F, p)
    e1, e2 = uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]
    area = np.abs(e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]) * W * H / 2
    np.testing.assert_allclose(area, (p - 1) ** 2 / 2, rtol=1e-9)
    px = uv[..., 0] * W - 0.5
    py = (1 - uv[..., 1]) * H - 0.5  # vt orientation: v = 1 - (row + 0.5) / H
    np.testing.assert_allclose(px, np.round(px), atol=1e-6)
    np.testing.assert_allclose(py, np.round(py), atol=1e-6)
    r, c = np.round(py).astype(np.int64), np.round(px).astype(np.int64)
    assert (owners[r, c] == np.arange(F)[:, None]).all()  # each corner sits on a texel its face owns
    # the no-bleed property, by brute force: bilinear lookups on a barycentric lattice of every triangle (corners, edges,
    # interior) read only texels of the face
    K = 6
    for i in range(K + 1):
        for j in range(K + 1 - i):
            w = np.array([1 - (i + j) / K, i / K, j / K])
            pts = np.einsum("k,fkd->fd", w, uv)
            assert footprint_ok(pts, owners, np.arange(F), W, H).all(), (i, j)


def test_vt_orientation_and_first_face():
    uv = T.uv_coordinates(2, 4)
    W, H = T.atlas_size(2, 4)
    assert (W, H) == (7, 4)
    # face 0: vertex 0 at the top-left texel centre (row 0 is the top: v close to 1), vertex 1 to its right, vertex 2 below
    np.testing.assert_allclose(uv[0], [[0.5 / 7, 1 - 0.5 / 4], [3.5 / 7, 1 - 0.5 / 4], [0.5 / 7, 1 - 3.5 / 4]])
    # face 1: the point reflection of face 0 in its block, three columns to the right
    np.testing.assert_allclose(uv[1], [[6.5 / 7, 1 - 3.5 / 4], [3.5 / 7, 1 - 3.5 / 4], [6.5 / 7, 1 - 0.5 / 4]])


def test_too_large_atlas_is_refused():
    F = 2 * 16384 * 16384 // 4
    with pytest.raises(T.AtlasTooLargeError, match=rf"{F} faces at --px-per-uv-triangle 4"):
        T.atlas_size(F, 4)
    for p in (1, 0, -3):
        with pytest.raises(ValueError, match="px_per_uv_triangle"):
            T.atlas_layout(10, p)
    with pytest.raises(ValueError):
        T.atlas_layout(0, 4)


# ---- the restatement of fnr_texel_rays -------------------------------------------------------------------------------
def closest_barycentrics(q, a, b, c):
    """Brute force: the closest point of triangle abc (2D, fp64) to q, as barycentrics -- the point itself when inside,
    else the best of the three clamped edge projections."""
    m = np.array([[b[0] - a[0], c[0] - a[0]], [b[1] - a[1], c[1] - a[1]]])
    s, t = np.linalg.solve(m, np.asarray(q) - a)
    if s >= -1e-12 and t >= -1e-12 and s + t <= 1 + 1e-12:
        return np.array([1 - s - t, s, t])
    best = None
    for (i, j) in ((0, 1), (1, 2), (2, 0)):
        P, Q = (a, b, c)[i], (a, b, c)[j]
        d = Q - P
        u = np.clip(np.dot(np.asarray(q) - P, d) / np.dot(d, d), 0, 1)
        pt = P + u * d
        dist = np.linalg.norm(pt - q)
        if best is None or dist < best[0] - 1e-12:
            w = np.zeros(3)
            w[i], w[j] = 1 - u, u
            best = (dist, w)
    return best[1]


@pytest.mark.parametrize("F, p", [(7, 2), (5, 4), (3, 7)])
def test_barycentrics_are_the_closest_point(F, p):
    _, W, H = T.atlas_layout(F, p)
    owners = T.texel_owners(F, p)
    face, w = T.texel_barycentrics(F, p)
    uv = T.uv_coordinates(F, p)
    tri = np.stack([uv[..., 0] * W - 0.5, (1 - uv[..., 1]) * H - 0.5], -1)  # texel-centre coordinates (col, row)
    for t in range(W * H):
        r, c = divmod(t, W)
        f = owners[r, c]
        if f < 0:
            assert face[t] == F - 1
            continue
        assert face[t] == f
        want = closest_barycentrics(np.array([c, r], float), *tri[f])
        np.testing.assert_allclose(w[t].astype(np.float64), want, atol=1e-6, err_msg=f"texel {(r, c)}")


def random_mesh(seed, F, V=None):
    rng = np.random.default_rng(seed)
    V = V or max(3, F)
    v = rng.uniform(-1, 1, (V, 3)).astype(np.float32)
    n = rng.standard_normal((V, 3)).astype(np.float32)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    f = rng.integers(0, V, (F, 3))
    return v, n, f


def test_ray_origin_and_direction():
    v, n, f = random_mesh(0, 9)
    W, H = T.atlas_size(9, 4)
    raylen = np.float32(0.37)
    o, d = T.restated_texel_rays(v, n, f, 4, W, H, raylen)
    assert o.dtype == np.float32 and o.shape == (W * H, 3)
    face, w = T.texel_barycentrics(9, 4)
    x = np.einsum("tk,tkd->td", w.astype(np.float64), v[f[face]].astype(np.float64))
    nn = np.einsum("tk,tkd->td", w.astype(np.float64), n[f[face]].astype(np.float64))
    nn /= np.linalg.norm(nn, axis=1, keepdims=True)
    np.testing.assert_allclose(np.linalg.norm(d, axis=1), 1, atol=1e-6)
    np.testing.assert_allclose(d, -nn, atol=1e-5)
    np.testing.assert_allclose(o - x, 0.5 * float(raylen) * nn, atol=1e-5)  # origin - x == 0.5 raylen n
    # a texel range is the same rays
    o2, d2 = T.restated_texel_rays(v, n, f, 4, W, H, raylen, texel_start=5, num_texels=17)
    assert np.array_equal(o2, o[5:22]) and np.array_equal(d2, d[5:22])
    with pytest.raises(ValueError):
        T.restated_texel_rays(v, n, f, 4, W + 1, H, raylen)


def test_vanishing_normals_fall_back_to_the_face_normal():
    """Opposite vertex normals cancel at the midpoint; the rule: |n| <= 1e-12 takes the right-hand face normal
    (v1 - v0) x (v2 - v0), and a degenerate face as well takes +z."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [3, 0, 0], [4, 0, 0]], np.float32)
    n = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 1], [3, 4, 5]])
    W, H = T.atlas_size(3, 4)
    o, d = T.restated_texel_rays(v, n, f, 4, W, H, 1.0)
    face, _ = T.texel_barycentrics(3, 4)
    assert (d[face == 0] == np.float32([0, 0, -1])).all()
    assert (d[face == 1] == np.float32([0, 0, 1])).all()
    assert (d[face == 2] == np.float32([0, 0, -1])).all()  # collinear vertices: +z
    # a cancelling pair of vertex normals: zero at the edge midpoint only
    n2 = np.array([[1, 0, 0], [-1, 0, 0], [0, 0, 1]], np.float32)
    W1, H1 = T.atlas_size(1, 3)
    _, d1 = T.restated_texel_rays(v[:3], n2, f[:1], 3, W1, H1, 1.0)
    face1, w1 = T.texel_barycentrics(1, 3)
    mid = (w1[:, 0] == w1[:, 1]) & (w1[:, 2] == 0) & (face1 == 0)
    assert mid.any() and (d1[mid] == np.float32([0, 0, -1])).all()


def test_mean_edge_on_a_hand_built_mesh():
    v = np.array([[0, 0, 0], [3, 4, 0], [0, 0, 2], [1, 1, 1]], np.float32)
    f = np.array([[0, 1, 2], [2, 0, 3], [3, 3, 0]])
    assert T.restated_mean_edge(v, f) == pytest.approx((5 + 2 + 0) / 3, rel=1e-15)


# ---- OBJ / MTL ---------------------------------------------------------------------------------------------------------
def test_obj_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    V, F = 200, 333
    v = (rng.standard_normal((V, 3)) * 10.0 ** rng.integers(-6, 6, (V, 1))).astype(np.float32)
    v[0] = [0, -0.0, 1e-45]
    v[1] = [np.finfo(np.float32).max, -np.finfo(np.float32).tiny, 9.999999e9]
    n = rng.standard_normal((V, 3)).astype(np.float32)
    f = rng.integers(0, V, (F, 3))
    uv = T.uv_coordinates(F, 4)
    T.write_textured_obj(tmp_path / "mesh.obj", "material_0.mtl", "material_0.png", v, n, f, uv)
    m = T.read_textured_obj(tmp_path / "mesh.obj")
    assert m["mtllib"] == "material_0.mtl" and m["usemtl"] == "material_0"
    assert np.array_equal(m["v"].astype(np.float32), v)  # positions round-trip exactly
    assert np.array_equal(m["vn"].astype(np.float32), n)
    assert m["vt"].shape == (3 * F, 2)
    np.testing.assert_allclose(m["vt"], uv.reshape(-1, 2), rtol=1e-8, atol=0)
    assert m["f"].shape == (F, 3, 3) and m["f"].min() >= 1
    np.testing.assert_array_equal(m["f"][:, :, 0] - 1, f)  # 1-based
    np.testing.assert_array_equal(m["f"][:, :, 2] - 1, f)
    np.testing.assert_array_equal(m["f"][:, :, 1] - 1, np.arange(3 * F).reshape(F, 3))  # three vt per face, face order
    mtl = (tmp_path / "material_0.mtl").read_text().splitlines()
    assert "newmtl material_0" in mtl and mtl[-1] == "map_Kd material_0.png"
    text = (tmp_path / "mesh.obj").read_text()
    assert text.startswith("mtllib material_0.mtl\nusemtl material_0\nv ")
    assert f"\nf {f[0, 0] + 1}/1/{f[0, 0] + 1} {f[0, 1] + 1}/2/{f[0, 1] + 1} " in text


def test_obj_bytes_of_one_triangle(tmp_path):
    T.write_textured_obj(tmp_path / "t.obj", "fruit_material_0.mtl", "fruit_material_0.png", [[0, 1.5, -2]], [[0, 0, 1]],
                         [[0, 0, 0]], [[[0.25, 1], [0.5, 0.75], [0, 0.125]]])
    assert (tmp_path / "t.obj").read_text() == (
        "mtllib fruit_material_0.mtl\nusemtl fruit_material_0\n"
        "v 0.00000000e+00 1.50000000e+00 -2.00000000e+00\n"
        "vt 2.50000000e-01 1.00000000e+00\nvt 5.00000000e-01 7.50000000e-01\nvt 0.00000000e+00 1.25000000e-01\n"
        "vn 0.00000000e+00 0.00000000e+00 1.00000000e+00\n"
        "f 1/1/1 1/2/1 1/3/1\n")
    assert "map_Kd fruit_material_0.png" in (tmp_path / "fruit_material_0.mtl").read_text()
    with pytest.raises(ValueError):
        T.write_textured_obj(tmp_path / "b.obj", "m.mtl", "m.png", [[0, 0, 0]], [[0, 0, 1]], [[0, 0, 1]], [[[0, 0]] * 3])
    with pytest.raises(ValueError):
        T.write_textured_obj(tmp_path / "b.obj", "m.mtl", "m.png", [[np.nan, 0, 0]], [[0, 0, 1]], [[0, 0, 0]], [[[0, 0]] * 3])


# ---- CLI ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("command", ["tsdf", "poisson"])
def test_cli_defaults_and_nerf_custom(command):
    import argparse

    from fruitnerf_b200.scripts import exporter as E

    sub = argparse.ArgumentParser().add_subparsers(dest="command")
    add, build = {"tsdf": (E.add_tsdf_parser, E.tsdf_exporter_from_args), "poisson": (E.add_poisson_parser, E.poisson_exporter_from_args)}[command]
    p = add(sub)
    exp = build(p.parse_args(["--load-config", "c.yml", "--output-dir", "o"]))
    assert exp.unwrap_method == "xatlas" and exp.px_per_uv_triangle == 4
    exp.validate()
    exp = build(p.parse_args(["--load-config", "c.yml", "--output-dir", "o", "--texture-method", "nerf", "--unwrap-method", "custom",
                              "--px-per-uv-triangle", "2"]))
    assert exp.texture_method == "nerf" and exp.unwrap_method == "custom" and exp.px_per_uv_triangle == 2
    exp.validate()
    exp.unwrap_method = "xatlas"
    with pytest.raises(ValueError, match="--unwrap-method custom"):
        exp.validate()


@pytest.mark.parametrize("command", ["tsdf", "poisson"])
@pytest.mark.parametrize("args, match", [
    (["--texture-method", "nerf", "--unwrap-method", "custom", "--px-per-uv-triangle", "1"], "px_per_uv_triangle"),
    (["--px-per-uv-triangle", "0"], "px_per_uv_triangle"),
    (["--texture-method", "nerf"], "xatlas"),
])
def test_cli_refusals(command, args, match, capsys, tmp_path):
    from fruitnerf_b200.scripts.exporter import entrypoint

    with pytest.raises(SystemExit) as e:
        entrypoint([command, "--load-config", str(tmp_path / "missing.yml"), "--output-dir", str(tmp_path / "out"), *args])
    assert e.value.code == 2
    assert match in capsys.readouterr().err
    assert not (tmp_path / "out").exists()


# ---- C ABI --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", PX)
@pytest.mark.parametrize("F", FACE_COUNTS + [2 ** 27])
def test_cabi_atlas_size_is_the_layout(native_lib, F, p):
    w, h = C.c_int64(0), C.c_int64(0)
    assert native_lib.fnr_texture_atlas_size(F, p, C.byref(w), C.byref(h)) == 0
    assert (w.value, h.value) == T.atlas_layout(F, p)[1:]


def test_cabi_refusals(native_lib):
    lib = native_lib
    P = 16  # any non-NULL address: nothing is dereferenced on a refusal
    W, H = T.atlas_size(5, 4)

    def rays(**kw):
        a = dict(v=P, n=P, f=P, F=5, p=4, W=W, H=H, raylen=0.5, t0=0, num=W * H, o=P, d=P)
        a.update(kw)
        return lib.fnr_texel_rays(a["v"], a["n"], a["f"], a["F"], a["p"], a["W"], a["H"], a["raylen"], a["t0"], a["num"], a["o"], a["d"], None)

    assert rays(num=0) == 0 and rays(t0=W * H, num=0) == 0
    for kw in (dict(v=None), dict(n=None), dict(f=None), dict(o=None), dict(d=None), dict(p=1), dict(p=0), dict(F=0), dict(F=-1),
               dict(W=W + 1), dict(H=H - 1), dict(t0=1), dict(t0=-1), dict(num=-1), dict(t0=W * H, num=1), dict(raylen=0.0),
               dict(raylen=-1.0), dict(raylen=float("inf")), dict(raylen=float("nan"))):
        assert rays(**kw) == -1, kw
        assert b"fnr_texel_rays" in lib.fnr_last_error()
    big = 2 * 16384 * 16384 // 4
    w, h = C.c_int64(0), C.c_int64(0)
    assert lib.fnr_texture_atlas_size(big, 4, C.byref(w), C.byref(h)) == 0 and max(w.value, h.value) > 16384
    assert rays(F=big, W=w.value, H=h.value, num=1) == -1 and b"at most 16384" in lib.fnr_last_error()
    assert lib.fnr_texture_atlas_size(0, 4, C.byref(w), C.byref(h)) == -1
    assert lib.fnr_texture_atlas_size(5, 1, C.byref(w), C.byref(h)) == -1
    assert lib.fnr_texture_atlas_size(5, 4, None, C.byref(h)) == -1
    assert lib.fnr_mesh_mean_edge(None, P, 5, P, None) == -1
    assert lib.fnr_mesh_mean_edge(P, None, 5, P, None) == -1
    assert lib.fnr_mesh_mean_edge(P, P, 5, None, None) == -1
    assert lib.fnr_mesh_mean_edge(P, P, 0, P, None) == -1
    assert b"fnr_mesh_mean_edge" in lib.fnr_last_error()
