"""The `charts` UV unwrap (DESIGN section 4.3r) on the CPU: the numpy restatement in texture.py checked by brute force on a
marched sphere, a cube, a mesh with degenerate and non-manifold faces, a self-overlapping helicoid and a mesh whose face
areas vary by more than 100x; the CLI options and the C-ABI refusals."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from fruitnerf_b200 import mesh as M
from fruitnerf_b200 import texture as T


# ---- meshes -------------------------------------------------------------------------------------------------------------
def marched_sphere(n=40, r=0.7):
    x = np.linspace(-1.0, 1.0, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    m = M.marching_cubes_numpy((np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - r).astype(np.float32), (-1.0, -1.0, -1.0), (2.0 / (n - 1),) * 3)
    return np.asarray(m["vertices"], np.float32), np.asarray(m["faces"], np.int64)


def cube():
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
    q = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]  # outward quads
    return v, np.array([t for a, b, c, d in q for t in ((a, b, c), (a, c, d))], np.int64)


def degenerate_nonmanifold():
    v, f = marched_sphere(n=16)
    extra = [f[0], [f[1, 0], f[1, 0], f[1, 1]], [f[2, 0], f[2, 1], f[2, 1]], [f[3, 0], f[3, 0], f[3, 0]]]  # a third face on
    v = np.concatenate([v, [[0.0, 0.0, 0.0], [0.1, 0.0, 0.0], [0.2, 0.0, 0.0]]]).astype(np.float32)  # f[0]'s edges, points
    V = len(v)
    extra.append([V - 3, V - 2, V - 1])  # a collinear (zero-area) face
    return v, np.concatenate([f, np.array(extra, np.int64)])


def helicoid(nu=40, nv=8, turns=2.0, pitch=0.05):
    """Two turns of a flat helicoid: every face is +z, so one chart overlaps itself in projection."""
    u = np.linspace(0, 2 * np.pi * turns, nu + 1)
    r = np.linspace(0.2, 1, nv + 1)
    U, R = np.meshgrid(u, r, indexing="ij")
    v = np.stack([R * np.cos(U), R * np.sin(U), pitch * U], -1).reshape(-1, 3).astype(np.float32)
    f = []
    for i in range(nu):
        for j in range(nv):
            a = i * (nv + 1) + j
            f += [[a, a + nv + 1, a + nv + 2], [a, a + nv + 2, a + 1]]
    return v, np.array(f, np.int64)


def graded_terrain(n=24):
    """A height field on a grid whose spacing grows geometrically: face areas vary by more than 100x."""
    x = np.cumsum(1.22 ** np.arange(n)) / 200.0
    X, Y = np.meshgrid(x, x, indexing="ij")
    v = np.stack([X, Y, 0.15 * np.sin(4 * X) * np.cos(3 * Y)], -1).reshape(-1, 3).astype(np.float32)
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            a = i * n + j
            f += [[a, a + n, a + n + 1], [a, a + n + 1, a + 1]]
    return v, np.array(f, np.int64)


MESHES = {"sphere": marched_sphere, "cube": cube, "degenerate": degenerate_nonmanifold, "helicoid": helicoid, "graded": graded_terrain}


def face_areas(v, f):
    t = np.asarray(v, np.float64)[f]
    return 0.5 * np.linalg.norm(np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]), axis=1)


def signed_area(p):
    return 0.5 * ((p[:, 1, 0] - p[:, 0, 0]) * (p[:, 2, 1] - p[:, 0, 1]) - (p[:, 1, 1] - p[:, 0, 1]) * (p[:, 2, 0] - p[:, 0, 0]))


_CACHE = {}


def unwrap(name, N=256):
    if (name, N) not in _CACHE:
        v, f = MESHES[name]()
        _CACHE[name, N] = (v, f, T.restated_chart_unwrap(v, f, N))
    return _CACHE[name, N]


def test_meshes_are_what_they_claim():
    a = face_areas(*graded_terrain())
    assert a.max() / a.min() > 100
    _, _, r = unwrap("helicoid")
    assert r["rounds"] >= 1  # the self-overlap was split
    v, f, r = unwrap("cube")
    assert r["num_charts"] == 6 and r["rounds"] == 0
    assert np.array_equal(np.bincount(r["labels"], minlength=6), [2] * 6)


# ---- properties ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MESHES))
def test_charts_are_connected_single_label_components(name):
    v, f, r = unwrap(name)
    charts, labels, C = r["charts"], r["labels"], r["num_charts"]
    assert charts.min() == 0 and charts.max() == C - 1
    # one label per chart
    assert all(len(np.unique(labels[charts == c])) == 1 for c in range(C))
    # connected through interior edges (exactly two half-edges), found by brute force
    halves = {}
    for fi, tri in enumerate(f.tolist()):
        for k in range(3):
            a, b = tri[k], tri[(k + 1) % 3]
            halves.setdefault((min(a, b), max(a, b)), []).append(fi)
    pairs = np.array([h for h in halves.values() if len(h) == 2 and charts[h[0]] == charts[h[1]]] or np.zeros((0, 2)), np.int64)
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(len(f), len(f)))
    n, comp = connected_components(g, directed=False)
    assert n == C
    assert all(len(np.unique(comp[charts == c])) == 1 for c in range(C))
    # numbered in order of the smallest face
    first = np.array([np.flatnonzero(charts == c)[0] for c in range(C)])
    assert (np.diff(first) > 0).all()


@pytest.mark.parametrize("name", list(MESHES))
def test_projection_is_area_proportional_and_not_flipped(name):
    v, f, r = unwrap(name)
    s, uv = r["scale"], r["uv"]
    vt = T.chart_vt(uv, 256)
    area3 = face_areas(v, f)
    good = area3 > 1e-12
    a_vt = signed_area(vt)
    assert (a_vt[good] > 0).all() and (a_vt >= 0).all()
    # edge lengths in texels are s times the projected lengths
    drop = r["labels"] // 2
    P = np.asarray(v, np.float64)[f]
    keep = np.array([[1, 2], [0, 2], [0, 1]])[drop]
    proj = np.take_along_axis(P, keep[:, None, :], axis=2)
    for k in range(3):
        e_uv = np.linalg.norm(uv[:, (k + 1) % 3] - uv[:, k], axis=1)
        e_p = np.linalg.norm(proj[:, (k + 1) % 3] - proj[:, k], axis=1)
        np.testing.assert_allclose(e_uv, s * e_p, rtol=1e-6, atol=1e-9)
    # UV area / 3D area in [s^2 / sqrt(3), s^2]
    ratio = -signed_area(uv)[good] / area3[good]
    assert (ratio >= s * s / math.sqrt(3) * (1 - 1e-6)).all() and (ratio <= s * s * (1 + 1e-6)).all()


@pytest.mark.parametrize("name", list(MESHES))
def test_rectangles_are_disjoint_and_packing_is_tight(name):
    v, f, r = unwrap(name)
    N, s = 256, r["scale"]
    labels, proj = T.chart_labels(v, f)
    ext, pmin = T.chart_extents(proj, r["charts"], r["num_charts"])
    w = np.floor(s * ext).astype(np.int64) + 1 + 2 * T.UNWRAP_MARGIN
    paint = np.zeros((N, N), np.int32)
    for (x, y), (cw, ch) in zip(r["offsets"], w):
        assert 0 <= x and x + cw <= N and 0 <= y and y + ch <= N
        paint[y:y + ch, x:x + cw] += 1
    assert paint.max() == 1
    # every triangle lies inside its chart's rectangle, a margin in
    o = r["offsets"][r["charts"]]
    assert (r["uv"] >= (o + T.UNWRAP_MARGIN)[:, None, :] - 1e-9).all()
    assert (r["uv"] <= (o + T.UNWRAP_MARGIN + s * ext[r["charts"]])[:, None, :] + 1e-9).all()
    # s packs, the next bisection step above it does not
    order = T.chart_order(ext)
    assert T.pack_charts(ext, order, s, N) is not None
    assert r["scale_fails"] > s and T.pack_charts(ext, order, r["scale_fails"], N) is None
    assert (r["scale_fails"] - s) <= 2 * (N / ext.max()) * 2.0 ** -T.UNWRAP_BISECTIONS  # one bisection step, up to rounding


@pytest.mark.parametrize("name", list(MESHES))
def test_no_texel_centre_is_inside_two_triangles(name):
    v, f, r = unwrap(name)
    N, uv = 256, r["uv"]
    count = np.zeros(N * N, np.int64)
    for fi in range(len(f)):
        x, y = uv[fi, :, 0], uv[fi, :, 1]
        cx, cy = np.meshgrid(np.arange(math.floor(x.min()), math.ceil(x.max()) + 1) + 0.5,
                             np.arange(math.floor(y.min()), math.ceil(y.max()) + 1) + 0.5)
        cx, cy = cx.ravel(), cy.ravel()
        inside = np.ones(len(cx), bool)
        for k in range(3):
            a, b = k, (k + 1) % 3
            inside &= (cx - x[a]) * (y[b] - y[a]) - (cy - y[a]) * (x[b] - x[a]) > 0
        np.add.at(count, cy[inside].astype(np.int64) * N + cx[inside].astype(np.int64), 1)
    assert count.max() <= 1


@pytest.mark.parametrize("name", list(MESHES))
def test_bilinear_lookups_stay_in_the_chart(name):
    v, f, r = unwrap(name)
    N, uv, owner, charts = 256, r["uv"], r["owner"], r["charts"]
    rng = np.random.default_rng(0)
    for _ in range(4):
        w = rng.dirichlet(np.ones(3), len(f))
        p = np.einsum("fk,fkd->fd", w, uv)
        x0, y0 = np.floor(p[:, 0] - 0.5).astype(np.int64), np.floor(p[:, 1] - 0.5).astype(np.int64)
        for dx in (0, 1):
            for dy in (0, 1):
                o = owner[(y0 + dy) * N + x0 + dx]
                assert (o >= 0).all()
                assert (charts[o] == charts).all()
    # owners agree with the compacted list, the barycentrics are a partition of one
    assert np.array_equal(np.flatnonzero(owner >= 0), r["texels"])
    assert np.array_equal(owner[r["texels"]], r["texel_faces"])
    b = r["barycentrics"].astype(np.float64)
    assert (b >= 0).all() and np.allclose(b.sum(axis=1), 1, atol=1e-6)


def test_owner_is_the_closest_face_within_the_gutter():
    v, f, r = unwrap("sphere")
    N, uv, owner = 256, r["uv"], r["owner"]
    rng = np.random.default_rng(1)
    texels = rng.choice(np.flatnonzero(owner >= 0), 300, replace=False)
    cx, cy = texels % N + 0.5, texels // N + 0.5
    # the distance from each sampled texel centre to every triangle of the mesh: the owner is the first closest face
    for t, x, y in zip(texels, cx, cy):
        d2, _ = T.chart_closest(uv, np.arange(len(f)), np.full(len(f), t % N), np.full(len(f), t // N))
        assert d2[owner[t]] == d2.min() and d2.min() <= T.UNWRAP_GUTTER ** 2
        assert owner[t] == np.flatnonzero(d2.astype(np.float32) == d2.astype(np.float32).min())[0]


def test_restated_rays_use_the_barycentrics():
    v, f, r = unwrap("cube")
    n = np.zeros_like(v)
    o, d = T.restated_chart_texel_rays(v, n, f, r["texel_faces"], r["barycentrics"], 0.5)
    x = np.einsum("tk,tkd->td", r["barycentrics"].astype(np.float64), v.astype(np.float64)[f[r["texel_faces"]]])
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    fn = fn / np.linalg.norm(fn, axis=1, keepdims=True)
    np.testing.assert_allclose(d, -fn[r["texel_faces"]], atol=1e-6)
    np.testing.assert_allclose(o, x + 0.25 * fn[r["texel_faces"]], atol=1e-6)


def test_obj_round_trips(tmp_path):
    v, f, r = unwrap("graded")
    vt = T.chart_vt(r["uv"], 256)
    T.write_textured_obj(tmp_path / "mesh.obj", "material_0.mtl", "material_0.png", v, np.zeros_like(v), f, vt)
    obj = T.read_textured_obj(tmp_path / "mesh.obj")
    assert np.array_equal(obj["f"][:, :, 0] - 1, f)
    np.testing.assert_allclose(obj["vt"][obj["f"][:, :, 1] - 1], vt, rtol=1e-8, atol=1e-12)


def test_refusals():
    v, f = cube()
    for N in (15, 16385, 0):
        with pytest.raises(ValueError, match="num_pixels_per_side"):
            T.restated_chart_unwrap(v, f, N)
    v, f = helicoid()
    with pytest.raises(T.AtlasTooLargeError) as e:
        T.restated_chart_unwrap(v, f, 16)  # more charts than 7 x 7 rectangles fit
    msg = str(e.value)
    assert "charts" in msg and "--num-pixels-per-side" in msg and "--target-num-faces" in msg
    with pytest.raises(T.AtlasTooLargeError, match="6 charts"):
        T.restated_chart_unwrap(*cube(), 16)  # four 7 x 7 rectangles fit into 16 x 16, six do not
    assert T.restated_chart_unwrap(*cube(), 21)["num_charts"] == 6  # nine do into 21 x 21


# ---- CLI ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("command", ["tsdf", "poisson"])
def test_cli_accepts_charts(command):
    import argparse

    from fruitnerf_b200.scripts import exporter as E

    sub = argparse.ArgumentParser().add_subparsers(dest="command")
    add, build = {"tsdf": (E.add_tsdf_parser, E.tsdf_exporter_from_args), "poisson": (E.add_poisson_parser, E.poisson_exporter_from_args)}[command]
    p = add(sub)
    base = ["--load-config", "c.yml", "--output-dir", "o", "--texture-method", "nerf"]
    exp = build(p.parse_args(base + ["--unwrap-method", "charts"]))
    assert exp.unwrap_method == "charts" and exp.num_pixels_per_side == 1024
    exp.validate()
    exp = build(p.parse_args(base + ["--unwrap-method", "charts", "--num-pixels-per-side", "2048", "--target-num-faces", "5000"]))
    assert exp.num_pixels_per_side == 2048 and exp.target_num_faces == 5000
    exp.validate()
    exp = build(p.parse_args(base + ["--unwrap-method", "custom", "--num-pixels-per-side", "3"]))
    exp.validate()  # the atlas side is only read by the charts unwrap


@pytest.mark.parametrize("command", ["tsdf", "poisson"])
@pytest.mark.parametrize("args, match", [
    (["--texture-method", "nerf", "--unwrap-method", "charts", "--num-pixels-per-side", "15"], "num_pixels_per_side"),
    (["--texture-method", "nerf", "--unwrap-method", "charts", "--num-pixels-per-side", "16385"], "num_pixels_per_side"),
    (["--texture-method", "nerf", "--unwrap-method", "xatlas"], "--unwrap-method custom"),
    (["--texture-method", "nerf"], "--unwrap-method charts"),
])
def test_cli_refusals(command, args, match, capsys, tmp_path):
    from fruitnerf_b200.scripts.exporter import entrypoint

    with pytest.raises(SystemExit) as e:
        entrypoint([command, "--load-config", str(tmp_path / "missing.yml"), "--output-dir", str(tmp_path / "out"), *args])
    assert e.value.code == 2
    assert match in capsys.readouterr().err
    assert not (tmp_path / "out").exists()


# ---- C ABI --------------------------------------------------------------------------------------------------------------
def test_cabi_refusals(native_lib):
    lib = native_lib
    P = 16  # any non-NULL address: nothing is dereferenced on a refusal
    size = C.c_size_t(0)
    for args in ((8, 12, 256, None), (8, 0, 256, C.byref(size)), (0, 12, 256, C.byref(size)), (8, 12, 15, C.byref(size)),
                 (8, 12, 16385, C.byref(size))):
        assert lib.fnr_chart_unwrap_scratch_bytes(*args) == -1, args
    assert lib.fnr_chart_unwrap_scratch_bytes(8, 2 ** 30, 256, C.byref(size)) == -2
    rounds, charts, scale, owned = C.c_int32(0), C.c_int64(0), C.c_double(0), C.c_int64(0)

    def run(**kw):
        a = dict(v=P, f=P, V=8, F=12, N=256, s=P, sb=1 << 40, out=P, rounds=C.byref(rounds), charts=C.byref(charts), scale=C.byref(scale),
                 owned=C.byref(owned))
        a.update(kw)
        o = a["out"]
        return lib.fnr_chart_unwrap(a["v"], a["f"], a["V"], a["F"], a["N"], a["s"], a["sb"], o, o, o, o, o, o, o, o, a["rounds"], a["charts"],
                                    a["scale"], a["owned"], None, None)

    for kw in (dict(v=None), dict(f=None), dict(out=None), dict(rounds=None), dict(charts=None), dict(scale=None), dict(owned=None),
               dict(F=0), dict(F=-1), dict(V=0), dict(N=15), dict(N=16385), dict(N=0), dict(s=None)):
        assert run(**kw) == -1, kw
        assert b"fnr_chart_unwrap" in lib.fnr_last_error()

    def rays(**kw):
        a = dict(v=P, n=P, f=P, F=12, tf=P, w=P, owned=100, raylen=0.5, t0=0, num=100, o=P, d=P)
        a.update(kw)
        return lib.fnr_chart_texel_rays(a["v"], a["n"], a["f"], a["F"], a["tf"], a["w"], a["owned"], a["raylen"], a["t0"], a["num"], a["o"],
                                        a["d"], None)

    assert rays(num=0) == 0 and rays(t0=100, num=0) == 0
    for kw in (dict(v=None), dict(n=None), dict(f=None), dict(tf=None), dict(w=None), dict(o=None), dict(d=None), dict(F=0), dict(t0=-1),
               dict(num=-1), dict(t0=1), dict(raylen=0.0), dict(raylen=-1.0), dict(raylen=float("inf")), dict(raylen=float("nan"))):
        assert rays(**kw) == -1, kw
        assert b"fnr_chart_texel_rays" in lib.fnr_last_error()
