"""Per-fruit measurement on the host (measure.py): analytic meshes from marching cubes of signed-distance grids (sphere,
torus, ellipsoid, a sphere cut by a plane, two touching spheres), degenerate groups, the restatement's labels and edge
counts against brute-force loops, the `measure` command and the C-ABI refusals.

Measured errors (restatement, voxel edge 1): sphere r = 15.3 volume -0.26 %, radius -0.11 %, |coverage - 1| = 2.2e-15;
torus R = 14, r = 5 volume -0.82 %; ellipsoid 18 x 14 x 11 volume -0.31 % (rms 1.8 voxels); caps coverage -1.4e-4
(r = 15.3, cos(theta) = 0.5), -4.0e-5 (r = 20.3, 0.3), +1.6e-5 (r = 20.3, -0.2) and volume_extrapolated -0.32 %, -0.16 %,
-0.14 %; touching spheres r = 12 split by their centres, radii -0.15 % and -0.17 %."""

import ctypes as C
import json
import math

import numpy as np
import pytest

from fruitnerf_b200 import measure as ME
from fruitnerf_b200 import mesh as M


def sdf_mesh(n, f):
    g = np.arange(n, dtype=np.float64)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    m = M.marching_cubes_numpy(f(X, Y, Z).astype(np.float32), (0.0, 0.0, 0.0), 1.0)
    return m["vertices"].astype(np.float64), m["faces"]


def sphere(r=15.3, c=(24.2, 23.7, 24.5), n=50):
    c = np.asarray(c)
    return sdf_mesh(n, lambda X, Y, Z: np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r)


def torus(R0=14.0, r0=5.0):
    return sdf_mesh(48, lambda X, Y, Z: np.sqrt((np.sqrt((X - 24) ** 2 + (Y - 24.3) ** 2) - R0) ** 2 + (Z - 23.8) ** 2) - r0)


def ellipsoid(a=18.0, b=14.0, c=11.0):
    # the first-order distance f / |grad f| of the implicit ellipsoid f = |x / axes| - 1
    def f(X, Y, Z):
        u, v, w = (X - 24.1) / a, (Y - 23.9) / b, (Z - 24.2) / c
        q = np.sqrt(u * u + v * v + w * w)
        g = np.sqrt((u / a) ** 2 + (v / b) ** 2 + (w / c) ** 2) / np.maximum(q, 1e-12)
        return (q - 1) / g
    return sdf_mesh(50, f)


def two_spheres(r=12.0, gap=-0.6):
    c0, c1 = np.array([16.2, 20.1, 20.3]), np.array([16.2 + 2 * r + gap, 20.1, 20.3])
    d = lambda X, Y, Z, c: np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r  # noqa: E731
    v, f = sdf_mesh(66, lambda X, Y, Z: np.minimum(d(X, Y, Z, c0), d(X, Y, Z, c1)))
    return v, f, np.stack([c0, c1])


def clip_above(v, f, z0):
    """The part of the mesh above the plane z = z0, faces crossing it cut exactly (cut vertices shared by edge)."""
    above = v[:, 2] > z0
    verts, cache, out = list(v), {}, list(f[above[f].all(1)])

    def cut(a, b):
        k = (min(a, b), max(a, b))
        if k not in cache:
            t = (z0 - v[a, 2]) / (v[b, 2] - v[a, 2])
            cache[k] = len(verts)
            verts.append(v[a] + t * (v[b] - v[a]))
        return cache[k]

    for tri in f[above[f].any(1) & ~above[f].all(1)]:
        for s in range(3):
            a, b, c = tri[s], tri[(s + 1) % 3], tri[(s + 2) % 3]
            if above[a] and not above[b] and not above[c]:
                out.append([a, cut(a, b), cut(c, a)])
            elif above[a] and above[b] and not above[c]:
                p, q = cut(b, c), cut(c, a)
                out += [[a, b, p], [a, p, q]]
    return np.array(verts), np.array(out, np.int64)


# ---- analytic meshes --------------------------------------------------------------------------------------------------
def test_sphere():
    r = 15.3
    v, f = sphere(r)
    res = ME.measure_fruits(v, f)
    assert res["num_groups"] == 1 and bool(res["closed"][0]) and res["fit_ok"][0] == 1
    assert res["boundary_edges"][0] == 0 and res["nonmanifold_edges"][0] == 0 and res["unassigned_faces"] == 0
    assert abs(res["coverage"][0] - 1) <= 1e-9
    truth = 4 / 3 * math.pi * r ** 3
    assert abs(res["volume"][0] / truth - 1) <= 0.01 and abs(res["radius"][0] / r - 1) <= 0.01
    assert res["volume_extrapolated"][0] == res["volume"][0]
    np.testing.assert_allclose(res["center"][0], (24.2, 23.7, 24.5), atol=0.01)
    np.testing.assert_allclose(res["equivalent_diameter"][0], (6 * res["volume_extrapolated"][0] / math.pi) ** (1 / 3))
    assert 0 < res["rms"][0] < 0.05


def test_torus():
    R0, r0 = 14.0, 5.0
    res = ME.measure_fruits(*torus(R0, r0))
    assert res["num_groups"] == 1 and bool(res["closed"][0])
    assert abs(res["volume"][0] / (2 * math.pi ** 2 * R0 * r0 ** 2) - 1) <= 0.01
    # the fitted centre lies in the hole, where the coverage is 0: a closed group reports its volume as is
    assert abs(res["coverage"][0]) < 1e-9
    assert res["volume_extrapolated"][0] == res["volume"][0]
    np.testing.assert_allclose(res["equivalent_diameter"][0], (6 * res["volume"][0] / math.pi) ** (1 / 3))


def test_ellipsoid():
    a, b, c = 18.0, 14.0, 11.0
    res = ME.measure_fruits(*ellipsoid(a, b, c))
    assert res["num_groups"] == 1 and bool(res["closed"][0])
    assert abs(res["volume"][0] / (4 / 3 * math.pi * a * b * c) - 1) <= 0.01
    assert res["rms"][0] > 0.5


@pytest.mark.parametrize("r,ct", [(15.3, 0.5), (20.3, 0.3), (20.3, -0.2)])
def test_sphere_cut_by_a_plane(r, ct):
    n = int(2 * r + 8)
    c = np.array([n / 2 - 0.3, n / 2 + 0.2, n / 2 + 0.1])
    v, f = clip_above(*sphere(r, c, n), c[2] + ct * r)
    res = ME.measure_fruits(v, f)
    assert res["num_groups"] == 1 and not res["closed"][0] and res["boundary_edges"][0] > 0 and res["fit_ok"][0] == 1
    assert abs(res["coverage"][0] - (1 - ct) / 2) <= 1e-3
    assert abs(res["volume_extrapolated"][0] / (4 / 3 * math.pi * r ** 3) - 1) <= 0.02


def test_two_touching_spheres():
    r = 12.0
    v, f, centres = two_spheres(r)
    comp = ME.measure_fruits(v, f)
    assert comp["num_groups"] == 1 and bool(comp["closed"][0])
    split = ME.measure_fruits(v, f, centres)
    assert split["num_groups"] == 2 and split["unassigned_faces"] == 0 and (split["faces"] > 0).all()
    assert (np.abs(split["radius"] / r - 1) <= 0.02).all() and (split["fit_ok"] == 1).all()
    assert (split["boundary_edges"] > 0).all()  # each half is open where the other begins
    np.testing.assert_allclose(split["area"].sum(), comp["area"][0], rtol=1e-12)
    near = ME.measure_fruits(v, f, centres, max_distance=0.8 * r)
    p = ME.face_centroids(v, f)
    far = np.linalg.norm(p[:, None] - centres[None], axis=2).min(1) > 0.8 * r
    assert far.sum() > 0 and near["unassigned_faces"] == int(far.sum())
    np.testing.assert_array_equal(near["face_group"] == -1, far)
    np.testing.assert_allclose(near["unassigned_area"], ME.face_areas(v, f)[far].sum(), rtol=1e-12)


def test_reversed_winding_negates_volume_and_coverage():
    v, f = sphere()
    a, b = ME.measure_fruits(v, f), ME.measure_fruits(v, f[:, ::-1])
    np.testing.assert_allclose(b["volume"], -a["volume"], rtol=1e-12)
    np.testing.assert_allclose(b["coverage"], -a["coverage"], rtol=1e-12)
    np.testing.assert_allclose(b["radius"], a["radius"], rtol=1e-12)
    assert b["volume_extrapolated"][0] == b["volume"][0] < 0 and np.isnan(b["equivalent_diameter"]).all()
    cap_v, cap_f = clip_above(v, f, 30.0)
    cap = ME.measure_fruits(cap_v, cap_f[:, ::-1])  # an open group with negative coverage: no extrapolated volume
    assert not cap["closed"][0] and cap["coverage"][0] < 0 and np.isnan(cap["volume_extrapolated"]).all()


def test_planar_groups_fail_the_fit():
    tri = (np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0]]), np.array([[0, 1, 2]]))
    rng = np.random.default_rng(0)
    n = rng.normal(size=3)
    n /= np.linalg.norm(n)
    u = np.cross(n, [1.0, 0, 0])
    u /= np.linalg.norm(u)
    w = np.cross(n, u)
    pts = rng.uniform(-1, 1, size=(8, 2))
    fan_v = np.array([3.0, -1, 2]) + pts[:, :1] * u + pts[:, 1:] * w
    fan = (fan_v, np.array([[0, k, k + 1] for k in range(1, 7)]))
    for v, f in (tri, fan):
        res = ME.measure_fruits(v, f)
        assert res["num_groups"] == 1 and res["fit_ok"][0] == 0
        np.testing.assert_allclose(res["center"][0], res["centroid"][0])
        assert abs(res["volume"][0]) < 1e-12  # the coverage of a plane seen from within it is +-1/2 or 0: not asserted


# ---- the restatement against brute force -------------------------------------------------------------------------------
def random_mesh(seed, V=60, F=90):
    """Random faces over a subset of the vertices (so some are unused), plus a non-manifold fan of four faces on one
    edge and a face reusing a vertex."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(V, 3))
    pool = rng.choice(V, size=V * 2 // 3, replace=False)
    f = np.stack([rng.choice(pool, 3, replace=False) for _ in range(F)])
    a, b = pool[0], pool[1]
    fan = np.array([[a, b, c] for c in pool[2:6]])
    return v, np.concatenate([f, fan, [[pool[7], pool[7], pool[8]]]]).astype(np.int64)


def brute_components(f, V):
    parent = list(range(V))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x

    for a, b, c in f:
        for p, q in ((a, b), (b, c)):
            rp, rq = find(p), find(q)
            if rp != rq:
                parent[max(rp, rq)] = min(rp, rq)
    roots = sorted({find(a) for a in f.reshape(-1)})
    ids = {r: k for k, r in enumerate(roots)}
    return np.array([ids[find(t[0])] for t in f]), len(roots)


def brute_edges(f, g, G):
    runs = {}
    for t, gt in zip(f, g):
        for k in range(3):
            a, b = int(t[k]), int(t[(k + 1) % 3])
            runs.setdefault((min(a, b), max(a, b)), []).append(int(gt))
    bnd, nm = np.zeros(G, np.int64), np.zeros(G, np.int64)
    for groups in runs.values():
        for x in set(groups):
            if x < 0:
                continue
            c = groups.count(x)
            bnd[x] += c == 1
            nm[x] += c >= 3
    return bnd, nm


@pytest.mark.parametrize("seed", range(4))
def test_restatement_matches_brute_force(seed):
    v, f = random_mesh(seed)
    lab, G = ME.restated_components(f, len(v))
    want, Gw = brute_components(f, len(v))
    assert G == Gw
    np.testing.assert_array_equal(lab, want)
    res = ME.restated_measure(v, f, lab, G)
    b, nm = brute_edges(f, lab, G)
    np.testing.assert_array_equal(res["boundary_edges"], b)
    np.testing.assert_array_equal(res["nonmanifold_edges"], nm)
    assert nm.sum() >= 1
    np.testing.assert_array_equal(res["faces"], np.bincount(lab, minlength=G))
    # centre mode: nearest centroid by a loop, ties to the lower index, beyond max_distance unassigned
    rng = np.random.default_rng(seed + 10)
    centres = rng.normal(size=(7, 3))
    centres[3] = centres[1]  # an exact tie
    got = ME.restated_assign(v, f, centres, 1.2)
    p = ME.face_centroids(v, f)
    for i in range(len(f)):
        d = [float(((p[i] - c) ** 2).sum()) for c in centres]
        k = int(np.argmin(d))
        assert got[i] == (k if d[k] <= 1.44 else -1) and got[i] != 3
    res = ME.restated_measure(v, f, got, 7)
    b, nm = brute_edges(f, got, 7)
    np.testing.assert_array_equal(res["boundary_edges"], b)
    np.testing.assert_array_equal(res["nonmanifold_edges"], nm)
    assert res["faces"][3] == 0 and np.isnan(res["sphere"][3]).all() and res["volume"][3] == 0
    assert res["unassigned_faces"][0] == int((got == -1).sum())


def test_driver_refusals():
    v, f = sphere()
    with pytest.raises(ValueError, match="max_distance"):
        ME.measure_fruits(v, f, np.zeros((1, 3)), max_distance=0.0)
    with pytest.raises(ValueError, match="finite"):
        ME.measure_fruits(v, f, np.array([[0.0, np.nan, 0.0]]))
    with pytest.raises(ValueError, match="face indices"):
        ME.measure_fruits(v, np.array([[0, 1, len(v)]]))
    with pytest.raises(ValueError, match="labels"):
        ME.restated_measure(v, f[:2], np.array([0, 1]), 1)


# ---- the command ------------------------------------------------------------------------------------------------------
def write_run(tmp_path, scale=0.4, rot_deg=30.0):
    from fruitnerf_b200.export.exporter_utils import write_mesh_ply

    v, f, centres = two_spheres()
    v = v / 66.0  # inside the unit cube, as the exported meshes
    centres = centres / 66.0
    write_mesh_ply(tmp_path / "fruit_mesh.ply", v, np.zeros_like(v), None, f)
    t = math.radians(rot_deg)
    R = np.array([[math.cos(t), -math.sin(t), 0], [math.sin(t), math.cos(t), 0], [0, 0, 1]])
    tr = np.array([0.1, -0.2, 0.3])
    (tmp_path / "dataparser_transforms.json").write_text(json.dumps({"transform": np.concatenate([R, tr[:, None]], 1).tolist(), "scale": scale}))
    (tmp_path / "count.json").write_text(json.dumps({"count": 2, "centers": (centres * 2 / scale).tolist()}))
    return v, f, centres, R, tr


def test_cli_defaults_and_frames(tmp_path):
    from fruitnerf_b200.scripts import measure as cli

    v, f, centres, R, tr = write_run(tmp_path)
    _, a = cli.parse_args(["--mesh", str(tmp_path / "fruit_mesh.ply")])
    assert (a.device, a.count_json, a.transform_json, a.max_distance, a.json, a.csv) == ("cuda:0", None, None, None, None, None)
    comp = cli.main(["--mesh", str(tmp_path / "fruit_mesh.ply"), "--device", "cpu", "--json", str(tmp_path / "c.json")])
    assert comp["mode"] == "components" and comp["num_groups"] == 1 and comp["frame"] == "dataparser"
    assert json.loads((tmp_path / "c.json").read_text()) == comp
    base = ["--mesh", str(tmp_path / "fruit_mesh.ply"), "--device", "cpu", "--count-json", str(tmp_path / "count.json"), "--transform-json",
            str(tmp_path / "dataparser_transforms.json")]
    out = cli.main([*base, "--csv", str(tmp_path / "m.csv")])
    assert out["mode"] == "centers" and out["num_groups"] == 2 and out["unassigned_faces"] == 0 and out["scale"] == 0.4
    lines = (tmp_path / "m.csv").read_text().splitlines()
    assert lines[0].split(",") == list(cli.COLUMNS) and len(lines) == 3
    # sizes in the capture's units, positions in the capture frame
    direct = ME.measure_fruits(v, f, centres)
    s = 0.4
    for k, row in enumerate(out["groups"]):
        assert row["id"] == k and row["faces"] == direct["faces"][k]
        np.testing.assert_allclose(row["radius"], direct["radius"][k] / s, rtol=1e-12)
        np.testing.assert_allclose(row["area"], direct["area"][k] / s ** 2, rtol=1e-12)
        np.testing.assert_allclose(row["volume"], direct["volume"][k] / s ** 3, rtol=1e-12)
        np.testing.assert_allclose(row["equivalent_diameter"], direct["equivalent_diameter"][k] / s, rtol=1e-12)
        back = s * (R @ np.array([row["center_x"], row["center_y"], row["center_z"]]) + tr)
        np.testing.assert_allclose(back, direct["center"][k], atol=1e-12)
    # --max-distance is in count-frame units: 0.8 r in the mesh frame is 0.8 r * 2 / scale there
    r = 12.0 / 66.0
    near = cli.main([*base, "--max-distance", str(0.8 * r * 2 / s)])
    want = ME.measure_fruits(v, f, centres, max_distance=0.8 * r)
    assert near["unassigned_faces"] == want["unassigned_faces"] > 0


@pytest.mark.parametrize("extra,msg", [
    (["--mesh", "{d}/missing.ply"], "no such file"),
    (["--mesh", "{d}/fruit_mesh.ply", "--count-json", "{d}/count.json"], "needs --transform-json"),
    (["--mesh", "{d}/fruit_mesh.ply", "--count-json", "{d}/count.json", "--transform-json", "{d}/dataparser_transforms.json",
      "--max-distance", "0"], "must be > 0"),
    (["--mesh", "{d}/fruit_mesh.ply", "--max-distance", "1"], "applies to centre mode"),
    (["--mesh", "{d}/empty.ply", "--device", "cpu"], "no faces"),
])
def test_cli_refusals(tmp_path, capsys, extra, msg):
    from fruitnerf_b200.export.exporter_utils import write_mesh_ply
    from fruitnerf_b200.scripts import measure as cli

    write_run(tmp_path)
    write_mesh_ply(tmp_path / "empty.ply", np.zeros((0, 3)), np.zeros((0, 3)), None, np.zeros((0, 3), np.int64))
    with pytest.raises(SystemExit) as e:
        cli.main([x.format(d=tmp_path) for x in extra])
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


# ---- the C ABI -------------------------------------------------------------------------------------------------------------
def test_cabi_refusals(native_lib):
    lib = native_lib
    n = C.c_size_t(0)
    assert lib.fnr_mesh_measure_scratch_bytes(10, 10, None) == -1
    assert lib.fnr_mesh_measure_scratch_bytes(-1, 10, C.byref(n)) == -1
    assert lib.fnr_mesh_measure_scratch_bytes(10, -1, C.byref(n)) == -1
    assert lib.fnr_mesh_measure_scratch_bytes(2 ** 31, 10, C.byref(n)) == -2
    assert lib.fnr_mesh_measure_scratch_bytes(10, 2 ** 30, C.byref(n)) == -2
    fake = C.c_void_p(16)  # never dereferenced: every call below is refused before any device work
    g = C.c_int64(0)
    assert lib.fnr_mesh_components(None, 10, 10, fake, 1 << 30, fake, C.byref(g), None) == -1
    assert b"fnr_mesh_components" in lib.fnr_last_error()
    assert lib.fnr_mesh_components(fake, 10, 10, fake, 1 << 30, fake, None, None) == -1
    assert lib.fnr_mesh_components(fake, -1, 10, fake, 1 << 30, fake, C.byref(g), None) == -1
    assert lib.fnr_mesh_components(fake, 10, 2 ** 31, fake, 1 << 30, fake, C.byref(g), None) == -2
    sb = 256
    for md in (0.0, -1.0, float("nan")):
        assert lib.fnr_mesh_assign_centers(fake, fake, 10, 10, fake, 3, md, fake, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, None, 10, 10, fake, 3, 1.0, fake, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, 10, None, 3, 1.0, fake, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, 10, fake, 3, 1.0, None, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, 10, fake, 3, 1.0, fake, sb - 1, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, 10, fake, -3, 1.0, fake, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, -1, fake, 3, 1.0, fake, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, -1, 10, fake, 3, 1.0, fake, sb, fake, None) == -1
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, 2 ** 31, fake, 3, 1.0, fake, sb, fake, None) == -2
    assert lib.fnr_mesh_assign_centers(fake, fake, 10, 10, fake, 2 ** 31, 1.0, fake, sb, fake, None) == -2
    outs = [fake] * 9
    assert lib.fnr_mesh_measure_groups(fake, fake, 10, 10, None, 2, fake, 1 << 30, *outs, fake, fake, None) == -1
    assert lib.fnr_mesh_measure_groups(fake, fake, 10, 10, fake, 2, fake, 1 << 30, *outs[:8], None, fake, fake, None) == -1
    assert lib.fnr_mesh_measure_groups(fake, fake, 10, 10, fake, 2, fake, 1 << 30, *outs, fake, None, None) == -1
    assert lib.fnr_mesh_measure_groups(fake, fake, 10, 10, fake, -1, fake, 1 << 30, *outs, fake, fake, None) == -1
    assert lib.fnr_mesh_measure_groups(fake, fake, 10, -10, fake, 2, fake, 1 << 30, *outs, fake, fake, None) == -1
    assert lib.fnr_mesh_measure_groups(fake, fake, 10, 10, fake, 2 ** 31, fake, 1 << 30, *outs, fake, fake, None) == -2
