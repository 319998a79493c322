"""Mesh decimation on the host: the numpy restatement of fnr_mesh_decimate (decimate.py) on marched meshes (face count,
manifoldness, topology, orientation, distance from the surface, volume), one round against brute force (selection,
independence, the prefix rule), the quadric cost against a direct sum of plane distances, the tetrahedron and the
octahedron, meshes already at the target, the CLI options and the C-ABI refusals of fnr_decimate.cu (these return before
any launch, so they run without a GPU)."""
import ctypes as C

import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from fruitnerf_b200 import decimate as D
from fruitnerf_b200 import measure
from fruitnerf_b200 import mesh as M


# ---- meshes -------------------------------------------------------------------------------------------------------------
def march(sdf, n=40, lo=-1.0, hi=1.0):
    x = np.linspace(lo, hi, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    m = M.marching_cubes_numpy(sdf(X, Y, Z).astype(np.float32), (lo, lo, lo), ((hi - lo) / (n - 1),) * 3)
    return m["vertices"].astype(np.float64), m["faces"]


def sphere_sdf(c=(0.0, 0.0, 0.0), r=0.7):
    return lambda X, Y, Z: np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r


def torus_sdf(R=0.55, r=0.22):
    return lambda X, Y, Z: np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R) ** 2 + Z ** 2) - r


AX = (0.8, 0.5, 0.35)


def ellipsoid_sdf(X, Y, Z):  # first-order distance of the level set
    a, b, c = AX
    g = (X / a) ** 2 + (Y / b) ** 2 + (Z / c) ** 2
    grad = 2 * np.sqrt((X / a ** 2) ** 2 + (Y / b ** 2) ** 2 + (Z / c ** 2) ** 2)
    return (g - 1) / np.maximum(grad, 1e-9)


def compact(v, f):
    used = np.zeros(len(v), bool)
    used[f.reshape(-1)] = True
    new = np.cumsum(used) - 1
    return v[used], new[f]


def clipped_sphere():
    v, f = march(sphere_sdf())
    return compact(v, f[v[f].mean(axis=1)[:, 2] < 0.35])


def two_spheres():
    s1, s2 = sphere_sdf((-0.45, 0, 0), 0.4), sphere_sdf((0.5, 0.1, 0), 0.35)
    return march(lambda X, Y, Z: np.minimum(s1(X, Y, Z), s2(X, Y, Z)))


def perturbed():
    v, f = march(sphere_sdf(r=0.6), n=14)
    rng = np.random.default_rng(3)
    return v + rng.normal(0, 0.01, v.shape), f


def two_sphere_distance(p):
    d1 = np.abs(np.linalg.norm(p - [-0.45, 0, 0], axis=1) - 0.4)
    d2 = np.abs(np.linalg.norm(p - [0.5, 0.1, 0], axis=1) - 0.35)
    return np.minimum(d1, d2)


# name -> (builder, distance from the analytic surface or None, closed)
MESHES = {
    "sphere": (lambda: march(sphere_sdf()), lambda p: np.abs(sphere_sdf()(*p.T)), True),
    "torus": (lambda: march(torus_sdf()), lambda p: np.abs(torus_sdf()(*p.T)), True),
    "ellipsoid": (lambda: march(ellipsoid_sdf), lambda p: np.abs(ellipsoid_sdf(*p.T)), True),
    "clipped_sphere": (clipped_sphere, lambda p: np.abs(sphere_sdf()(*p.T)), False),
    "two_spheres": (two_spheres, two_sphere_distance, True),
    "perturbed": (perturbed, None, True),
}
FRACTIONS = (0.5, 0.1, 0.01)
# Largest vertex distance from the analytic surface, in units of the grid spacing, and the largest relative change of the
# enclosed volume, at each fraction of the faces kept.  Measured with the restatement over these meshes: the worst
# distance is 0.023 / 0.144 / 5.51 cells (the last on the clipped sphere at 53 faces) and the worst volume change
# 0.07 % / 2.1 % / 33 % (two spheres at 42 faces); the bounds leave about 1.5x.
DIST_BOUND = {0.5: 0.035, 0.1: 0.22, 0.01: 8.0}
VOLUME_BOUND = {0.5: 0.0011, 0.1: 0.031, 0.01: 0.5}

_cache = {}


def decimated(name, frac):
    if (name, frac) not in _cache:
        v, f = MESHES[name][0]()
        N = max(1, int(round(len(f) * frac)))
        _cache[(name, frac)] = (v, f, N, D.restated_decimate(v, f, N))
    return _cache[(name, frac)]


# ---- topology -----------------------------------------------------------------------------------------------------------
def edge_table(f):
    a = f.reshape(-1)
    b = f[:, [1, 2, 0]].reshape(-1)
    key = np.minimum(a, b) * (f.max() + 1) + np.maximum(a, b)
    uniq, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    return a, b, inv, cnt


def boundary_loops(f):
    a, b, inv, cnt = edge_table(f)
    bd = cnt[inv] == 1
    if not bd.any():
        return 0
    n = f.max() + 1
    g = coo_matrix((np.ones(bd.sum()), (a[bd], b[bd])), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    return len(np.unique(lab[a[bd]]))


def components_euler(v, f):
    n = len(v)
    g = coo_matrix((np.ones(2 * len(f)), (np.concatenate([f[:, 0], f[:, 1]]), np.concatenate([f[:, 1], f[:, 2]]))), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    out = []
    for c in np.unique(lab[f[:, 0]]):
        fc = f[lab[f[:, 0]] == c]
        nv = len(np.unique(fc))
        _, _, _, cnt = edge_table(fc)
        out.append(nv - len(cnt) + len(fc))
    return sorted(out)


def check_manifold(f, nv):
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all()
    assert len(np.unique(np.sort(f, axis=1), axis=0)) == len(f)
    assert np.array_equal(np.unique(f), np.arange(nv))
    a, b, inv, cnt = edge_table(f)
    assert cnt.max() <= 2
    # an interior edge is crossed once each way
    directed = a * (f.max() + 1) + b
    inner = cnt[inv] == 2
    assert len(np.unique(directed[inner])) == inner.sum()


@pytest.mark.parametrize("frac", FRACTIONS)
@pytest.mark.parametrize("name", list(MESHES))
def test_restatement_on_marched_meshes(name, frac):
    v, f, N, r = decimated(name, frac)
    ov, of = r["vertices"], r["faces"]
    no_edge_left = len(of) > N + 1 and not D.decimation_round(*_state(ov, of), N)["valid"].any()
    assert len(of) in (N, N + 1) or no_edge_left
    check_manifold(of, len(ov))
    assert boundary_loops(of) == boundary_loops(f)
    assert components_euler(ov, of) == components_euler(v, f)
    assert r["normals"].shape == ov.shape
    if name == "sphere" and frac >= 0.1:  # at 70 faces a face may lean past 90 degrees from the radius without a flip
        nf = D._face_normals(ov, of)
        assert (D._dot(nf, ov[of].mean(axis=1)) > 0).all()
    h = 2.0 / 39 if name != "perturbed" else 2.0 / 13
    dist = MESHES[name][1]
    if dist is not None:
        assert dist(ov).max() <= DIST_BOUND[frac] * h
    if MESHES[name][2] and name != "perturbed":
        vol0 = measure.restated_measure(v, f, np.zeros(len(f), np.int32), 1)["volume"][0]
        vol1 = measure.restated_measure(ov, of, np.zeros(len(of), np.int32), 1)["volume"][0]
        assert abs(vol1 / vol0 - 1) <= VOLUME_BOUND[frac]


def _state(v, f):
    return v, D.initial_quadrics(v, f), f


# ---- one round against brute force --------------------------------------------------------------------------------------
def random_manifold(seed):
    v, f = march(sphere_sdf(r=0.55 + 0.05 * seed), n=10 + seed)
    rng = np.random.default_rng(seed)
    return v + rng.normal(0, 0.02, v.shape), f


@pytest.mark.parametrize("seed", range(4))
def test_one_round_against_brute_force(seed):
    v, f = random_manifold(seed)
    P, Q, _ = _state(v, f)
    N = len(f) // 2
    r = D.decimation_round(P, Q, f, N)
    a, b, valid, rank = r["a"], r["b"], r["valid"], r["rank"]
    assert valid.any()
    # ranks: (cost, edge order) of the valid edges
    vi = np.flatnonzero(valid)
    order = sorted(vi, key=lambda e: (r["cost"][e], e))
    assert [rank[e] for e in order] == list(range(len(vi)))
    # neighbours and stars by brute force
    nb = [set() for _ in range(len(v))]
    star = [set() for _ in range(len(v))]
    for i, face in enumerate(f):
        for x in face:
            star[x].add(i)
            nb[x].update(y for y in face if y != x)
    best = {x: min([rank[e] for e in vi if x in (a[e], b[e])], default=None) for x in range(len(v))}
    for e in vi:
        ring = ({a[e], b[e]} | nb[a[e]] | nb[b[e]])
        least = min(best[x] for x in ring if best[x] is not None)
        assert r["selected"][e] == (rank[e] == least)
    sel = np.flatnonzero(r["selected"])
    touched = [star[a[e]] | star[b[e]] for e in sel]
    for i in range(len(sel)):
        for j in range(i + 1, len(sel)):
            assert not (touched[i] & touched[j])
    # the prefix rule: the kept edges are the selected ones in rank order before the count reaches N + 1
    for target in (len(f) - 3, len(f) - 10, N):
        rr = D.decimation_round(P, Q, f, target)
        kept = np.flatnonzero(rr["kept"])
        count = len(f)
        for e in sorted(sel, key=lambda e: rank[e]):
            if count <= target + 1:
                assert e not in kept
                continue
            assert e in kept
            count -= r["count"][e]
        assert len(rr["faces"]) == count
        if sum(r["count"][sel]) >= len(f) - target:
            assert count in (target, target + 1)


def test_quadric_cost_is_the_sum_of_plane_distances():
    v, f = clipped_sphere()
    Q = D.initial_quadrics(v, f)
    E = D.edges_of(f, len(v))
    rng = np.random.default_rng(0)
    x = v + rng.normal(0, 0.05, v.shape)
    got = D.quadric_cost(Q, x)
    want = np.zeros(len(v))
    for i, face in enumerate(f):
        p = v[face]
        n = np.cross(p[1] - p[0], p[2] - p[0])
        area = np.linalg.norm(n) / 2
        u = n / np.linalg.norm(n)
        for k, vert in enumerate(face):
            want[vert] += area * np.dot(u, x[vert] - p[0]) ** 2
    bd = E["h0"][E["count"] == 1]
    for h in bd:
        face = f[h // 3]
        k = h % 3
        p = v[face]
        n = np.cross(p[1] - p[0], p[2] - p[0])
        e = p[(k + 1) % 3] - p[k]
        m = np.cross(e, n)
        m /= np.linalg.norm(m)
        for vert in (face[k], face[(k + 1) % 3]):
            want[vert] += D.BOUNDARY_WEIGHT * np.dot(e, e) * np.dot(m, x[vert] - p[k]) ** 2
    assert np.allclose(got, want, rtol=1e-9, atol=1e-15)


TETRA = (np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], float), np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]]))
OCTA = (np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], float),
        np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]))


@pytest.mark.parametrize("mesh", [TETRA, OCTA], ids=["tetrahedron", "octahedron"])
@pytest.mark.parametrize("target", [1, 2, 3, 4])
def test_no_doubled_faces(mesh, target):
    r = D.restated_decimate(*mesh, target)
    f = r["faces"]
    assert len(np.unique(np.sort(f, axis=1), axis=0)) == len(f)
    assert len(f) >= 4  # a closed surface stops at the tetrahedron
    check_manifold(f, len(r["vertices"]))


@pytest.mark.parametrize("name", ["sphere", "clipped_sphere"])
def test_mesh_at_the_target_is_unchanged(name):
    v, f = MESHES[name][0]()
    for N in (len(f), len(f) + 5, len(f) - 1):
        r = D.restated_decimate(v, f, N)
        assert r["rounds"] == 0
        assert np.array_equal(r["faces"], f) and np.array_equal(r["vertices"], v)
        assert np.array_equal(r["normals"], D.vertex_normals(v, f))


def test_restatement_refuses():
    v, f = TETRA
    with pytest.raises(ValueError, match=">= 1"):
        D.restated_decimate(v, f, 0)
    with pytest.raises(ValueError, match="face indices"):
        D.restated_decimate(v, f + 1, 2)


# ---- CLI ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("command", ["tsdf", "poisson"])
def test_cli_option_parses(command):
    import argparse

    from fruitnerf_b200.scripts import exporter as X

    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="command")
    add = X.add_tsdf_parser if command == "tsdf" else X.add_poisson_parser
    make = X.tsdf_exporter_from_args if command == "tsdf" else X.poisson_exporter_from_args
    add(sub)
    base = [command, "--load-config", "c.yml", "--output-dir", "o"]
    assert make(ap.parse_args(base)).target_num_faces is None
    exp = make(ap.parse_args(base + ["--texture-method", "nerf", "--unwrap-method", "custom", "--target-num-faces", "50000"]))
    assert exp.target_num_faces == 50000
    exp.validate()


@pytest.mark.parametrize("command", ["tsdf", "poisson"])
@pytest.mark.parametrize("args, match", [
    (["--texture-method", "nerf", "--unwrap-method", "custom", "--target-num-faces", "0"], "target_num_faces"),
    (["--texture-method", "nerf", "--unwrap-method", "custom", "--target-num-faces", "-5"], "target_num_faces"),
    (["--target-num-faces", "1000"], "--texture-method nerf"),
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
    nv, nf, rounds = C.c_int64(0), C.c_int64(0), C.c_int32(0)

    def call(**kw):
        a = dict(v=P, f=P, V=8, F=12, N=4, s=P, sb=1 << 30, ov=P, on=P, of=P, nv=C.byref(nv), nf=C.byref(nf), r=C.byref(rounds))
        a.update(kw)
        return lib.fnr_mesh_decimate(a["v"], a["f"], a["V"], a["F"], a["N"], a["s"], a["sb"], a["ov"], a["on"], a["of"], a["nv"], a["nf"],
                                     a["r"], None)

    for kw in (dict(v=None), dict(f=None), dict(ov=None), dict(on=None), dict(of=None), dict(nv=None), dict(nf=None), dict(r=None),
               dict(V=-1), dict(F=-1), dict(N=0), dict(N=-3)):
        assert call(**kw) == -1, kw
        assert b"fnr_mesh_decimate" in lib.fnr_last_error()
    assert call(V=2 ** 31) == -2 and b"exceed" in lib.fnr_last_error()
    assert call(F=(2 ** 31 - 1) // 3 + 1) == -2
    size = C.c_size_t(0)
    assert lib.fnr_mesh_decimate_scratch_bytes(8, 12, None) == -1
    assert lib.fnr_mesh_decimate_scratch_bytes(-1, 12, C.byref(size)) == -1
    assert lib.fnr_mesh_decimate_scratch_bytes(8, 2 ** 30, C.byref(size)) == -2
    assert b"fnr_mesh_decimate_scratch_bytes" in lib.fnr_last_error()
