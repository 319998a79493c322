"""Deterministic synthetic inputs (parameters, ray batches) for tests, smoke and bench.

Values come from integer hashing, not from a random-number generator, so the very same bits are
produced on any machine / torch version: golden fixtures made in the build container stay valid
on the GPU box.  Workload definition follows SURVEY.md section 8(d) / BASELINE.md section 3.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch
from torch import Tensor

_M32 = 0xFFFFFFFF


def hash_uniform(n: int, salt: int, device="cpu") -> Tensor:
    """n float32 values in [-1, 1), a pure function of (index, salt)."""
    x = torch.arange(n, dtype=torch.int64, device=device)
    x = (x * 2654435761 + (salt * 974711 + 12345)) & _M32
    x = x ^ (x >> 15)
    x = (x * 2246822519) & _M32
    x = x ^ (x >> 13)
    x = (x * 3266489917) & _M32
    x = x ^ (x >> 16)
    return (x.to(torch.float64) / 2147483648.0 - 1.0).to(torch.float32)


def hash_normalish(n: int, salt: int, device="cpu") -> Tensor:
    """Roughly N(0,1): sum of 4 uniforms on [-1,1) scaled to unit variance."""
    u = sum(hash_uniform(n, salt * 7 + k, device) for k in range(4))
    return (u * math.sqrt(3.0 / 4.0)).to(torch.float32)


def field_state(
    geo: int = 15,
    sem_dims=(15, 64, 64),
    log2_hashmap_size: int = 19,
    num_levels: int = 16,
    features: int = 2,
    num_images: int = 100,
    table_scale: float = 1e-3,
    weight_gain: float = 1.0,
    aabb=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)),
    device="cpu",
) -> Dict[str, Tensor]:
    """State dict (reference key names) of a FruitField with hash-generated values.

    Linear layers get the nn.Linear default scale U(-1/sqrt(in), 1/sqrt(in)) (times weight_gain),
    the table U(-1,1)*table_scale, the embedding ~N(0,1)."""
    sd: Dict[str, Tensor] = {}
    salt = [1000]

    def nxt():
        salt[0] += 1
        return salt[0]

    rows = num_levels * 2**log2_hashmap_size
    sd["mlp_base_grid.hash_table"] = (hash_uniform(rows * features, nxt(), device) * table_scale).view(rows, features)

    def linear(key, fan_in, fan_out):
        k = weight_gain / math.sqrt(fan_in)
        sd[f"{key}.weight"] = (hash_uniform(fan_in * fan_out, nxt(), device) * k).view(fan_out, fan_in)
        sd[f"{key}.bias"] = hash_uniform(fan_out, nxt(), device) * k

    base = (num_levels * features, 64, 1 + geo)
    for i in range(2):
        linear(f"mlp_base_mlp.layers.{i}", base[i], base[i + 1])
    for i in range(len(sem_dims) - 1):
        linear(f"mlp_semantics.layers.{i}", sem_dims[i], sem_dims[i + 1])
    linear("field_head_semantics.net", sem_dims[-1], 1)
    col = (16 + geo + 32, 64, 64, 3)
    for i in range(3):
        linear(f"mlp_head.layers.{i}", col[i], col[i + 1])
    sd["embedding_appearance.embedding.weight"] = hash_normalish(num_images * 32, nxt(), device).view(num_images, 32)
    sd["aabb"] = torch.tensor(aabb, dtype=torch.float32, device=device)
    return sd


SMALL = dict(geo=15, sem_dims=(15, 64, 64), log2_hashmap_size=19, max_res=2048)
BIG = dict(geo=30, sem_dims=(30, 128, 128, 64), log2_hashmap_size=21, max_res=4096)


def ray_batch(R: int, S: int, salt: int = 0, near: float = 0.05, far: float = 2.0, num_images: int = 100, device="cpu"):
    """SURVEY.md 8(d) workload: origins U([-0.5,0.5]^3), unit directions, uniform bins on
    [near, far] with one jitter per ray, camera indices in [0, num_images)."""
    o = hash_uniform(R * 3, 11 + salt, device).view(R, 3) * 0.5
    d = hash_normalish(R * 3, 23 + salt, device).view(R, 3)
    d = d / d.norm(dim=-1, keepdim=True).clamp_min(1e-6)
    jitter = (hash_uniform(R, 37 + salt, device).view(R, 1) + 1.0) * 0.5  # [0,1)
    edges = (torch.arange(S + 1, dtype=torch.float32, device=device)[None, :] + jitter * 0.999) / (S + 1)
    t = near + (far - near) * edges
    starts, ends = t[:, :-1].contiguous(), t[:, 1:].contiguous()
    cam = ((hash_uniform(R, 41 + salt, device) + 1.0) * 0.5 * num_images).to(torch.int64).clamp_(0, num_images - 1)
    return o.contiguous(), d.contiguous(), starts, ends, cam


def targets(R: int, salt: int = 0, device="cpu") -> Tuple[Tensor, Tensor]:
    """image ~ U(0,1) [R,3]; fruit_mask ~ Bernoulli(0.1) [R,1] (fruit_nerf.py:359-366 inputs)."""
    img = (hash_uniform(R * 3, 53 + salt, device).view(R, 3) + 1.0) * 0.5
    mask = ((hash_uniform(R, 59 + salt, device).view(R, 1) + 1.0) * 0.5 < 0.1).to(torch.float32)
    return img, mask


def density_state(num_levels: int = 5, log2_hashmap_size: int = 17, hidden: int = 16, table_scale: float = 0.5, weight_gain: float = 1.5,
                  salt: int = 5000, aabb=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), device="cpu") -> Dict[str, Tensor]:
    """State dict (nerfstudio torch-path key names) of a HashMLPDensityField proposal network, hash-generated."""
    rows = num_levels * 2**log2_hashmap_size
    sd = {"encoding.hash_table": (hash_uniform(rows * 2, salt + 1, device) * table_scale).view(rows, 2)}
    k0, k1 = weight_gain / math.sqrt(2 * num_levels), weight_gain / math.sqrt(hidden)
    sd["mlp_base.1.layers.0.weight"] = (hash_uniform(hidden * 2 * num_levels, salt + 2, device) * k0).view(hidden, 2 * num_levels)
    sd["mlp_base.1.layers.0.bias"] = hash_uniform(hidden, salt + 3, device) * k0
    sd["mlp_base.1.layers.1.weight"] = (hash_uniform(hidden, salt + 4, device) * k1).view(1, hidden)
    sd["mlp_base.1.layers.1.bias"] = hash_uniform(1, salt + 5, device) * k1
    sd["aabb"] = torch.tensor(aabb, dtype=torch.float32, device=device)
    return sd


def fruit_shell_cloud(n: int, seed: int = 0, points_per_fruit: int = 4000, fruit_radius: float = 0.035, spacing: float = 0.15,
                      noise_fraction: float = 0.02):
    """[n,3] float64 numpy cloud that looks like an exported semantic cloud of a tree: n // points_per_fruit fruit shells
    (radius ``fruit_radius`` with 3 % radial jitter) on a jittered lattice of pitch ``spacing``, plus a fraction of
    uniform noise over the same box, in shuffled order.  With the defaults its density suits the reference's real-tree
    counting parameters (clustering/config_real.py).  Unlike the hashed inputs above it comes from numpy's seeded
    generator: clustering tests compare the CPU and GPU paths on the same machine."""
    import numpy as np

    rng = np.random.default_rng(seed)
    k = max(1, n // points_per_fruit)
    side = math.ceil(k ** (1.0 / 3.0) - 1e-9)
    cell = np.stack(np.unravel_index(np.arange(k), (side, side, side)), axis=1).astype(np.float64)
    centers = cell * spacing + rng.uniform(-0.15 * spacing, 0.15 * spacing, (k, 3))
    n_noise = int(n * noise_fraction)
    fruit = rng.integers(0, k, n - n_noise)
    dirs = rng.standard_normal((n - n_noise, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    radii = fruit_radius * (1.0 + 0.03 * rng.standard_normal((n - n_noise, 1)))
    shells = centers[fruit] + dirs * radii
    lo, hi = centers.min(axis=0) - 2 * fruit_radius, centers.max(axis=0) + 2 * fruit_radius
    noise = rng.uniform(lo, hi, (n_noise, 3))
    return np.concatenate([shells, noise])[rng.permutation(n)]


def sphere_template(radius: float = 0.035, n: int = 1000):
    """[n,3] float64 fruit template: n points of a Fibonacci lattice on a sphere of ``radius`` about the origin (their
    mean is the origin to rounding).  Stands in for the reference's scanned fruit templates in tests and benchmarks."""
    import numpy as np

    i = np.arange(n, dtype=np.float64) + 0.5
    z = 1.0 - 2.0 * i / n
    r = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    phi = i * (math.pi * (3.0 - math.sqrt(5.0)))
    return radius * np.stack([r * np.cos(phi), r * np.sin(phi), z], axis=1)


def touching_fruit_cloud(seed: int = 0, singles: int = 3, pairs: int = 3, triples: int = 2, fragments: int = 2, fruit_radius: float = 0.035,
                         points_per_fruit: int = 4000, fragment_radius: float = 0.012, points_per_fragment: int = 800,
                         overlap: float = 0.95, spacing: float = 0.3, jitter: float = 0.02):
    """(points [n,3] float64, true fruit centres [K,3]) of a tree-like semantic cloud for the split stage of the count:
    single fruit shells, touching pairs and triples (centres ``overlap`` * 2 * ``fruit_radius`` apart, in random
    orientations) and fragments (shells of ``fragment_radius``, well under 0.3 of a fruit's volume, which are no fruit).
    Shells have ``jitter`` relative radial noise; the groups sit on a lattice of pitch ``spacing`` with random offsets,
    far enough apart that DBSCAN never joins two of them.  At the defaults the density suits the reference's real-tree
    counting parameters (clustering/config_real.py).  numpy's seeded generator, points in shuffled order."""
    import numpy as np

    rng = np.random.default_rng(seed)
    kinds = ["single"] * singles + ["pair"] * pairs + ["triple"] * triples + ["fragment"] * fragments
    side = max(1, math.ceil(len(kinds) ** (1.0 / 3.0) - 1e-9))
    shells, centres = [], []

    def shell(c, radius, n):
        d = rng.standard_normal((n, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        return c + d * (radius * (1.0 + jitter * rng.standard_normal((n, 1))))

    for g, kind in enumerate(rng.permutation(kinds)):
        anchor = np.array(np.unravel_index(g, (side, side, side)), dtype=np.float64) * spacing + rng.uniform(-0.05, 0.05, 3) * spacing
        if kind == "fragment":
            shells.append(shell(anchor, fragment_radius, points_per_fragment))
            continue
        k = {"single": 1, "pair": 2, "triple": 3}[kind]
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))  # random orientation of the group
        step = overlap * 2.0 * fruit_radius
        offsets = np.array([[0.0, 0.0, 0.0], [step, 0.0, 0.0], [step / 2.0, step * math.sqrt(3.0) / 2.0, 0.0]])[:k]
        for c in (offsets - offsets.mean(axis=0)) @ q.T + anchor:
            centres.append(c)
            shells.append(shell(c, fruit_radius, points_per_fruit))
    pts = np.concatenate(shells)
    return pts[rng.permutation(pts.shape[0])], np.array(centres)
