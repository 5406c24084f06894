"""Seeded synthetic point-cloud pairs shaped like the reference's datasets.

There is no network for 3DMatch / ModelNet40, so every benchmark and parity test
runs on synthetic pairs whose *statistics* follow the real data measured in
SURVEY.md 8d: 3DMatch fragments are voxel-averaged at 2.5 cm, hold 17-25k points
and see ~30 neighbours inside r = 6.25 cm; the pyramid then yields ~10k / ~2.7k /
~0.7k points.  Seeds follow SURVEY.md: seed = 1000 * config + pair_index.
All outputs are numpy float32; generation is pure numpy (PCG64) and therefore
bit-identical on the build container and the GPU box.
"""
from __future__ import annotations

import numpy as np


def random_rotation(rng, max_deg=45.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = np.deg2rad(rng.uniform(-max_deg, max_deg))
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)


def _voxel_average(pts, dl):
    """Barycentre per voxel (what the dataset's 2.5 cm pre-voxelisation does)."""
    key = np.floor(pts / dl).astype(np.int64)
    key -= key.min(0)
    dims = key.max(0) + 1
    flat = (key[:, 0] * dims[1] + key[:, 1]) * dims[2] + key[:, 2]
    uniq, inv = np.unique(flat, return_inverse=True)
    out = np.zeros((len(uniq), 3))
    np.add.at(out, inv, pts)
    cnt = np.bincount(inv, minlength=len(uniq))[:, None]
    return out / cnt


def _room_surfaces(rng, extent, n_planes, n_boxes):
    """List of (origin, u, v) parallelogram patches: walls/floor pieces + box faces."""
    patches = []
    ex = np.asarray(extent, dtype=np.float64)
    for _ in range(n_planes):
        ax = rng.integers(0, 3)
        o = rng.uniform(0, 1, 3) * ex * 0.5
        o[ax] = rng.choice([0.0, ex[ax]]) if rng.random() < 0.6 else rng.uniform(0, ex[ax])
        u = np.zeros(3); v = np.zeros(3)
        a1, a2 = [a for a in range(3) if a != ax]
        u[a1] = rng.uniform(0.5, 1.0) * ex[a1] * 0.9
        v[a2] = rng.uniform(0.5, 1.0) * ex[a2] * 0.9
        patches.append((o, u, v))
    for _ in range(n_boxes):
        size = rng.uniform(0.25, 0.8, 3)
        o = rng.uniform(0, 1, 3) * (ex - size)
        R = random_rotation(rng, 30.0)
        e = [R[:, i] * size[i] for i in range(3)]
        for i, (a, b) in enumerate(((0, 1), (0, 2), (1, 2))):
            c = 3 - a - b
            patches.append((o, e[a], e[b]))
            patches.append((o + e[c], e[a], e[b]))
    return patches


def _sample_patches(rng, patches, density):
    pts = []
    for o, u, v in patches:
        area = np.linalg.norm(np.cross(u, v))
        n = max(8, int(area * density))
        ab = rng.random((n, 2))
        pts.append(o + ab[:, :1] * u + ab[:, 1:] * v)
    return np.concatenate(pts, 0)


_PTS_PER_M2 = 3000.0


def make_3dmatch_pair(seed: int, n_target: int = 20000, overlap=(0.3, 0.6), voxel=0.025,
                      noise=0.006):
    """One 3DMatch-like pair.  Returns dict(src_xyz, tgt_xyz, pose (3,4) src->tgt)."""
    rng = np.random.default_rng(seed)
    extent = np.array([3.0, 2.3, 2.7])
    patches = _room_surfaces(rng, extent, rng.integers(5, 9), rng.integers(3, 7))
    ov = rng.uniform(*overlap)
    frac = 1.0 / (2.0 - ov)                        # each crop covers `frac` of the span
    # Scale the room so that one crop holds ~n_target voxel-averaged points: a noisy
    # surface fills ~1.9 voxel layers, i.e. ~3000 points per m^2 at 2.5 cm.
    area = sum(np.linalg.norm(np.cross(u, v)) for _, u, v in patches)
    s = np.sqrt(n_target / (_PTS_PER_M2 * frac * area))
    patches = [(o * s, u * s, v * s) for o, u, v in patches]
    scene = _sample_patches(rng, patches, density=16000.0)
    scene = scene + rng.normal(scale=noise, size=scene.shape)
    # two overlapping crops along a random (mostly horizontal) direction
    d = rng.normal(size=3); d[2] *= 0.2; d /= np.linalg.norm(d)
    proj = scene @ d
    lo, hi = proj.min(), proj.max()
    span = hi - lo
    src = scene[proj <= lo + frac * span]
    tgt = scene[proj >= hi - frac * span]
    clouds = []
    for c in (src, tgt):
        c = _voxel_average(c, voxel)
        clouds.append(c[rng.permutation(len(c))])  # real fragments come in hash order
    R = random_rotation(rng, 45.0)
    t = rng.uniform(-0.5, 0.5, 3)
    src_xyz = clouds[0]
    tgt_xyz = clouds[1]
    # src lives in its own frame: tgt = R src + t
    src_xyz = (src_xyz - t) @ R                      # R^T (x - t)
    tgt_xyz = tgt_xyz + rng.normal(scale=0.005, size=tgt_xyz.shape)   # augment_noise 0.005
    pose = np.concatenate([R, t[:, None]], 1)
    return dict(src_xyz=src_xyz.astype(np.float32), tgt_xyz=tgt_xyz.astype(np.float32),
                pose=pose.astype(np.float32))


def make_modelnet_pair(seed: int, n_points: int = 1024, keep: float = 0.7):
    """One ModelNet-like pair: a union of ellipsoid / box surfaces in the unit cube,
    each cloud cropped to `keep` by a random half-space (conf/modelnet.yaml:16-19)."""
    rng = np.random.default_rng(seed)
    parts = []
    n_shapes = rng.integers(3, 6)
    for _ in range(n_shapes):
        c = rng.uniform(-0.4, 0.4, 3)
        s = rng.uniform(0.15, 0.45, 3)
        n = n_points
        if rng.random() < 0.5:
            v = rng.normal(size=(n, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
            parts.append(c + v * s)
        else:
            f = rng.integers(0, 3, n); sign = rng.choice([-1.0, 1.0], n)
            p = rng.uniform(-1, 1, (n, 3)); p[np.arange(n), f] = sign
            parts.append(c + p * s)
    shape = np.concatenate(parts, 0)
    shape /= np.abs(shape).max() * 1.0
    clouds = []
    for _ in range(2):
        p = shape[rng.choice(len(shape), n_points, replace=False)]
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        proj = p @ d
        p = p[proj <= np.quantile(proj, keep)]
        clouds.append(p + rng.normal(scale=0.005, size=p.shape))
    R = random_rotation(rng, 45.0)
    t = rng.uniform(-0.5, 0.5, 3)
    src = (clouds[0] - t) @ R
    pose = np.concatenate([R, t[:, None]], 1)
    return dict(src_xyz=src.astype(np.float32), tgt_xyz=clouds[1].astype(np.float32),
                pose=pose.astype(np.float32))


def make_batch(config_id: int, n_pairs: int, first_pair: int = 0, n_target: int | None = None):
    """Batch for BASELINE.json config `config_id` (1-5): dict of lists src_xyz / tgt_xyz / pose."""
    out = dict(src_xyz=[], tgt_xyz=[], pose=[])
    for i in range(first_pair, first_pair + n_pairs):
        seed = 1000 * config_id + i
        if config_id == 1:
            p = make_modelnet_pair(seed)
        elif config_id == 5:
            p = make_3dmatch_pair(seed, n_target or 30000, overlap=(0.1, 0.3))
        else:
            p = make_3dmatch_pair(seed, n_target or 20000)
        for k in out:
            out[k].append(p[k])
    return out


def make_modelnet_shapes(n_shapes: int, seed: int = 0, n_points: int = 2048, n_dup: int = 8) -> np.ndarray:
    """(n_shapes, n_points, 3) float32 ModelNet40-like shapes (the h5 files hold 2048 points per shape): unions of
    ellipsoid and box surfaces inside the unit ball, with `n_dup` points repeated so that crop distances tie."""
    rng = np.random.default_rng(seed)
    out = np.empty((n_shapes, n_points, 3), np.float32)
    for s in range(n_shapes):
        parts = []
        k = int(rng.integers(2, 5))
        sizes = np.diff(np.sort(np.concatenate([[0, n_points], rng.choice(np.arange(1, n_points), k - 1, replace=False)])))
        for n in sizes:
            c, r = rng.uniform(-0.3, 0.3, 3), rng.uniform(0.15, 0.45, 3)
            if rng.random() < 0.5:
                v = rng.normal(size=(n, 3)); v /= np.linalg.norm(v, axis=1, keepdims=True)
                parts.append(c + v * r)
            else:
                f = rng.integers(0, 3, n); sign = rng.choice([-1.0, 1.0], n)
                p = rng.uniform(-1, 1, (n, 3)); p[np.arange(n), f] = sign
                parts.append(c + p * r)
        shape = np.concatenate(parts, 0)
        shape /= np.linalg.norm(shape, axis=1).max()
        if n_dup:
            dst = rng.choice(n_points, n_dup, replace=False)
            shape[dst] = shape[rng.choice(np.setdiff1d(np.arange(n_points), dst), n_dup, replace=False)]
        out[s] = shape
    return out
