"""Float64 numpy restatement of the training-data path (not collected: no test_ prefix).

* `nearest_within`: brute force, chunked: for every point of `a` the nearest point of `b` with float64 squared
  distance ((dx dx + dy dy) + dz dz) strictly below r * r, the lowest index on equal distances, or -1.
* `overlap`: utils/pointcloud.py:8-65 on the source moved by the pose (((r0 x + r1 y) + r2 z) + t per coordinate):
  masks, the mutual correspondences with the reference's `src_corr > 0` quirk, and both nearest-index arrays.
* The four transforms of data_loaders/transforms.py:15-149 with EXPLICIT draws instead of the global random
  streams: `rigid_perturb`, `jitter`, `shuffle_points`, `random_swap`.
"""
from __future__ import annotations

import numpy as np


def nearest_within(a: np.ndarray, b: np.ndarray, r: float, chunk: int = 512) -> np.ndarray:
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    out = np.full(a.shape[0], -1, np.int64)
    if b.shape[0] == 0:
        return out
    r2 = r * r
    for s in range(0, a.shape[0], chunk):
        q = a[s:s + chunk]
        dx, dy, dz = (q[:, None, k] - b[None, :, k] for k in range(3))
        d2 = (dx * dx + dy * dy) + dz * dz
        j = np.argmin(d2, axis=1)                       # first index of the minimum: lowest index on ties
        best = d2[np.arange(q.shape[0]), j]
        out[s:s + chunk] = np.where(best < r2, j, -1)
    return out


def align(src: np.ndarray, pose: np.ndarray) -> np.ndarray:
    """pose (3,4) applied to src (n,3) with the kernel's operation order."""
    x, y, z = src[:, 0], src[:, 1], src[:, 2]
    return np.stack([((pose[a, 0] * x + pose[a, 1] * y) + pose[a, 2] * z) + pose[a, 3] for a in range(3)], axis=1)


def overlap(src: np.ndarray, tgt: np.ndarray, pose: np.ndarray, r: float):
    """-> src_mask, tgt_mask, corr (2, M) int64, s2t, t2s."""
    sa = align(np.asarray(src, np.float64), np.asarray(pose, np.float64))
    s2t = nearest_within(sa, tgt, r)
    t2s = nearest_within(tgt, sa, r)
    mutual = (s2t > 0) & (t2s[np.maximum(s2t, 0)] == np.arange(len(s2t))) if len(t2s) else s2t > 0
    corr = np.stack([np.nonzero(mutual)[0], s2t[mutual]]).astype(np.int64)
    return s2t >= 0, t2s >= 0, corr, s2t, t2s


# ------------------------------------------------------------------------------------------------ transforms
def se3_inv(p):
    r = p[:, :3].T
    return np.concatenate([r, -(r @ p[:, 3:4])], axis=1)


def se3_cat(a, b):
    return np.concatenate([a[:, :3] @ b[:, :3], a[:, :3] @ b[:, 3:4] + a[:, 3:4]], axis=1)


def se3_transform(p, xyz):
    return xyz @ p[:, :3].T + p[:, 3]


def axis_angle(axis, angle):
    k = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    return np.eye(3) + np.sin(angle) * k + (1.0 - np.cos(angle)) * (k @ k)


def sphere(phi, cos_theta):
    """so3_common.uniform_2_sphere given its two uniforms."""
    t = np.arccos(cos_theta)
    return np.array([np.sin(t) * np.cos(phi), np.sin(t) * np.sin(phi), np.cos(t)])


def pose_small(phi, cos_theta, theta_n, trans_n, std=0.1):
    """SE3.sample_small(std) given its draws: uniform(0, 2 pi), uniform(-1, 1), randn(), randn(3, 1)."""
    rot = axis_angle(sphere(phi, cos_theta), theta_n * std * np.pi / np.sqrt(3))
    return np.concatenate([rot, np.reshape(trans_n, (3, 1)) * std / np.sqrt(3)], axis=1)


def pose_large(euler):
    from scipy.spatial.transform import Rotation
    return np.concatenate([Rotation.from_euler('zyx', euler).as_matrix(), np.zeros((3, 1))], axis=1)


def rigid_perturb(data, perturb, perturb_source: bool, centre: bool):
    """RigidPerturb given the perturbation (3,4) and the side; centre: the 'small' mode's rotation about the
    perturbed cloud's centroid."""
    d = dict(data)
    if centre:
        c = np.mean(d['src_xyz'] if perturb_source else d['tgt_xyz'], axis=0)
        perturb = se3_cat(se3_cat(np.concatenate([np.eye(3), c[:, None]], 1), perturb),
                          np.concatenate([np.eye(3), -c[:, None]], 1))
    if perturb_source:
        d['pose'] = se3_cat(d['pose'], se3_inv(perturb))
        d['src_xyz'] = se3_transform(perturb, d['src_xyz'])
    else:
        d['pose'] = se3_cat(perturb, d['pose'])
        d['tgt_xyz'] = se3_transform(perturb, d['tgt_xyz'])
    return d


def jitter(data, noise_src, noise_tgt):
    d = dict(data)
    d['src_xyz'] = d['src_xyz'] + noise_src
    d['tgt_xyz'] = d['tgt_xyz'] + noise_tgt
    return d


def shuffle_points(data, src_idx, tgt_idx):
    """ShufflePoints given the (already truncated) index arrays."""
    d = dict(data)
    if 'correspondences' in d:
        srev = np.full(d['src_xyz'].shape[0], -1, np.int64); srev[src_idx] = np.arange(len(src_idx))
        trev = np.full(d['tgt_xyz'].shape[0], -1, np.int64); trev[tgt_idx] = np.arange(len(tgt_idx))
        c = np.stack([srev[d['correspondences'][0]], trev[d['correspondences'][1]]]).reshape(2, -1)
        d['correspondences'] = c[:, np.all(c >= 0, axis=0)]
    for k, idx in (('src_xyz', src_idx), ('src_overlap', src_idx), ('tgt_xyz', tgt_idx), ('tgt_overlap', tgt_idx)):
        if k in d:
            d[k] = d[k][idx]
    return d


def random_swap(data, swap: bool):
    d = dict(data)
    if swap:
        for a, b in (('src_xyz', 'tgt_xyz'), ('src_overlap', 'tgt_overlap'), ('src_path', 'tgt_path')):
            if a in d:
                d[a], d[b] = d[b], d[a]
        if 'correspondences' in d:
            d['correspondences'] = d['correspondences'][::-1].copy()
        if 'pose' in d:
            d['pose'] = se3_inv(d['pose'])
    return d


def real_pairs(golden_dir: str):
    """The two real 3DMatch benchmark pairs as (src, tgt, pose (3,4), row) in float64, with the info rows' mapping:
    the row's source cloud is the fixture's `tgt_xyz` when the fixture's `src_file` is the row's target."""
    import json
    import os
    rows = json.load(open(os.path.join(golden_dir, 'real', 'test_3DMatch_info_rows.json')))
    out = []
    for r in rows:
        inp = np.load(os.path.join(golden_dir, 'real', r['fixture'] + '_input.npz'))
        cloud = {}
        for rel in (r['src'], r['tgt']):
            which = 'src_xyz' if os.path.basename(rel) == os.path.basename(str(inp['src_file'])) else 'tgt_xyz'
            cloud[rel] = inp[which].astype(np.float64)
        pose = np.concatenate([np.array(r['rot'], np.float64), np.array(r['trans'], np.float64).reshape(3, 1)], 1)
        out.append((cloud[r['src']], cloud[r['tgt']], pose, r))
    return out
