"""Float64 numpy restatement of voxel down-sampling (`ops.voxel_down_sample`) and of multi-scale ICP (`eval.icp_refine`
with voxels=); not collected: no test_ prefix.

Down-sampling (Open3D's voxel_down_sample, with this library's order rule):

* Per cloud: lo = the per-axis minimum, origin = lo - 0.5 V, v = floor((p - origin) / V) per axis (numpy's float64
  subtraction and division, each rounded to nearest).  An index outside 0..65535 or a non-finite coordinate is
  refused (ValueError here, REGTR_STATUS_KEY_RANGE on the device).
* One row per occupied voxel in ascending (vx, vy, vz); the row is the sum of the member points in ascending point index,
  added one by one, divided by the count.  Attributes (colours) alike.

Multi-scale ICP, per level l of voxels V_l (strictly decreasing; a last V = 0 means the full clouds): both clouds (and
their colours) down-sampled at V_l, then the single-level method at radius R_l (default V_l; the positional radius at
V = 0) for at most I_l iterations, starting from the previous level's pose (level 0 from init).  Normals at 2 R_l with
normal_max_nn neighbours (the target's; both clouds' for generalized), colour gradients at 2 R_l with 30 neighbours.
"""
from __future__ import annotations

import numpy as np

import colored_icp_oracle as C
import gicp_oracle as G
import icp_oracle as I
import icp_plane_oracle as N

MAX_INDEX = 65535


def voxel_indices(xyz, voxel: float) -> np.ndarray:
    """(n,3) float64 points -> (n,3) int64 voxel indices of the bounding-box-anchored grid."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    if xyz.shape[0] == 0:
        return np.zeros((0, 3), np.int64)
    origin = xyz.min(axis=0) - 0.5 * voxel
    v = np.floor((xyz - origin) / voxel)
    if not np.isfinite(xyz).all() or not ((v >= 0) & (v <= MAX_INDEX)).all():
        raise ValueError(f'voxel_down_sample: a voxel index beyond 0..{MAX_INDEX} or a non-finite coordinate')
    return v.astype(np.int64)


def voxel_down_sample(xyz, voxel: float, attr=None):
    """One cloud -> (points (m,3), attributes (m,3) or None, members: list of m ascending index arrays)."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    v = voxel_indices(xyz, voxel)
    key = (v[:, 0] << 32) | (v[:, 1] << 16) | v[:, 2]
    order = np.argsort(key, kind='stable')
    _, start, counts = np.unique(key[order], return_index=True, return_counts=True)
    cols = [xyz] + ([] if attr is None else [np.asarray(attr, np.float64).reshape(-1, 3)])
    sums = [np.zeros((len(start), 3)) for _ in cols]
    for k in range(int(counts.max()) if len(counts) else 0):       # k-th member of every voxel that has one
        g = np.nonzero(counts > k)[0]
        for s, c in zip(sums, cols):
            s[g] += c[order[start[g] + k]]
    means = [s / counts[:, None] for s in sums]
    members = [order[a:a + n] for a, n in zip(start, counts)]
    return means[0], (means[1] if attr is not None else None), members


def level_plan(voxels, radii=None, level_iters=None, radius: float = None, max_iteration: int = 30):
    """-> [(V_l, R_l, I_l)]: radii default to the voxels (the positional radius at V = 0), iterations to
    max_iteration."""
    L = len(voxels)
    radii = [None] * L if radii is None else list(radii)
    iters = [max_iteration] * L if level_iters is None else list(level_iters)
    return [(float(v), float(r if r is not None else (v if v > 0 else radius)), int(i))
            for v, r, i in zip(voxels, radii, iters)]


def single_level(method, src, tgt, init, r, max_iteration, normal_max_nn=30, colors=None, lambda_geometric=0.968,
                 epsilon=1e-3, loss='l2', loss_k=None):
    """`icp_refine`'s single-level body for one pair: -> the oracle's dict(pose, fitness, rmse, k, iterations)."""
    if method == 'point_to_point':
        return I.icp(src, tgt, init, r, max_iteration)
    nt, _ = N.estimate_normals(tgt, 2.0 * r, normal_max_nn)
    if method == 'point_to_plane':
        if loss == 'l2':
            return N.icp(src, tgt, nt, init, r, max_iteration)
        return G.icp(src, tgt, nt, init, r, max_iteration, method='point_to_plane', loss=loss, loss_k=loss_k)
    if method == 'generalized':
        ns, _ = N.estimate_normals(src, 2.0 * r, normal_max_nn)
        return G.icp(src, tgt, nt, init, r, max_iteration, src_normals=ns, epsilon=epsilon, loss=loss, loss_k=loss_k)
    grad = C.color_gradients(tgt, nt, colors[1], 2.0 * r, 30)
    return C.icp(src, tgt, nt, colors[0], colors[1], grad, init, r, max_iteration, lambda_geometric=lambda_geometric,
                 loss=loss, loss_k=loss_k)


def multiscale_icp(src, tgt, init, voxels, radii=None, level_iters=None, radius: float = None,
                   max_iteration: int = 30, method: str = 'point_to_point', colors=None, **kw):
    """One pair through the pyramid: -> dict(pose (3,4), fitness, rmse, k, iterations of the last level, levels (L,4)
    = fitness, rmse, k, iterations per level).  colors=(src_rgb, tgt_rgb) with method='colored'; kw: normal_max_nn,
    lambda_geometric, epsilon, loss, loss_k."""
    T = np.asarray(init, np.float64).reshape(3, 4)
    levels, o = [], None
    for v, r, it in level_plan(voxels, radii, level_iters, radius, max_iteration):
        if v > 0:
            s, sc, _ = voxel_down_sample(src, v, None if colors is None else colors[0])
            t, tc, _ = voxel_down_sample(tgt, v, None if colors is None else colors[1])
        else:
            s, t = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
            sc, tc = (None, None) if colors is None else colors
        o = single_level(method, s, t, T, r, it, colors=(sc, tc), **kw)
        T = o['pose']
        levels.append([o['fitness'], o['rmse'], o['k'], o['iterations']])
    return dict(o, levels=np.array(levels, np.float64))
