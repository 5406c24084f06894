"""Float64 numpy restatement of the outlier filters (include/regtr_b200.h, "Outlier removal"): the exact (d2, index)
k-nearest neighbours, Open3D's RemoveStatisticalOutliers with the library's chunked summation order, the radius rule
of RemoveRadiusOutliers and the stable compaction of regtr_select_points.

Every d2 is (dx dx + dy dy) + dz dz with each operation rounded on its own (numpy does not contract), so the results
are the device's bits.  Large clouds take their candidates from scipy's cKDTree and are then ranked by the exact rule;
`knn(..., brute=True)` ranks every point of the cloud.
"""
from __future__ import annotations

import numpy as np

STAT_CHUNK = 256


def d2_rows(q, p):
    """d2 between q (n,3) and p (n,...,3) rows, the library's rounding."""
    d = q - p
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _rank(xyz, cand, k):
    """Rows of candidate indices (n,w) -> the k smallest (d2, index) per row: (idx (n,k), d2 (n,k))."""
    cand = np.sort(cand, axis=1)                                     # ascending index, then a stable sort by d2
    d2 = d2_rows(xyz[:, None, :], xyz[cand])
    order = np.argsort(d2, axis=1, kind='stable')
    idx = np.take_along_axis(cand, order, 1)[:, :k]
    return idx, np.take_along_axis(d2, order, 1)[:, :k]


def knn(xyz, k: int, brute: bool = False):
    """The min(k, n) nearest neighbours of every point of one cloud, itself included, ascending (d2, index).
    -> (idx (n,m) int64, d2 (n,m) float64)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64)
    n = xyz.shape[0]
    m = min(k, n)
    if n == 0:
        return np.zeros((0, 0), np.int64), np.zeros((0, 0))
    if brute or n <= 4096:
        out_i, out_d = np.empty((n, m), np.int64), np.empty((n, m))
        for a in range(0, n, 256):
            b = min(a + 256, n)
            d2 = d2_rows(xyz[a:b, None, :], xyz[None, :, :])
            order = np.argsort(d2, axis=1, kind='stable')[:, :m]      # ties: the lower index (stable on 0..n-1)
            out_i[a:b] = order
            out_d[a:b] = np.take_along_axis(d2, order, 1)
        return out_i, out_d
    from scipy.spatial import cKDTree
    tree = cKDTree(xyz)
    w = min(n, m + 8)
    dist, cand = tree.query(xyz, k=w)
    dist, cand = dist.reshape(n, w), cand.reshape(n, w)
    idx, d2 = _rank(xyz, cand, m)
    # complete where every point outside the w candidates is provably farther than the m-th key
    ok = np.full(n, True) if w == n else dist[:, w - 1] > np.sqrt(d2[:, m - 1]) * (1 + 1e-9) + 1e-300
    for i in np.flatnonzero(~ok):
        near = np.array(tree.query_ball_point(xyz[i], np.sqrt(d2[i, m - 1]) * (1 + 1e-9) + 1e-300), np.int64)
        idx[i], d2[i] = _rank_one(xyz, i, near, m)
    return idx, d2


def _rank_one(xyz, i, cand, m):
    cand = np.sort(cand)
    d2 = d2_rows(xyz[i][None, :], xyz[cand])
    order = np.argsort(d2, kind='stable')[:m]
    return cand[order], d2[order]


def knn_avg(xyz, k: int, brute: bool = False):
    """avg_i = (sum of sqrt(d2) in ascending key order) / m per point."""
    _, d2 = knn(xyz, k, brute)
    s = np.zeros(d2.shape[0])
    for e in range(d2.shape[1]):
        s = s + np.sqrt(d2[:, e])
    return s / max(d2.shape[1], 1)


def chunk_sum(v):
    """The header's order: chunks of 256 anchored at v[0], each by the tree e[i] += e[i + h], h = 128..1, partials
    added in ascending order from 0."""
    v = np.asarray(v, np.float64)
    nch = -(-v.shape[0] // STAT_CHUNK)
    e = np.zeros(nch * STAT_CHUNK)
    e[:v.shape[0]] = v
    e = e.reshape(nch, STAT_CHUNK)
    while e.shape[1] > 1:
        h = e.shape[1] // 2
        e = e[:, :h] + e[:, h:]
    s = 0.0
    for p in e[:, 0]:
        s = s + p
    return np.float64(s)


def cloud_stats(avg, std_ratio: float):
    """(cloud_mean, std_dev, threshold) of one cloud's avg, Open3D's rule in the header's summation order."""
    avg = np.asarray(avg, np.float64)
    valid = np.float64(avg.shape[0])
    pos = avg > 0
    with np.errstate(invalid='ignore', divide='ignore'):
        mean = chunk_sum(np.where(pos, avg, 0.0)) / valid
        dev = avg - mean
        sq = chunk_sum(np.where(pos, dev * dev, 0.0))
        sd = np.sqrt(sq / (valid - 1.0))
        thr = mean + np.float64(std_ratio) * sd
    return np.float64(mean), np.float64(sd), np.float64(thr)


def statistical_outlier(xyz, nb_neighbors: int, std_ratio: float, brute: bool = False):
    """One cloud -> (avg (n,), keep (n,) int32, (mean, std, threshold))."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    avg = knn_avg(xyz, nb_neighbors, brute)
    st = cloud_stats(avg, std_ratio)
    with np.errstate(invalid='ignore'):
        keep = ((avg > 0) & (avg < st[2])).astype(np.int32)
    return avg, keep, st


def radius_counts(xyz, radius: float, brute: bool = False):
    """Points of the cloud with d2 strictly below radius^2, the point itself included."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
    n = xyz.shape[0]
    r2 = np.float64(radius) * np.float64(radius)
    if n == 0:
        return np.zeros(0, np.int32)
    if brute or n <= 4096:
        out = np.empty(n, np.int32)
        for a in range(0, n, 256):
            b = min(a + 256, n)
            out[a:b] = (d2_rows(xyz[a:b, None, :], xyz[None, :, :]) < r2).sum(1)
        return out
    from scipy.spatial import cKDTree
    tree = cKDTree(xyz)
    near = tree.query_ball_point(xyz, radius * (1 + 1e-9) + 1e-300)
    out = np.empty(n, np.int32)
    for i, nb in enumerate(near):
        nb = np.asarray(nb, np.int64)
        out[i] = int((d2_rows(xyz[i][None, :], xyz[nb]) < r2).sum())
    return out


def radius_outlier(xyz, nb_points: int, radius: float, brute: bool = False):
    """One cloud -> (counts (n,) int32, keep (n,) int32)."""
    counts = radius_counts(xyz, radius, brute)
    return counts, (counts >= nb_points).astype(np.int32)


def select_points(xyz, keep, colors=None):
    """Stable compaction of one cloud -> (kept xyz, kept colours or None, kept indices)."""
    idx = np.flatnonzero(np.asarray(keep) != 0)
    return (np.asarray(xyz, np.float64).reshape(-1, 3)[idx],
            None if colors is None else np.asarray(colors, np.float64).reshape(-1, 3)[idx], idx)


def outlier_scan(seed: int, n: int = 300000, frac: float = 0.01, noise: float = 0.002):
    """A seeded synthetic scan: n points on the six faces of a 4 x 3 x 2.5 m room (area-weighted, Gaussian noise of
    `noise` m along every axis), a fraction `frac` of them replaced by points uniform in the room's box grown by
    0.5 m, in random order.  -> (xyz (n,3) float64, outlier mask (n,) bool)."""
    rng = np.random.default_rng(seed)
    size = np.array([4.0, 3.0, 2.5])
    n_out = int(round(n * frac))
    faces = [(a, side) for a in range(3) for side in (0.0, 1.0)]
    area = np.array([np.prod(np.delete(size, a)) for a, _ in faces])
    pick = rng.choice(len(faces), n - n_out, p=area / area.sum())
    pts = rng.random((n - n_out, 3)) * size
    for f, (a, side) in enumerate(faces):
        pts[pick == f, a] = side * size[a]
    pts += rng.normal(scale=noise, size=pts.shape)
    out = rng.random((n_out, 3)) * (size + 1.0) - 0.5
    xyz = np.concatenate([pts, out])
    mask = np.concatenate([np.zeros(n - n_out, bool), np.ones(n_out, bool)])
    order = rng.permutation(n)
    return xyz[order], mask[order]
