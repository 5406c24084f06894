"""Float64 numpy + scipy restatement of FPFH features and their matching (`ops.fpfh`, `ops.feature_match`,
`ops.feature_correspondences`; not collected: no test_ prefix).

Open3D's ComputeFPFHFeature(KDTreeSearchParamHybrid(r, max_nn)) and the matching of
registration_ransac_based_on_feature_matching, with the library's rules:

* Neighbours: `icp_plane_oracle.neighbours` (own cloud, d2 = (dx dx + dy dy) + dz dz strictly below r * r, the point
  itself included, the max_nn smallest by (d2, index)).  Fewer than 2 neighbours: a zero SPFH and FPFH row.
* Pair feature (p1, n1, p2, n2), every product and sum rounded on its own, dot products (x x + y y) + z z:
  d = p2 - p1 (zero feature when |d| = 0); a1 = n1.d / |d|, a2 = n2.d / |d|; when |a1| < |a2| (Open3D's
  acos(|a1|) > acos(|a2|) without the acos), n1 <-> n2, d -> -d, f2 = -a2, else f2 = a1; v = d x n1 (zero feature
  when |v| = 0), v /= |v|; w = n1 x v; f1 = v.n2; f0 = atan2(w.n2, n1.n2).
* SPFH: entries k >= 1 (entry 0 skipped whatever it is) add 100 / (count - 1) to bins floor(11 (f0 + pi) / 2pi),
  11 + floor(11 (f1 + 1) 0.5), 22 + floor(11 (f2 + 1) 0.5), each floor clamped to 0..10, in entry order.
* FPFH: entries k >= 1 with d2 != 0, in order, add val = spfh[j][b] / d2 to feature[b] and to sum[b // 11]; then
  feature[b] = feature[b] * (100 / sum if sum != 0 else 0) + spfh[i][b].
* Matching: d2(i, j) = sum over k = 0..32 of (a_k - b_k)^2, accumulated column by column as the device does; the
  forward match of source i is the lowest (d2, j), the reverse match of target j the lowest (d2, i) (numpy's argmin
  keeps the first minimum); match i is mutual when reverse[forward[i]] == i.  The mask is the mutual set, or every
  match without the mutual filter or when fewer than min_mutual (3 ransac_n) are mutual.

The device reproduces every bit except the ulps of libdevice's atan2; the tests hold it to 1e-9 and to identical bins.
"""
from __future__ import annotations

import numpy as np

import icp_plane_oracle as PO
import ransac_oracle as RO

DIM = 33


def dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross3(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def pair_features(p1, n1, p2, n2):
    """(m,3) arrays each -> (m,3) (f0, f1, f2), zero rows for the zero feature."""
    p1, n1, p2, n2 = (np.asarray(x, np.float64).reshape(-1, 3) for x in (p1, n1, p2, n2))
    d = p2 - p1
    dn = np.sqrt(dot3(d, d))
    ok = dn != 0.0
    dd = np.where(ok, dn, 1.0)
    a1, a2 = dot3(n1, d) / dd, dot3(n2, d) / dd
    sw = (np.abs(a1) < np.abs(a2))[:, None]
    m1, m2, d = np.where(sw, n2, n1), np.where(sw, n1, n2), np.where(sw, -d, d)
    f2 = np.where(sw[:, 0], -a2, a1)
    v = cross3(d, m1)
    vn = np.sqrt(dot3(v, v))
    ok &= vn != 0.0
    v = v / np.where(vn != 0.0, vn, 1.0)[:, None]
    w = cross3(m1, v)
    out = np.stack([np.arctan2(dot3(w, m2), dot3(m1, m2)), dot3(v, m2), f2], -1)
    out[~ok] = 0.0
    return out


def bins(pf):
    """(m,3) pair features -> (m,3) bin indices 0..32."""
    def clamp(x):
        return np.clip(np.floor(x), 0, 10).astype(np.int64)
    return np.stack([clamp(11.0 * (pf[:, 0] + np.pi) / (2.0 * np.pi)),
                     11 + clamp(11.0 * (pf[:, 1] + 1.0) * 0.5),
                     22 + clamp(11.0 * (pf[:, 2] + 1.0) * 0.5)], -1)


def fpfh(xyz, normals, r: float, max_nn: int = 100):
    """One cloud -> dict(feature (n,33), spfh (n,33), counts (n,), bins (m,3) of every SPFH entry (q, j))."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    nrm = np.asarray(normals, np.float64).reshape(-1, 3)
    n = xyz.shape[0]
    q, j, d2 = PO.neighbours(xyz, r, max_nn)
    cnt = np.bincount(q, minlength=n)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    later = np.arange(q.shape[0]) != start[q]                     # entries k >= 1
    sel = later & (cnt[q] > 1)
    qq, jj, dd = q[sel], j[sel], d2[sel]
    b = bins(pair_features(xyz[qq], nrm[qq], xyz[jj], nrm[jj]))
    inc = 100.0 / np.maximum(cnt[qq] - 1, 1)
    spfh = np.zeros((n, DIM))
    for c in range(3):
        np.add.at(spfh, (qq, b[:, c]), inc)                       # sequential, in entry order
    feat = np.zeros((n, DIM))
    sums = np.zeros((n, 3))
    nz = dd != 0.0
    qn, jn, dn = qq[nz], jj[nz], dd[nz]
    val = spfh[jn] / dn[:, None]
    # np.add.at applies its rows one after the other: per point, feature[b] in entry order and sum[t] in (entry, bin)
    # order, as the device adds them
    np.add.at(feat, qn, val)
    for t in range(3):
        np.add.at(sums[:, t], np.repeat(qn, 11), val[:, 11 * t:11 * t + 11].reshape(-1))
    scale = np.where(sums != 0.0, 100.0 / np.where(sums != 0.0, sums, 1.0), 0.0)
    feat = feat * np.repeat(scale, 11, axis=1) + spfh
    feat[cnt < 2] = 0.0
    return dict(feature=feat, spfh=spfh, counts=cnt, bins=b, pairs=(qq, jj))


def feature_d2(fs, ft):
    """(n_s,33), (n_t,33) -> (n_s,n_t) d2, accumulated over k = 0..32 in order."""
    fs = np.asarray(fs, np.float64)
    ft = np.asarray(ft, np.float64)
    d2 = np.zeros((fs.shape[0], ft.shape[0]))
    for k in range(DIM):
        t = fs[:, k, None] - ft[None, :, k]
        d2 += t * t
    return d2


def feature_match(fs, ft, mutual_filter: bool = True, min_mutual: int = 9):
    """-> dict(nn (n_s,), reverse (n_t,), mask (n_s,) bool, n_mutual)."""
    d2 = feature_d2(fs, ft)
    nn = np.argmin(d2, axis=1) if d2.shape[1] else np.full(d2.shape[0], -1)
    rev = np.argmin(d2, axis=0) if d2.shape[0] else np.zeros(d2.shape[1], np.int64)
    mutual = rev[nn] == np.arange(d2.shape[0]) if d2.shape[1] else np.zeros(d2.shape[0], bool)
    n_mutual = int(mutual.sum())
    mask = mutual if mutual_filter and n_mutual >= min_mutual else np.ones(d2.shape[0], bool)
    return dict(nn=nn, reverse=rev, mask=mask, n_mutual=n_mutual)


def ransac_feature_matching(src, tgt, fs, ft, mutual_filter: bool, r: float, ransac_n: int = 3, **kw):
    """Open3D's registration_ransac_based_on_feature_matching: `feature_match`, then `ransac_oracle.ransac` over
    src[i] -> tgt[nn[i]] with the mask.  -> (ransac_oracle's dict, feature_match's dict)."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    m = feature_match(fs, ft, mutual_filter, 3 * ransac_n)
    o = RO.ransac(src, tgt, src, tgt[m['nn']], r, ransac_n=ransac_n, mask=m['mask'], **kw)
    return o, m
