"""FPFH and feature matching on the host: the float64 oracle (tests/fpfh_oracle.py) against a naive scalar
transcription of Open3D's loops (pair features, SPFH, FPFH, matching with the mutual filter and its fallback) on small
clouds with duplicate and isolated points, zero normals, collinear neighbours and features on the bins' clamp edges;
one pair feature by hand; invariance under a rigid motion; feature-space ties; `ops`' argument checks; the --fpfh
command lines; the launch counts; and the spills of the FPFH kernels."""
import functools
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import fpfh_oracle as FO
import train_data_oracle as O
from conftest import ROOT
from regtr_b200 import eval as E
from regtr_b200 import lib, ops
from regtr_b200 import register as R


# ------------------------------------------------------------------------------------- naive transcription of Open3D

def naive_neighbours(xyz, i, r, max_nn):
    """KDTreeFlann::SearchHybrid restated: (index, d2) of the points strictly within r, by (d2, index), max_nn."""
    hits = []
    for j in range(len(xyz)):
        dx, dy, dz = (xyz[i][a] - xyz[j][a] for a in range(3))
        d2 = (dx * dx + dy * dy) + dz * dz
        if d2 < r * r:
            hits.append((d2, j))
    hits.sort()
    return [j for _, j in hits[:max_nn]], [d for d, _ in hits[:max_nn]]


def naive_pair_features(p1, n1, p2, n2):
    """ComputePairFeatures, with Open3D's acos test."""
    dot = lambda a, b: (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]
    cross = lambda a, b: [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    d = [p2[a] - p1[a] for a in range(3)]
    r = math.sqrt(dot(d, d))
    if r == 0.0:
        return [0.0, 0.0, 0.0]
    m1, m2 = list(n1), list(n2)
    a1, a2 = dot(m1, d) / r, dot(m2, d) / r
    if math.acos(min(abs(a1), 1.0)) > math.acos(min(abs(a2), 1.0)):
        m1, m2, d, f2 = list(n2), list(n1), [-x for x in d], -a2
    else:
        f2 = a1
    v = cross(d, m1)
    vn = math.sqrt(dot(v, v))
    if vn == 0.0:
        return [0.0, 0.0, 0.0]
    v = [x / vn for x in v]
    w = cross(m1, v)
    return [math.atan2(dot(w, m2), dot(m1, m2)), dot(v, m2), f2]


def naive_fpfh(xyz, nrm, r, max_nn):
    """ComputeSPFHFeature and ComputeFPFHFeature, loop for loop."""
    n = len(xyz)
    spfh = np.zeros((n, 33))
    nbr = [naive_neighbours(xyz, i, r, max_nn) for i in range(n)]
    for i in range(n):
        idx, _ = nbr[i]
        if len(idx) > 1:
            inc = 100.0 / (len(idx) - 1)
            for k in range(1, len(idx)):
                pf = naive_pair_features(xyz[i], nrm[i], xyz[idx[k]], nrm[idx[k]])
                h = int(math.floor(11 * (pf[0] + math.pi) / (2.0 * math.pi)))
                spfh[i, min(max(h, 0), 10)] += inc
                h = int(math.floor(11 * (pf[1] + 1.0) * 0.5))
                spfh[i, min(max(h, 0), 10) + 11] += inc
                h = int(math.floor(11 * (pf[2] + 1.0) * 0.5))
                spfh[i, min(max(h, 0), 10) + 22] += inc
    feat = np.zeros((n, 33))
    for i in range(n):
        idx, dist = nbr[i]
        if len(idx) > 1:
            s = [0.0, 0.0, 0.0]
            for k in range(1, len(idx)):
                if dist[k] == 0.0:
                    continue
                for j in range(33):
                    val = spfh[idx[k], j] / dist[k]
                    s[j // 11] += val
                    feat[i, j] += val
            s = [100.0 / x if x != 0.0 else x for x in s]
            for j in range(33):
                feat[i, j] = feat[i, j] * s[j // 11] + spfh[i, j]
    return feat, np.array([len(b[0]) for b in nbr])


def naive_match(fs, ft, mutual_filter, ransac_n=3):
    """The matching of RegistrationRANSACBasedOnFeatureMatching: 1-NN both ways, the mutual set, the fallback."""
    def nn(q, pts):
        best, bj = None, -1
        for j, p in enumerate(pts):
            d = 0.0
            for k in range(33):
                d += (q[k] - p[k]) ** 2
            if best is None or d < best:
                best, bj = d, j
        return bj
    ij = [nn(f, ft) for f in fs]
    mask = np.ones(len(fs), bool)
    if mutual_filter:
        ji = [nn(f, fs) for f in ft]
        mutual = np.array([ji[j] == i for i, j in enumerate(ij)])
        if mutual.sum() >= 3 * ransac_n:
            mask = mutual
    return np.array(ij), mask


# ------------------------------------------------------------------------------------------------ clouds

def edge_cloud():
    """Hand-made pairs whose features sit on the clamp edges: f0 = +pi and -pi, f1 = +1 and -1; and collinear points
    with normals along their line (|v| = 0)."""
    xyz = np.array([[0, 0, 0], [1, 0, 0], [10, 0, 0], [9, 0, 0], [20, 0, 0], [21, 0, 0], [30, 0, 0], [31, 0, 0],
                    [40, 0, 0], [41, 0, 0], [42, 0, 0]], np.float64)
    nrm = np.array([[0, 0, 1], [0, 0, -1],                  # atan2(+0, -1) = +pi: bin 11 clamped to 10
                    [0, 0, 1], [0, -0.0, -1],               # atan2(-0, -1) = -pi: bin 0
                    [0, 0, 1], [0, -1, 0],                  # f1 = v . n2 = +1: bin 11 clamped to 10
                    [0, 0, 1], [0, 1, 0],                   # f1 = -1
                    [1, 0, 0], [1, 0, 0], [-1, 0, 0]], np.float64)   # collinear, normals along the line
    return xyz, nrm


def random_cloud(seed, n=160):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0.0, 0.4, (n, 3))
    xyz[:, 2] *= 0.2
    xyz[10:14] = xyz[20:24]                                 # duplicates (entry 0 may be a lower-indexed twin)
    xyz[30] = [5.0, 5.0, 5.0]                               # isolated
    xyz[31] = [-5.0, 5.0, 5.0]
    xyz[32] = [-5.0, 5.05, 5.0]                             # a pair: 2 neighbours each
    nrm = rng.normal(size=(n, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[40:50] = 0.0                                        # zero normals (fewer than 3 neighbours)
    return xyz, nrm


def test_pair_features_against_open3d_including_the_clamp_edges():
    xyz, nrm = edge_cloud()
    pf = FO.pair_features(xyz[0::2][:5], nrm[0::2][:5], xyz[1::2][:5], nrm[1::2][:5])
    for k in range(5):
        assert np.array_equal(pf[k], naive_pair_features(xyz[2 * k], nrm[2 * k], xyz[2 * k + 1], nrm[2 * k + 1]))
    assert pf[0, 0] == math.pi and pf[1, 0] == -math.pi and pf[2, 1] == 1.0 and pf[3, 1] == -1.0
    assert np.array_equal(FO.bins(pf[:4])[:, :2], [[10, 16], [0, 16], [5, 21], [5, 11]])
    assert np.array_equal(pf[4], [0.0, 0.0, 0.0])                 # n1 along d: v = 0


def test_one_pair_feature_by_hand():
    """p1 = 0, n1 = z, p2 = (2,0,0), n2 = (0.6,0,0.8): |a1| = 0 < |a2| = 0.6 swaps the roles: d = (-2,0,0), n1 = n2,
    v = d x n1 / |.| = (0,1,0), w = n1 x v = (-0.8,0,0.6); f0 = atan2(0.6, 0.8), f1 = 0, f2 = -0.6."""
    pf = FO.pair_features([0, 0, 0], [0, 0, 1], [2, 0, 0], [0.6, 0, 0.8])[0]
    assert np.allclose(pf, [math.atan2(0.6, 0.8), 0.0, -0.6], atol=1e-15, rtol=0)


@pytest.mark.parametrize('seed', [1, 2])
def test_fpfh_oracle_against_open3d_loops(seed):
    for xyz, nrm, r in (random_cloud(seed) + (0.1,), edge_cloud() + (1.5,)):
        o = FO.fpfh(xyz, nrm, r, 12)
        feat, cnt = naive_fpfh(xyz, nrm, r, 12)
        assert np.array_equal(o['counts'], cnt)
        assert np.abs(o['feature'] - feat).max() <= 1e-9
        assert (cnt < 2).any() and (cnt >= 12).any() or r == 1.5
    o = FO.fpfh(*random_cloud(seed), 0.1, 12)
    assert np.all(o['feature'][30] == 0.0)                         # isolated: zero row
    assert o['counts'][31] == 2 and o['feature'][31].sum() > 0


def test_fpfh_is_invariant_under_a_rigid_motion():
    xyz, nrm = random_cloud(5, 300)
    nrm[40:50] = nrm[50:60]
    T = np.eye(3, 4)
    T[:, :3] = O.axis_angle(np.array([0.36, 0.48, 0.8]), 0.7)
    T[:, 3] = [0.3, -0.2, 0.1]
    a = FO.fpfh(xyz, nrm, 0.1, 30)
    b = FO.fpfh(xyz @ T[:, :3].T + T[:, 3], nrm @ T[:, :3].T, 0.1, 30)
    assert np.array_equal(a['counts'], b['counts'])
    assert np.abs(a['feature'] - b['feature']).max() <= 1e-6


def test_feature_matching_oracle_against_open3d_with_ties_and_the_fallback():
    rng = np.random.default_rng(3)
    ft = rng.integers(0, 2, size=(40, 33)).astype(np.float64)
    ft[5] = ft[2]                                                # an exact tie: the lower index
    ft[7:9] = 0.0
    fs = np.concatenate([ft[[5, 2, 8, 7, 0, 1]], rng.integers(0, 2, size=(30, 33))]).astype(np.float64)
    for mutual in (True, False):
        o = FO.feature_match(fs, ft, mutual, 9)
        ij, mask = naive_match(fs, ft, mutual)
        assert np.array_equal(o['nn'], ij) and np.array_equal(o['mask'], mask)
        assert o['nn'][0] == 2 and o['nn'][1] == 2 and o['nn'][2] == 7 and o['nn'][3] == 7
    o = FO.feature_match(fs[:8], ft[:8], True, 9)                 # fewer than 3 ransac_n mutual: every match
    assert 0 < o['n_mutual'] < 9 and o['mask'].all()
    ij, mask = naive_match(fs[:8], ft[:8], True)
    assert mask.all() and np.array_equal(o['nn'], ij)


def test_feature_distance_accumulates_column_by_column():
    rng = np.random.default_rng(4)
    fs, ft = rng.normal(size=(5, 33)), rng.normal(size=(6, 33))
    d2 = FO.feature_d2(fs, ft)
    for i in range(5):
        for j in range(6):
            acc = 0.0
            for k in range(33):
                t = fs[i, k] - ft[j, k]
                acc = acc + t * t
            assert d2[i, j] == acc


# ------------------------------------------------------------------------------------------------ ops arguments

@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError('the library was loaded: an argument error must come first')
    monkeypatch.setattr(ops._lib, 'load', refuse)


def test_ops_reject_bad_arguments_before_any_launch(no_library):
    c, n = np.zeros((4, 3)), np.zeros((4, 3))
    f = np.zeros((4, 33))
    with pytest.raises(ValueError, match='radius'):
        ops.fpfh([c], [n], 0.0)
    for bad in (0, 129):
        with pytest.raises(ValueError, match='max_nn'):
            ops.fpfh([c], [n], 0.1, bad)
    with pytest.raises(ValueError, match='normals'):
        ops.fpfh([c], [n[:3]], 0.1)
    with pytest.raises(ValueError, match='as many'):
        ops.fpfh([c, c], [n], 0.1)
    with pytest.raises(ValueError, match=r'\(n,33\)'):
        ops.feature_match([np.zeros((4, 32))], [f], [c])
    with pytest.raises(ValueError, match='target cloud'):
        ops.feature_match([f], [f], [c[:3]])
    with pytest.raises(ValueError, match='as many'):
        ops.feature_match([f, f], [f], [c])
    with pytest.raises(ValueError, match='source cloud'):
        ops.feature_correspondences([c[:3]], [c], [f], [f])
    with pytest.raises(ValueError, match='confidence'):
        ops.ransac_feature_matching([c], [c], [f], [f], True, 0.1, confidence=2.0)
    with pytest.raises(TypeError):
        ops.ransac_feature_matching([c], [c], [f], [f], True, 0.1, no_such_option=1)


def test_launch_counts():
    assert ops.fpfh_launches() == 1 + 4 + 3
    assert ops.feature_match_launches() == 3
    header = open(lib.HEADER).read()
    assert '1 + 4 + 3 launches whatever C' in header


# ------------------------------------------------------------------------------------------------ command lines

def test_register_fpfh_command_line(capsys):
    with pytest.raises(SystemExit) as e:
        R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.05', '--ckpt', 'c/ckpt/m.pth'])
    assert e.value.code == 2 and '--ckpt is not allowed' in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        R.parse_args(['a.ply', 'b.ply'])
    assert e.value.code == 2 and '--ckpt' in capsys.readouterr().err
    for bad in (['--fpfh', '0'], ['--fpfh', '0.05', '--fpfh_max_nn', '129'], ['--fpfh', '0.05', '--ransac', '0']):
        with pytest.raises(SystemExit):
            R.parse_args(['a.ply', 'b.ply'] + bad)
    opt = R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.04'])
    assert opt.fpfh_radius == pytest.approx(0.2) and opt.ransac == pytest.approx(0.06)
    assert opt.ransac_dist == opt.ransac and opt.fit_radius == opt.ransac and opt.normal_radius is None
    kw = E.fpfh_kwargs(opt)
    assert kw == dict(fpfh_radius=opt.fpfh_radius, fpfh_max_nn=100, mutual_filter=True, ransac_radius=opt.ransac,
                      max_iteration=100000, confidence=0.999, ransac_n=3, edge_length=0.9, distance=opt.ransac,
                      seed=0)
    opt = R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.04', '--fpfh_radius', '0.3', '--fpfh_max_nn', '64',
                        '--fpfh_no_mutual', '--ransac', '0.1', '--ransac_dist', '0', '--fit_radius', '0.02'])
    assert (opt.fpfh_radius, opt.fpfh_max_nn, opt.ransac, opt.ransac_dist, opt.fit_radius) == (0.3, 64, 0.1, 0.0, 0.02)
    assert E.fpfh_kwargs(opt)['mutual_filter'] is False
    opt = R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth'])         # without --fpfh: as before
    assert opt.fpfh is None and opt.ransac is None and opt.fit_radius is None


def test_eval_3dmatch_fpfh_command_line(capsys):
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import eval_3dmatch
    finally:
        sys.path.pop(0)
    base = ['--root', 'r', '--info', 'i.pkl', '--gt', 'g']
    with pytest.raises(SystemExit) as e:
        eval_3dmatch.main(base + ['--fpfh', '0.05', '--ckpt', 'm.pth'])
    assert e.value.code == 2 and '--ckpt is not allowed' in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        eval_3dmatch.main(base)
    assert e.value.code == 2


def test_fpfh_forward_passes_its_options(monkeypatch):
    seen = {}

    def stub(src_list, tgt_list, voxel, icp_radius=None, icp_kwargs=None, **kw):
        import torch
        seen.update(voxel=voxel, icp_radius=icp_radius, icp_kwargs=icp_kwargs, **kw)
        return dict(pose=torch.zeros((2, 3, 4), dtype=torch.float64), pose_fpfh=torch.ones((2, 3, 4)))
    monkeypatch.setattr(E, 'fpfh_register', stub)
    out = E.fpfh_forward(0.05, icp_radius=0.02, icp_kwargs={'max_iteration': 5}, max_iteration=7)(
        {'src_xyz': ['a', 'b'], 'tgt_xyz': ['c', 'd']})
    assert out['pose'].shape == (1, 2, 3, 4) and out['pose_fpfh'].shape == (1, 2, 3, 4)
    assert seen == dict(voxel=0.05, icp_radius=0.02, icp_kwargs={'max_iteration': 5}, max_iteration=7)
    assert set(E.fpfh_forward(0.05)({'src_xyz': ['a'], 'tgt_xyz': ['c']})) == {'pose'}


# ------------------------------------------------------------------------------------------------ kernels

FPFH_KERNELS = ('k_fpfh_init', 'k_fpfh_select', 'k_fpfh_spfh', 'k_fpfh_feature', 'k_fm_sweep', 'k_fm_reduce',
                'k_fm_finalize')


@functools.lru_cache(maxsize=None)
def fpfh_ptxas():
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'fpfh.cu'),
                                                        '-o', os.path.join(tmp, 'fpfh.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    return text, entries


def test_fpfh_kernels_do_not_spill():
    """fpfh.cu's entry functions are exactly FPFH_KERNELS; none spills, nor does any device function they call, and
    none has a stack frame."""
    text, entries = fpfh_ptxas()
    assert len(entries) == len(FPFH_KERNELS), [e[0] for e in entries]
    for k in FPFH_KERNELS:
        assert len([e for e in entries if k + 'E' in e[0]]) == 1, k
    for name, stack, st, ld in entries:
        assert (stack, st, ld) == ('0', '0', '0'), (name, stack, st, ld)
    assert set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
