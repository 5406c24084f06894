"""Fast Global Registration on the host: the float64 oracle (tests/fgr_oracle.py) against a naive transcription of
Open3D's three loops (InitialMatching, AdvancedMatching's tuple test, OptimizePairwiseRegistration); the GNC parameter
schedule by hand; exact poses from noise-free correspondences under both scale modes; the edge cases; one trial's
draws by hand; `ops`' argument checks; the --fgr command lines and wrappers; the launch counts; and the registers of
the FGR kernels."""
import functools
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import fgr_oracle as G
import fpfh_oracle as FO
import train_data_oracle as O
from conftest import ROOT
from dropout_rule import philox
from regtr_b200 import eval as E
from regtr_b200 import lib, ops
from regtr_b200 import multiway as M
from regtr_b200 import register as R


# ------------------------------------------------------------------------------------- naive transcription of Open3D

def naive_initial_matching(fs, ft):
    """InitialMatching's cross check: nearest neighbours both ways in feature space, the mutual pairs collected in a
    dict keyed by the source index (Open3D's std::map), read back in key order."""
    def nn(q, pts):
        best, bj = None, -1
        for j, p in enumerate(pts):
            d = 0.0
            for k in range(len(q)):
                d += (q[k] - p[k]) ** 2
            if best is None or d < best:
                best, bj = d, j
        return bj
    i_to_j = {}
    corres_ji = []
    for j in range(len(ft)):
        i = nn(ft[j], fs)
        if i not in i_to_j:
            i_to_j[i] = nn(fs[i], ft)
        corres_ji.append((i, j))
    mutual = {i: j for i, j in corres_ji if i_to_j[i] == j}
    return [(i, mutual[i]) for i in sorted(mutual)]


def naive_normalise(src, tgt, use_absolute_scale):
    means, scale = [], 0.0
    for cloud in (src, tgt):
        m = [0.0, 0.0, 0.0]
        for p in cloud:
            m = [m[a] + p[a] for a in range(3)]
        m = [x / len(cloud) for x in m]
        means.append(np.array(m))
        for p in cloud:
            scale = max(scale, math.sqrt(sum((p[a] - m[a]) ** 2 for a in range(3))))
    return (means, 1.0, scale) if use_absolute_scale else (means, scale, 1.0)


def naive_tuples(ps, pt, corres, seed, pair, tuple_scale, cap):
    """AdvancedMatching's tuple test, fed the library's draws one trial at a time."""
    n = len(corres)
    out, cnt, k = [], 0, 0
    for k in range(100 * n):
        r = G.tuple_draws(seed, pair, [k], n)[0]
        i = [corres[x][0] for x in r]
        j = [corres[x][1] for x in r]
        li = [np.linalg.norm(ps[i[e]] - ps[i[(e + 1) % 3]]) for e in range(3)]
        lj = [np.linalg.norm(pt[j[e]] - pt[j[(e + 1) % 3]]) for e in range(3)]
        if all(li[e] * tuple_scale < lj[e] < li[e] / tuple_scale for e in range(3)):
            out += [(i[e], j[e]) for e in range(3)]
            cnt += 1
        if cnt >= cap:
            return out, cnt, k + 1
    return out, cnt, 100 * n


def naive_optimize(ps, pt, corres, par, iters=64, dist=0.025, division=1.4, decrease_mu=True):
    """OptimizePairwiseRegistration: the normal equations by np.outer, solved by np.linalg.cholesky, the target copy
    moved by every delta."""
    if len(corres) < 10:
        return np.eye(4)
    copy = pt.copy()
    trans = np.eye(4)
    for itr in range(iters):
        JTJ, JTr = np.zeros((6, 6)), np.zeros(6)
        for i, j in corres:
            p, q = ps[i], copy[j]
            rpq = p - q
            s = (par / (rpq @ rpq + par)) ** 2
            for row, J in enumerate(([0, -q[2], q[1], -1, 0, 0], [q[2], 0, -q[0], 0, -1, 0],
                                     [-q[1], q[0], 0, 0, 0, -1])):
                J = np.array(J, np.float64)
                JTJ += np.outer(J, J) * s
                JTr += J * rpq[row] * s
        if abs(np.linalg.det(JTJ)) >= 1e-6:
            Lc = np.linalg.cholesky(JTJ)
            x = np.linalg.solve(Lc.T, np.linalg.solve(Lc, -JTr))
            delta = G.rigid_from_vec6(x)
            trans = delta @ trans
            copy = copy @ delta[:3, :3].T + delta[:3, 3]
        if decrease_mu and itr % 4 == 0 and par > dist:
            par /= division
    return trans


def naive_fgr(src, tgt, corres, tuple_test, use_absolute_scale=False, seed=0, pair=0, tuple_scale=0.95, cap=1000,
              **kw):
    (mu_s, mu_t), sg, par0 = naive_normalise(src, tgt, use_absolute_scale)
    ps, pt = (src - mu_s) / sg, (tgt - mu_t) / sg
    tuples, trials = 0, 0
    if tuple_test:
        corres, tuples, trials = naive_tuples(ps, pt, corres, seed, pair, tuple_scale, cap)
    T = naive_optimize(ps, pt, corres, par0, **kw)
    if len(corres) < 10:
        return np.eye(3, 4), len(corres), tuples, trials
    return G.original_scale(T, mu_s, mu_t, sg), len(corres), tuples, trials


# ------------------------------------------------------------------------------------------------ pairs

def rigid(rng, deg=25.0):
    axis = rng.normal(size=3)
    T = np.eye(3, 4)
    T[:, :3] = O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))
    T[:, 3] = rng.uniform(-0.3, 0.3, 3)
    return T


def feature_pair(seed, n=120, outliers=0.3):
    """src, tgt = the source moved and jittered, features that match j -> j except for a share of outliers."""
    rng = np.random.default_rng(seed)
    src = rng.uniform(0.0, 1.0, (n, 3)) * [1.0, 0.8, 0.5]
    T = rigid(rng)
    tgt = src @ T[:, :3].T + T[:, 3] + rng.normal(scale=0.003, size=(n, 3))
    fs = rng.normal(size=(n, 33))
    ft = fs + 0.02 * rng.normal(size=(n, 33))
    bad = rng.random(n) < outliers
    ft[bad] = rng.normal(size=(int(bad.sum()), 33))
    return src, tgt, fs, ft, T


@pytest.mark.parametrize('seed', [1, 2])
@pytest.mark.parametrize('tuple_test', [True, False])
def test_oracle_against_open3d_loops(seed, tuple_test):
    src, tgt, fs, ft, _ = feature_pair(seed)
    corres = naive_initial_matching(fs, ft)
    o, m = G.fgr_feature_matching(src, tgt, fs, ft, tuple_test=tuple_test, seed=seed, pair=3, maximum_tuple_count=60)
    assert [(i, int(m['nn'][i])) for i in np.nonzero(m['mask'])[0]] == corres
    pose, n_corr, tuples, trials = naive_fgr(src, tgt, corres, tuple_test, seed=seed, pair=3, cap=60)
    assert (o['n_corr'], o['tuples'], o['trials']) == (n_corr, tuples, trials)
    assert np.abs(o['pose'] - pose).max() <= 1e-12, np.abs(o['pose'] - pose).max()
    if tuple_test:
        assert tuples == 60 and trials < 100 * len(corres)


def test_oracle_against_open3d_loops_with_absolute_scale_and_fixed_mu():
    src, tgt, fs, ft, _ = feature_pair(5)
    src, tgt = 4.0 * src, 4.0 * tgt
    corres = naive_initial_matching(fs, ft)
    o, _ = G.fgr_feature_matching(src, tgt, fs, ft, tuple_test=False, use_absolute_scale=True, decrease_mu=False,
                                  iteration_number=20)
    assert o['par0'] > 1.0 and o['par'] == o['par0']
    pose, _, _, _ = naive_fgr(src, tgt, corres, False, use_absolute_scale=True, iters=20, decrease_mu=False)
    assert np.abs(o['pose'] - pose).max() <= 1e-12


def test_par_schedule_by_hand():
    """par0 = 1, distance 0.025, divisor 1.4: divided at iterations 0, 4, ..., 40 (1.4^-10 = 0.0346 > 0.025 is
    divided once more, 1.4^-11 = 0.0247 stops), so iteration i runs at 1.4^-ceil(i / 4) up to i = 41."""
    seq, final = G.par_schedule(1.0, 64, 0.025, 1.4)
    want, p = [], 1.0
    for i in range(64):
        want.append(p)
        if i % 4 == 0 and i <= 40:
            p = p / 1.4
    assert seq == want and final == p
    assert seq[0] == 1.0 and seq[1] == 1.0 / 1.4 and seq[5] == 1.0 / 1.4 / 1.4 and seq[41] == seq[63]
    assert abs(final - 1.4 ** -11) <= 1e-15 and final < 0.025 < seq[40]
    seq, final = G.par_schedule(1.0, 64, 0.025, 1.4, decrease_mu=False)
    assert seq == [1.0] * 64 and final == 1.0
    seq, final = G.par_schedule(3.0, 10, 0.5, 2.0)
    assert seq == [3.0, 1.5, 1.5, 1.5, 1.5, 0.75, 0.75, 0.75, 0.75, 0.375] and final == 0.375
    src, tgt, fs, ft, _ = feature_pair(1)
    o, _ = G.fgr_feature_matching(src, tgt, fs, ft, tuple_test=False)
    assert o['par'] == G.par_schedule(1.0, 64, 0.025, 1.4)[1]


@pytest.mark.parametrize('absolute', [False, True])
def test_noise_free_correspondences_give_the_pose_back(absolute):
    rng = np.random.default_rng(9)
    src = rng.uniform(-1.0, 1.0, (400, 3)) * [3.0, 2.0, 1.0] + [5.0, -2.0, 1.0]
    T = rigid(rng, 40.0)
    tgt = src @ T[:, :3].T + T[:, 3]
    o = G.fgr(src, tgt, src, tgt, use_absolute_scale=absolute)
    assert (o['sigma_g'] == 1.0 and o['par0'] > 1.0) if absolute else (o['par0'] == 1.0 and o['sigma_g'] > 1.0)
    assert np.abs(o['pose'] - T).max() <= 1e-10, np.abs(o['pose'] - T).max()


def test_edge_cases():
    src, tgt, fs, ft, T = feature_pair(4)
    o = G.fgr(src, tgt, src[:9], tgt[:9])                              # fewer than 10: identity
    assert np.array_equal(o['pose'], np.eye(3, 4)) and o['n_corr'] == 9 and o['par'] == 1.0
    o = G.fgr(src, tgt, src[:12], tgt[:12], mask=np.arange(12) < 9)
    assert np.array_equal(o['pose'], np.eye(3, 4)) and o['n_corr'] == 9
    o = G.fgr(src, tgt, src[:0], tgt[:0], tuple_test=True)             # n = 0: no trials
    assert (o['n_corr'], o['tuples'], o['trials']) == (0, 0, 0)
    o = G.fgr(src, tgt, src, tgt, tuple_test=True, maximum_tuple_count=7, seed=3)
    assert o['tuples'] == 7 and o['n_corr'] == 21
    a, c = (src - o['mu_s']) / o['sigma_g'], (tgt - o['mu_t']) / o['sigma_g']
    draws = G.tuple_draws(3, 0, np.arange(o['trials']), len(src))
    ok = G.tuple_passes(a, c, draws, 0.95)
    assert ok.sum() == 7 and ok[-1]                                   # the walk ends on the pass reaching the cap
    assert np.array_equal(o['idx'], draws[ok].reshape(-1))
    o = G.fgr(src, tgt, src, tgt, tuple_test=True, tuple_scale=1.0)  # nothing passes l s < l < l / s at s = 1
    assert (o['tuples'], o['trials'], o['n_corr']) == (0, 100 * len(src), 0)
    assert np.array_equal(o['pose'], np.eye(3, 4))


def test_one_trial_by_hand():
    """Trial k = 5 of global pair 7 under seed 2^32 + 9 among n = 1000 correspondences: Philox4x32-10 at counter
    (5, 7, 0, 'FGRT') with key (9, 1), index e = (w_e * 1000) >> 32."""
    seed = (1 << 32) + 9
    w = philox((np.uint64(5), 7, 0, 0x46475254), 9, 1)
    assert G.WORD3 == int.from_bytes(b'FGRT', 'big')
    want = [(int(w[e]) * 1000) >> 32 for e in range(3)]
    assert G.tuple_draws(seed, 7, [5], 1000)[0].tolist() == want
    assert all(0 <= x < 1000 for x in want)


def test_block_sum_is_the_halving_tree_of_the_warps():
    rng = np.random.default_rng(0)
    v = rng.normal(size=256)
    w = [G.tree(v[32 * k:32 * k + 32]) for k in range(8)]
    assert G.block_sum(v) == ((w[0] + w[4]) + (w[2] + w[6])) + ((w[1] + w[5]) + (w[3] + w[7]))


# ------------------------------------------------------------------------------------------------ ops arguments

@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError('the library was loaded: an argument error must come first')
    monkeypatch.setattr(ops._lib, 'load', refuse)


def test_ops_reject_bad_arguments_before_any_launch(no_library):
    c, f = np.zeros((12, 3)), np.zeros((12, 33))
    bad = [(dict(maximum_correspondence_distance=0.0), 'maximum_correspondence_distance'),
           (dict(maximum_correspondence_distance=float('inf')), 'maximum_correspondence_distance'),
           (dict(division_factor=0.0), 'division_factor'), (dict(division_factor=-1.0), 'division_factor'),
           (dict(maximum_tuple_count=0), 'maximum_tuple_count'), (dict(tuple_scale=0.0), 'tuple_scale'),
           (dict(tuple_scale=1.5), 'tuple_scale'), (dict(iteration_number=-1), 'iteration_number'),
           (dict(seed=-1), 'seed'), (dict(seed=2 ** 64), 'seed'), (dict(pair_base=-1), 'pair_base'),
           (dict(pair_base=2 ** 31), 'pair_base')]
    for kw, what in bad:
        with pytest.raises(ValueError, match=what):
            ops.fgr([c], [c], [c], [c], **kw)
        with pytest.raises(ValueError, match=what):
            ops.fgr_feature_matching([c], [c], [f], [f], **kw)
    with pytest.raises(ValueError, match='as many'):
        ops.fgr([c, c], [c], [c], [c])
    with pytest.raises(ValueError, match=r'\(m,3\)'):
        ops.fgr([c], [c], [c], [c[:5]])
    with pytest.raises(ValueError, match='mask'):
        ops.fgr([c], [c], [c], [c], [np.ones(5, bool)])
    with pytest.raises(ValueError, match='correspondence arrays'):
        ops.fgr([c], [c], [c, c], [c, c])
    with pytest.raises(ValueError, match='source cloud'):
        ops.fgr_feature_matching([c[:5]], [c], [f], [f])
    with pytest.raises(TypeError):
        ops.fgr_feature_matching([c], [c], [f], [f], no_such_option=1)


def test_launch_counts_and_header():
    assert ops.fgr_launches() == 2
    header = open(lib.HEADER).read()
    assert '2 launches whatever the data' in header
    assert 'regtr_fgr' in lib.SIGNATURES and 'regtr_fgr_ws_bytes' in lib.SIGNATURES
    assert ops.FGR_MAX_CORR == 21474836 and 100 * ops.FGR_MAX_CORR < 2 ** 31
    assert '#define REGTR_FGR_MAX_CORR 21474836' in header and '#define REGTR_FGR_MAX_TUPLES (1 << 20)' in header


# ------------------------------------------------------------------------------------------------ command lines

def test_register_fgr_usage_errors(capsys):
    with pytest.raises(SystemExit) as e:
        R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--fgr', '--ransac', '0.05'])
    assert e.value.code == 2 and 'exclusive' in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.05', '--fgr', '--fpfh_no_mutual'])
    assert e.value.code == 2 and '--fpfh_no_mutual' in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.05', '--fgr', '--ransac', '0.1'])
    assert e.value.code == 2 and 'exclusive' in capsys.readouterr().err
    for bad in (['--fgr_dist', '0'], ['--fgr_division', '0'], ['--fgr_tuple_scale', '1.5'], ['--fgr_max_tuples', '0'],
                ['--fgr_iters', '-1'], ['--fgr_seed', '-1'], ['--fgr_no_tuple_test']):
        with pytest.raises(SystemExit):
            R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--fgr'] + bad)


def test_register_fgr_flags():
    opt = R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.04', '--fgr'])
    assert opt.ransac is None and opt.fgr_dist == pytest.approx(0.02) and opt.fit_radius == pytest.approx(0.06)
    kw = E.fpfh_kwargs(opt)
    assert kw == dict(fpfh_radius=opt.fpfh_radius, fpfh_max_nn=100, method='fgr',
                      fgr_kwargs=dict(maximum_correspondence_distance=opt.fgr_dist, iteration_number=64,
                                      division_factor=1.4, decrease_mu=True, use_absolute_scale=False,
                                      tuple_test=True, tuple_scale=0.95, maximum_tuple_count=1000, seed=0))
    opt = R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.04', '--fgr', '--fgr_no_tuple_test', '--fgr_dist', '0.1',
                        '--fgr_iters', '8', '--fgr_no_decrease_mu', '--fgr_absolute_scale', '--fgr_seed', '4'])
    kw = E.fgr_kwargs(opt)
    assert kw['tuple_test'] is False and kw['maximum_correspondence_distance'] == 0.1 and kw['iteration_number'] == 8
    assert kw['decrease_mu'] is False and kw['use_absolute_scale'] is True and kw['seed'] == 4
    opt = R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--fgr', '--fgr_tuple_test',
                        '--fgr_max_tuples', '50', '--fgr_tuple_scale', '0.9', '--fgr_division', '2'])
    kw = E.fgr_kwargs(opt)
    assert opt.fgr_dist == 0.025 and kw['tuple_test'] is True and kw['maximum_tuple_count'] == 50
    assert kw['tuple_scale'] == 0.9 and kw['division_factor'] == 2.0
    assert E.fgr_kwargs(R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--fgr']))['tuple_test'] is False
    opt = R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth'])         # without --fgr: as before
    assert opt.fgr is False and opt.fgr_dist is None and opt.ransac is None


def test_multiway_and_eval_3dmatch_fgr_usage_errors(capsys):
    import sys
    with pytest.raises(SystemExit) as e:
        M.main(['a.npy', 'b.npy', '--ckpt', 'm.pth', '--out', 'o', '--fgr', '--ransac', '0.05'])
    assert e.value.code == 2 and 'exclusive' in capsys.readouterr().err
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import eval_3dmatch
    finally:
        sys.path.pop(0)
    base = ['--root', 'r', '--info', 'i.pkl', '--gt', 'g']
    for extra, msg in ((['--ckpt', 'm.pth', '--fgr', '--ransac', '0.05'], 'exclusive'),
                       (['--fpfh', '0.05', '--fgr', '--fpfh_no_mutual'], '--fpfh_no_mutual')):
        with pytest.raises(SystemExit) as e:
            eval_3dmatch.main(base + extra)
        assert e.value.code == 2 and msg in capsys.readouterr().err


def test_fpfh_forward_passes_the_fgr_options(monkeypatch):
    seen = {}

    def stub(src_list, tgt_list, voxel, icp_radius=None, icp_kwargs=None, **kw):
        import torch
        seen.update(voxel=voxel, icp_radius=icp_radius, **kw)
        return dict(pose=torch.zeros((1, 3, 4), dtype=torch.float64), pose_fpfh=torch.ones((1, 3, 4)))
    monkeypatch.setattr(E, 'fpfh_register', stub)
    opt = R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.05', '--fgr', '--fgr_iters', '9'])
    E.fpfh_forward(0.05, icp_radius=0.02, **E.fpfh_kwargs(opt))({'src_xyz': ['a'], 'tgt_xyz': ['c']})
    assert seen['method'] == 'fgr' and seen['fgr_kwargs']['iteration_number'] == 9 and seen['icp_radius'] == 0.02
    assert seen['fgr_kwargs']['maximum_correspondence_distance'] == pytest.approx(0.025)


def test_fgr_forward_passes_its_options():
    import torch
    seen = {}

    def fgr(src_list, tgt_list, cs, ct, cm, pair_base=0, **kw):
        seen.update(src=src_list, cs=cs, cm=cm, pair_base=pair_base, **kw)
        return torch.full((2, 3, 4), 2.0, dtype=torch.float64), torch.zeros((2, 4))

    def corr(pred, overlap):
        seen['overlap'] = overlap
        return ['a'], ['c'], ['m']

    def icp(src_list, tgt_list, init, radius, max_iteration=30, **kw):
        seen.update(icp_init=init.clone(), icp_radius=radius, icp_iters=max_iteration)
        return torch.full((2, 3, 4), 3.0, dtype=torch.float64), torch.zeros((2, 4))
    pred = {'pose': torch.ones((6, 2, 3, 4), dtype=torch.float32)}
    fwd = E.fgr_forward(lambda b: pred, 0.3, fgr=fgr, correspondences=corr, icp_radius=0.05,
                        icp_kwargs={'max_iteration': 4}, icp=icp, maximum_correspondence_distance=0.01, tuple_test=True)
    out = fwd({'src_xyz': ['s0', 's1'], 'tgt_xyz': ['t0', 't1']})
    assert seen['overlap'] == 0.3 and seen['cs'] == ['a'] and seen['cm'] == ['m'] and seen['pair_base'] == 0
    assert seen['maximum_correspondence_distance'] == 0.01 and seen['tuple_test'] is True
    assert seen['icp_radius'] == 0.05 and seen['icp_iters'] == 4 and torch.all(seen['icp_init'] == 2.0)
    assert torch.all(out['pose'] == 3.0) and torch.all(out['pose_fgr'] == 2.0) and torch.all(out['pose_coarse'] == 1.0)
    out = E.fgr_forward(lambda b: pred, fgr=fgr, correspondences=corr)({'src_xyz': ['s'], 'tgt_xyz': ['t']})
    assert 'pose_fgr' not in out and torch.all(out['pose'] == 2.0)


# ------------------------------------------------------------------------------------------------ kernels

FGR_KERNELS = ('k_fgr_prepare', 'k_fgr_solve')


@functools.lru_cache(maxsize=None)
def fgr_ptxas():
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'fgr.cu'),
                                                        '-o', os.path.join(tmp, 'fgr.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    return text, entries


def test_fgr_kernels_do_not_spill():
    """fgr.cu's entry functions are exactly FGR_KERNELS and nothing spills.  The preparation has no stack frame; the
    solve's only frame is the 40 bytes of double sincos's large-argument reduction (rigid_from_vec6, as in ICP's
    point-to-plane update)."""
    text, entries = fgr_ptxas()
    assert len(entries) == len(FGR_KERNELS), [e[0] for e in entries]
    for k in FGR_KERNELS:
        assert len([e for e in entries if k + 'E' in e[0]]) == 1, k
    for name, stack, st, ld in entries:
        assert (st, ld) == ('0', '0'), (name, st, ld)
        assert stack == ('0' if 'k_fgr_prepare' in name else '40'), (name, stack)
    assert set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
    assert 'internal_trig_reduction_slowpathd' in text
