"""RANSAC over correspondences on the host: the float64 oracle (tests/ransac_oracle.py) against a naive transcription
of Open3D's loop, its draws, checkers and stop rule; `ops.ransac`'s argument checks and chunk schedule;
`ops.regtr_correspondences`; the --ransac flags of the three command lines; the `ransac_forward` wrapper and its
RANSAC -> ICP composition; and the spills of the RANSAC kernels."""
import functools
import math
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import icp_oracle as I
import ransac_oracle as RO
import train_data_oracle as O
from conftest import ROOT
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import ops
from regtr_b200 import register as R


def rigid(rng, deg=30.0):
    axis = rng.normal(size=3)
    T = np.eye(3, 4)
    T[:, :3] = O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))
    T[:, 3] = rng.uniform(-0.5, 0.5, 3)
    return T


def problem(seed, n_src=300, m=40, outliers=0.5, noise=0.002):
    """A source / target pair related by T and m correspondences, a share of them random."""
    rng = np.random.default_rng(seed)
    T = rigid(rng)
    src = rng.uniform(-1.0, 1.0, (n_src, 3))
    tgt = I.transform(T, src) + rng.normal(scale=noise, size=(n_src, 3))
    pick = rng.integers(0, n_src, m)
    a = src[pick]
    c = tgt[pick].copy()
    bad = rng.random(m) < outliers
    c[bad] = tgt[rng.integers(0, n_src, int(bad.sum()))]
    return src, tgt, a, c, T


# ------------------------------------------------------------------------------------------------ draws

def _philox_scalar(c, k):
    """Philox4x32-10 on Python ints, written out independently of dropout_rule."""
    c, k = list(c), list(k)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c[3] ^ k[1]) & 0xFFFFFFFF,
             p0 & 0xFFFFFFFF]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return c


def test_one_draw_by_hand():
    """Hypothesis 7 of global pair 3, seed 0x0123456789abcdef, n = 1000: draw j = 5 is word 1 of the block at counter
    (7, 3, 1, 'RSAC'), scaled by mulhi32."""
    seed, n = 0x0123456789ABCDEF, 1000
    w = _philox_scalar((7, 3, 1, 0x52534143), (seed & 0xFFFFFFFF, seed >> 32))
    want = (w[1] * n) >> 32
    got = RO.draws(seed, 3, [7], n, 6)
    assert got[0, 5] == want
    assert all(got[0, j] == (_philox_scalar((7, 3, 0, 0x52534143), (seed & 0xFFFFFFFF, seed >> 32))[j] * n) >> 32
               for j in range(4))
    assert 0x52534143.to_bytes(4, 'big') == b'RSAC'


def test_draws_are_uniform_and_per_hypothesis():
    d = RO.draws(5, 0, np.arange(4000), 10, 3)
    assert d.min() == 0 and d.max() == 9
    counts = np.bincount(d.ravel(), minlength=10)
    assert counts.min() > 1000 and counts.max() < 1400
    assert np.array_equal(RO.draws(5, 0, [123], 10, 3)[0], d[123])
    assert not np.array_equal(RO.draws(5, 1, [123], 10, 3)[0], d[123])          # another pair draws otherwise


# ------------------------------------------------------------------------------------------------ checkers

def test_edge_checker_on_hand_built_samples():
    a = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    assert RO.edge_ok(a, a + 5.0, 0.9)
    assert RO.edge_ok(a, a * 0.95, 0.9)                          # every edge ratio 0.95 >= 0.9
    assert not RO.edge_ok(a, a * 0.85, 0.9)
    assert RO.edge_ok(a, a * 0.85, 0.0) and RO.edge_ok(a, a * 0.85, None)    # off
    c = a.copy()
    c[2] = [0.0, 1.2, 0.0]                                       # one stretched edge
    assert not RO.edge_ok(a, c, 0.9) and RO.edge_ok(a, c, 0.8)


def test_distance_checker_and_exact_recovery():
    rng = np.random.default_rng(1)
    T = rigid(rng)
    a = rng.uniform(-1, 1, (4, 3))
    c = I.transform(T, a)
    ok, E_ = RO.hypothesis(a, c, [0, 1, 2, 3], 0.9, 1e-9)
    assert ok and np.abs(E_ - T).max() < 1e-12
    c2 = c.copy()
    c2[3] += [0.0, 0.0, 0.05]
    ok, T2 = RO.hypothesis(a, c2, [0, 1, 2, 3], None, None)
    assert ok
    res = RO.norm3(I.transform(T2, a) - c2)
    assert RO.distance_ok(T2, a, c2, res.max() * 1.0001) and not RO.distance_ok(T2, a, c2, res.max() * 0.9999)
    assert RO.hypothesis(a, c2, [0, 1, 2, 3], None, res.max() * 0.5)[0] is False


def test_degenerate_samples_are_rejected():
    a = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    assert RO.hypothesis(a, a, [0, 1, 2], None, None)[0] is False              # collinear: S[1] = 0
    assert RO.hypothesis(a, a, [0, 1, 3], None, None)[0] is True
    assert RO.hypothesis(a, a, [0, 3, 0], None, None)[0] is False              # repeated index
    same = np.zeros((3, 3))
    assert RO.hypothesis(same, same + 1.0, [0, 1, 2], None, None)[0] is False  # S[0] = 0 too


# ------------------------------------------------------------------------------------------------ stop rule

def test_est_k_edge_cases():
    assert RO.est_k_update(1000, 0.5, 0.999, 3) == math.ceil(math.log(0.001) / math.log(1 - 0.125))
    assert RO.est_k_update(1000, 1.0, 0.999, 3) == 0                  # fitness 1: stop at once
    assert RO.est_k_update(1000, 0.5, 1.0, 3) == 1000                 # confidence 1: d = +inf
    assert RO.est_k_update(1000, 1e-7, 0.999, 3) == 1000              # 1 - f^3 rounds to 1: d = -inf, unchanged
    assert RO.est_k_update(1000, 0.0, 0.999, 3) == 1000               # fitness 0
    assert RO.est_k_update(1000, 0.5, 0.0, 3) == 0                    # confidence 0: d = -0.0
    assert RO.est_k_update(10, 0.5, 0.999, 3) == 10                   # d >= est_k: unchanged
    assert RO.est_k_update(1000, 1.0, 1.0, 3) == 1000                 # 0 / 0: unchanged


def naive_open3d(src, tgt, a, c, r, max_iteration, confidence, ransac_n, edge, dist, seed, pair):
    """Open3D's loop, one thread: for itr < max_iteration, skipped once itr >= est_k_global; checkers after the
    estimation, in the list's order; IsBetterRANSACThan; est_k_local from the improvement.  The deviations:
    degenerate samples rejected, d = -inf ignored."""
    n = a.shape[0]
    out = dict(pose=np.eye(3, 4), fitness=0.0, rmse=0.0, iterations=0, validations=0, best=-1)
    if ransac_n < 3 or n < ransac_n or r <= 0.0:
        return out
    est_k_global, total_validation, walked = max_iteration, 0, 0
    for itr in range(max_iteration):
        if itr < est_k_global:
            walked += 1
            idx = RO.draws(seed, pair, [itr], n, ransac_n)[0]
            if len(set(idx.tolist())) < ransac_n or RO.degenerate(a[idx], c[idx]):
                continue
            T = I.umeyama(a[idx], c[idx])
            checks = [lambda: RO.edge_ok(a[idx], c[idx], edge), lambda: RO.distance_ok(T, a[idx], c[idx], dist)]
            if not all(ch() for ch in checks):
                continue
            nn, d2 = I.correspondences(I.transform(T, src), tgt, r)
            k = int((nn >= 0).sum())
            fit = k / src.shape[0]
            rmse = math.sqrt(RO.fixed_sum(np.where(nn >= 0, d2, 0.0)) / k) if k else 0.0
            est_k_local = est_k_global
            if fit > out['fitness'] or (fit == out['fitness'] and rmse < out['rmse']):
                out.update(pose=T, fitness=fit, rmse=rmse, best=itr)
                pw = fit ** 1
                for _ in range(ransac_n - 1):
                    pw *= fit
                with np.errstate(divide='ignore', invalid='ignore'):
                    d = float(np.float64(np.log(1.0 - confidence)) / np.float64(np.log(1.0 - pw)))
                if d < est_k_global and not d == -math.inf:
                    est_k_local = int(math.ceil(d))
            total_validation += 1
            est_k_global = min(est_k_global, est_k_local)
    out.update(iterations=walked, validations=total_validation)
    return out


@pytest.mark.parametrize('case', [
    dict(seed=1), dict(seed=2, outliers=0.8, m=60), dict(seed=3, edge=None), dict(seed=4, dist=0.01),
    dict(seed=5, ransac_n=4), dict(seed=6, ransac_n=5, outliers=0.3), dict(seed=7, max_iteration=0),
    dict(seed=8, m=2), dict(seed=9, m=0), dict(seed=10, confidence=1.0, max_iteration=60),
    dict(seed=11, outliers=0.0), dict(seed=12, mask=True), dict(seed=13, ransac_n=2), dict(seed=14, r=0.0),
])
def test_oracle_equals_naive_open3d_loop(case):
    case = dict(case)
    seed = case.pop('seed')
    src, tgt, a, c, _ = problem(seed, m=case.pop('m', 40), outliers=case.pop('outliers', 0.5))
    mask = None
    if case.pop('mask', False):
        mask = np.random.default_rng(seed).random(a.shape[0]) < 0.7
    kw = dict(r=0.02, max_iteration=300, confidence=0.999, ransac_n=3, edge=0.9, dist=None)
    kw.update(case)
    got = RO.ransac(src, tgt, a, c, kw['r'], kw['max_iteration'], kw['confidence'], kw['ransac_n'], kw['edge'],
                    kw['dist'], mask, seed=77, pair=seed)
    aa, cc = (a, c) if mask is None else (a[mask], c[mask])
    want = naive_open3d(src, tgt, aa, cc, kw['r'], kw['max_iteration'], kw['confidence'], kw['ransac_n'], kw['edge'],
                        kw['dist'], 77, seed)
    for key in ('fitness', 'rmse', 'iterations', 'validations', 'best'):
        assert got[key] == want[key], (key, got[key], want[key])
    assert np.array_equal(got['pose'], want['pose'])


def test_oracle_finds_the_pose_and_stops_on_clean_data():
    src, tgt, a, c, T = problem(21, outliers=0.0, noise=0.0)
    got = RO.ransac(src, tgt, a, c, 0.02, 1000, 0.999, 3, 0.9, None, seed=0, pair=0)
    first = next(k for k in range(1000) if RO.hypothesis(a, c, RO.draws(0, 0, [k], a.shape[0], 3)[0], 0.9)[0])
    assert got['fitness'] == 1.0 and got['best'] == first
    assert got['iterations'] == first + 1 and got['validations'] == 1          # fitness 1 stops at once
    assert np.abs(got['pose'] - T).max() < 1e-9


def test_fast_matches_equal_the_ball_query():
    rng = np.random.default_rng(6)
    lattice = rng.integers(0, 25, (4000, 3)) * 0.01                  # duplicates and exact ties
    for p, t, r in ((rng.uniform(0, 0.25, (3000, 3)), lattice, 0.02),
                    (rng.integers(0, 25, (2000, 3)) * 0.01 + 0.005, lattice, 0.02),
                    (rng.uniform(-1, 1, (500, 3)), rng.uniform(-1, 1, (300, 3)), 0.3),
                    (rng.uniform(-1, 1, (50, 3)), rng.uniform(-1, 1, (3, 3)), 5.0)):
        want = I.correspondences(p, t, r)
        got = RO.matches(p, t, r)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_fixed_sum_order():
    rng = np.random.default_rng(2)
    for n in (0, 1, 255, 1024, 1025, 5000, 40000):
        v = rng.random(n)
        assert abs(RO.fixed_sum(v) - v.sum()) <= 1e-12 * max(1.0, v.sum())
    v = rng.random(1000)
    chains = np.zeros(256)
    for i in range(1000):                                # regtr_registration_fit's order for one block
        chains[i % 256] += v[i]
    h = 128
    while h:
        chains[:h] = chains[:h] + chains[h:2 * h]
        h //= 2
    assert RO.fixed_sum(v) == chains[0]


# ------------------------------------------------------------------------------------------------ ops layer

def test_chunk_schedule_and_launches():
    for mi, fc in ((0, 256), (1, 1), (100, 7), (1000, 256), (100000, 256), (100000, 1), (100000, 8192), (5, 4096)):
        ch = ops.ransac_chunks(mi, fc)
        assert sum(s for _, s in ch) == mi and all(s > 0 for _, s in ch)
        assert all(ch[i + 1][0] == ch[i][0] + ch[i][1] for i in range(len(ch) - 1))
        assert all(s == min(fc << c, ops.RANSAC_CHUNK_MAX) for c, (_, s) in enumerate(ch[:-1]))
        assert ops.ransac_launches(mi, fc) == 6 + 3 * len(ch)
    assert len(ops.ransac_chunks(100000, 256)) == 17                # 6 doubling chunks, then 8192 at most
    assert ops.ransac_launches(1000, 256, ransac_n=2) == 0
    assert ops.ransac_launches(1000, 256, max_correspondence_distance=0.0) == 0


@pytest.mark.parametrize('kw, msg', [
    (dict(max_iteration=-1), 'max_iteration'), (dict(max_iteration=2.5), 'max_iteration'),
    (dict(confidence=1.5), 'confidence'), (dict(confidence=-0.1), 'confidence'),
    (dict(ransac_n=17), 'ransac_n'), (dict(edge_length=-0.1), 'edge_length'),
    (dict(edge_length=float('nan')), 'edge_length'), (dict(distance=float('inf')), 'distance'),
    (dict(seed=-1), 'seed'), (dict(seed=2 ** 64), 'seed'), (dict(pair_base=-2), 'pair_base'),
    (dict(first_chunk=0), 'first_chunk'), (dict(first_chunk=8193), 'first_chunk'),
])
def test_ransac_rejects_bad_arguments_before_any_launch(kw, msg):
    src, tgt, a, c, _ = problem(3)
    before = ops.LAUNCHES
    with pytest.raises(ValueError, match=msg):
        ops.ransac([src], [tgt], [a], [c], 0.02, **kw)
    assert ops.LAUNCHES == before


def test_ransac_rejects_bad_shapes():
    src, tgt, a, c, _ = problem(3)
    with pytest.raises(ValueError, match='correspondence arrays'):
        ops.ransac([src], [tgt], [a, a], [c, c], 0.02)
    with pytest.raises(ValueError, match='expected two'):
        ops.ransac([src], [tgt], [a], [c[:-1]], 0.02)
    with pytest.raises(ValueError, match='expected two'):
        ops.ransac([src], [tgt], [a[:, :2]], [c[:, :2]], 0.02)
    with pytest.raises(ValueError, match='mask'):
        ops.ransac([src], [tgt], [a], [c], 0.02, corr_mask=[np.ones(3, bool)])
    with pytest.raises(ValueError, match='as many source as target'):
        ops.ransac([src], [], [a], [c], 0.02)


def fake_pred(rng, sizes, L=2):
    pred = {k: [] for k in ('src_kp', 'tgt_kp', 'src_kp_warped', 'tgt_kp_warped', 'src_overlap', 'tgt_overlap')}
    for ns, nt in sizes:
        for side, n in (('src', ns), ('tgt', nt)):
            pred[f'{side}_kp'].append(torch.from_numpy(rng.normal(size=(n, 3))).float())
            pred[f'{side}_kp_warped'].append(torch.from_numpy(rng.normal(size=(L, n, 3))).float())
            pred[f'{side}_overlap'].append(torch.from_numpy(rng.normal(size=(L, n, 1))).float())
    return pred


def test_regtr_correspondences_layout():
    rng = np.random.default_rng(4)
    pred = fake_pred(rng, [(5, 7), (3, 2)])
    cs, ct, cm = ops.regtr_correspondences(pred, 0.6)
    for b, (ns, nt) in enumerate([(5, 7), (3, 2)]):
        assert cs[b].shape == (ns + nt, 3) and ct[b].shape == (ns + nt, 3) and cm[b].shape == (ns + nt,)
        assert torch.equal(cs[b][:ns], pred['src_kp'][b]) and torch.equal(ct[b][:ns], pred['src_kp_warped'][b][-1])
        assert torch.equal(cs[b][ns:], pred['tgt_kp_warped'][b][-1]) and torch.equal(ct[b][ns:], pred['tgt_kp'][b])
        logit = torch.cat([pred['src_overlap'][b][-1][:, 0], pred['tgt_overlap'][b][-1][:, 0]])
        assert torch.equal(cm[b], torch.sigmoid(logit) > 0.6)


# ------------------------------------------------------------------------------------------------ command lines

def _eval_3dmatch():
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import eval_3dmatch
    finally:
        sys.path.pop(0)
    return eval_3dmatch


CLIS = {
    'register': lambda: (R.parser(), R.main, ['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth']),
    'multiway': lambda: (MW.parser(), MW.main, ['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--out', 'o']),
    'eval_3dmatch': lambda: (_eval_3dmatch().parser(), _eval_3dmatch().main,
                             ['--root', 'r', '--info', 'i.pkl', '--gt', 'g', '--ckpt', 'm.pth']),
}


@pytest.mark.parametrize('cli', sorted(CLIS))
def test_every_command_line_parses_the_ransac_flags(cli):
    ap, _, args = CLIS[cli]()
    opt = ap.parse_args(args)
    assert opt.ransac is None
    E.check_ransac_arguments(ap, opt)
    opt = ap.parse_args(args + ['--ransac', '0.05', '--ransac_iters', '5000', '--ransac_confidence', '0.99',
                                '--ransac_n', '4', '--ransac_edge', '0', '--ransac_dist', '0.1', '--ransac_overlap',
                                '0.3', '--ransac_seed', '9', '--icp', '0.02'])
    E.check_ransac_arguments(ap, opt)
    assert E.ransac_kwargs(opt) == dict(max_iteration=5000, confidence=0.99, ransac_n=4, edge_length=0.0,
                                        distance=0.1, overlap=0.3, seed=9)
    assert opt.ransac == 0.05 and opt.icp == 0.02
    d = ap.parse_args(args + ['--ransac', '0.05'])
    assert E.ransac_kwargs(d) == dict(max_iteration=100000, confidence=0.999, ransac_n=3, edge_length=0.9,
                                      distance=None, overlap=0.5, seed=0)


@pytest.mark.parametrize('cli', sorted(CLIS))
@pytest.mark.parametrize('bad, msg', [
    (['--ransac', '0'], '--ransac 0.0 must be > 0'), (['--ransac', '0.05', '--ransac_n', '2'], '--ransac_n 2'),
    (['--ransac', '0.05', '--ransac_confidence', '2'], '--ransac_confidence 2.0'),
    (['--ransac', '0.05', '--ransac_iters', '-1'], '--ransac_iters -1'),
    (['--ransac', '0.05', '--ransac_edge', '-1'], '--ransac_edge -1.0'),
    (['--ransac', '0.05', '--ransac_dist', 'nan'], '--ransac_dist nan'),
])
def test_every_command_line_rejects_bad_ransac_options(cli, bad, msg, capsys):
    """At parse time, before any model or data is loaded: a usage error (exit status 2)."""
    _, main, args = CLIS[cli]()
    with pytest.raises(SystemExit) as e:
        main(args + bad)
    assert e.value.code == 2 and msg in capsys.readouterr().err


# ------------------------------------------------------------------------------------------------ wrappers

def test_ransac_forward_and_icp_composition():
    rng = np.random.default_rng(5)
    B, L = 2, 3
    probs = [problem(30 + b) for b in range(B)]
    net = torch.from_numpy(np.stack([np.stack([p[4] for p in probs])] * L)).float()     # (L,B,3,4)
    net_before = net.clone()
    batch = {'src_xyz': [torch.from_numpy(p[0]).float() for p in probs],
             'tgt_xyz': [torch.from_numpy(p[1]).float() for p in probs]}
    calls = []

    def correspondences(pred, overlap):
        calls.append(('corr', overlap))
        return [p[2] for p in probs], [p[3] for p in probs], None

    def oracle_ransac(src_list, tgt_list, cs, ct, radius, max_iteration, **kw):
        calls.append(('ransac', radius, max_iteration, kw['seed'], kw['pair_base'], kw['edge_length']))
        pose, res = RO.ransac_batch([s.numpy().astype(np.float64) for s in src_list],
                                    [t.numpy().astype(np.float64) for t in tgt_list], cs, ct, radius, max_iteration,
                                    kw['confidence'], kw['ransac_n'], kw['edge_length'], kw['distance'],
                                    kw['corr_mask'], kw['seed'], kw['pair_base'])
        return torch.from_numpy(pose), torch.from_numpy(res)

    inits = []

    def stub_icp(src_list, tgt_list, init, radius, max_iteration, **kw):
        inits.append((init.clone(), radius, max_iteration, kw))
        return init + 1.0, torch.zeros((len(src_list), 4), dtype=torch.float64)

    run = E.ransac_forward(lambda b: {'pose': net, 'src_kp': 'kept'}, 0.02, 500, seed=3, overlap=0.4,
                           ransac=oracle_ransac, correspondences=correspondences)
    pred = run(batch)
    assert calls == [('corr', 0.4), ('ransac', 0.02, 500, 3, 0, 0.9)]
    want, _ = oracle_ransac(batch['src_xyz'], batch['tgt_xyz'], [p[2] for p in probs], [p[3] for p in probs], 0.02,
                            500, confidence=0.999, ransac_n=3, edge_length=0.9, distance=None, corr_mask=None, seed=3,
                            pair_base=0)
    assert pred['pose'].shape == (1, B, 3, 4) and pred['pose'].dtype == torch.float64
    assert torch.equal(pred['pose'][0], want)
    assert torch.equal(pred['pose_coarse'][0], net[-1].double()) and 'pose_ransac' not in pred
    assert pred['src_kp'] == 'kept' and torch.equal(net, net_before)
    m = E.compute_metrics(pred, net[-1].double())
    assert set(m) == {'rot_err_deg', 'trans_err', 'rot_err_deg_coarse', 'trans_err_coarse'}

    run = E.ransac_forward(lambda b: {'pose': net}, 0.02, 500, seed=3, overlap=0.4, ransac=oracle_ransac,
                           correspondences=correspondences, icp_radius=0.01, icp=stub_icp,
                           icp_kwargs=dict(max_iteration=7))
    pred = run(batch)
    assert len(inits) == 1 and inits[0][1:] == (0.01, 7, {})
    assert torch.equal(inits[0][0], want)                                   # ICP starts from the RANSAC pose
    assert torch.equal(pred['pose'][0], want + 1.0) and torch.equal(pred['pose_ransac'][0], want)
    assert torch.equal(pred['pose_coarse'][0], net[-1].double())
    assert {'rot_err_deg_ransac', 'rot_err_deg_coarse'} <= set(E.compute_metrics(pred, net[-1].double()))


def test_ransac_refine_passes_the_mask_and_pair_base():
    seen = {}

    def stub(src_list, tgt_list, cs, ct, radius, max_iteration, **kw):
        seen.update(kw, radius=radius, max_iteration=max_iteration, cs=cs)
        return 'pose', 'result'

    out = E.ransac_refine('pred', ['s'], ['t'], 0.03, 10, pair_base=5, ransac=stub,
                          correspondences=lambda p, o: (['a'], ['c'], ['m']))
    assert out == ('pose', 'result')
    assert seen['corr_mask'] == ['m'] and seen['pair_base'] == 5 and seen['cs'] == ['a'] and seen['radius'] == 0.03


# ------------------------------------------------------------------------------------------------ kernels

RANSAC_KERNELS = ('k_ransac_init', 'k_ransac_compact', 'k_ransac_generate', 'k_ransac_validate', 'k_ransac_scan')


@functools.lru_cache(maxsize=None)
def ransac_ptxas():
    """ransac.cu compiled with -Xptxas -v: (output, {kernel: (stack, spill stores, spill loads)})."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'ransac.cu'),
                                                        '-o', os.path.join(tmp, 'ransac.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(entries) == len(RANSAC_KERNELS), [e[0] for e in entries]
    stats = {}
    for k in RANSAC_KERNELS:
        hit = [e for e in entries if k + 'E' in e[0]]
        assert len(hit) == 1, (k, [e[0] for e in entries])
        stats[k] = hit[0][1:]
    return text, stats


def test_ransac_kernels_do_not_spill():
    """ransac.cu's entry functions are exactly RANSAC_KERNELS; none spills, nor does any device function they call;
    only the hypothesis generator (its sample indices and the SVD) has a stack frame."""
    text, stats = ransac_ptxas()
    for k, (_, st, ld) in stats.items():
        assert (st, ld) == ('0', '0'), (k, st, ld)
    assert set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
    for k in RANSAC_KERNELS:
        assert (stats[k][0] == '0') == (k != 'k_ransac_generate'), (k, stats[k])
