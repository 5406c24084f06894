"""Generalized ICP and robust kernels on the host: the float64 oracle (tests/gicp_oracle.py) against independent
constructions of the covariance and the weights, recovery of a known transform, the robust kernels' resistance to an
off-surface block, the CLI flags of register, multiway, eval_3dmatch and bench_icp, and the 3DMatch benchmark
wrapper's generalized layout.  (The ICP kernels' stack and spill check is in test_icp_host.py.)"""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import gicp_oracle as G
import icp_oracle as I
import icp_plane_oracle as N
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import register as R
from test_icp_plane_host import inverse, pose34, room

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_covariance_matches_open3d_construction_and_zero_normal_gives_identity():
    rng = np.random.default_rng(1)
    for eps in (1e-3, 0.1, 1.0):
        n = rng.normal(size=(50, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        got = G.covariance(n, eps)
        for m, c in zip(n, got):
            rx = Rotation.align_vectors([m], [[1.0, 0.0, 0.0]])[0].as_matrix()     # e1 -> n
            want = rx @ np.diag([eps, 1.0, 1.0]) @ rx.T
            assert np.abs(c - want).max() < 1e-14
    assert np.array_equal(G.covariance(np.zeros((1, 3)), 1e-3)[0], np.eye(3))


def test_information_square_root_whitens_m():
    rng = np.random.default_rng(2)
    a, b = rng.normal(size=(200, 3)), rng.normal(size=(200, 3))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    b[:20] = a[:20]                                               # coincident normals: the most anisotropic M
    M = G.covariance(a, 1e-3) + G.covariance(b, 1e-3)
    W, ok = G.information_sqrt(M)
    assert ok.all()
    assert np.abs(W @ M @ W - np.eye(3)).max() < 1e-11
    assert np.abs(W - W.transpose(0, 2, 1)).max() < 1e-13
    # non-unit normals can make M indefinite: that correspondence leaves the update
    _, ok = G.information_sqrt(G.covariance(np.array([[3.0, 0.0, 0.0]]), 1e-3) + np.eye(3)[None])
    assert not ok[0]
    _, ok = G.information_sqrt(np.full((1, 3, 3), np.nan))
    assert not ok[0]


def test_weights_match_their_formulas_and_boundaries():
    k = 0.02
    r = np.array([-0.05, -0.02, -0.01, 0.0, 0.005, 0.02, 0.03])
    assert np.array_equal(G.weight('l2', k, r), np.ones(7))
    hub = G.weight('huber', k, r)
    assert hub[3] == 1.0 and hub[1] == 1.0 and hub[5] == 1.0          # |r| = k is inside
    assert hub[0] == k / 0.05 and hub[6] == k / 0.03
    for i, x in enumerate(r):
        assert G.weight('cauchy', k, x) == 1.0 / (1.0 + (x / k) ** 2)
        assert G.weight('gm', k, x) == k / (k + x * x) ** 2
    tk = G.weight('tukey', k, r)
    assert tk[1] == 0.0 and tk[5] == 0.0 and tk[3] == 1.0           # |r| = k: (1 - 1)^2 = 0, inside the branch
    assert tk[0] == 0.0 and tk[6] == 0.0
    assert tk[2] == (1.0 - 0.25) ** 2 and tk[4] == (1.0 - 0.0625) ** 2
    assert np.isfinite(G.weight('huber', k, np.array([0.0]))).all()


def test_generalized_recovers_a_rigid_transform_on_a_noiseless_pair():
    rng = np.random.default_rng(5)
    tgt = room(rng)
    gt = pose34([0.2, -0.4, 0.9], 3.0, [0.03, -0.02, 0.01])
    src = I.transform(inverse(gt), tgt)
    nt, _ = N.estimate_normals(tgt, 0.15, 30)
    ns, _ = N.estimate_normals(src, 0.15, 30)
    for loss, k in (('l2', None), ('tukey', 0.05)):
        out = G.icp(src, tgt, nt, np.eye(3, 4), 0.2, 100, 1e-12, 1e-12, src_normals=ns, loss=loss, loss_k=k)
        assert np.abs(out['pose'] - gt).max() < 1e-10, (loss, np.abs(out['pose'] - gt).max())
        assert out['fitness'] == 1.0 and out['rmse'] < 1e-10 and 0 < out['iterations'] < 100
    # L2 point-to-plane through this oracle is icp_plane_oracle's
    a = G.icp(src, tgt, nt, np.eye(3, 4), 0.2, 5, method='point_to_plane')
    b = N.icp(src, tgt, nt, np.eye(3, 4), 0.2, 5)
    assert np.abs(a['pose'] - b['pose']).max() < 1e-12 and a['iterations'] == b['iterations']


def test_tukey_resists_an_off_surface_block():
    """A block of source points pushed 2 cm off the floor, inside the max distance: Tukey with k = 1 cm ignores it;
    L2 is pulled towards it."""
    rng = np.random.default_rng(6)
    tgt = room(rng)
    gt = pose34([0.3, 0.1, 1.0], 2.0, [0.02, 0.01, -0.01])
    src_in_tgt = tgt.copy()
    block = (np.abs(src_in_tgt[:, 2]) < 1e-12) & (src_in_tgt[:, 0] > 0.0)          # half of the floor
    assert block.sum() > 500
    src_in_tgt[block, 2] += 0.02
    src = I.transform(inverse(gt), src_in_tgt)
    nt, _ = N.estimate_normals(tgt, 0.15, 30)
    ns, _ = N.estimate_normals(src, 0.15, 30)
    init = I.compose(pose34([1.0, 0.0, 0.0], 0.5, [0.005, 0.0, 0.005]), gt)
    def err(out):
        return np.linalg.norm(out['pose'][:, 3] - gt[:, 3]) + np.linalg.norm(out['pose'][:, :3] - gt[:, :3])
    for method, extra in (('point_to_plane', {}), ('generalized', dict(src_normals=ns))):
        l2 = G.icp(src, tgt, nt, init, 0.05, 50, method=method, **extra)
        tk = G.icp(src, tgt, nt, init, 0.05, 50, method=method, loss='tukey', loss_k=0.01, **extra)
        assert err(tk) < 0.5 * err(l2), (method, err(tk), err(l2))
        assert err(tk) < 1e-3, (method, err(tk))


def test_register_and_multiway_parsers_accept_the_generalized_flags():
    args = ['--ckpt', 'c/ckpt/m.pth', '--icp', '0.0375', '--icp_method', 'generalized', '--icp_epsilon', '0.01',
            '--icp_loss', 'tukey', '--icp_loss_k', '0.02']
    for ap, pos in ((R.parser(), ['a.ply', 'b.ply']), (MW.parser(), ['a.ply', 'b.ply', '--out', 'o'])):
        opt = ap.parse_args(pos + args)
        assert (opt.icp_method, opt.icp_epsilon, opt.icp_loss, opt.icp_loss_k) == ('generalized', 0.01, 'tukey', 0.02)
        opt = ap.parse_args(pos + ['--ckpt', 'c/ckpt/m.pth'])
        assert (opt.icp_method, opt.icp_epsilon, opt.icp_loss, opt.icp_loss_k) == ('point_to_point', 1e-3, 'l2', None)
        for loss in ('l2', 'huber', 'cauchy', 'gm', 'tukey'):
            assert ap.parse_args(pos + ['--ckpt', 'x', '--icp_loss', loss, '--icp_loss_k', '1']).icp_loss == loss
        with pytest.raises(SystemExit):
            ap.parse_args(pos + ['--ckpt', 'x', '--icp_loss', 'l1'])
    with pytest.raises(SystemExit):                                     # a robust loss without its k
        R.main(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.03', '--icp_loss', 'huber'])


def test_bench_and_eval_scripts_accept_the_generalized_flags():
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import bench_icp
    finally:
        sys.path.pop(0)
    opt = bench_icp.parser().parse_args(['--method', 'generalized', '--loss', 'tukey', '--loss_k', '0.01'])
    assert (opt.method, opt.loss, opt.loss_k, opt.epsilon) == ('generalized', 'tukey', 0.01, 1e-3)
    opt = bench_icp.parser().parse_args([])
    assert (opt.method, opt.loss, opt.loss_k) == ('point_to_point', 'l2', None)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'scripts', 'eval_3dmatch.py'), '--help'],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    for flag in ('--icp_epsilon', '--icp_loss {l2,huber,cauchy,gm,tukey}', '--icp_loss_k'):
        assert flag in r.stdout, flag
    assert 'generalized' in r.stdout


def _eval_3dmatch():
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import eval_3dmatch
    finally:
        sys.path.pop(0)
    return eval_3dmatch


@pytest.mark.parametrize('cli', ['register', 'multiway', 'eval_3dmatch'])
def test_every_command_line_rejects_a_robust_loss_without_its_k(cli, capsys):
    """At parse time, before any model or data is loaded: a usage error (exit status 2)."""
    ap, main, args = {
        'register': lambda: (R.parser(), R.main, ['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth']),
        'multiway': lambda: (MW.parser(), MW.main, ['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--out', 'o']),
        'eval_3dmatch': lambda: (_eval_3dmatch().parser(), _eval_3dmatch().main,
                                 ['--root', 'r', '--info', 'i.pkl', '--gt', 'g', '--ckpt', 'm.pth']),
    }[cli]()
    args += ['--icp', '0.03', '--icp_method', 'point_to_plane', '--icp_loss', 'huber']
    with pytest.raises(SystemExit) as e:
        main(args)
    assert e.value.code == 2 and '--icp_loss huber needs --icp_loss_k' in capsys.readouterr().err
    opt = ap.parse_args(args + ['--icp_loss_k', '0.02'])
    E.check_icp_arguments(ap, opt)
    assert (opt.icp_loss, opt.icp_loss_k) == ('huber', 0.02)


def test_benchmark_wrapper_generalized_layout_on_cpu():
    rng = np.random.default_rng(11)
    B, L = 2, 3
    tgts = [room(rng, 300) * 0.5 for _ in range(B)]
    gts = [pose34([0, 0, 1], 2.0, [0.01, 0, 0]), pose34([1, 0, 0], -1.5, [0, 0.02, 0])]
    srcs = [torch.from_numpy(I.transform(inverse(g), t)).float() for t, g in zip(tgts, gts)]
    net = torch.from_numpy(np.stack([np.stack(gts)] * L)).float()
    batch = {'src_xyz': srcs, 'tgt_xyz': [torch.from_numpy(t).float() for t in tgts],
             'pose': torch.from_numpy(np.stack(gts)).float()}
    calls = []

    def oracle_normals(clouds, radius, max_nn):
        calls.append(('normals', len(clouds), radius, max_nn))
        return [N.estimate_normals(c.numpy(), radius, max_nn)[0] for c in clouds]

    def oracle_icp(src_list, tgt_list, init, radius, max_iteration, method, tgt_normals, src_normals,
                   epsilon=1e-3, loss='l2', loss_k=None):
        calls.append(('icp', radius, max_iteration, method, epsilon, loss, loss_k))
        return G.icp_batch([s.numpy() for s in src_list], [t.numpy() for t in tgt_list], tgt_normals, init.numpy(),
                           radius, max_iteration, src_normals_list=src_normals, epsilon=epsilon, loss=loss,
                           loss_k=loss_k)

    run = E.icp_forward(lambda b: {'pose': net}, 0.05, 7, icp=oracle_icp, method='generalized', normal_max_nn=20,
                        estimate_normals=oracle_normals)
    pred = run(batch)
    assert calls == [('normals', 2 * B, 0.1, 20), ('icp', 0.05, 7, 'generalized', 1e-3, 'l2', None)]
    assert pred['pose'].shape == (1, B, 3, 4) and pred['pose'].dtype == torch.float64
    normals = oracle_normals(batch['src_xyz'] + batch['tgt_xyz'], 0.1, 20)
    want, _ = G.icp_batch([s.numpy() for s in srcs], [t.numpy() for t in batch['tgt_xyz']], normals[B:],
                          net[-1].double().numpy(), 0.05, 7,
                          src_normals_list=normals[:B])
    assert np.array_equal(pred['pose'][0].numpy(), want)
    calls.clear()
    E.icp_forward(lambda b: {'pose': net}, 0.05, 7, icp=oracle_icp, method='generalized', epsilon=0.01, loss='huber',
                  loss_k=0.02, estimate_normals=oracle_normals)(batch)
    assert calls[1] == ('icp', 0.05, 7, 'generalized', 0.01, 'huber', 0.02)
    # point_to_plane with a loss: only the loss arguments are added to today's call
    seen = []
    E.icp_forward(lambda b: {'pose': net}, 0.05, 7, method='point_to_plane', loss='tukey', loss_k=0.01,
                  icp=lambda *a, **kw: (seen.append(sorted(kw)), (net[-1].double(), None))[1],
                  estimate_normals=oracle_normals)(batch)
    assert seen == [['loss', 'loss_k', 'method', 'tgt_normals']]
    with pytest.raises(ValueError):
        E.icp_forward(lambda b: b, 0.05, method='gicp')
