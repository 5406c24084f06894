"""Generalized ICP (`ops.icp` with method='generalized') and robust point-to-plane ICP (a loss other than 'l2') on the
device against the float64 oracle (tests/gicp_oracle.py) on the real 3DMatch fixtures and on synthetic pairs: the
final pose, iteration count, correspondences and RMSE, the state after 0..3 iterations, batching, reruns, the launch
count, the L2 bit-identities, the errors, `python -m regtr_b200.register --icp_method generalized` end to end and
`multiway.register_pairs` with generalized ICP."""
import os

import numpy as np
import pytest
import torch

import gicp_oracle as G
from regtr_b200 import lib, ops
from regtr_b200 import multiway as MW
from regtr_b200 import pointio as P
from regtr_b200 import register as R
from regtr_b200 import synthetic as S
from test_gpu_icp import RADIUS, _run_register, real_pairs, synthetic_pairs
from test_gpu_icp_plane import REAL

pytestmark = pytest.mark.gpu
NR = 2.0 * RADIUS
K_DIFF = []
LOSSES = [('huber', 0.005), ('cauchy', 0.01), ('gm', 0.01), ('tukey', 0.01)]
CASES = [('generalized', 'l2', None)] + [(m, l, k) for m in ('point_to_plane', 'generalized') for l, k in LOSSES]


def with_normals(pairs):
    """(src, tgt, init) -> (src, tgt, init, src normals, tgt normals) from one estimate_normals call."""
    B = len(pairs)
    n = ops.estimate_normals([s for s, _, _ in pairs] + [t for _, t, _ in pairs], NR)
    return [(s, t, p, n[b].cpu().numpy(), n[B + b].cpu().numpy()) for b, (s, t, p) in enumerate(pairs)]


def device(pairs5, method, loss='l2', loss_k=None, max_iteration=30, **kw):
    init = torch.from_numpy(np.stack([q[2] for q in pairs5])).cuda()
    return ops.icp([q[0] for q in pairs5], [q[1] for q in pairs5], init, RADIUS, max_iteration, method=method,
                   tgt_normals=[q[4] for q in pairs5],
                   src_normals=[q[3] for q in pairs5] if method == 'generalized' else None, loss=loss, loss_k=loss_k,
                   **kw)


def check(pose, res, pairs5, method, loss='l2', loss_k=None, max_iteration=30):
    pose, res = pose.cpu().numpy(), res.cpu().numpy()
    for b, (s, t, p, ns, nt) in enumerate(pairs5):
        o = G.icp(s, t, nt, p, RADIUS, max_iteration, method=method, src_normals=ns, loss=loss, loss_k=loss_k)
        rot_err = np.linalg.norm(pose[b, :, :3] - o['pose'][:, :3])
        trans_err = np.linalg.norm(pose[b, :, 3] - o['pose'][:, 3])
        what = (method, loss, b)
        assert rot_err <= 1e-9 and trans_err <= 1e-9, (what, rot_err, trans_err)
        assert int(res[b, 3]) == o['iterations'], (what, res[b], o['iterations'])
        K_DIFF.append(abs(int(res[b, 2]) - o['k']))
        assert abs(int(res[b, 2]) - o['k']) <= 2, (what, res[b, 2], o['k'])
        assert abs(res[b, 1] - o['rmse']) <= 1e-12 * o['rmse'], (what, res[b, 1], o['rmse'])
        assert res[b, 0] == res[b, 2] / len(s)
    return res


@pytest.mark.parametrize('method,loss,loss_k', CASES)
def test_real_and_synthetic_pairs_against_the_oracle(method, loss, loss_k):
    pairs5 = with_normals(real_pairs() + synthetic_pairs())
    pose, res = device(pairs5, method, loss, loss_k)
    r = check(pose, res, pairs5, method, loss, loss_k)
    print(f'{method} {loss}: iterations {r[:, 3].astype(int).tolist()}')


@pytest.mark.parametrize('method,loss,loss_k', [CASES[0], ('point_to_plane', 'tukey', 0.01),
                                                ('generalized', 'huber', 0.005)])
def test_state_after_each_of_the_first_iterations(method, loss, loss_k):
    pairs5 = with_normals(real_pairs()[:1] + synthetic_pairs((4003,)))
    for it in range(4):
        pose, res = device(pairs5, method, loss, loss_k, it)
        r = check(pose, res, pairs5, method, loss, loss_k, it)
        assert (r[:, 3] == it).all()
        if it == 0:
            assert np.array_equal(pose.cpu().numpy(), np.stack([q[2] for q in pairs5]))


@pytest.mark.parametrize('method,loss,loss_k', [CASES[0], ('point_to_plane', 'cauchy', 0.01),
                                                ('generalized', 'tukey', 0.01)])
def test_batch_equals_one_call_per_pair_and_reruns_are_identical(method, loss, loss_k):
    real = real_pairs()
    syn = synthetic_pairs((4004,))[0]
    far = (syn[0][:3000], syn[1][:5000] + 40.0, syn[2])              # no correspondences at all
    pairs5 = with_normals([real[0], far, (real[1][0][:7001], real[1][1], real[1][2]), syn])
    pose, res = device(pairs5, method, loss, loss_k)
    again = device(pairs5, method, loss, loss_k)
    assert torch.equal(pose, again[0]) and torch.equal(res, again[1])
    for b, q in enumerate(pairs5):
        p1, r1 = device([q], method, loss, loss_k)
        assert torch.equal(p1[0], pose[b]) and torch.equal(r1[0], res[b]), b
    assert res[1].cpu().numpy().tolist() == [0.0, 0.0, 0.0, 1.0]
    assert np.array_equal(pose[1].cpu().numpy(), far[2])


def test_launch_count_does_not_depend_on_method_batch_or_convergence():
    pairs5 = with_normals(synthetic_pairs((4005,)))
    loose = dict(relative_fitness=1e-2, relative_rmse=1e-2)
    never = dict(relative_fitness=0.0, relative_rmse=0.0)
    for method, loss, loss_k in (CASES[0], ('point_to_plane', 'tukey', 0.01)):
        counts = []
        for batch, kw, done_early in ((pairs5, loose, True), (pairs5 * 8, loose, True), (pairs5, never, False),
                                      (pairs5 * 8, never, False)):
            before = ops.LAUNCHES
            _, res = device(batch, method, loss, loss_k, 30, **kw)
            torch.cuda.synchronize()
            counts.append(ops.LAUNCHES - before)
            iters = res[:, 3].cpu().numpy()
            assert (iters < 30).all() if done_early else (iters == 30).all(), iters
        assert counts == [ops.icp_launches(30)] * 4, counts


def test_l2_identities():
    """Huber with k above every residual weights everything by exactly 1: the bits of L2 point-to-plane.  An explicit
    loss='l2' is the default call.  In generalized ICP the same weights give L2's result up to rounding (the compiler
    may order the L2 instantiation's operations differently)."""
    pairs5 = with_normals(real_pairs() + synthetic_pairs((4006,)))
    a = device(pairs5, 'point_to_plane')
    b = device(pairs5, 'point_to_plane', 'huber', 1e6)
    c = ops.icp([q[0] for q in pairs5], [q[1] for q in pairs5],
                torch.from_numpy(np.stack([q[2] for q in pairs5])).cuda(), RADIUS, 30, method='point_to_plane',
                tgt_normals=[q[4] for q in pairs5])
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, c))
    d = device(pairs5, 'generalized', 'huber', 1e6)
    e = device(pairs5, 'generalized')
    assert torch.equal(d[1][:, 3], e[1][:, 3]) and torch.equal(d[1][:, 2], e[1][:, 2])
    assert (d[0] - e[0]).abs().max().item() <= 1e-9
    assert not torch.equal(a[0], e[0])


def test_errors():
    rb = ops.overlap_coord_bound(RADIUS)
    src = np.array([[0.0, 0.0, 0.0], [rb * 1.001, 0.0, 0.0]])
    tgt = np.array([[0.01, 0.0, 0.0]])
    eye = torch.from_numpy(np.eye(3, 4)[None])
    nt = [np.array([[0.0, 0.0, 1.0]])]
    ns = [np.zeros((1, 3))]
    with pytest.raises(lib.RegtrLibError, match='icp: a coordinate'):
        ops.icp([src], [tgt], eye, RADIUS, method='generalized', tgt_normals=nt, src_normals=[np.zeros((2, 3))])
    with pytest.raises(lib.RegtrLibError, match='icp: a coordinate'):
        ops.icp([src], [tgt], eye, RADIUS, method='point_to_plane', tgt_normals=nt, loss='tukey', loss_k=0.01)
    ok = dict(method='generalized', tgt_normals=nt, src_normals=ns)
    with pytest.raises(ValueError, match='source normals'):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='generalized', tgt_normals=nt)
    with pytest.raises(ValueError, match='target normals'):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='generalized', src_normals=ns)
    with pytest.raises(ValueError):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='generalized', tgt_normals=nt, src_normals=[np.zeros((2, 3))])
    with pytest.raises(ValueError):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='generalized', tgt_normals=nt, src_normals=ns * 2)
    for eps in (0.0, -1e-3, 1.5, float('nan')):
        with pytest.raises(ValueError, match='epsilon'):
            ops.icp([src[:1]], [tgt], eye, RADIUS, epsilon=eps, **ok)
    with pytest.raises(ValueError, match='loss'):
        ops.icp([src[:1]], [tgt], eye, RADIUS, loss='l1', loss_k=1.0, **ok)
    for k in (None, 0.0, -1.0, float('inf'), float('nan')):
        with pytest.raises(ValueError, match='loss_k'):
            ops.icp([src[:1]], [tgt], eye, RADIUS, loss='huber', loss_k=k, **ok)
    with pytest.raises(ValueError, match='point_to_point'):
        ops.icp([src[:1]], [tgt], eye, RADIUS, loss='tukey', loss_k=0.01)
    pose, res = ops.icp([src[:1]], [tgt], eye, RADIUS, epsilon=1.0, **ok)
    assert torch.isfinite(pose).all() and res[0, 2].item() == 1.0


def test_report_largest_k_difference():
    print(f'largest |k_device - k_oracle|: {max(K_DIFF) if K_DIFF else "n/a"}')
    assert not K_DIFF or max(K_DIFF) <= 2


def test_register_cli_with_generalized_tukey_icp(tmp_path):
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config('modelnet')
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': random_state_dict(cfg, 43), 'step': 1}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, 'modelnet', str(run / 'config.yaml'))
    src_file = os.path.join(REAL, 'modelnet_test_2_0.ply')
    tgt_file = os.path.join(REAL, 'modelnet_test_2_1.ply')
    s, t = P.load_point_cloud(src_file), P.load_point_cloud(tgt_file)
    radius, k = 0.05, 0.02
    line = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'gicp',
                         ['--icp', str(radius), '--icp_method', 'generalized', '--icp_loss', 'tukey',
                          '--icp_loss_k', str(k)])
    res = np.load(str(tmp_path / 'gicp' / 'result.npz'))
    coarse = res['pose'][-1]
    assert np.array_equal(res['pose_coarse'], coarse)
    ns, nt = ops.estimate_normals([s, t], 2.0 * radius, 30)
    pose, out = ops.icp([s], [t], torch.from_numpy(coarse[None]).cuda(), radius, 30, method='generalized',
                        tgt_normals=[nt], src_normals=[ns], loss='tukey', loss_k=k)
    pose, out = pose[0].cpu().numpy(), out[0].cpu().numpy()
    assert np.array_equal(res['pose_icp'], pose) and np.array_equal(res['icp'], out)
    assert open(tmp_path / 'gicp' / 'pose.txt').read() == R.pose_text(pose)
    assert (line['icp_method'], line['icp_loss'], line['icp_loss_k'], line['icp_epsilon'], line['icp_iterations']) == \
        ('generalized', 'tukey', k, 1e-3, int(out[3]))


class _FakeModel:
    """register_pairs' view of a model: the scene's true relative poses, perturbed, as the final layer's poses."""

    def __init__(self, poses, fragments):
        self.device = torch.device('cuda:0')
        self.poses, self.frags = poses, [torch.from_numpy(f).float() for f in fragments]

    def _index(self, x):
        return next(k for k, f in enumerate(self.frags) if x.shape == f.shape and torch.equal(x.cpu(), f))

    def __call__(self, batch):
        out = []
        for s, t in zip(batch['src_xyz'], batch['tgt_xyz']):
            j, i = self._index(s), self._index(t)
            rel = np.linalg.inv(self.poses[i]) @ self.poses[j]               # source j -> target i
            d = np.eye(4)
            d[:3, 3] = [0.01, -0.005, 0.008]
            out.append((d @ rel)[:3])
        return {'pose': torch.from_numpy(np.stack(out))[None].to(self.device)}


def test_multiway_register_pairs_with_generalized_icp():
    sc = S.make_scene(9, 4, n_target=4000)
    frags = [f.astype(np.float64) for f in sc['fragments']]
    model = _FakeModel(sc['poses'], sc['fragments'])
    radius = 0.05
    got = MW.register_pairs(model, frags, 4, radius, 30, 'generalized', icp_loss='huber', icp_loss_k=0.01)
    coarse = MW.register_pairs(model, frags, 4)
    normals = ops.estimate_normals(frags, 2.0 * radius, 30)
    for k, (i, j) in enumerate(MW.all_pairs(len(frags))):
        pose, _ = ops.icp([frags[j]], [frags[i]], torch.from_numpy(coarse[k:k + 1]).cuda(), radius, 30,
                          method='generalized', tgt_normals=[normals[i]], src_normals=[normals[j]], loss='huber',
                          loss_k=0.01)
        assert np.array_equal(got[k], pose[0].cpu().numpy()), (i, j)
