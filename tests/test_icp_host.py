"""Point-to-point ICP on the host: the float64 oracle (tests/icp_oracle.py) against brute force and known transforms,
its edge cases, the CLI flags of `python -m regtr_b200.register`, and the 3DMatch benchmark's ICP wrapper; and the
spills and stack frames of every ICP kernel in icp.cu."""
import functools
import os
import re
import subprocess
import tempfile

import numpy as np
import torch

import icp_oracle as I
import train_data_oracle as O
from regtr_b200 import eval as E
from regtr_b200 import register as R


def rot(axis, deg):
    axis = np.asarray(axis, np.float64)
    return O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))


def pose34(axis, deg, t):
    p = np.eye(3, 4)
    p[:, :3] = rot(axis, deg)
    p[:, 3] = t
    return p


def test_correspondences_equal_brute_force():
    rng = np.random.default_rng(3)
    for n, m, r in ((300, 250, 0.15), (50, 400, 0.08), (200, 1, 0.5)):
        p = rng.uniform(-1, 1, (n, 3))
        t = rng.uniform(-1, 1, (m, 3))
        t[: m // 10] = t[m // 10: 2 * (m // 10)]          # duplicated targets: ties go to the lowest index
        nn, d2 = I.correspondences(p, t, r)
        ref = O.nearest_within(p, t, r)
        assert np.array_equal(nn, ref)
        m_ = ref >= 0
        dx, dy, dz = (p[m_, a] - t[ref[m_], a] for a in range(3))
        assert np.array_equal(d2[m_], (dx * dx + dy * dy) + dz * dz)
        assert np.isinf(d2[~m_]).all()
    # exactly on the radius is not a correspondence (strict)
    nn, _ = I.correspondences(np.array([[0.0, 0.0, 0.0]]), np.array([[0.5, 0.0, 0.0]]), 0.5)
    assert nn.tolist() == [-1]


def test_recovers_a_rigid_transform_on_a_noiseless_pair():
    rng = np.random.default_rng(5)
    tgt = rng.uniform(-1, 1, (2000, 3)) * [1.0, 0.8, 0.6]
    gt = pose34([0.2, -0.4, 0.9], 3.0, [0.03, -0.02, 0.01])
    inv = np.eye(3, 4)
    inv[:, :3] = gt[:, :3].T
    inv[:, 3] = -gt[:, :3].T @ gt[:, 3]
    src = I.transform(inv, tgt)                              # gt maps src exactly onto tgt
    init = np.eye(3, 4)
    out = I.icp(src, tgt, init, 0.2, max_iteration=100, relative_fitness=1e-12, relative_rmse=1e-12)
    assert np.abs(out['pose'] - gt).max() < 1e-10, np.abs(out['pose'] - gt).max()
    assert out['fitness'] == 1.0 and out['rmse'] < 1e-10 and out['k'] == 2000
    assert 0 < out['iterations'] < 100                    # the stop test ends it


def test_no_correspondences_and_zero_iterations_return_init():
    rng = np.random.default_rng(7)
    src = rng.uniform(-1, 1, (100, 3))
    init = pose34([1, 1, 0], 5.0, [0.1, 0.2, 0.3])
    far = I.icp(src, src + 50.0, init, 0.1)
    assert np.array_equal(far['pose'], init)
    assert far['fitness'] == 0.0 and far['rmse'] == 0.0 and far['k'] == 0
    assert far['iterations'] == 1                          # the identity update, then no change: converged
    zero = I.icp(src, src, init, 0.5, max_iteration=0)
    assert np.array_equal(zero['pose'], init) and zero['iterations'] == 0
    assert zero['fitness'] > 0                             # the initial correspondences are still reported
    empty = I.icp(np.zeros((0, 3)), src, init, 0.5)
    assert np.array_equal(empty['pose'], init) and (empty['fitness'], empty['rmse'], empty['k']) == (0.0, 0.0, 0)
    pose, res = I.icp_batch([src, src], [src + 50.0, src], np.stack([init, init]), 0.1, max_iteration=0)
    assert np.array_equal(pose, np.stack([init, init])) and res.shape == (2, 4)
    assert res[0].tolist() == [0.0, 0.0, 0.0, 0.0]


def test_register_parser_accepts_icp_flags():
    ap = R.parser()
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.0375', '--icp_iters', '12'])
    assert opt.icp == 0.0375 and opt.icp_iters == 12
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth'])
    assert opt.icp is None and opt.icp_iters == 30


def test_benchmark_wrapper_layout_on_cpu():
    rng = np.random.default_rng(11)
    B, L = 2, 3
    tgts = [rng.uniform(-1, 1, (400, 3)) for _ in range(B)]
    gts = [pose34([0, 0, 1], 2.0, [0.01, 0, 0]), pose34([1, 0, 0], -1.5, [0, 0.02, 0])]
    srcs = []
    for t, g in zip(tgts, gts):
        inv = np.eye(3, 4)
        inv[:, :3] = g[:, :3].T
        inv[:, 3] = -g[:, :3].T @ g[:, 3]
        srcs.append(torch.from_numpy(I.transform(inv, t)).float())
    net = torch.from_numpy(np.stack([np.stack(gts)] * L)).float()        # (L,B,3,4) network poses
    net_before = net.clone()
    batch = {'src_xyz': srcs, 'tgt_xyz': [torch.from_numpy(t).float() for t in tgts],
             'pose': torch.from_numpy(np.stack(gts)).float()}
    calls = []

    def oracle_icp(src_list, tgt_list, init, radius, max_iteration):
        calls.append((radius, max_iteration))
        return I.icp_batch([s.numpy() for s in src_list], [t.numpy() for t in tgt_list], init.numpy(), radius,
                           max_iteration)

    run = E.icp_forward(lambda b: {'pose': net, 'src_kp': 'kept'}, 0.05, 7, icp=oracle_icp)
    pred = run(batch)
    assert calls == [(0.05, 7)]
    assert pred['pose'].shape == (1, B, 3, 4) and pred['pose'].dtype == torch.float64
    assert pred['pose_coarse'].shape == (1, B, 3, 4) and torch.equal(pred['pose_coarse'][0], net[-1].double())
    assert pred['src_kp'] == 'kept' and torch.equal(net, net_before)              # the forward's outputs untouched
    want, _ = oracle_icp(batch['src_xyz'], batch['tgt_xyz'], net[-1].double(), 0.05, 7)
    assert np.array_equal(pred['pose'][0].numpy(), want)
    m = E.compute_metrics(pred, batch['pose'].double())
    assert set(m) == {'rot_err_deg', 'trans_err', 'rot_err_deg_coarse', 'trans_err_coarse'}
    assert all(v.shape == (1, B) for v in m.values())
    agg = E.aggregate_metrics([m])
    assert 'rot_err_deg_final' in agg and 'rot_err_deg_coarse_final' in agg


ICP_KERNELS = ('k_icp_init', 'k_icp_nn', 'k_icp_reduce_point', 'k_icp_reduce_planeILNS_9PlaneModeE0',
               'k_icp_reduce_planeILNS_9PlaneModeE1', 'k_icp_reduce_planeILNS_9PlaneModeE2', 'k_icp_updateILb0',
               'k_icp_updateILb1')


@functools.lru_cache(maxsize=None)
def icp_ptxas():
    """icp.cu compiled with -Xptxas -v: (ptxas output, {kernel of ICP_KERNELS: (stack, spill stores, spill loads)})."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'icp.cu'),
                                                        '-o', os.path.join(tmp, 'icp.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(entries) == len(ICP_KERNELS), [e[0] for e in entries]
    stats = {}
    for k in ICP_KERNELS:
        hit = [e for e in entries if k + 'E' in e[0]]
        assert len(hit) == 1, (k, [e[0] for e in entries])
        stats[k] = hit[0][1:]
    return text, stats


def test_icp_kernels_do_not_spill():
    """icp.cu's entry functions are exactly ICP_KERNELS; none spills, nor does any device function they call."""
    text, stats = icp_ptxas()
    for k, (_, st, ld) in stats.items():
        assert (st, ld) == ('0', '0'), (k, st, ld)
    assert set(re.findall(r'bytes spill (?:stores|loads)', text)) and \
        set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}


def test_icp_kernels_have_no_stack_frame():
    """Every ICP kernel but the two updates runs without a stack frame: in generalized ICP's reduction that means the
    unsorted Jacobi sweeps keep M, A and V in registers."""
    _, stats = icp_ptxas()
    for k in ICP_KERNELS[:6]:
        assert stats[k][0] == '0', (k, stats[k])
