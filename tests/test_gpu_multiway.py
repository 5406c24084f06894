"""Multiway registration on the device: `ops.registration_information` and `ops.pose_graph_optimize` against the
float64 oracle (tests/posegraph_oracle.py), the optimiser's batch, rerun, launch and error properties, a synthetic
scene through the post-network API and the 3DMatch benchmark, and `python -m regtr_b200.multiway` end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import posegraph_oracle as PG
from conftest import GOLDEN, ROOT
from regtr_b200 import eval as E
from regtr_b200 import lib, ops
from regtr_b200 import multiway as M
from regtr_b200 import pointio as PIO
from regtr_b200 import synthetic as S

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')


def real_pairs():
    out = []
    for fx, scene in (('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'),
                      ('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3')):
        keys, traj = E.read_trajectory(os.path.join(REAL, 'benchmarks', '3DMatch', scene, 'gt.log'))
        inp = np.load(os.path.join(REAL, fx + '_input.npz'))
        src_is_file_src = os.path.basename(str(inp['src_file'])) == f'cloud_bin_{int(keys[0][1])}.pth'
        a, b = inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64)
        out.append((a, b, traj[0][:3]) if src_is_file_src else (b, a, traj[0][:3]))
    return out


def test_information_matches_the_restatement_on_real_and_synthetic_pairs():
    pairs = real_pairs()
    p = S.make_3dmatch_pair(77, 6000)
    pairs.append((p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), p['pose'].astype(np.float64)))
    r = 0.0375
    pose = torch.from_numpy(np.stack([q for _, _, q in pairs])).cuda()
    fit, info = ops.registration_information([s for s, _, _ in pairs], [t for _, t, _ in pairs], pose, r)
    assert torch.equal(fit, ops.registration_fit([s for s, _, _ in pairs], [t for _, t, _ in pairs], pose, r))
    info = info.cpu().numpy()
    for b, (s, t, q) in enumerate(pairs):
        want = PG.information(s, t, q, r)
        assert want[5, 5] > 100 and info[b, 5, 5] == want[5, 5], b
        assert np.abs(info[b] - want).max() <= 1e-12 * np.abs(want).max(), (b, np.abs(info[b] - want).max())
        assert round(float(fit[b, 0]) * len(s)) == want[5, 5]
        one = ops.registration_information([s], [t], torch.from_numpy(q[None]).cuda(), r)[1].cpu().numpy()
        assert np.array_equal(one[0], info[b])                                # independent of the batch


def run_device(graphs, d, **kw):
    return ops.pose_graph_optimize([g['init'] for g in graphs], [g['edges'] for g in graphs],
                                   [g['X'] for g in graphs], [g['info'] for g in graphs],
                                   [g['uncertain'] for g in graphs], d, **kw)


def check_against_oracle(g, P, conf, kept, res, d):
    want = PG.optimize(g['init'], g['edges'], g['X'], g['info'], g['uncertain'], d)
    P = P.cpu().numpy()
    assert np.array_equal(kept.cpu().numpy(), want['kept'])
    assert res[:2].tolist() == want['result'][:2].tolist(), (res, want['result'])
    assert np.abs(P - want['poses']).max() < 1e-9, np.abs(P - want['poses']).max()
    assert abs(res[2] - want['result'][2]) <= 1e-9 * max(1.0, abs(want['result'][2]))
    c = conf.cpu().numpy()
    assert np.all(np.abs(c - want['confidence']) <= 1e-9 * np.abs(want['confidence']) + 1e-15), \
        np.abs(c - want['confidence']).max()
    return want


def one_node():
    return dict(init=np.eye(4)[None], edges=np.zeros((0, 2), np.int64), X=np.zeros((0, 4, 4)),
                info=np.zeros((0, 6, 6)), uncertain=np.zeros(0, bool), truth=np.eye(4)[None])


CASES = {
    'n1': one_node,
    'n2': lambda: PG.noisy_graph(10, 2),
    'chain6_loops': lambda: PG.noisy_graph(11, 6, loop_span=3, wrong_frac=0.3),
    'n40_all_pairs': lambda: PG.noisy_graph(12, 40, all_pairs=True, wrong_frac=0.1, n_pts=60),
    'n256': lambda: PG.noisy_graph(13, 256, loop_span=3, wrong_frac=0.1, n_pts=60),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_optimizer_matches_the_oracle(case):
    g = CASES[case]()
    d = 0.05
    P, conf, kept, res = run_device([g], d)
    want = check_against_oracle(g, P[0], conf[0], kept[0], res[0].cpu().numpy(), d)
    assert np.array_equal(P[0][0].cpu().numpy(), g['init'][0][:3])          # the reference node, bit for bit
    if 'wrong' in g and g['wrong'].any():
        assert np.array_equal(~want['kept'], g['wrong'])


def test_a_batch_of_graphs_gives_the_bits_of_each_alone_and_reruns_agree():
    gs = [PG.noisy_graph(20, 7, loop_span=3, wrong_frac=0.3), PG.noisy_graph(21, 3), PG.noisy_graph(22, 12, 4, 0.2)]
    P, conf, kept, res = run_device(gs, 0.05)
    P2, conf2, kept2, res2 = run_device(gs, 0.05)
    assert torch.equal(res, res2) and all(torch.equal(a, b) for a, b in zip(P, P2))
    for k, g in enumerate(gs):
        check_against_oracle(g, P[k], conf[k], kept[k], res[k].cpu().numpy(), 0.05)
        Pa, ca, ka, ra = run_device([g], 0.05)
        assert torch.equal(Pa[0], P[k]) and torch.equal(ca[0], conf[k]) and torch.equal(ka[0], kept[k])
        assert torch.equal(ra[0], res[k])


def kernel_launches(fn):
    """(kernels named k_pose_graph, all device kernels) that fn launches, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and 'memcpy' not in e.name.lower() and 'memset' not in e.name.lower()]
    return sum('k_pose_graph' in n for n in names), out


def test_launches_do_not_depend_on_convergence():
    """A graph that is converged on entry (0 iterations) and one that runs to max_iteration in both passes: one
    k_pose_graph launch each, counted on the device."""
    fast = PG.noisy_graph(30, 5, noise_deg=0.0, noise_t=0.0)
    fast['init'] = fast['truth']
    slow = PG.noisy_graph(31, 8, loop_span=3, wrong_frac=0.3)
    kw_slow = dict(max_iteration=3, min_relative_increment=0.0, min_relative_residual_increment=0.0,
                   min_right_term=0.0, min_residual=0.0)
    n_fast, (_, _, _, res_fast) = kernel_launches(lambda: run_device([fast], 0.05))
    n_slow, (P, conf, kept, res_slow) = kernel_launches(lambda: run_device([slow], 0.05, **kw_slow))
    assert res_fast[0, :2].tolist() == [0.0, 0.0]
    assert res_slow[0, :2].tolist() == [3.0, 3.0]                            # both passes ran to max_iteration
    want = PG.optimize(slow['init'], slow['edges'], slow['X'], slow['info'], slow['uncertain'], 0.05, **kw_slow)
    assert want['result'][:2].tolist() == [3.0, 3.0]
    assert np.abs(P[0].cpu().numpy() - want['poses']).max() < 1e-9
    assert n_fast == n_slow == 1


def test_rejected_factorisations_match_the_oracle():
    """An indefinite information matrix on one odometry edge makes H + lambda I indefinite, so the first attempts'
    Cholesky fails and lambda grows; every thread of the CTA must take the same path through those attempts."""
    for seed, scale in ((11, 1.5), (14, 3.0)):
        g = PG.noisy_graph(seed, 6, loop_span=3, wrong_frac=0.3)
        e = int(np.flatnonzero(~g['uncertain'])[0])
        g['info'][e, 0, 0] -= scale * g['info'][e, 0, 0]
        P1, conf1, kept1, res1 = run_device([g], 0.05)
        want = check_against_oracle(g, P1[0], conf1[0], kept1[0], res1[0].cpu().numpy(), 0.05)
        assert want['failed_factorisations'] > 0, seed
        P, conf, kept, res = run_device([g, PG.noisy_graph(seed + 1, 5)], 0.05)         # alone or in a batch
        assert torch.equal(P[0], P1[0]) and torch.equal(conf[0], conf1[0]) and torch.equal(res[0], res1[0])


def test_bad_inputs_raise():
    g = PG.noisy_graph(40, 4)
    bad = dict(g, edges=g['edges'].copy())
    bad['edges'][1] = (2, 2)
    with pytest.raises(lib.RegtrLibError, match='rejected'):
        run_device([bad], 0.05)
    bad = dict(g, edges=g['edges'].copy())
    bad['edges'][0] = (0, 9)
    status = ops.new_status(torch.device('cuda'))
    P, conf, kept, res = run_device([g, bad], 0.05, status=status)
    assert int(status.item()) & ops.STATUS_INPUT
    assert np.isnan(res[1, 2].item()) and np.array_equal(P[1].cpu().numpy(), g['init'][:, :3])
    check_against_oracle(g, P[0], conf[0], kept[0], res[0].cpu().numpy(), 0.05)      # the good graph is unaffected
    nan_x = dict(g, X=g['X'].copy())
    nan_x['X'][0, 0, 0] = np.nan
    with pytest.raises(lib.RegtrLibError):
        run_device([nan_x], 0.05)
    big = PG.noisy_graph(41, 257, loop_span=1, n_pts=10)
    with pytest.raises(lib.RegtrLibError, match='UNSUPPORTED'):
        run_device([big], 0.05)


def scene_inputs(seed, n, noise_deg=0.2, noise_t=0.004, n_wrong=2):
    sc = S.make_scene(seed, n, n_target=5000)
    rng = np.random.default_rng(seed)
    truth = sc['poses']
    pairs = M.all_pairs(n)
    T = np.stack([PG.random_pose(rng, noise_deg, noise_t) @ PG.rinv(truth[i]) @ truth[j] for i, j in pairs])
    loops = [p for p, (i, j) in enumerate(pairs) if j - i == 2]
    wrong = rng.choice(loops, n_wrong, replace=False)
    for p in wrong:
        T[p] = PG.random_pose(rng, 30.0, 0.5) @ T[p]
    return sc, T, set(int(p) for p in wrong)


def test_scene_from_known_poses_recovers_the_truth_and_scores_full_recall(tmp_path):
    n = 8
    sc, T, wrong = scene_inputs(5, n)
    res = M.optimize_scene(sc['fragments'], T, 0.0375, min_overlap=0.3)
    pairs = [tuple(p) for p in res['pairs']]
    edge_pair = [pairs.index((int(t), int(s))) for s, t in res['edges']]
    assert res['n_odometry'] == n - 1 and res['n_loop'] >= len(wrong)
    for k, p in enumerate(edge_pair):
        if p in wrong:
            assert not res['kept'][k], p
    assert all(res['kept'][k] for k, p in enumerate(edge_pair) if p not in wrong)
    assert PG.pose_error(res['poses'], sc['poses']) < 0.02
    assert np.array_equal(res['poses'][0], np.eye(4))
    # gt.log / gt.info from the truth, est.log from the optimised poses: every pair is recalled
    M.write_outputs(res, str(tmp_path / 'est'), 'synthetic-scene')
    gt = tmp_path / 'gt' / 'synthetic-scene'
    gt.mkdir(parents=True)
    with open(gt / 'gt.log', 'w') as fh, open(gt / 'gt.info', 'w') as fi:
        for i, j in pairs:
            fh.write(f'{i}\t{j}\t{n}\n')
            fh.write(''.join('\t'.join(f'{v:.12f}' for v in row) + '\n' for row in M.relative_pose(sc['poses'], i, j)))
            info = PG.info_of_points(np.asarray(sc['fragments'][j], np.float64)[::50]) / 100.0 + np.eye(6)
            fi.write(f'{i}\t{j}\t{n}\n')
            fi.write(''.join(' '.join(f'{v:.6f}' for v in row) + '\n' for row in info))
    _, recall, per_scene = E.benchmark_3dmatch(str(tmp_path / 'est'), str(tmp_path / 'gt'))
    assert recall == 1.0 and per_scene['synthetic-scene']['precision'] == 1.0


@pytest.mark.parametrize('extra', [[], ['--icp', '0.05', '--voxel', '0.05']])
def test_multiway_cli_end_to_end(tmp_path, extra):
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': random_state_dict(cfg, 5), 'step': 1}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, '3dmatch', str(run / 'config.yaml'))
    sc = S.make_scene(9, 5, n_target=4000)
    files = []
    for k, f in enumerate(sc['fragments']):
        path = tmp_path / 'frags' / 'my-scene' / f'cloud_bin_{k}.npy'
        path.parent.mkdir(parents=True, exist_ok=True)
        np.save(path, f)
        files.append(str(path))
    out = tmp_path / 'out'
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', 'regtr_b200.multiway'] + files +
                       ['--ckpt', str(run / 'ckpt' / 'model-best.pth'), '--out', str(out), '--batch_pairs', '4'] + extra,
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line['n_fragments'] == 5 and line['pairs'] == 10 and line['edges_odometry'] == 4
    res = np.load(out / 'result.npz')
    assert res['poses'].shape == (5, 4, 4) and np.array_equal(res['poses'][0], np.eye(4))
    assert res['fit'].shape == (10, 4) and res['information'].shape == (len(res['edges']), 6, 6)
    keys, traj = E.read_trajectory(str(out / 'my-scene' / 'est.log'))
    for (i, j), k, T in zip(M.all_pairs(5), keys, traj):
        assert (int(k[0]), int(k[1])) == (i, j)
        assert np.abs(T - M.relative_pose(res['poses'], i, j)).max() < 1e-11
    if '--voxel' in extra:
        pts = PIO.read_ply(str(out / 'scene.ply'))
        pts = pts[0] if isinstance(pts, tuple) else pts
        assert len(pts) > 100
    else:
        assert not (out / 'scene.ply').exists()
