"""Fast Global Registration on the device (`ops.fgr`, `ops.fgr_feature_matching`, `eval.fpfh_register(method='fgr')`,
`eval.fgr_forward`) against the float64 restatement (tests/fgr_oracle.py) on the real 3DMatch fixtures' FPFH matches
and on synthetic correspondences, its determinism alone and in a batch, its launch count, its accuracy against known
and gt.log poses, and the `register`, `multiway` and `eval_3dmatch.py` --fgr paths end to end."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import fgr_oracle as G
from conftest import GOLDEN, ROOT
from regtr_b200 import eval as E
from regtr_b200 import ops
from regtr_b200 import pointio as P
from regtr_b200.synthetic import make_3dmatch_pair
from test_gpu_fpfh import GT_PAIRS, V, device_features, errors, fixture_clouds
from test_gpu_ransac import _checkpoint, correspondences, rigid
from test_gpu_register import gt_log_pair

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')

FEATURES = None


def fixture_features():
    """(name, src_down, tgt_down, src_feat, tgt_feat, gt pose or None) of the three fixtures at V, host float64."""
    global FEATURES
    if FEATURES is None:
        FEATURES = []
        for name, s, t, g in fixture_clouds():
            xyz, _, feat, _ = device_features([s, t], V)
            FEATURES.append((name, xyz[0], xyz[1], feat[0], feat[1], g))
    return FEATURES


def check_against_oracle(pose, res, o):
    assert (int(res[0]), int(res[1]), int(res[2])) == (o['n_corr'], o['tuples'], o['trials']), (res, o['n_corr'],
                                                                                                o['tuples'], o['trials'])
    assert abs(res[3] - o['par']) <= 1e-15 * max(1.0, o['par']), (res[3], o['par'])
    assert np.abs(pose - o['pose']).max() <= 1e-9, np.abs(pose - o['pose']).max()


OPTIONS = [dict(), dict(tuple_test=False), dict(use_absolute_scale=True), dict(decrease_mu=False),
           dict(maximum_tuple_count=200, seed=5)]


@pytest.mark.parametrize('kw', OPTIONS, ids=['default', 'no_tuple_test', 'absolute_scale', 'fixed_mu', 'cap_200'])
def test_feature_matching_against_the_oracle_on_the_real_fixtures(kw):
    for name, s, t, fs, ft, _ in fixture_features():
        kw = dict(kw, maximum_correspondence_distance=0.5 * V)
        pose, res, n_mut = ops.fgr_feature_matching([s], [t], [fs], [ft], **kw)
        o, m = G.fgr_feature_matching(s, t, fs, ft, **kw)
        assert int(n_mut[0]) == m['n_mutual']
        check_against_oracle(pose.cpu().numpy()[0], res.cpu().numpy()[0], o)
        if kw.get('tuple_test', True):
            assert o['n_corr'] == 3 * o['tuples'] >= 30 and o['trials'] > 0, (name, o['tuples'], o['trials'])
            if o['tuples'] < kw.get('maximum_tuple_count', 1000):
                assert o['trials'] == 100 * m['n_mutual']


def synthetic_pairs():
    """(name, src, tgt, pose): two real fixtures with their gt.log pose and two synthetic 3DMatch-shaped pairs."""
    out = []
    for fx, scene, _ in GT_PAIRS:
        s, t, p = gt_log_pair(fx, scene)
        out.append((fx, s, t, np.asarray(p, np.float64)))
    for seed in (4001, 4002):
        p = make_3dmatch_pair(seed)
        out.append((f'synthetic_{seed}', p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64),
                    np.asarray(p['pose'], np.float64)))
    return out


@pytest.mark.parametrize('outliers', [0.5, 0.2, 0.05])
def test_correspondences_against_the_oracle(outliers):
    for k, (name, s, t, p) in enumerate(synthetic_pairs()):
        a, c = correspondences(s, t, p, 1500, outliers, 20 + k)
        mask = np.random.default_rng(k).random(len(a)) < 0.9
        for kw in (dict(), dict(tuple_test=True, seed=7)):
            pose, res = ops.fgr([s], [t], [a], [c], [mask], **kw)
            o = G.fgr(s, t, a, c, mask, **kw)
            check_against_oracle(pose.cpu().numpy()[0], res.cpu().numpy()[0], o)
        rot, trans = errors(pose.cpu().numpy()[0], p)
        print(name, outliers, 'fgr', rot, trans)
        if outliers <= 0.2:
            assert rot < 5.0 and trans < 0.1, (name, outliers, rot, trans)


def test_edge_cases_on_the_device():
    s, t = np.random.default_rng(1).random((500, 3)), np.random.default_rng(2).random((400, 3))
    a, c = s[:30], t[:30]
    pose, res = ops.fgr([s], [t], [a[:9]], [c[:9]])
    assert np.array_equal(pose.cpu().numpy()[0], np.eye(3, 4)) and res.cpu().numpy()[0].tolist() == [9, 0, 0, 1.0]
    pose, res = ops.fgr([s], [t], [a[:0]], [c[:0]], tuple_test=True)
    assert np.array_equal(pose.cpu().numpy()[0], np.eye(3, 4)) and res.cpu().numpy()[0].tolist() == [0, 0, 0, 1.0]
    for kw in (dict(tuple_test=True, tuple_scale=1.0), dict(tuple_test=True, maximum_tuple_count=3, tuple_scale=0.5),
               dict(iteration_number=0), dict(use_absolute_scale=True, tuple_test=True)):
        pose, res = ops.fgr([s], [t], [a], [c], **kw)
        check_against_oracle(pose.cpu().numpy()[0], res.cpu().numpy()[0], G.fgr(s, t, a, c, **kw))
    before = ops.LAUNCHES
    ops.fgr([s], [t], [a], [c])
    assert ops.LAUNCHES - before == ops.fgr_launches() == 2


def test_bit_identity_alone_in_a_batch_and_across_pair_base_splits():
    pairs = synthetic_pairs()
    cs, ct = [], []
    for k, (name, s, t, p) in enumerate(pairs):
        a, c = correspondences(s, t, p, 1200, 0.4, 40 + k)
        cs.append(a)
        ct.append(c)
    src, tgt = [x[1] for x in pairs], [x[2] for x in pairs]
    kw = dict(tuple_test=True, seed=(1 << 40) + 3)
    pose, res = ops.fgr(src, tgt, cs, ct, pair_base=10, **kw)
    for b in range(len(pairs)):
        pb, rb = ops.fgr([src[b]], [tgt[b]], [cs[b]], [ct[b]], pair_base=10 + b, **kw)
        assert torch.equal(pb[0], pose[b]) and torch.equal(rb[0], res[b])
    p2, r2 = ops.fgr(src[2:], tgt[2:], cs[2:], ct[2:], pair_base=12, **kw)
    assert torch.equal(p2, pose[2:]) and torch.equal(r2, res[2:])
    p3, r3 = ops.fgr(src[:1], tgt[:1], cs[:1], ct[:1], pair_base=11, **kw)    # another global pair: other draws
    assert int(r3[0, 2]) != int(res[0, 2]) or not torch.equal(p3[0], pose[0])
    o = G.fgr(src[1], tgt[1], cs[1], ct[1], pair=11, **kw)
    check_against_oracle(pose.cpu().numpy()[1], res.cpu().numpy()[1], o)


def crop_pair(seed):
    """A real fixture cloud, rigidly moved, both sides cropped to about 70 % overlap and given 1 cm noise."""
    rng = np.random.default_rng(seed)
    _, s, _, _ = fixture_clouds()[0]
    T = rigid(rng, 45.0)
    axis = np.argmax(np.ptp(s, 0))
    lo, hi = np.quantile(s[:, axis], [0.3, 0.7])
    src = s[s[:, axis] < hi]
    tgt = s[s[:, axis] > lo] @ T[:, :3].T + T[:, 3]
    src = src + rng.normal(scale=0.01 / np.sqrt(3.0), size=src.shape)
    tgt = tgt + rng.normal(scale=0.01 / np.sqrt(3.0), size=tgt.shape)
    return src, tgt, T


def test_known_pose_through_fpfh_matches():
    for seed in (1, 2):
        s, t, T = crop_pair(seed)
        out = E.fpfh_register([s], [t], V, method='fgr')
        rot, trans = errors(out['pose_fpfh'].cpu().numpy()[0], T)
        print('cropped', seed, rot, trans, out['fgr'].cpu().numpy()[0], int(out['n_mutual'][0]))
        assert rot < 2.0 and trans < 0.05, (seed, rot, trans)


def test_accuracy_against_the_ground_truth():
    """FGR, and ICP at 0.05 after it, on the gt.log pairs against benchmark_dgr's thresholds (15 degrees, 0.3 m)."""
    for fx, scene, _ in GT_PAIRS:
        s, t, g = gt_log_pair(fx, scene)
        g = np.asarray(g, np.float64)
        out = E.fpfh_register([s], [t], V, method='fgr', icp_radius=0.05)
        rot, trans = errors(out['pose_fpfh'].cpu().numpy()[0], g)
        rot_i, trans_i = errors(out['pose'].cpu().numpy()[0], g)
        print(fx, 'fgr', rot, trans, out['fgr'].cpu().numpy()[0], int(out['n_mutual'][0]), 'icp', rot_i, trans_i)
        assert rot < 15.0 and trans < 0.3, (fx, rot, trans)
        assert rot_i < 15.0 and trans_i < 0.3, (fx, rot_i, trans_i)


def run_cli(args, timeout=900):
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable] + args, capture_output=True, text=True, cwd=ROOT, env=env, timeout=timeout)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_register_cli_with_fpfh_and_fgr_end_to_end(tmp_path):
    fx, scene, _ = GT_PAIRS[0]
    s, t, _ = gt_log_pair(fx, scene)
    np.save(tmp_path / 's.npy', s)
    np.save(tmp_path / 't.npy', t)
    out_dir = tmp_path / 'out'
    line = run_cli(['-m', 'regtr_b200.register', str(tmp_path / 's.npy'), str(tmp_path / 't.npy'), '--fpfh', str(V),
                    '--fgr', '--icp', '0.05', '--out', str(out_dir)])
    for k in ('fpfh_voxel', 'n_mutual', 'fgr_correspondences', 'fgr_tuples', 'fgr_trials', 'fgr_par', 'fgr_dist',
              'icp_fitness', 'pose'):
        assert k in line, k
    assert not any(k.startswith('ransac') for k in line)
    assert sorted(os.listdir(out_dir)) == ['pose.txt', 'result.npz', 'src_registered.ply']
    res = np.load(out_dir / 'result.npz')
    assert set(res.files) == {'pose_fpfh', 'fgr', 'n_mutual', 'fit', 'pose_icp', 'icp'}
    want = E.fpfh_register([s], [t], V, method='fgr', icp_radius=0.05)
    assert np.array_equal(res['pose_fpfh'], want['pose_fpfh'][0].cpu().numpy())
    assert np.array_equal(res['fgr'], want['fgr'][0].cpu().numpy())
    assert np.array_equal(res['pose_icp'], want['pose'][0].cpu().numpy())
    assert line['fgr_dist'] == 0.5 * V and line['fit_radius'] == 1.5 * V and line['fgr_tuples'] == int(res['fgr'][1])


@pytest.mark.parametrize('extra', [[], ['--icp', '0.05']])
def test_register_cli_with_a_checkpoint_and_fgr_end_to_end(tmp_path, extra):
    cfg, ckpt = _checkpoint(tmp_path, 'modelnet', 41)
    src_file = os.path.join(REAL, 'modelnet_test_2_0.ply')
    tgt_file = os.path.join(REAL, 'modelnet_test_2_1.ply')
    out_dir = tmp_path / 'out'
    line = run_cli(['-m', 'regtr_b200.register', src_file, tgt_file, '--ckpt', ckpt, '--out', str(out_dir), '--fgr',
                    '--fgr_overlap', '0.3', '--fgr_tuple_test', '--fgr_max_tuples', '100'] + extra)
    res = np.load(str(out_dir / 'result.npz'))
    s, t = P.load_point_cloud(src_file), P.load_point_cloud(tgt_file)
    m = np.concatenate([res['src_overlap'], res['tgt_overlap']]) > 0.3
    cs = np.concatenate([res['src_kp'], res['tgt_kp_warped']])
    ct = np.concatenate([res['src_kp_warped'], res['tgt_kp']])
    pose, rs = ops.fgr([s], [t], [cs], [ct], [m], tuple_test=True, maximum_tuple_count=100)
    assert np.array_equal(res['pose_fgr'], pose[0].cpu().numpy())
    assert np.array_equal(res['fgr'], rs[0].cpu().numpy())
    assert np.array_equal(res['pose_coarse'], res['pose'][-1])
    assert line['fgr_correspondences'] == int(rs[0, 0]) and line['fgr_dist'] == 0.025
    final = res['pose_icp'] if extra else res['pose_fgr']
    assert np.array_equal(np.array(line['pose']), np.vstack([final, [0, 0, 0, 1]]))
    if extra:
        want, _ = ops.icp([s], [t], pose, 0.05, 30)
        assert np.array_equal(res['pose_icp'], want[0].cpu().numpy())


def test_multiway_cli_with_fgr_end_to_end(tmp_path):
    from regtr_b200 import synthetic as S
    _, ckpt = _checkpoint(tmp_path, '3dmatch', 5)
    sc = S.make_scene(9, 4, n_target=4000)
    files = []
    for k, f in enumerate(sc['fragments']):
        path = tmp_path / 'frags' / 'my-scene' / f'cloud_bin_{k}.npy'
        path.parent.mkdir(parents=True, exist_ok=True)
        np.save(path, f)
        files.append(str(path))
    out = tmp_path / 'out'
    line = run_cli(['-m', 'regtr_b200.multiway'] + files + ['--ckpt', ckpt, '--out', str(out), '--batch_pairs', '4',
                                                            '--fgr', '--icp', '0.05'], timeout=1800)
    assert line['n_fragments'] == 4 and line['pairs'] == 6
    assert np.load(out / 'result.npz')['poses'].shape == (4, 4, 4)


def test_fpfh_fgr_forward_through_the_3dmatch_benchmark(tmp_path):
    from regtr_b200 import data as D
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import eval_3dmatch
    finally:
        sys.path.pop(0)
    rows = json.load(open(os.path.join(REAL, 'test_3DMatch_info_rows.json')))
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    for r in rows:
        inp = np.load(os.path.join(REAL, r['fixture'] + '_input.npz'))
        for rel in (r['src'], r['tgt']):
            which = 'src_xyz' if os.path.basename(rel) == os.path.basename(str(inp['src_file'])) else 'tgt_xyz'
            path = tmp_path / 'indoor' / rel
            os.makedirs(path.parent, exist_ok=True)
            torch.save(inp[which].astype(np.float64), path)
        infos['rot'].append(np.array(r['rot'])); infos['trans'].append(np.array(r['trans']))
        infos['src'].append(r['src']); infos['tgt'].append(r['tgt']); infos['overlap'].append(r['overlap'])
    with open(tmp_path / 'info.pkl', 'wb') as f:
        pickle.dump(infos, f)
    gt_dir = os.path.join(REAL, 'benchmarks', '3DMatch')
    ap = eval_3dmatch.parser()
    args = ap.parse_args(['--root', str(tmp_path / 'indoor'), '--info', str(tmp_path / 'info.pkl'), '--gt', gt_dir,
                          '--fpfh', str(V), '--fgr', '--out', str(tmp_path / 'log')])
    E.check_fgr_arguments(ap, args)
    E.check_fpfh_arguments(ap, args)
    kw = E.fpfh_kwargs(args)
    assert kw['method'] == 'fgr' and args.ransac is None
    ds = D.ThreeDMatchPairs(str(tmp_path / 'indoor'), str(tmp_path / 'info.pkl'), pin=True)
    res = E.run_3dmatch_benchmark(D.PairStream(ds, [[0], [1]], workers=2), E.fpfh_forward(V, **kw),
                                  str(tmp_path / 'log'), '3DMatch', gt_dir)
    assert 'Mean median RRE' in res['summary']
    for r in rows:
        scene = r['src'].split('/')[1]
        pairs, traj = E.read_trajectory(os.path.join(str(tmp_path / 'log'), '3DMatch', scene, 'est.log'))
        assert len(pairs) == 1 and traj.shape == (1, 4, 4) and np.isfinite(traj).all()
        R = traj[0, :3, :3]
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-9
    eval_3dmatch.main(['--root', str(tmp_path / 'indoor'), '--info', str(tmp_path / 'info.pkl'), '--gt', gt_dir,
                       '--fpfh', str(V), '--fgr', '--out', str(tmp_path / 'log2'), '--workers', '1'])
    for r in rows:
        scene = r['src'].split('/')[1]
        a = E.read_trajectory(os.path.join(str(tmp_path / 'log'), '3DMatch', scene, 'est.log'))[1]
        b = E.read_trajectory(os.path.join(str(tmp_path / 'log2'), '3DMatch', scene, 'est.log'))[1]
        assert np.array_equal(a, b)
