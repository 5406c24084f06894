"""FPFH features, feature matching and RANSAC over feature matches on the device (`ops.fpfh`, `ops.feature_match`,
`ops.ransac_feature_matching`, `eval.fpfh_register`) against the float64 restatement (tests/fpfh_oracle.py) on the real
3DMatch fixtures and synthetic features, their determinism, launch counts and range status, their accuracy against
the fixtures' gt.log poses, and the `register --fpfh` and `eval_3dmatch.py --fpfh` paths end to end."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import fpfh_oracle as FO
import ransac_oracle as RO
from conftest import GOLDEN, ROOT
from regtr_b200 import eval as E
from regtr_b200 import lib, ops
from test_gpu_register import gt_log_pair

pytestmark = pytest.mark.gpu

REAL = os.path.join(GOLDEN, 'real')
V = 0.05
GT_PAIRS = (('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen', (100000, 0.999)),
            ('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3', (20000, 1.0)))


def fixture_clouds():
    """(name, src, tgt, gt pose or None) of the three real 3DMatch fixtures."""
    out = [(fx, *gt_log_pair(fx, scene)) for fx, scene, _ in GT_PAIRS]
    inp = np.load(os.path.join(REAL, 'real_3dmatch_sun3d_home_38_41_input.npz'))
    out.append(('real_3dmatch_sun3d_home_38_41', inp['src_xyz'].astype(np.float64),
                inp['tgt_xyz'].astype(np.float64), None))
    return out


def device_features(clouds, voxel=None, radius=5 * V, max_nn=100):
    """Downsampled (voxel) or full clouds -> (clouds, normals, features, counts) as host float64 arrays."""
    clouds = E.fpfh_downsample(clouds, voxel) if voxel else [torch.as_tensor(c) for c in clouds]
    nr = 2 * (voxel or 0.025)
    normals = ops.estimate_normals(clouds, nr, 30)
    feats, counts = ops.fpfh(clouds, normals, radius, max_nn, return_counts=True)
    host = lambda ts: [t.cpu().numpy().astype(np.float64) for t in ts]
    return host(clouds), host(normals), host(feats), [c.cpu().numpy() for c in counts]


def check_features(xyz, nrm, feat, cnt, radius, max_nn=100):
    o = FO.fpfh(xyz, nrm, radius, max_nn)
    assert np.array_equal(cnt, o['counts'])
    err = np.abs(feat - o['feature'])
    flipped = int((err.max(1) > 1e-6).sum())             # a different bin decision moves a row by far more
    assert flipped == 0 and err.max() <= 1e-9, (flipped, err.max())


@pytest.mark.parametrize('voxel', [V, None])
def test_fpfh_against_the_oracle_on_the_real_fixtures(voxel):
    for name, s, t, _ in fixture_clouds():
        xyz, nrm, feat, cnt = device_features([s, t], voxel, 5 * (voxel or 0.025))
        for k in range(2):
            check_features(xyz[k], nrm[k], feat[k], cnt[k], 5 * (voxel or 0.025))
        if voxel:
            assert cnt[0].mean() > 50, (name, cnt[0].mean())           # the hybrid search is nearly saturated


def check_match(fs, ft, mutual_filter=True, min_mutual=9):
    tgt = np.random.default_rng(0).normal(size=(len(ft), 3))
    nn, corr, mask, n_mut = ops.feature_match([fs], [ft], [tgt], mutual_filter, min_mutual)
    o = FO.feature_match(fs, ft, mutual_filter, min_mutual)
    assert np.array_equal(nn[0].cpu().numpy(), o['nn'])
    assert np.array_equal(mask[0].cpu().numpy(), o['mask'])
    assert int(n_mut[0]) == o['n_mutual']
    assert np.array_equal(corr[0].cpu().numpy(), tgt[o['nn']])
    return o


def test_feature_matching_against_the_oracle_on_the_real_fixtures():
    for name, s, t, _ in fixture_clouds():
        _, _, feat, _ = device_features([s, t], V)
        o = check_match(feat[0], feat[1])
        assert o['n_mutual'] > 300, (name, o['n_mutual'])


def test_feature_matching_with_planted_ties():
    rng = np.random.default_rng(7)
    ft = rng.integers(0, 3, size=(700, 33)).astype(np.float64)
    ft[100:110] = 0.0                                          # isolated points' all-zero features
    ft[300:340] = ft[200:240]                                  # exact duplicates: the lower index wins
    fs = ft[rng.integers(0, 700, 900)].copy()
    fs[:20] = 0.0
    fs[500:] = rng.integers(0, 3, size=(400, 33))
    for mutual in (True, False):
        o = check_match(fs, ft, mutual)
        assert (o['nn'] < 300).sum() > 0 and not np.isin(o['nn'], np.arange(101, 110)).any()
    o = check_match(fs, ft, True, min_mutual=10 ** 6)          # Open3D's fallback: every match
    assert o['mask'].all()
    big = rng.normal(size=(1500, 33))                          # several row blocks and column chunks
    check_match(big[:1300] + 1e-3 * rng.normal(size=(1300, 33)), big)


def test_ransac_feature_matching_against_the_oracle():
    for (fx, scene, _), (name, s, t, _) in zip(GT_PAIRS, fixture_clouds()):
        xyz, _, feat, _ = device_features([s, t], V)
        kw = dict(max_iteration=100000, confidence=0.999, edge_length=0.9, distance=1.5 * V, seed=0)
        pose, res, n_mut = ops.ransac_feature_matching([xyz[0]], [xyz[1]], [feat[0]], [feat[1]], True, 1.5 * V, **kw)
        o, m = FO.ransac_feature_matching(xyz[0], xyz[1], feat[0], feat[1], True, 1.5 * V, **kw)
        res = res.cpu().numpy()[0]
        assert int(n_mut[0]) == m['n_mutual']
        assert int(res[4]) == o['best'] and int(res[2]) == o['iterations'] and int(res[3]) == o['validations']
        assert round(res[0] * len(xyz[0])) == round(o['fitness'] * len(xyz[0]))
        assert np.abs(pose.cpu().numpy()[0] - o['pose']).max() <= 1e-9 and abs(res[1] - o['rmse']) <= 1e-9


def test_determinism_alone_and_in_a_batch():
    fx = fixture_clouds()
    clouds = [c for _, s, t, _ in fx for c in (s, t)]
    down = [d.cpu() for d in E.fpfh_downsample(clouds, V)]
    normals = ops.estimate_normals(down, 2 * V, 30)
    stacked = ops.fpfh(down, normals, 5 * V)
    for k in (0, 3, 5):
        alone = ops.fpfh([down[k]], [normals[k]], 5 * V)[0]
        assert torch.equal(alone, stacked[k])
    fs, ft, tx = stacked[0::2], stacked[1::2], down[1::2]
    batch = ops.feature_match(fs, ft, tx)
    for b in range(3):
        one = ops.feature_match([fs[b]], [ft[b]], [tx[b]])
        for a, c in zip(one[:3], batch[:3]):
            assert torch.equal(a[0], c[b])
        assert int(one[3][0]) == int(batch[3][b])


def test_launch_counts_and_range_status():
    s = np.random.default_rng(3).random((3000, 3))
    n = ops.estimate_normals([s], 0.1, 30)
    before = ops.LAUNCHES
    f = ops.fpfh([s], n, 0.2)
    assert ops.LAUNCHES - before == ops.fpfh_launches() == 8
    before = ops.LAUNCHES
    ops.feature_match(f, f, [s])
    assert ops.LAUNCHES - before == ops.feature_match_launches() == 3
    far = s.copy()
    far[5] = [1e9, 0.0, 0.0]
    with pytest.raises(lib.RegtrLibError):
        ops.fpfh([far], n, 0.2)
    status = ops.new_status(torch.device('cuda'))
    ops.fpfh([far], n, 0.2, status=status)
    assert int(status.item()) & ops.STATUS_RANGE


def errors(p, g):
    cos = (np.trace(p[:, :3].T @ g[:, :3]) - 1.0) / 2.0
    return np.degrees(np.arccos(np.clip(cos, -1, 1))), np.linalg.norm(p[:, 3] - g[:, 3])


def test_accuracy_against_the_ground_truth():
    """benchmark_dgr's success thresholds (15 degrees, 0.3 m), and ICP after RANSAC is no worse."""
    for (fx, scene, (iters, conf)) in GT_PAIRS:
        s, t, g = gt_log_pair(fx, scene)
        g = np.asarray(g, np.float64)
        out = E.fpfh_register([s], [t], V, max_iteration=iters, confidence=conf, icp_radius=0.05)
        rot, trans = errors(out['pose_fpfh'].cpu().numpy()[0], g)
        print(fx, 'ransac', rot, trans, out['ransac'].cpu().numpy()[0], int(out['n_mutual'][0]))
        assert rot < 15.0 and trans < 0.3, (fx, rot, trans)
        rot_i, trans_i = errors(out['pose'].cpu().numpy()[0], g)
        print(fx, 'icp', rot_i, trans_i)
        assert rot_i <= rot + 0.1 and trans_i <= trans + 0.005, (fx, rot, trans, rot_i, trans_i)


def test_register_cli_with_fpfh_end_to_end(tmp_path):
    fx, scene, _ = GT_PAIRS[0]
    s, t, _ = gt_log_pair(fx, scene)
    np.save(tmp_path / 's.npy', s)
    np.save(tmp_path / 't.npy', t)
    out_dir = tmp_path / 'out'
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', 'regtr_b200.register', str(tmp_path / 's.npy'), str(tmp_path / 't.npy'),
                        '--fpfh', str(V), '--icp', '0.05', '--out', str(out_dir)],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for k in ('fpfh_voxel', 'n_src_down', 'n_tgt_down', 'n_mutual', 'ransac_fitness', 'icp_fitness', 'pose'):
        assert k in line, k
    assert sorted(os.listdir(out_dir)) == ['pose.txt', 'result.npz', 'src_registered.ply']
    res = np.load(out_dir / 'result.npz')
    assert set(res.files) == {'pose_fpfh', 'ransac', 'n_mutual', 'fit', 'pose_icp', 'icp'}
    want = E.fpfh_register([s], [t], V, icp_radius=0.05)
    assert np.array_equal(res['pose_fpfh'], want['pose_fpfh'][0].cpu().numpy())
    assert int(res['n_mutual']) == line['n_mutual'] == int(want['n_mutual'][0])
    assert line['fpfh_voxel'] == V and line['ransac_radius'] == 1.5 * V and line['fit_radius'] == 1.5 * V


def test_fpfh_forward_through_the_3dmatch_benchmark(tmp_path):
    from regtr_b200 import data as D
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
    ds = D.ThreeDMatchPairs(str(tmp_path / 'indoor'), str(tmp_path / 'info.pkl'), pin=True)
    gt_dir = os.path.join(REAL, 'benchmarks', '3DMatch')
    forward = E.fpfh_forward(V, max_iteration=20000, confidence=1.0)
    res = E.run_3dmatch_benchmark(D.PairStream(ds, [[0], [1]], workers=2), forward, str(tmp_path / 'log'),
                                  '3DMatch', gt_dir)
    assert 'Mean median RRE' in res['summary']
    for r in rows:
        scene = r['src'].split('/')[1]
        pairs, traj = E.read_trajectory(os.path.join(str(tmp_path / 'log'), '3DMatch', scene, 'est.log'))
        assert len(pairs) == 1 and traj.shape == (1, 4, 4) and np.isfinite(traj).all()
        assert np.allclose(traj[0, 3], [0, 0, 0, 1])
        R = traj[0, :3, :3]
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-9
