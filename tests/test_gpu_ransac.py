"""RANSAC over correspondences on the device (`ops.ransac`, regtr_ransac) against the float64 oracle
(tests/ransac_oracle.py) on the real 3DMatch fixtures and synthetic pairs: winning hypothesis, hypotheses walked and
validated, inlier count, pose and RMSE; bit identity across chunk schedules, batches and reruns; the edge cases and
both checkers; agreement with `ops.registration_fit`; the launch count; the range check; RANSAC against weighted
Kabsch at 80% outliers; and `register --ransac` / `multiway --ransac` end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import icp_oracle as I
import ransac_oracle as RO
import train_data_oracle as O
from conftest import GOLDEN, ROOT
from regtr_b200 import lib, ops
from regtr_b200 import pointio as P
from regtr_b200.synthetic import make_3dmatch_pair
from test_gpu_register import gt_log_pair

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')
RADIUS = 0.0375


def rigid(rng, deg=30.0):
    axis = rng.normal(size=3)
    T = np.eye(3, 4)
    T[:, :3] = O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))
    T[:, 3] = rng.uniform(-0.5, 0.5, 3)
    return T


def pairs():
    """(name, src, tgt, pose): the two real fixtures with a gt.log pose, the third with the oracle ICP's pose from the
    identity (the fixtures hold no ground truth for it), and two synthetic 3DMatch-shaped pairs."""
    out = []
    for fx, scene in (('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'),
                      ('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3')):
        s, t, p = gt_log_pair(fx, scene)
        out.append((fx, s, t, np.asarray(p, np.float64)))
    inp = np.load(os.path.join(REAL, 'real_3dmatch_sun3d_home_38_41_input.npz'))
    s, t = inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64)
    out.append(('real_3dmatch_sun3d_home_38_41', s, t, I.icp(s, t, np.eye(3, 4), RADIUS, 30)['pose']))
    for seed in (4001, 4002):
        p = make_3dmatch_pair(seed)
        out.append((f'synthetic_{seed}', p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64),
                    np.asarray(p['pose'], np.float64)))
    return out


PAIRS = None


def get_pairs():
    global PAIRS
    if PAIRS is None:
        PAIRS = pairs()
    return PAIRS


def correspondences(src, tgt, pose, m, outliers, seed, noise=0.005):
    """m correspondences from the pose plus noise; a share `outliers` of them end at a random target point."""
    rng = np.random.default_rng(seed)
    a = src[rng.integers(0, len(src), m)]
    c = I.transform(pose, a) + rng.normal(scale=noise / np.sqrt(3.0), size=(m, 3))
    bad = rng.random(m) < outliers
    c[bad] = tgt[rng.integers(0, len(tgt), int(bad.sum()))]
    return a, c


def device(src_list, tgt_list, cs, ct, **kw):
    pose, res = ops.ransac(src_list, tgt_list, cs, ct, kw.pop('r', RADIUS), **kw)
    return pose.cpu().numpy(), res.cpu().numpy()


def check_against_oracle(pose, res, o, src, tgt):
    assert int(res[4]) == o['best'] and int(res[2]) == o['iterations'] and int(res[3]) == o['validations'], \
        (res, o['best'], o['iterations'], o['validations'])
    assert round(res[0] * len(src)) == round(o['fitness'] * len(src))               # the same inlier count
    assert np.abs(pose - o['pose']).max() <= 1e-9, np.abs(pose - o['pose']).max()
    assert abs(res[1] - o['rmse']) <= 1e-9, (res[1], o['rmse'])


@pytest.mark.parametrize('outliers', [0.5, 0.2, 0.05])
def test_against_the_oracle(outliers):
    """Every 4th point of each cloud validates, so that the oracle's hundreds of validations stay affordable."""
    for k, (name, s, t, p) in enumerate(get_pairs()):
        s, t = s[::4], t[::4]
        a, c = correspondences(s, t, p, 300, outliers, 10 + k)
        pose, res = device([s], [t], [a], [c], seed=11)
        o = RO.ransac(s, t, a, c, RADIUS, seed=11, pair=0)
        check_against_oracle(pose[0], res[0], o, s, t)
        assert o['validations'] >= 1 and o['fitness'] > 0.05, (name, o['fitness'])


def synthetic_corr(seed, m, outliers, n_pts=6000):
    p = make_3dmatch_pair(seed, n_target=n_pts)
    s, t, pose = p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), np.asarray(p['pose'], np.float64)
    a, c = correspondences(s, t, pose, m, outliers, seed)
    return s, t, a, c, pose


def test_schedule_independence():
    """first_chunk 1, 7, 256 and 4096 give the same bits, with an early stop and with every hypothesis walked."""
    s, t, a, c, _ = synthetic_corr(5001, 400, 0.5)
    for kw in (dict(max_iteration=100000), dict(max_iteration=3000, confidence=1.0),
               dict(max_iteration=2000, confidence=1.0, edge_length=None)):
        outs = [device([s], [t], [a], [c], first_chunk=fc, seed=3, **kw) for fc in (1, 7, 256, 4096)]
        for pose, res in outs[1:]:
            assert np.array_equal(pose, outs[0][0]) and np.array_equal(res, outs[0][1]), (kw, res, outs[0][1])
    assert int(outs[0][1][0, 2]) == 2000


def test_batch_independence():
    """Five pairs with unequal m and some masks in one call equal each pair alone with the matching pair_base."""
    items = []
    for k, (m, outl) in enumerate(((300, 0.5), (50, 0.2), (700, 0.6), (3, 0.0), (200, 0.3))):
        s, t, a, c, _ = synthetic_corr(5100 + k, m, outl, n_pts=3000 + 1000 * k)
        mask = np.random.default_rng(k).random(m) < (0.8 if k % 2 else 1.1)
        items.append((s, t, a, c, mask))
    cols = list(zip(*items))
    pose, res = device(list(cols[0]), list(cols[1]), list(cols[2]), list(cols[3]), corr_mask=list(cols[4]),
                       seed=21, pair_base=4, first_chunk=64)
    for b, (s, t, a, c, mask) in enumerate(items):
        p1, r1 = device([s], [t], [a], [c], corr_mask=[mask], seed=21, pair_base=4 + b, first_chunk=256)
        assert np.array_equal(p1[0], pose[b]) and np.array_equal(r1[0], res[b]), (b, r1, res[b])
        o = RO.ransac(s, t, a, c, RADIUS, mask=mask, seed=21, pair=4 + b)
        check_against_oracle(pose[b], res[b], o, s, t)


def test_edge_cases():
    s, t, a, c, _ = synthetic_corr(5201, 100, 0.3)
    empty = np.concatenate([np.eye(3, 4)[None]])
    for kw in (dict(corr_mask=[np.zeros(100, bool)]), dict(max_iteration=0), dict(ransac_n=2), dict(r=0.0)):
        pose, res = device([s], [t], [a], [c], **kw)
        assert np.array_equal(pose, empty) and np.array_equal(res[0], [0, 0, 0, 0, -1]), kw
    mask = np.zeros(100, bool)
    mask[[5, 60]] = True                                           # two valid correspondences < ransac_n
    pose, res = device([s], [t], [a], [c], corr_mask=[mask])
    assert np.array_equal(pose, empty) and np.array_equal(res[0], [0, 0, 0, 0, -1])
    mask[70] = True                                                # exactly ransac_n
    pose, res = device([s], [t], [a], [c], corr_mask=[mask], max_iteration=50)
    check_against_oracle(pose[0], res[0], RO.ransac(s, t, a, c, RADIUS, 50, mask=mask), s, t)
    pose, res = device([s], [t], [a[:0]], [c[:0]])
    assert np.array_equal(res[0], [0, 0, 0, 0, -1])


def test_clean_correspondences_stop_after_the_first_valid_hypothesis():
    rng = np.random.default_rng(7)
    T = rigid(rng)
    src = rng.uniform(-1.0, 1.0, (5000, 3))
    tgt = I.transform(T, src)
    a = src[:200]
    c = tgt[:200]
    pose, res = device([src], [tgt], [a], [c], seed=5)
    first = next(k for k in range(1000) if RO.hypothesis(a, c, RO.draws(5, 0, [k], 200, 3)[0], 0.9)[0])
    assert res[0, 0] == 1.0 and int(res[0, 4]) == first and int(res[0, 2]) == first + 1 and int(res[0, 3]) == 1
    assert np.abs(pose[0] - T).max() < 1e-9


@pytest.mark.parametrize('edge, dist', [(None, None), (0.9, None), (None, 0.02), (0.95, 0.01), (0.5, 0.1)])
def test_checkers_on_and_off(edge, dist):
    s, t, a, c, _ = synthetic_corr(5301, 300, 0.6)
    pose, res = device([s], [t], [a], [c], edge_length=edge, distance=dist, seed=2, max_iteration=20000)
    o = RO.ransac(s, t, a, c, RADIUS, 20000, edge_length=edge, distance=dist, seed=2)
    check_against_oracle(pose[0], res[0], o, s, t)


def lattice_case():
    """A source patch of a planar lattice inside a larger target lattice: every in-plane motion of the patch matches
    all its points.  90% of the correspondences follow c = a / 2 + (0.3, 0.3, 0), not a rigid motion, so a sample of
    them gives an in-plane pose with fitness 1 that stops RANSAC at once, unless the edge-length checker rejects it."""
    g = np.arange(0, 1.0001, 0.02)
    src = np.array([[x, y, 0.0] for x in g for y in g])
    G = np.arange(-1.0, 2.0001, 0.02)
    tgt = np.array([[x, y, 0.0] for x in G for y in G])
    rng = np.random.default_rng(0)
    a = src[rng.integers(0, len(src), 200)]
    c = a.copy()
    wrong = rng.random(200) < 0.9
    c[wrong] = 0.5 * a[wrong] + np.array([0.3, 0.3, 0.0])
    return src, tgt, a, c


def test_only_the_edge_checker_keeps_ransac_off_a_wrong_sample():
    src, tgt, a, c = lattice_case()
    for edge in (None, 0.9):
        pose, res = device([src], [tgt], [a], [c], r=0.03, max_iteration=1000, edge_length=edge)
        o = RO.ransac(src, tgt, a, c, 0.03, 1000, edge_length=edge)
        check_against_oracle(pose[0], res[0], o, src, tgt)
        assert res[0, 0] == 1.0
        err = np.abs(pose[0] - np.eye(3, 4)).max()
        assert (err > 0.02) if edge is None else (err < 1e-9), (edge, err)


def test_registration_fit_launches_rerun_and_range():
    s, t, a, c, _ = synthetic_corr(5401, 300, 0.5, n_pts=20000)
    small = s[:900]
    for src in (s, small):
        before = ops.LAUNCHES
        pose, res = ops.ransac([src], [t], [a], [c], RADIUS, seed=8, first_chunk=32)
        assert ops.LAUNCHES - before == ops.ransac_launches(100000, 32)
        fit = ops.registration_fit([src], [t], pose, RADIUS).cpu().numpy()[0]
        res = res.cpu().numpy()[0]
        assert res[0] == fit[0]
        if len(src) <= 1024:
            assert res[1] == fit[1]                                # one block: regtr_registration_fit's order
        else:
            assert abs(res[1] - fit[1]) <= 1e-12 * fit[1]
        p2, r2 = ops.ransac([src], [t], [a], [c], RADIUS, seed=8, first_chunk=32)
        assert torch.equal(p2, pose) and np.array_equal(r2.cpu().numpy()[0], res)
    far = t.copy()
    far[0] = [1e9, 0.0, 0.0]
    with pytest.raises(lib.RegtrLibError):
        ops.ransac([s], [far], [a], [c], RADIUS)
    status = ops.new_status(torch.device('cuda'))
    ops.ransac([s], [far], [a], [c], RADIUS, status=status)
    assert int(status.item()) & ops.STATUS_RANGE


def test_ransac_beats_weighted_kabsch_at_80_percent_outliers():
    s, t, a, c, gt = synthetic_corr(5501, 500, 0.8, n_pts=20000)
    w = torch.ones(len(a), dtype=torch.float32, device='cuda')
    kb = ops.kabsch(torch.from_numpy(a).float().cuda(), torch.from_numpy(c).float().cuda(), w,
                    torch.tensor([0, len(a)], dtype=torch.int32, device='cuda')).cpu().numpy()[0].astype(np.float64)
    pose, res = device([s], [t], [a], [c], seed=1)

    def errors(p):
        cos = (np.trace(p[:, :3].T @ gt[:, :3]) - 1.0) / 2.0
        return np.degrees(np.arccos(np.clip(cos, -1, 1))), np.linalg.norm(p[:, 3] - gt[:, 3])
    assert errors(kb)[0] > 10.0, errors(kb)
    rot, trans = errors(pose[0])
    assert rot < 1.0 and trans < 0.05, (rot, trans, res)


def _checkpoint(tmp_path, name, seed):
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config(name)
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': random_state_dict(cfg, seed), 'step': 1}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, name, str(run / 'config.yaml'))
    return cfg, str(run / 'ckpt' / 'model-best.pth')


@pytest.mark.parametrize('extra', [[], ['--icp', '0.05']])
def test_register_cli_with_ransac_end_to_end(tmp_path, extra):
    cfg, ckpt = _checkpoint(tmp_path, 'modelnet', 41)
    src_file = os.path.join(REAL, 'modelnet_test_2_0.ply')
    tgt_file = os.path.join(REAL, 'modelnet_test_2_1.ply')
    out_dir = tmp_path / 'out'
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', 'regtr_b200.register', src_file, tgt_file, '--ckpt', ckpt,
                        '--out', str(out_dir), '--ransac', '0.05', '--ransac_overlap', '0.3', '--ransac_iters',
                        '20000'] + extra, capture_output=True, text=True, cwd=ROOT, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    res = np.load(str(out_dir / 'result.npz'))
    s, t = P.load_point_cloud(src_file), P.load_point_cloud(tgt_file)
    m = np.concatenate([res['src_overlap'], res['tgt_overlap']]) > 0.3
    cs = np.concatenate([res['src_kp'], res['tgt_kp_warped']])
    ct = np.concatenate([res['src_kp_warped'], res['tgt_kp']])
    pose, rs = ops.ransac([s], [t], [cs], [ct], 0.05, 20000, corr_mask=[m])
    assert np.array_equal(res['pose_ransac'], pose[0].cpu().numpy())
    assert np.array_equal(res['ransac'], rs[0].cpu().numpy())
    assert np.array_equal(res['pose_coarse'], res['pose'][-1])
    assert line['ransac_iterations'] == int(rs[0, 2]) and line['ransac_radius'] == 0.05
    final = res['pose_icp'] if extra else res['pose_ransac']
    assert np.array_equal(np.array(line['pose']), np.vstack([final, [0, 0, 0, 1]]))
    if extra:
        want, _ = ops.icp([s], [t], pose, 0.05, 30)
        assert np.array_equal(res['pose_icp'], want[0].cpu().numpy())


def test_multiway_cli_with_ransac_end_to_end(tmp_path):
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
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', 'regtr_b200.multiway'] + files +
                       ['--ckpt', ckpt, '--out', str(out), '--batch_pairs', '4', '--ransac', '0.05',
                        '--ransac_iters', '5000', '--icp', '0.05'],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line['n_fragments'] == 4 and line['pairs'] == 6
    assert np.load(out / 'result.npz')['poses'].shape == (4, 4, 4)
