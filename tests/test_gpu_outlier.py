"""Outlier removal on the device (`ops.remove_statistical_outlier`, `ops.remove_radius_outlier`: regtr_statistical_outlier,
regtr_radius_outlier and regtr_select_points) against the float64 oracle (tests/outlier_oracle.py), bit for bit: the
per-point averages and counts, keep flags, per-cloud statistics, packed rows, colours and indices, on the real 3DMatch
fixtures, a 300k-point synthetic scan with 1 % outliers and hand-built cases; the same bits alone or stacked, on a
rerun and for a tiny (brute-force fallback), the default and a huge kNN cell; the range statuses; and `register` (both
paths) and `multiway` with the outlier flags against the same commands on clouds filtered first."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import outlier_oracle as O
from regtr_b200 import lib, ops
from regtr_b200 import pointio as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = os.path.join(ROOT, 'tests', 'golden', 'real')
FIXTURES = ['real_3dmatch_redkitchen_0_5', 'real_3dmatch_sun3d_home_38_41', 'real_3dmatch_sun3d_hotel3_8_15']
K, S, N, R = 20, 2.0, 16, 0.05


def real_clouds():
    out = []
    for f in FIXTURES:
        d = np.load(os.path.join(REAL, f + '_input.npz'))
        out += [d['src_xyz'].astype(np.float64), d['tgt_xyz'].astype(np.float64)]
    return out


def hand_built():
    rng = np.random.default_rng(21)
    g = np.stack(np.meshgrid(np.arange(30), np.arange(30), indexing='ij'), -1).reshape(-1, 2) * 0.01
    pts = rng.random((300, 3))
    return [np.tile([[1.0, 2.0, 3.0]], (40, 1)),                                 # all identical
            np.concatenate([pts, np.tile(pts[:1], (30, 1))]),                   # 31 copies of point 0
            rng.random((7, 3)),                                                 # k > n
            np.array([[0.5, -0.5, 0.25]]),                                      # one point
            np.zeros((0, 3)),                                                   # empty, inside the stack
            np.concatenate([g, np.zeros((g.shape[0], 1))], 1),                  # planar lattice (ties)
            np.concatenate([rng.random((12, 3)) * 0.1, rng.random((50, 3)) * 0.1 + 40.0]),   # far clusters
            np.array([[0.0, 0.0, 0.0], [0.05, 0.0, 0.0], [0.0, 0.025, 0.0], [3.0, 0.0, 0.0]])]  # exactly R apart


def colours_of(clouds, seed=3):
    rng = np.random.default_rng(seed)
    return [rng.random(c.shape) for c in clouds]


def check_stat(clouds, colours, out, k, s):
    kept, kc, ki, det = out
    for b, c in enumerate(clouds):
        avg, keep, st = O.statistical_outlier(c, k, s)
        assert np.array_equal(det['avg'][b].cpu().numpy(), avg), b
        assert np.array_equal(det['keep'][b].cpu().numpy(), keep), b
        assert np.array_equal(det['stats'][b].cpu().numpy(), np.array(st), equal_nan=True), (b, det['stats'][b], st)
        xyz, col, idx = O.select_points(c, keep, None if colours is None else colours[b])
        assert np.array_equal(ki[b].cpu().numpy(), idx) and np.array_equal(kept[b].cpu().numpy(), xyz), b
        if colours is not None:
            assert np.array_equal(kc[b].cpu().numpy(), col), b


def check_radius(clouds, colours, out, n, r):
    kept, kc, ki, det = out
    for b, c in enumerate(clouds):
        counts, keep = O.radius_outlier(c, n, r)
        assert np.array_equal(det['counts'][b].cpu().numpy(), counts), b
        assert np.array_equal(det['keep'][b].cpu().numpy(), keep), b
        xyz, col, idx = O.select_points(c, keep, None if colours is None else colours[b])
        assert np.array_equal(ki[b].cpu().numpy(), idx) and np.array_equal(kept[b].cpu().numpy(), xyz), b
        if colours is not None:
            assert np.array_equal(kc[b].cpu().numpy(), col), b


def same(a, b):
    for x, y in zip(a[:3], b[:3]):
        if x is None:
            assert y is None
            continue
        assert all(torch.equal(u, v) for u, v in zip(x, y))
    for key in a[3]:
        if key == 'stats':
            assert np.array_equal(a[3][key].cpu().numpy(), b[3][key].cpu().numpy(), equal_nan=True)
        else:
            assert all(torch.equal(u, v) for u, v in zip(a[3][key], b[3][key]))


def test_statistical_on_the_real_fixtures():
    clouds = real_clouds()
    cols = colours_of(clouds)
    before = ops.LAUNCHES
    out = ops.remove_statistical_outlier(clouds, K, S, colors=cols, return_details=True)
    assert ops.LAUNCHES - before == ops.statistical_outlier_launches() + ops.select_points_launches()
    check_stat(clouds, cols, out, K, S)
    same(out, ops.remove_statistical_outlier(clouds, K, S, colors=cols, return_details=True))
    for b in (0, 3):                                                            # alone = stacked
        alone = ops.remove_statistical_outlier([clouds[b]], K, S, colors=[cols[b]], return_details=True)
        assert torch.equal(alone[0][0], out[0][b]) and torch.equal(alone[2][0], out[2][b])
        assert torch.equal(alone[3]['avg'][0], out[3]['avg'][b])
        assert np.array_equal(alone[3]['stats'][0].cpu().numpy(), out[3]['stats'][b].cpu().numpy())


@pytest.mark.parametrize('cell', [1e-7, 100.0, 0.02])
def test_statistical_any_cell(cell):
    """A tiny cell leaves every query to the brute-force sweep, a huge one puts each cloud in one cell; 2 cm walks
    several rings.  The bits are the default cell's."""
    clouds = real_clouds()[::2] + hand_built()
    ref = ops.remove_statistical_outlier(clouds, K, S, return_details=True)
    got = ops.remove_statistical_outlier(clouds, K, S, return_details=True, knn_cell_size=cell)
    same(ref, got)
    check_stat(clouds, None, got, K, S)


@pytest.mark.parametrize('k', [1, 5, 33, 64])
def test_statistical_hand_built(k):
    clouds = hand_built()
    cols = colours_of(clouds, 4)
    out = ops.remove_statistical_outlier(clouds, k, 1.0, colors=cols, return_details=True)
    check_stat(clouds, cols, out, k, 1.0)
    assert out[0][0].shape[0] == 0 and out[0][3].shape[0] == 0 and out[0][4].shape[0] == 0


def test_radius_on_the_real_fixtures_and_hand_built():
    clouds = real_clouds() + hand_built()
    cols = colours_of(clouds)
    before = ops.LAUNCHES
    out = ops.remove_radius_outlier(clouds, N, R, colors=cols, return_details=True)
    assert ops.LAUNCHES - before == ops.radius_outlier_launches() + ops.select_points_launches()
    check_radius(clouds, cols, out, N, R)
    same(out, ops.remove_radius_outlier(clouds, N, R, colors=cols, return_details=True))
    alone = ops.remove_radius_outlier([clouds[2]], N, R, return_details=True)
    assert torch.equal(alone[0][0], out[0][2]) and torch.equal(alone[3]['counts'][0], out[3]['counts'][2])
    exact = ops.remove_radius_outlier([clouds[-1]], 2, R, return_details=True)
    assert exact[3]['counts'][0].tolist() == [2, 1, 2, 1]                       # 0.05 apart is not within 0.05


def test_synthetic_scan_with_outliers():
    xyz, mask = O.outlier_scan(11)
    out = ops.remove_statistical_outlier([xyz], K, S, return_details=True)
    check_stat([xyz], None, out, K, S)
    rad = ops.remove_radius_outlier([xyz], N, R, return_details=True)
    check_radius([xyz], None, rad, N, R)
    for o in (out, rad):
        dropped = np.ones(xyz.shape[0], bool)
        dropped[o[2][0].cpu().numpy()] = False
        assert dropped[mask].mean() > 0.8 and dropped[~mask].mean() < 0.01     # some outliers land on the walls


def test_range_statuses():
    good = np.random.default_rng(1).random((100, 3))
    for bad in (np.nan, np.inf, 1e31):
        x = good.copy()
        x[7, 1] = bad
        with pytest.raises(lib.RegtrLibError):
            ops.remove_statistical_outlier([good, x], K, S)
        st = ops.new_status(torch.device('cuda'))
        ops.remove_statistical_outlier([x], K, S, status=st)
        assert int(st.item()) & ops.STATUS_RANGE
    far = good.copy()
    far[3, 0] = 2.0 * ops.overlap_coord_bound(R)
    with pytest.raises(lib.RegtrLibError):
        ops.remove_radius_outlier([far], N, R)
    for bad in (np.nan, np.inf):
        x = good.copy()
        x[0, 2] = bad
        with pytest.raises(lib.RegtrLibError):
            ops.remove_radius_outlier([x], N, R)
    big = good * 1e6                                                            # finite and far: the cell adapts
    same(ops.remove_statistical_outlier([big], K, S, return_details=True),
         ops.remove_statistical_outlier([big], K, S, return_details=True, knn_cell_size=1e-9))


def test_argument_errors():
    c = [np.zeros((4, 3))]
    for k, s in ((0, 1.0), (65, 1.0), (5, 0.0), (5, float('nan')), (5, -1.0)):
        with pytest.raises(ValueError):
            ops.remove_statistical_outlier(c, k, s)
    for n, r in ((0, 0.1), (3, 0.0), (3, float('inf'))):
        with pytest.raises(ValueError):
            ops.remove_radius_outlier(c, n, r)


# ----------------------------------------------------------------------------------------- command lines

def _run(module, args, tmp_path):
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', module] + args, capture_output=True, text=True, cwd=ROOT, env=env,
                       timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _noisy(xyz, seed):
    """xyz with 2 % uniform outliers inserted at random rows."""
    rng = np.random.default_rng(seed)
    lo, hi = xyz.min(0), xyz.max(0)
    out = rng.random((max(1, xyz.shape[0] // 50), 3)) * (hi - lo) + lo
    allp = np.concatenate([xyz, out])
    return allp[rng.permutation(allp.shape[0])]


def _prefilter(clouds, stat, rad):
    kept, _, _ = ops.remove_statistical_outlier(clouds, *stat)
    kept, _, _ = ops.remove_radius_outlier([k.cpu().numpy() for k in kept], *rad)
    return [k.cpu().numpy() for k in kept]


def _compare_npz(a, b, skip=()):
    a, b = np.load(a), np.load(b)
    assert sorted(set(a.files) - set(skip)) == sorted(b.files)
    for k in b.files:
        assert np.array_equal(a[k], b[k]), k


def test_register_with_outlier_flags(tmp_path):
    from test_gpu_colored_icp import _checkpoint
    cfg, run = _checkpoint(tmp_path)
    stat, rad = (10, 1.5), (4, 0.08)
    raw = [_noisy(P.load_point_cloud(os.path.join(REAL, f'modelnet_test_2_{i}.ply')), 30 + i) for i in (0, 1)]
    files, pre = [], []
    for i, (x, y) in enumerate(zip(raw, _prefilter(raw, stat, rad))):
        files.append(str(tmp_path / f'raw{i}.npy'))
        pre.append(str(tmp_path / f'pre{i}.npy'))
        np.save(files[-1], x)
        np.save(pre[-1], y)
    flags = ['--remove_statistical_outlier', str(stat[0]), str(stat[1]), '--remove_radius_outlier', str(rad[0]),
             str(rad[1])]
    ckpt = ['--ckpt', str(run / 'ckpt' / 'model-best.pth'), '--icp', '0.05']
    for name, extra in (('net', ckpt), ('fpfh', ['--fpfh', '0.05', '--icp', '0.05'])):
        a = _run('regtr_b200.register', files + extra + flags + ['--out', str(tmp_path / f'{name}_flags')], tmp_path)
        b = _run('regtr_b200.register', pre + extra + ['--out', str(tmp_path / f'{name}_pre')], tmp_path)
        extra_keys = {'n_src_read', 'n_tgt_read', 'n_src_filtered', 'n_tgt_filtered'}
        assert set(a) - set(b) == extra_keys and set(b) <= set(a)
        assert {k: a[k] for k in b} == b
        assert (a['n_src_read'], a['n_tgt_read']) == (raw[0].shape[0], raw[1].shape[0])
        _compare_npz(tmp_path / f'{name}_flags' / 'result.npz', tmp_path / f'{name}_pre' / 'result.npz',
                     ('src_index', 'tgt_index'))
        res = np.load(tmp_path / f'{name}_flags' / 'result.npz')
        for side, x, y in (('src', raw[0], pre[0]), ('tgt', raw[1], pre[1])):
            idx = res[f'{side}_index']
            assert np.array_equal(x[idx], np.load(y)) and a[f'n_{side}_filtered'] == idx.shape[0]
        with open(tmp_path / f'{name}_flags' / 'pose.txt') as fa, open(tmp_path / f'{name}_pre' / 'pose.txt') as fb:
            assert fa.read() == fb.read()


def test_multiway_with_outlier_flags(tmp_path):
    from regtr_b200 import synthetic as SY
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': random_state_dict(cfg, 5), 'step': 1}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, '3dmatch', str(run / 'config.yaml'))
    raw = [_noisy(f, 40 + k) for k, f in enumerate(SY.make_scene(9, 3, n_target=3000)['fragments'])]
    stat, rad = (K, S), (N, 0.1)
    pre = _prefilter(raw, stat, rad)
    runs = {}
    for name, clouds in (('flags', raw), ('pre', pre)):
        files = []
        for k, f in enumerate(clouds):
            path = tmp_path / name / 'my-scene' / f'cloud_bin_{k}.npy'
            path.parent.mkdir(parents=True, exist_ok=True)
            np.save(path, f)
            files.append(str(path))
        extra = ['--remove_statistical_outlier', str(K), str(S), '--remove_radius_outlier', str(N), '0.1'] \
            if name == 'flags' else []
        runs[name] = _run('regtr_b200.multiway', files + ['--ckpt', str(run / 'ckpt' / 'model-best.pth'), '--out',
                                                          str(tmp_path / f'out_{name}'), '--voxel', '0.05'] + extra,
                          tmp_path)
    assert runs['flags'] == runs['pre']
    _compare_npz(tmp_path / 'out_flags' / 'result.npz', tmp_path / 'out_pre' / 'result.npz',
                 ('point_index', 'point_offsets'))
    res = np.load(tmp_path / 'out_flags' / 'result.npz')
    offs = res['point_offsets']
    assert offs.tolist() == [0] + np.cumsum([p.shape[0] for p in pre]).tolist()
    for k, (x, y) in enumerate(zip(raw, pre)):
        assert np.array_equal(x[res['point_index'][offs[k]:offs[k + 1]]], y)
    for f in ('scene.ply', os.path.join('my-scene', 'est.log')):
        with open(tmp_path / 'out_flags' / f, 'rb') as fa, open(tmp_path / 'out_pre' / f, 'rb') as fb:
            assert fa.read() == fb.read(), f
