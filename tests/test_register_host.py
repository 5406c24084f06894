"""CPU tests of the point-cloud files, the register CLI's host rules and the DGR benchmark (regtr_b200/pointio.py,
regtr_b200/register.py, eval.benchmark_dgr, scripts/evaluate_3dmatch.py).  The DGR fixture comes from the
reference's unmodified benchmark_dgr (tests/golden/make_dgr_golden.py)."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden
from regtr_b200 import eval as E
from regtr_b200 import pointio as P
from regtr_b200 import register as R
from regtr_b200.config import Cfg, load_config

REAL = os.path.join(GOLDEN, 'real')


# ------------------------------------------------------------------------------------------------ PLY
def test_ply_reader_matches_the_reference_demo_inputs():
    inp = np.load(os.path.join(REAL, 'real_modelnet_2_input.npz'))
    for side, k in (('src_xyz', 0), ('tgt_xyz', 1)):
        xyz = P.load_point_cloud(os.path.join(REAL, f'modelnet_test_2_{k}.ply'))
        assert xyz.dtype == np.float64 and xyz.shape == (717, 3)
        assert np.array_equal(xyz.astype(np.float32), inp[side])


def test_write_ply_roundtrip(tmp_path):
    rng = np.random.default_rng(0)
    xyz = rng.normal(size=(50, 3))
    ov = rng.random(50).astype(np.float32)
    path = str(tmp_path / 'a.ply')
    P.write_ply(path, xyz, {'overlap': ov})
    assert np.array_equal(P.load_point_cloud(path), xyz)
    head = open(path, 'rb').read(300).split(b'end_header\n')[0].decode()
    assert 'format binary_little_endian 1.0' in head and 'property double x' in head and 'property float overlap' in head
    rec = np.frombuffer(open(path, 'rb').read().split(b'end_header\n', 1)[1],
                        dtype=[('x', '<f8'), ('y', '<f8'), ('z', '<f8'), ('overlap', '<f4')])
    assert np.array_equal(rec['overlap'], ov)
    P.write_ply(str(tmp_path / 'e.ply'), np.zeros((0, 3)))
    assert P.load_point_cloud(str(tmp_path / 'e.ply')).shape == (0, 3)


def _ply(path, fmt, props, rows, pre=None):
    """A PLY file with vertex properties `props` [(type, name)] and `rows` (list of tuples), optionally preceded by
    an element `pre` = (name, [(type, name)], rows) stored before the vertices."""
    order = {'binary_little_endian': '<', 'binary_big_endian': '>'}.get(fmt)
    code = {'float': 'f4', 'double': 'f8', 'int': 'i4', 'uchar': 'u1', 'short': 'i2', 'uint16': 'u2', 'int8': 'i1'}
    head = ['ply', f'format {fmt} 1.0', 'comment test']
    body = b''
    for name, pr, rw in ([pre] if pre else []) + [('vertex', props, rows)]:
        head.append(f'element {name} {len(rw)}')
        head += [f'property {t} {n}' for t, n in pr]
        if order is None:
            body += ''.join(' '.join(repr(v) for v in r) + '\n' for r in rw).encode()
        else:
            dt = np.dtype([(n, order + code[t]) for t, n in pr])
            body += np.array([tuple(r) for r in rw], dtype=dt).tobytes()
    head.append('end_header')
    with open(path, 'wb') as f:
        f.write(('\n'.join(head) + '\n').encode() + body)


@pytest.mark.parametrize('fmt', ['ascii', 'binary_big_endian', 'binary_little_endian'])
def test_ply_formats_types_and_skipped_properties(tmp_path, fmt):
    rows = [(3, 0.5, -1.25, 7, 2.0, 200), (-4, 1.5, 0.125, -2, 3.5, 17), (12, -0.75, 8.0, 5, -1.0, 0)]
    props = [('int', 'x'), ('float', 'nx'), ('double', 'y'), ('short', 'intensity'), ('float', 'z'), ('uchar', 'red')]
    pre = ('camera', [('double', 'fx'), ('uint16', 'w')], [(1.5, 640)])
    path = str(tmp_path / 'p.ply')
    _ply(path, fmt, props, rows, pre)
    want = np.array([[r[0], r[2], r[4]] for r in rows], dtype=np.float64)
    assert np.array_equal(P.load_point_cloud(path), want)
    # faces after the vertices (with their list property) are fine
    with open(path, 'rb') as f:
        data = f.read()
    if fmt == 'ascii':
        data = data.replace(b'end_header\n', b'element face 1\nproperty list uchar int vertex_indices\nend_header\n')
        data += b'3 0 1 2\n'
        with open(path, 'wb') as f:
            f.write(data)
        assert np.array_equal(P.load_point_cloud(path), want)


def test_ply_rejections(tmp_path):
    p = str(tmp_path / 'l.ply')
    with open(p, 'wb') as f:
        f.write(b'ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nproperty float z\n'
                b'property list uchar int idx\nend_header\n1 2 3 1 5\n')
    with pytest.raises(ValueError, match='list'):
        P.load_point_cloud(p)
    with open(p, 'wb') as f:
        f.write(b'ply\nformat ascii 1.0\nelement face 1\nproperty list uchar int vertex_indices\n'
                b'element vertex 1\nproperty float x\nproperty float y\nproperty float z\nend_header\n3 0 1 2\n1 2 3\n')
    with pytest.raises(ValueError, match='list'):
        P.load_point_cloud(p)
    full = open(os.path.join(REAL, 'modelnet_test_2_0.ply'), 'rb').read()
    head = full.split(b'end_header')[0]
    with open(p, 'wb') as f:
        f.write(head)                                                   # the header without end_header
    with pytest.raises(ValueError, match='end_header'):
        P.load_point_cloud(p)
    with open(p, 'wb') as f:
        f.write(full[:-10])                                             # truncated data
    with pytest.raises(ValueError, match='ends after'):
        P.load_point_cloud(p)
    for bad in (b'plx\n', b'ply\nformat binary_middle_endian 1.0\nend_header\n',
                b'ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nend_header\n1 2\n',
                b'ply\nformat ascii 1.0\nelement vertex 1\nproperty quad x\nend_header\n'):
        with open(p, 'wb') as f:
            f.write(bad)
        with pytest.raises(ValueError):
            P.load_point_cloud(p)


# ------------------------------------------------------------------------------------------------ other formats
def test_pth_ndarray_and_tensor_load(tmp_path):
    x = np.random.default_rng(1).normal(size=(40, 3))
    torch.save(x, str(tmp_path / 'a.pth'))
    assert np.array_equal(P.load_point_cloud(str(tmp_path / 'a.pth')), x)
    torch.save(torch.from_numpy(x).float(), str(tmp_path / 't.pth'))
    assert np.array_equal(P.load_point_cloud(str(tmp_path / 't.pth')), x.astype(np.float32).astype(np.float64))


class _Payload:
    def __reduce__(self):
        return (os.system, ('echo pwned',))


def test_pth_refuses_other_globals(tmp_path):
    p = str(tmp_path / 'evil.pth')
    torch.save({'xyz': np.zeros((2, 3)), 'x': _Payload()}, p)
    with pytest.raises(pickle.UnpicklingError):
        P.load_point_cloud(p)
    torch.save(np.zeros((2, 3), dtype=object), p)
    with pytest.raises(Exception):
        P.load_point_cloud(p)


def test_bin_npy_and_unknown(tmp_path):
    a = np.arange(40, dtype=np.float32).reshape(10, 4)
    a.tofile(str(tmp_path / 'k.bin'))
    assert np.array_equal(P.load_point_cloud(str(tmp_path / 'k.bin')), a[:, :3].astype(np.float64))
    np.save(str(tmp_path / 'n.npy'), a.astype(np.float64))
    assert np.array_equal(P.load_point_cloud(str(tmp_path / 'n.npy')), a[:, :3])
    with pytest.raises(ValueError, match='format'):
        P.load_point_cloud(str(tmp_path / 'x.xyz'))


# ------------------------------------------------------------------------------------------------ register CLI rules
def test_config_discovery_and_crop(tmp_path):
    ck = tmp_path / 'run' / 'ckpt' / 'model-best.pth'
    assert R.config_path(str(ck)) == tmp_path / 'run' / 'config.yaml'
    assert str(R.config_path(str(ck), 'other.yaml')) == 'other.yaml'
    (tmp_path / 'run').mkdir()
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    write_config(get_config('modelnet'), 'modelnet', str(tmp_path / 'run' / 'config.yaml'))
    assert load_config(str(R.config_path(str(ck)))) == get_config('modelnet')
    xyz = np.array([[0.0, 0, 0], [1.0, 0, 0], [0.6, 0.8, 0], [2.0, 0, 0]])
    assert np.array_equal(R.crop(Cfg(overlap_radius=0.1), xyz), xyz)
    assert np.array_equal(R.crop(Cfg(crop_radius=1.0), xyz), xyz[[0]])           # strictly inside
    assert np.array_equal(R.crop(Cfg(crop_radius=1.5), xyz), xyz[:3])


def test_pose_text_is_est_log_format():
    p = np.array([[1, 0, 0, 0.5], [0, 1, 0, -0.25], [0, 0, 1, 1e-3]], np.float32)
    txt = R.pose_text(p)
    rows = txt.splitlines()
    assert len(rows) == 4 and rows[3] == '0.000000000000\t0.000000000000\t0.000000000000\t1.000000000000'
    assert rows[0].split('\t')[3] == '0.500000000000'


# ------------------------------------------------------------------------------------------------ DGR benchmark
@pytest.fixture(scope='module')
def dgr():
    return load_golden('eval_dgr')


def _materialise(fx, case, root):
    scenes = [str(s) for s in fx[f'{case}_scenes']]
    for scene in scenes:
        os.makedirs(os.path.join(root, 'est', scene), exist_ok=True)
        with open(os.path.join(root, 'est', scene, 'est.log'), 'wb') as f:
            f.write(fx[f'{case}_est_{scene}'].tobytes())
        if f'{case}_gt_{scene}' in fx:
            os.makedirs(os.path.join(root, 'gt', scene), exist_ok=True)
            with open(os.path.join(root, 'gt', scene, 'gt.log'), 'wb') as f:
                f.write(fx[f'{case}_gt_{scene}'].tobytes())
    gt = os.path.join(root, 'gt') if f'{case}_gt_{scenes[0]}' in fx else os.path.join(REAL, 'benchmarks', '3DMatch')
    return scenes, os.path.join(root, 'est'), gt


@pytest.mark.parametrize('case', ['real', 'synth'])
def test_benchmark_dgr_matches_reference(tmp_path, dgr, case):
    scenes, est, gt = _materialise(dgr, case, str(tmp_path))
    s, per = E.benchmark_dgr(est, gt)
    assert s == dgr[f'{case}_summary'].tobytes().decode('utf-8')
    for scene in scenes:
        np.testing.assert_allclose(per[scene]['rre'], dgr[f'{case}_rre_{scene}'], rtol=0, atol=1e-12)
        np.testing.assert_allclose(per[scene]['rte'], dgr[f'{case}_rte_{scene}'], rtol=0, atol=1e-12)
        assert np.array_equal(per[scene]['success'],
                              (dgr[f'{case}_rre_{scene}'] < 15) & (dgr[f'{case}_rte_{scene}'] < 0.3))
    if case == 'real':
        assert 'nan' in s                          # a scene without a success, as the reference prints it


def _run_script(args):
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    return subprocess.run([sys.executable, os.path.join(ROOT, 'scripts', 'evaluate_3dmatch.py')] + args,
                          capture_output=True, text=True, env=env, cwd=ROOT, timeout=300)


def test_evaluate_3dmatch_script_both_modes(tmp_path):
    gt_root = os.path.join(REAL, 'benchmarks')
    bench_gt = os.path.join(gt_root, '3DMatch')
    w = E.EstLogWriter(str(tmp_path), '3DMatch')
    rng = np.random.default_rng(5)
    for k, scene in enumerate(sorted(os.listdir(bench_gt))):
        keys, traj = E.read_trajectory(os.path.join(bench_gt, scene, 'gt.log'))
        i, j = int(keys[0][0]), int(keys[0][1])
        d = np.eye(4)
        d[:3, 3] = rng.normal(size=3) * (0.01 if k == 0 else 0.5)
        w.append(scene, j, i, traj[0] @ d)
    r = _run_script(['--results_dir', str(tmp_path), '--gt', gt_root, '--use_dgr'])
    assert r.returncode == 0, r.stderr
    want, per = E.benchmark_dgr(w.root, bench_gt)
    assert r.stdout == want + '\n'
    assert os.path.exists(tmp_path / 'individual_errors_dgr.csv')
    r = _run_script(['--results_dir', str(tmp_path), '--gt', gt_root])
    assert r.returncode == 0, r.stderr
    want, _, per = E.benchmark_3dmatch(w.root, bench_gt)
    assert r.stdout == want + '\n'
    rows = open(tmp_path / 'individual_errors.csv').read().splitlines()
    assert rows[0] == 'scene,src,tgt,errors' and len(rows) == 1 + len(per)
