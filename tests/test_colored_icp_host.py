"""Colored ICP without a GPU: the PLY colour reader and writer, the float64 oracle (tests/colored_icp_oracle.py) on
planes where the answer is known, the command lines' flags and usage errors, `eval.icp_refine`'s call layout, and the
compiler's report on color.cu."""
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import colored_icp_oracle as C
import gicp_oracle as G
import icp_oracle as I
import icp_plane_oracle as N
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import pointio as P
from regtr_b200 import register as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ply(path, fmt, props, rows):
    """A PLY file with one vertex element of (name, ply type) props and rows (list of tuples)."""
    codes = {'uchar': 'u1', 'ushort': 'u2', 'float': 'f4', 'double': 'f8', 'int': 'i4'}
    head = ['ply', f'format {fmt} 1.0', f'element vertex {len(rows)}']
    head += [f'property {t} {n}' for n, t in props] + ['end_header']
    with open(path, 'wb') as fh:
        fh.write(('\n'.join(head) + '\n').encode('ascii'))
        if fmt == 'ascii':
            fh.write(''.join(' '.join(str(v) for v in r) + '\n' for r in rows).encode('ascii'))
        else:
            o = '<' if fmt == 'binary_little_endian' else '>'
            dt = np.dtype([(n, o + codes[t]) for n, t in props])
            fh.write(np.array([tuple(r) for r in rows], dtype=dt).tobytes())


XYZ = [(0.5, -1.25, 2.0), (3.0, 0.0, -0.75), (1e-3, 2.5, 7.0)]


@pytest.mark.parametrize('fmt', ['ascii', 'binary_little_endian', 'binary_big_endian'])
@pytest.mark.parametrize('ctype,vals,scale', [('uchar', [0, 128, 255], 255.0), ('ushort', [0, 1000, 65535], 65535.0),
                                              ('float', [0.0, 0.25, 1.0], 1.0), ('double', [0.0, 0.125, 1.0], 1.0)])
def test_ply_colour_reader(tmp_path, fmt, ctype, vals, scale):
    props = [('x', 'double'), ('y', 'double'), ('z', 'double'), ('nx', 'float'),
             ('red', ctype), ('green', ctype), ('blue', ctype)]
    rows = [XYZ[i] + (0.5,) + (vals[i], vals[(i + 1) % 3], vals[(i + 2) % 3]) for i in range(3)]
    path = str(tmp_path / 'c.ply')
    _ply(path, fmt, props, rows)
    xyz, rgb = P.load_point_cloud_colors(path)
    assert xyz.dtype == np.float64 and rgb.dtype == np.float64 and rgb.shape == (3, 3)
    assert np.array_equal(xyz, np.array(XYZ))
    want = np.array([[vals[i], vals[(i + 1) % 3], vals[(i + 2) % 3]] for i in range(3)], np.float64)
    want = want.astype(np.float32).astype(np.float64) if ctype == 'float' else want
    assert np.array_equal(rgb, want / scale)
    # read_ply and load_point_cloud still return the coordinates alone
    assert np.array_equal(P.read_ply(path), np.array(XYZ)) and np.array_equal(P.load_point_cloud(path), np.array(XYZ))


def test_ply_colour_reader_rejects_bad_channels(tmp_path):
    base = [('x', 'float'), ('y', 'float'), ('z', 'float')]
    for props, what in ((base + [('red', 'uchar'), ('green', 'uchar')], "'blue'"),
                        (base, "'red'"),
                        (base + [('red', 'uchar'), ('green', 'int'), ('blue', 'uchar')], "'green'")):
        path = str(tmp_path / 'bad.ply')
        _ply(path, 'binary_little_endian', props, [(1, 2, 3) + (5,) * (len(props) - 3)])
        with pytest.raises(ValueError, match=re.escape(path) + '.*' + what):
            P.load_point_cloud_colors(path)
    for ext, data in (('.npy', None), ('.bin', None), ('.pth', None)):
        with pytest.raises(ValueError, match='carry no colour'):
            P.load_point_cloud_colors(str(tmp_path / ('x' + ext)))


def test_write_ply_colours_round_trip_and_plain_output_unchanged(tmp_path):
    xyz = np.array(XYZ)
    plain = str(tmp_path / 'plain.ply')
    P.write_ply(plain, xyz, {'overlap': np.array([0.5, 1.0, 0.0])})
    head = ('ply\nformat binary_little_endian 1.0\ncomment Created by regtr_b200\nelement vertex 3\n'
            'property double x\nproperty double y\nproperty double z\nproperty float overlap\nend_header\n')
    rec = np.empty(3, np.dtype([('x', '<f8'), ('y', '<f8'), ('z', '<f8'), ('overlap', '<f4')]))
    for a, k in enumerate('xyz'):
        rec[k] = xyz[:, a]
    rec['overlap'] = [0.5, 1.0, 0.0]
    assert open(plain, 'rb').read() == head.encode('ascii') + rec.tobytes()
    rgb = np.array([[0.0, 0.5, 1.0], [1.0, 0.2, 0.7], [0.3, 0.3, 0.3]])
    path = str(tmp_path / 'c.ply')
    P.write_ply(path, xyz, colors=rgb)
    x2, c2 = P.load_point_cloud_colors(path)
    assert np.array_equal(x2, xyz) and np.array_equal(c2, np.round(rgb * 255.0) / 255.0)
    assert np.array_equal(P.load_point_cloud(path), xyz)
    with pytest.raises(ValueError):
        P.write_ply(path, xyz, colors=rgb[:2])


def plane(rng, n_side=40, step=0.01, z=1.0, jitter=0.3):
    """A jittered grid of n_side^2 points on the plane z = const."""
    g = np.stack(np.meshgrid(np.arange(n_side), np.arange(n_side), indexing='ij'), -1).reshape(-1, 2) * step
    g = g + rng.uniform(-jitter, jitter, g.shape) * step
    return np.concatenate([g, np.full((g.shape[0], 1), z)], axis=1)


def test_oracle_gradient_of_a_linear_ramp_is_its_in_plane_gradient():
    """Intensity a x + b y + c on the plane z = 1: the gradient is (a, b, 0) wherever the point has 4 neighbours."""
    rng = np.random.default_rng(3)
    xyz = plane(rng, 20)
    a, b = 0.7, -0.4
    it = 0.3 + a * xyz[:, 0] + b * xyz[:, 1]
    rgb = np.repeat(it[:, None], 3, axis=1)
    nrm, cnt = N.estimate_normals(xyz, 0.03, 30)
    grad = C.color_gradients(xyz, nrm, rgb, 0.03, 30)
    ok = cnt >= 4
    assert ok.mean() > 0.9
    assert np.abs(grad[ok] - np.array([a, b, 0.0])).max() < 1e-9
    assert not grad[~ok].any()
    # a zero normal gives a zero gradient
    nrm[5] = 0.0
    assert not C.color_gradients(xyz, nrm, rgb, 0.03, 30)[5].any()


def test_colored_icp_recovers_an_in_plane_offset_that_point_to_plane_cannot():
    """A textured plane (tests' procedural texture) sampled twice and displaced within the plane: geometry gives
    point-to-plane nothing to hold on to, colour gives colored ICP the offset."""
    rng = np.random.default_rng(5)
    tgt = plane(rng, 50)
    src = plane(rng, 50) + np.array([0.004, 0.003, 0.0])
    gt = np.eye(3, 4)                                   # the clouds are already aligned in world coordinates
    scol, tcol = C.colour_pair(src, tgt, gt, scale=0.5)
    init = np.eye(3, 4)
    init[:, 3] = [0.02, -0.015, 0.0]
    nrm, _ = N.estimate_normals(tgt, 0.05, 30)
    grad = C.color_gradients(tgt, nrm, tcol, 0.05, 30)
    col = C.icp(src, tgt, nrm, scol, tcol, grad, init, 0.05, 60)
    p2p = G.icp(src, tgt, nrm, init, 0.05, 60, method='point_to_plane')
    col_err = np.linalg.norm(col['pose'][:, 3] - gt[:, 3])
    p2p_err = np.linalg.norm(p2p['pose'][:, 3] - gt[:, 3])
    assert col_err < 2e-3 and p2p_err > 0.02, (col_err, p2p_err)
    assert np.abs(col['pose'][:, :3] - np.eye(3)).max() < 1e-2


def test_lambda_one_is_point_to_plane():
    rng = np.random.default_rng(9)
    p, q = rng.normal(size=(50, 3)), rng.normal(size=(50, 3))
    n = rng.normal(size=(50, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    n[7] = 0.0
    grad, it_q, is_p = rng.normal(size=(50, 3)), rng.uniform(size=50), rng.uniform(size=50)
    for loss, k in (('l2', None), ('huber', 0.3)):
        jtj, jtr = C.colored_system(p, q, n, grad, it_q, is_p, 1.0, loss, k)
        want = G.plane_system(p, q, n, loss, k)
        assert np.allclose(jtj, want[0], rtol=0, atol=1e-12) and np.allclose(jtr, want[1], rtol=0, atol=1e-12)
    jtj, _ = C.colored_system(p, q, n, grad, it_q, is_p, 0.5)
    assert not np.allclose(jtj, G.plane_system(p, q, n)[0])


def test_register_and_multiway_accept_the_colored_flags():
    opt = R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.03', '--icp_method', 'colored',
                        '--icp_lambda_geometric', '0.5'])
    assert (opt.icp_method, opt.icp_lambda_geometric) == ('colored', 0.5)
    assert E.icp_kwargs(opt)['lambda_geometric'] == 0.5 and E.icp_kwargs(opt)['method'] == 'colored'
    assert R.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth']).icp_lambda_geometric == 0.968
    assert 'lambda_geometric' not in E.icp_kwargs(R.parse_args(['a.ply', 'b.ply', '--ckpt', 'x', '--icp', '0.03']))
    ap = MW.parser()
    opt = ap.parse_args(['a.ply', 'b.ply', 'c.ply', '--ckpt', 'x', '--out', 'o', '--icp', '0.03', '--icp_method',
                         'colored', '--icp_lambda_geometric', '1'])
    E.check_icp_arguments(ap, opt, colors=True)
    assert (opt.icp_method, opt.icp_lambda_geometric) == ('colored', 1.0)


def _eval_3dmatch():
    sys.path.insert(0, os.path.join(ROOT, 'scripts'))
    try:
        import eval_3dmatch
    finally:
        sys.path.pop(0)
    return eval_3dmatch


def test_eval_3dmatch_rejects_colored(capsys):
    with pytest.raises(SystemExit) as e:
        _eval_3dmatch().main(['--root', 'r', '--info', 'i.pkl', '--gt', 'g', '--ckpt', 'm.pth', '--icp', '0.03',
                              '--icp_method', 'colored'])
    assert e.value.code == 2 and 'colored needs coloured clouds' in capsys.readouterr().err


@pytest.mark.parametrize('lam', ['-0.1', '1.5', 'nan'])
def test_lambda_out_of_range_is_a_usage_error(lam, capsys):
    with pytest.raises(SystemExit) as e:
        R.main(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.03', '--icp_method', 'colored',
                '--icp_lambda_geometric', lam])
    assert e.value.code == 2 and '--icp_lambda_geometric' in capsys.readouterr().err


def test_an_uncoloured_file_is_a_usage_error_before_the_checkpoint(tmp_path, capsys):
    """The checkpoint does not exist: the usage error must come first, and it names the file."""
    xyz = np.random.default_rng(0).normal(size=(20, 3))
    plain, coloured = str(tmp_path / 'plain.ply'), str(tmp_path / 'col.ply')
    P.write_ply(plain, xyz)
    P.write_ply(coloured, xyz, colors=np.full((20, 3), 0.5))
    npy = str(tmp_path / 'a.npy')
    np.save(npy, xyz)
    for argv, bad in (([coloured, plain], plain), ([npy, coloured], npy)):
        with pytest.raises(SystemExit) as e:
            R.main(argv + ['--ckpt', str(tmp_path / 'none' / 'ckpt' / 'm.pth'), '--icp', '0.03', '--icp_method',
                           'colored'])
        err = capsys.readouterr().err
        assert e.value.code == 2 and bad in err, err
    with pytest.raises(SystemExit) as e:
        MW.main([coloured, coloured, plain, '--ckpt', str(tmp_path / 'none' / 'ckpt' / 'm.pth'), '--out',
                 str(tmp_path / 'o'), '--icp', '0.03', '--icp_method', 'colored'])
    err = capsys.readouterr().err
    assert e.value.code == 2 and plain in err, err


def test_icp_refine_colored_call_layout():
    """Target normals as point_to_plane estimates them, gradients at 2 R with 30 neighbours, then one icp call with the
    colours, the gradients and lambda_geometric."""
    rng = np.random.default_rng(1)
    src, tgt = [plane(rng, 10)], [plane(rng, 10)]
    scol, tcol = [C.texture(src[0])], [C.texture(tgt[0])]
    calls = []

    def normals(clouds, r, max_nn):
        calls.append(('normals', len(clouds), r, max_nn))
        return [N.estimate_normals(c, r, max_nn)[0] for c in clouds]

    def gradients(clouds, nrm, cols, r, max_nn):
        calls.append(('gradients', len(clouds), r, max_nn))
        return [C.color_gradients(c, n, k, r, max_nn) for c, n, k in zip(clouds, nrm, cols)]

    def icp(s, t, init, r, it, **kw):
        calls.append(('icp', r, it, sorted(kw), kw['lambda_geometric']))
        return C.icp_batch(s, t, kw['tgt_normals'], kw['src_colors'], kw['tgt_colors'], kw['tgt_color_gradients'],
                           init, r, it, lambda_geometric=kw['lambda_geometric'])

    pose, _ = E.icp_refine(src, tgt, np.eye(3, 4)[None], 0.02, 5, 'colored', colors=(scol, tcol),
                           lambda_geometric=0.9, icp=icp, estimate_normals=normals, color_gradients=gradients)
    assert calls == [('normals', 1, 0.04, 30), ('gradients', 1, 0.04, 30),
                     ('icp', 0.02, 5, ['lambda_geometric', 'method', 'src_colors', 'tgt_color_gradients',
                                       'tgt_colors', 'tgt_normals'], 0.9)]
    assert pose.shape == (1, 3, 4)
    with pytest.raises(ValueError, match='colors'):
        E.icp_refine(src, tgt, np.eye(3, 4)[None], 0.02, 5, 'colored', icp=icp, estimate_normals=normals)
    with pytest.raises(ValueError, match='src_colors'):
        E.icp_forward(lambda b: {'pose': torch.eye(3, 4)[None, None]}, 0.02, method='colored')(
            {'src_xyz': src, 'tgt_xyz': tgt})


def test_color_kernels_do_not_spill():
    """color.cu's entry functions: the init, the gradients and the colored reduction, none spilling; the colored
    reduction fits two 256-thread CTAs per SM (at most 128 registers)."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'color.cu'),
                                                        '-o', os.path.join(tmp, 'color.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) "
                         r"registers", text)
    names = sorted(('k_color_init' in e[0], 'k_color_gradients' in e[0], 'PlaneModeE3E' in e[0]) for e in entries)
    assert len(entries) == 3 and names == [(False, False, True), (False, True, False), (True, False, False)], entries
    for name, _, st, ld, regs in entries:
        assert (st, ld) == ('0', '0'), (name, st, ld)
        if 'PlaneModeE3E' in name:
            assert int(regs) <= 128, regs
    assert set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
