"""ModelNet40 on the host: the crop-chain restatement against the reference's transforms (tests/golden/
modelnet_transforms.npz, made by make_modelnet_golden.py), the dataset's file and category rules, the reference's
quirks, and the training CLI up to the device."""
import os
import types

import numpy as np
import pytest
import torch

from regtr_b200 import modelnet as M
from regtr_b200.config import get_config

HERE = os.path.dirname(os.path.abspath(__file__))
FIELDS = ('src_xyz', 'tgt_xyz', 'src_overlap', 'tgt_overlap', 'correspondences', 'pose')


@pytest.fixture(scope='module')
def golden():
    return np.load(os.path.join(HERE, 'golden', 'modelnet_transforms.npz'))


def _cases(z, kind):
    return sorted({k.split('/')[0] for k in z.files if k.startswith(kind)})


def test_deterministic_pairs_match_the_reference_bit_for_bit(golden):
    cases = _cases(golden, 'test')
    assert len(cases) == 6
    for c in cases:
        idx, partial = int(golden[c + '/idx']), list(golden[c + '/partial'])
        it = M.crop_chain(golden['shapes'][idx], partial, 45.0, 0.5, np.random.RandomState(idx), idx=idx,
                          deterministic=True)
        for k in FIELDS:
            assert it[k].dtype == golden[f'{c}/{k}'].dtype, (c, k)
            np.testing.assert_array_equal(it[k], golden[f'{c}/{k}'], err_msg=f'{c} {k}')


class Replay:
    """The recorded np.random draws of one train case, served in order to crop_chain."""

    def __init__(self, z, case):
        self.z = z
        self.keys = sorted(k for k in z.files if k.startswith(case + '/draw'))
        self.i = 0

    def _next(self, name):
        key = self.keys[self.i]
        assert key.endswith('_' + name), (key, name)
        self.i += 1
        v = self.z[key]
        return v[()] if v.ndim == 0 else v

    def uniform(self, low=0.0, high=1.0, size=None):
        return self._next('uniform')

    def choice(self, a, size=None, replace=True):
        v = self._next('choice')
        assert len(v) == size and not replace
        return v

    def normal(self, loc=0.0, scale=1.0, size=None):
        v = self._next('normal')
        assert v.shape == size and scale == M.JITTER_SCALE
        return v

    def permutation(self, n):
        v = self._next('permutation')
        assert len(v) == n
        return v

    def seed(self, s):
        raise AssertionError('the train chain does not reseed')


def test_train_chain_fed_the_recorded_draws_matches_the_reference(golden):
    cases = _cases(golden, 'train')
    assert len(cases) == 2
    for c in cases:
        idx, partial = int(golden[c + '/idx']), list(golden[c + '/partial'])
        rep = Replay(golden, c)
        it = M.crop_chain(golden['shapes'][idx], partial, 45.0, 0.5, rep, idx=idx)
        assert rep.i == len(rep.keys)
        for k in FIELDS:
            np.testing.assert_array_equal(it[k], golden[f'{c}/{k}'], err_msg=f'{c} {k}')


def test_reference_quirks():
    shapes = np.load(os.path.join(HERE, 'golden', 'modelnet_transforms.npz'))['shapes']
    raw = shapes[0]
    # both sizes are 717 whatever num_points / partial say
    for partial in ([0.7, 0.7], [0.5, 0.5], [0.7, 0.5]):
        it = M.crop_chain(raw, partial, 45.0, 0.5, np.random.RandomState(0), deterministic=True)
        assert it['src_xyz'].shape == it['tgt_xyz'].shape == (717, 3)
    # both clouds are cropped with p_keep[0]: the second proportion changes nothing
    a = M.crop_chain(raw, [0.7, 0.7], 45.0, 0.5, np.random.RandomState(3), idx=3, deterministic=True)
    b = M.crop_chain(raw, [0.7, 0.2], 45.0, 0.5, np.random.RandomState(3), idx=3, deterministic=True)
    for k in FIELDS:
        np.testing.assert_array_equal(a[k], b[k])
    assert ((a['crop_masks'].sum(axis=1) > 1400) & (a['crop_masks'].sum(axis=1) <= 2048 - 615)).all()
    # the jitter is RandomJitter's default N(0, 0.01^2) clipped to 0.05, not cfg.augment_noise (0.005)
    pose = a['pose'].astype(np.float64)
    rot = pose[:, :3].T                                   # the source transform is the inverse of the pose
    clean = raw[a['src_raw_idx']].astype(np.float64) @ rot.T - rot @ pose[:, 3]
    noise = np.concatenate([a['src_xyz'] - clean, a['tgt_xyz'] - raw[a['tgt_raw_idx']]])
    assert np.abs(noise).max() <= 0.05 + 1e-5
    assert 0.008 < noise.std() < 0.0115
    # overlap masks follow from the other side's crop
    np.testing.assert_array_equal(a['src_overlap'], a['crop_masks'][1][a['src_raw_idx']])
    np.testing.assert_array_equal(a['tgt_overlap'], a['crop_masks'][0][a['tgt_raw_idx']])


def test_partials_that_leave_too_few_points_and_other_noise_types_are_rejected():
    with pytest.raises(ValueError, match='717'):
        M.check_partial([0.3, 0.3], 2048)
    with pytest.raises(ValueError):
        M.check_partial([0.7], 2048)
    assert M.check_partial([0.5, 0.5], 2048) == np.float32(0.5)
    assert M.percentile_position(2048, np.float32(0.5)) == (-1, 0.0)
    k, g = M.percentile_position(2048, np.float32(0.7))
    d = np.random.default_rng(0).normal(size=2048)
    s = np.sort(d)
    thr = s[k] + (s[k + 1] - s[k]) * g if g < 0.5 else s[k + 1] - (s[k + 1] - s[k]) * (1 - g)
    assert thr == np.percentile(d, (1.0 - np.float32(0.7)) * 100)
    cfg = get_config('modelnet', noise_type='jitter')
    shapes = M.ModelNetShapes.from_arrays(np.zeros((1, 2048, 3), np.float32))
    with pytest.raises(NotImplementedError, match='RandomCrop'):
        M.ModelNetPairs(shapes, cfg)


def _fake_root(tmp_path, n_per_file=(5, 4)):
    """A ModelNet40 root with shape_names.txt, train/test file lists (with the reference's prefix) and fake h5 data."""
    root = tmp_path / 'modelnet40_ply_hdf5_2048'
    root.mkdir()
    (root / 'shape_names.txt').write_text('airplane\nbathtub\nbed\nbench\n')
    files, rng = {}, np.random.default_rng(0)
    for subset in ('train', 'test'):
        names = [f'ply_data_{subset}{i}.h5' for i in range(len(n_per_file))]
        (root / f'{subset}_files.txt').write_text(''.join(f'data/modelnet40_ply_hdf5_2048/{n}\n' for n in names))
        for n, count in zip(names, n_per_file):
            files[str(root / n)] = {'data': rng.normal(size=(count, 2048, 3)).astype(np.float32),
                                    'normal': rng.normal(size=(count, 2048, 3)).astype(np.float32),
                                    'label': rng.integers(0, 4, size=(count, 1)).astype(np.uint8)}
    fake = types.SimpleNamespace(File=lambda fname, mode='r': files[fname])
    return root, files, fake


def test_dataset_file_lists_categories_and_idx(tmp_path, monkeypatch):
    root, files, fake = _fake_root(tmp_path)
    monkeypatch.setattr(M, 'h5_reader', lambda: fake)
    cat = tmp_path / 'half.txt'
    cat.write_text('bench\nairplane\n')
    cats = M.read_categories(str(cat))
    assert cats == ['airplane', 'bench'] and M.read_categories('') is None
    ds = M.ModelNetShapes(str(root), 'train', cats)
    want_pts, want_lab = [], []
    for i in range(2):
        f = files[str(root / f'ply_data_train{i}.h5')]
        lab = f['label'].flatten().astype(np.int64)
        keep = np.isin(lab, [0, 3])
        want_pts.append(f['data'][keep]); want_lab.append(lab[keep])
    np.testing.assert_array_equal(ds.points, np.concatenate(want_pts))
    np.testing.assert_array_equal(ds.labels, np.concatenate(want_lab))
    assert ds.classes == ['airplane', 'bench'] and len(ds) == len(ds.labels)
    everything = M.ModelNetShapes(str(root), 'test')
    assert len(everything) == 9 and everything.classes == ['airplane', 'bathtub', 'bed', 'bench']
    # idx is the item index after filtering: pair i is the deterministic chain of shape i seeded with i
    cfg = get_config('modelnet')
    pairs = M.ModelNetPairs(M.ModelNetShapes.from_arrays(ds.points[:3]), cfg)
    for i in range(3):
        it = M.crop_chain(ds.points[i], cfg.partial, cfg.rot_mag, cfg.trans_mag, np.random.RandomState(i), idx=i,
                          deterministic=True)
        assert int(pairs[i]['idx']) == i
        np.testing.assert_array_equal(pairs[i]['src_xyz'].numpy(), it['src_xyz'])


def test_h5_read_without_h5py_says_so(monkeypatch):
    import builtins
    real = builtins.__import__

    def no_h5py(name, *a, **k):
        if name == 'h5py':
            raise ImportError('no h5py')
        return real(name, *a, **k)
    monkeypatch.setattr(builtins, '__import__', no_h5py)
    with pytest.raises(NotImplementedError, match='h5'):
        M.read_h5_files(['x.h5'], None)


def test_modelnet_config_has_the_reference_dataset_keys():
    cfg = get_config('modelnet')
    assert cfg.root == '../data/modelnet40_ply_hdf5_2048'
    assert cfg.train_categoryfile == cfg.val_categoryfile == 'datasets/modelnet/modelnet40_half1.txt'
    assert cfg.test_categoryfile == 'datasets/modelnet/modelnet40_half2.txt'
    assert (cfg.partial, cfg.num_points, cfg.noise_type, cfg.rot_mag, cfg.trans_mag) == ([0.7, 0.7], 1024, 'crop', 45.0, 0.5)
    assert (cfg.train_batch_size, cfg.val_batch_size, cfg.test_batch_size, cfg.niter) == (4, 4, 1, -400)


def test_train_cli_builds_both_modelnet_datasets(tmp_path, monkeypatch):
    from regtr_b200 import train
    root, files, fake = _fake_root(tmp_path)
    monkeypatch.setattr(M, 'h5_reader', lambda: fake)
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    (tmp_path / 'datasets' / 'modelnet').mkdir(parents=True)
    (tmp_path / 'datasets' / 'modelnet' / 'modelnet40_half1.txt').write_text('airplane\nbathtub\n')
    (tmp_path / 'datasets' / 'modelnet' / 'modelnet40_half2.txt').write_text('bed\nbench\n')
    cfg = get_config('modelnet', root=str(root))
    train.write_config(cfg, 'modelnet', str(tmp_path / 'cfg.yaml'))
    built = {}
    real_pairs = M.ModelNetPairs

    def pairs(shapes, cfg_, partial=None):
        built['val'] = shapes
        return real_pairs(shapes, cfg_, partial)
    monkeypatch.setattr(M, 'ModelNetPairs', pairs)
    monkeypatch.chdir(tmp_path)
    with pytest.raises(RuntimeError, match='Trainer needs a CUDA device'):
        train.main(['--config', str(tmp_path / 'cfg.yaml'), '--logdir', str(tmp_path / 'logs')])
    lab = np.concatenate([files[str(root / f'ply_data_test{i}.h5')]['label'].flatten() for i in range(2)])
    assert len(built['val']) == int(np.isin(lab, [0, 1]).sum())


def test_modelnet_args_layout_matches_the_header(tmp_path):
    """offsetof / sizeof of regtr_modelnet_args, compiled from the header, against the numpy dtype ops fills."""
    import re
    import shutil
    import subprocess
    from regtr_b200 import lib, ops
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    text = open(lib.HEADER).read()
    assert int(re.search(r'#define REGTR_MODELNET_MAX_PTS (\d+)', text).group(1)) == ops.MODELNET_MAX_PTS
    assert int(re.search(r'#define REGTR_MODELNET_PARAMS (\d+)', text).group(1)) == ops.MODELNET_PARAMS
    dt = ops.MODELNET_ARGS
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{lib.HEADER}"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(regtr_modelnet_args));']
    lines += [f'printf("{f} %zu\\n", offsetof(regtr_modelnet_args, {f}));' for f in dt.names]
    lines += ['return 0;', '}']
    (tmp_path / 'l.c').write_text('\n'.join(lines))
    subprocess.run([cc, str(tmp_path / 'l.c'), '-o', str(tmp_path / 'l')], check=True)
    got = dict(l.split() for l in subprocess.run([str(tmp_path / 'l')], capture_output=True, text=True,
                                                  check=True).stdout.splitlines())
    assert int(got['size']) == dt.itemsize
    for f in dt.names:
        assert int(got[f]) == dt.fields[f][1], f
