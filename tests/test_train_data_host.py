"""CPU checks of the training-data path: the float64 oracle against the reference's own transforms
(tests/golden/augment.npz) and against data.compute_overlap, the host sampler of augment.TrainingPrep, and the
float64 mode of ThreeDMatchPairs."""
import os
import pickle

import numpy as np
import pytest
import torch
from scipy import stats
from scipy.spatial.transform import Rotation

import train_data_oracle as O
from regtr_b200 import augment as A
from regtr_b200 import data as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
RADIUS = 0.0375


def _cases():
    z = np.load(os.path.join(GOLDEN, 'augment.npz'))
    n = len({k.split('/')[0] for k in z.files})
    for i in range(n):
        p = f'case{i}/'
        yield {k[len(p):]: z[k] for k in z.files if k.startswith(p)}


def _draws(case):
    return [case[k] for k in sorted(k for k in case if k.startswith('draw'))]


def test_oracle_transforms_reproduce_reference():
    seen = set()
    for c in _cases():
        mode, max_pts = str(c['mode']), int(c['max_pts'])
        d = list(_draws(c))
        data = dict(src_xyz=c['in_src'], tgt_xyz=c['in_tgt'], pose=c['in_pose'], src_overlap=c['in_src_overlap'],
                    tgt_overlap=c['in_tgt_overlap'], correspondences=c['in_corr'])
        if mode == 'small':
            P = O.pose_small(d[0], d[1], d[2], d[3])
            d = d[4:]
        elif mode == 'large':
            P = O.pose_large(d[0] * np.pi * 2)             # np.random.rand(3) * np.pi * 2
            d = d[1:]
        if mode != 'none':
            data = O.rigid_perturb(data, P, bool(d[0] > 0.5), centre=mode == 'small')
            d = d[1:]
        data = O.jitter(data, d[0].astype(np.float64) * 0.005, d[1].astype(np.float64) * 0.005)
        data = O.shuffle_points(data, d[2][:max_pts], d[3][:max_pts])
        swap = bool(d[4] > 0.5)
        assert swap == bool(c['swapped'])
        data = O.random_swap(data, swap)
        for k in ('src_overlap', 'tgt_overlap', 'correspondences'):
            assert np.array_equal(data[k], c['out_' + k]), k
        for k in ('src_xyz', 'tgt_xyz'):
            ref = c['out_' + k].astype(np.float64)
            assert np.abs(data[k] - ref).max() <= 1e-6 * np.abs(ref).max(), k
        assert np.abs(data['pose'] - c['out_pose']).max() <= 1e-6 * max(1.0, np.abs(c['out_pose']).max())
        seen.add((mode, max_pts < len(c['in_src']), swap))
    assert {m for m, _, _ in seen} == {'small', 'large', 'none'}
    assert {(t, s) for _, t, s in seen} == {(a, b) for a in (False, True) for b in (False, True)}


def test_oracle_overlap_equals_compute_overlap_seeded():
    rng = np.random.default_rng(11)
    for n in (50, 700):
        tgt = rng.uniform(0, 0.5, size=(n, 3))
        src = np.concatenate([tgt[: n // 2] + rng.normal(scale=0.01, size=(n // 2, 3)), rng.uniform(1, 2, (20, 3))])
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        pose = np.concatenate([q, rng.normal(size=(3, 1))], axis=1)
        src_in = (src - pose[:, 3]) @ q                      # pose maps src_in back onto src
        sm, tm, corr, _, _ = O.overlap(src_in, tgt, pose, 0.05)
        rsm, rtm, rcorr = D.compute_overlap(O.align(src_in, pose), tgt, 0.05)
        assert np.array_equal(sm, rsm) and np.array_equal(tm, rtm) and np.array_equal(corr, rcorr)


def test_oracle_overlap_on_the_real_pairs():
    for src, tgt, pose, row in O.real_pairs(GOLDEN):
        sm, tm, corr, s2t, t2s = O.overlap(src, tgt, pose, RADIUS)
        rsm, rtm, rcorr = D.compute_overlap(src @ pose[:, :3].T + pose[:, 3], tgt, RADIUS)
        assert np.array_equal(sm, rsm) and np.array_equal(tm, rtm) and np.array_equal(corr, rcorr)
        assert 0.44 <= sm.mean() <= 0.59 and 0.44 <= tm.mean() <= 0.59, (sm.mean(), tm.mean())
        assert 3500 <= corr.shape[1] <= 6000


def test_oracle_nearest_within_rules():
    b = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.25, 0.0, 0.0], [0.25, 0.0, 0.0]])
    a = np.array([[0.25, 0.0, 0.0], [0.75, 0.0, 0.0], [0.125, 0.0, 0.0], [2.0, 0.0, 0.0]])
    # exactly r = 0.25 away does not count; ties go to the lowest index
    assert O.nearest_within(a, b, 0.25).tolist() == [2, -1, 0, -1]


def test_host_sampler_distributions():
    B, steps = 8, 500
    d = [A.sample_draws(3, s, B) for s in range(steps)]
    angle = np.concatenate([x['angle'] for x in d])
    trans = np.concatenate([x['trans'] for x in d]).ravel()
    axis = np.concatenate([x['axis'] for x in d])
    assert stats.kstest(angle, stats.norm(0, 0.1 * np.pi / np.sqrt(3)).cdf).pvalue > 1e-3
    assert stats.kstest(trans, stats.norm(0, 0.1 / np.sqrt(3)).cdf).pvalue > 1e-3
    assert stats.kstest(axis[:, 2], stats.uniform(-1, 2).cdf).pvalue > 1e-3       # uniform on the sphere
    assert np.allclose(np.linalg.norm(axis, axis=1), 1.0)
    euler = np.concatenate([x['euler'] for x in d]).ravel()
    assert stats.kstest(euler, stats.uniform(0, 2 * np.pi).cdf).pvalue > 1e-3
    n = B * steps
    for k in ('perturb_source', 'swap'):
        hits = int(np.concatenate([x[k] for x in d]).sum())
        lo, hi = stats.binom.ppf([1e-4, 1 - 1e-4], n, 0.5)
        assert lo <= hits <= hi, (k, hits)


def test_host_draws_depend_on_seed_step_and_pair_only():
    a, b = A.sample_draws(5, 9, 6), A.sample_draws(5, 9, 2)
    for k in a:
        assert np.array_equal(a[k][:2], b[k]), k
    assert not np.array_equal(A.sample_draws(5, 10, 2)['angle'], b['angle'])
    # the perturbation of every mode is built from the same block
    for mode in ('small', 'large', 'none'):
        P = A.perturbations(a, mode)
        assert P.shape == (6, 3, 4)
        assert np.allclose(P[:, :, :3] @ P[:, :, :3].transpose(0, 2, 1), np.eye(3), atol=1e-12)
    P = A.perturbations(a, 'small')
    for i in range(6):
        assert np.allclose(P[i, :, :3], O.axis_angle(a['axis'][i], a['angle'][i]), atol=1e-14)
        assert np.allclose(P[i, :, 3], a['trans'][i])
    P = A.perturbations(a, 'large')
    assert np.allclose(P[:, :, :3], Rotation.from_euler('zyx', a['euler']).as_matrix(), atol=1e-13)
    assert np.all(P[:, :, 3] == 0)


def _write_pairs(tmp_path):
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    for i, (src, tgt, pose, row) in enumerate(O.real_pairs(GOLDEN)):
        for rel, x in ((row['src'], src), (row['tgt'], tgt)):
            os.makedirs(tmp_path / os.path.dirname(rel), exist_ok=True)
            torch.save(x, tmp_path / rel)
        infos['rot'].append(pose[:, :3]); infos['trans'].append(pose[:, 3:])
        infos['src'].append(row['src']); infos['tgt'].append(row['tgt']); infos['overlap'].append(row['overlap'])
    with open(tmp_path / 'info.pkl', 'wb') as f:
        pickle.dump(infos, f)
    return str(tmp_path), str(tmp_path / 'info.pkl')


def test_threedmatch_pairs_float64(tmp_path):
    root, info = _write_pairs(tmp_path)
    ds = D.ThreeDMatchPairs(root, info, float64=True)
    it = ds[0]
    assert it['src_xyz'].dtype == it['tgt_xyz'].dtype == it['pose'].dtype == torch.float64
    assert set(it) == {'src_xyz', 'tgt_xyz', 'pose', 'idx', 'src_path', 'tgt_path', 'overlap_p'}
    src, tgt, pose, _ = O.real_pairs(GOLDEN)[0]
    assert np.array_equal(it['src_xyz'].numpy(), src) and np.array_equal(it['pose'].numpy(), pose)
    b = D.collate_pair([ds[0], ds[1]])
    assert b['pose'].dtype == torch.float64 and b['pose'].shape == (2, 3, 4)
    assert D.ThreeDMatchPairs(root, info)[0]['src_xyz'].dtype == torch.float32       # default unchanged
    with pytest.raises(ValueError):
        D.ThreeDMatchPairs(root, info, float64=True, overlap_radius=RADIUS)
