"""Training batches on the device (regtr_b200.augment.TrainingPrep): overlap ground truth against the float64
oracle, the shuffle's permutation, perturbation / swap / jitter against the oracle's transforms, determinism, no
host sync, and one training step of the whole path on the two real 3DMatch pairs."""
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import stats

import train_data_oracle as O
from regtr_b200 import augment as A
from regtr_b200 import data as D
from regtr_b200 import ops
from regtr_b200.synthetic import make_3dmatch_pair

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
R = 0.0375


def cfg(radius=R, mode='small', noise=0.005):
    return SimpleNamespace(overlap_radius=radius, perturb_pose=mode, augment_noise=noise)


def batch_of(pairs, pin=True):
    f = (lambda t: t.pin_memory()) if pin else (lambda t: t)
    return {'src_xyz': [f(torch.from_numpy(np.ascontiguousarray(s, np.float64))) for s, _, _ in pairs],
            'tgt_xyz': [f(torch.from_numpy(np.ascontiguousarray(t, np.float64))) for _, t, _ in pairs],
            'pose': torch.from_numpy(np.stack([np.asarray(p, np.float64) for _, _, p in pairs])),
            'src_path': [f's{b}' for b in range(len(pairs))], 'tgt_path': [f't{b}' for b in range(len(pairs))],
            'idx': list(range(len(pairs)))}


def synth(seed, n=20000):
    p = make_3dmatch_pair(seed, n_target=n)
    return p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), p['pose'].astype(np.float64)


def host(out, key):
    return [t.cpu().numpy() for t in out[key]]


def assert_overlap_exact(out, pairs):
    for b, (s, t, p) in enumerate(pairs):
        sm, tm, corr, _, _ = O.overlap(s, t, p, R)
        assert np.array_equal(out['src_overlap'][b].cpu().numpy(), sm), b
        assert np.array_equal(out['tgt_overlap'][b].cpu().numpy(), tm), b
        assert np.array_equal(out['correspondences'][b].cpu().numpy(), corr), b
        assert np.array_equal(out['src_xyz'][b].cpu().numpy(), s.astype(np.float32))


@pytest.mark.parametrize('sizes', [(20000,), (20000, 9000, 14000)])
def test_overlap_exact_vs_oracle_synthetic(sizes):
    pairs = [synth(100 + i, n) for i, n in enumerate(sizes)]
    out = A.TrainingPrep(cfg())(batch_of(pairs), augment=False)
    assert_overlap_exact(out, pairs)
    assert np.array_equal(out['pose'].cpu().numpy(), np.stack([p for _, _, p in pairs]).astype(np.float32))
    # the nearest indices themselves
    xyz = torch.from_numpy(np.concatenate([s for s, _, _ in pairs] + [t for _, t, _ in pairs])).cuda()
    lens = [len(s) for s, _, _ in pairs] + [len(t) for _, t, _ in pairs]
    nn = ops.overlap_nn(xyz, ops.make_offsets(lens, xyz.device), len(pairs),
                        torch.from_numpy(np.stack([p for _, _, p in pairs])).cuda(), R,
                        ops.new_status(xyz.device)).cpu().numpy()
    o = np.concatenate([[0], np.cumsum(lens)])
    B = len(pairs)
    for b, (s, t, p) in enumerate(pairs):
        _, _, _, s2t, t2s = O.overlap(s, t, p, R)
        assert np.array_equal(nn[o[b]:o[b + 1]], s2t) and np.array_equal(nn[o[B + b]:o[B + b + 1]], t2s)


def test_overlap_exact_on_the_real_pairs():
    pairs = [(s, t, p) for s, t, p, _ in O.real_pairs(GOLDEN)]
    out = A.TrainingPrep(cfg())(batch_of(pairs), augment=False)
    assert_overlap_exact(out, pairs)
    for b, (s, t, p) in enumerate(pairs):
        sm, tm, corr = D.compute_overlap(s @ p[:, :3].T + p[:, 3], t, R)
        assert np.array_equal(out['src_overlap'][b].cpu().numpy(), sm)
        assert np.array_equal(out['tgt_overlap'][b].cpu().numpy(), tm)
        assert np.array_equal(out['correspondences'][b].cpu().numpy(), corr)


def test_overlap_edge_cases():
    eye = np.eye(3, 4)
    tgt = np.array([[0.0, 0, 0], [0.5, 0, 0], [0.25, 0, 0], [0.25, 0, 0]])
    src = np.array([[0.25, 0, 0], [0.75, 0, 0], [0.125, 0, 0], [2.0, 0, 0]])
    pairs = [(src, tgt, eye), (np.zeros((0, 3)), tgt, eye), (src[:1], tgt[:1], eye), (src, np.zeros((0, 3)), eye),
             (src[2:3], tgt[:1], eye)]
    out = A.TrainingPrep(cfg(radius=0.25))(batch_of(pairs), augment=False)
    for b, (s, t, p) in enumerate(pairs):
        sm, tm, corr, _, _ = O.overlap(s, t, p, 0.25)
        assert np.array_equal(out['src_overlap'][b].cpu().numpy(), sm), b
        assert np.array_equal(out['tgt_overlap'][b].cpu().numpy(), tm), b
        assert np.array_equal(out['correspondences'][b].cpu().numpy().reshape(2, -1), corr), b
    # exactly r away does not count, ties go to the lowest index, a match to target 0 is never a correspondence
    assert out['src_overlap'][0].tolist() == [True, False, True, False]
    assert out['correspondences'][0].tolist() == [[0], [2]]
    assert out['correspondences'][4].shape == (2, 0) and out['src_overlap'][4].tolist() == [True]


def test_batch_invariance():
    pairs = [synth(200 + i, n) for i, n in enumerate((6000, 11000, 3000))]
    prep = A.TrainingPrep(cfg())
    full = prep(batch_of(pairs), augment=False)
    for b in range(3):
        one = prep(batch_of(pairs[b:b + 1]), augment=False)
        for k in ('src_xyz', 'tgt_xyz', 'src_overlap', 'tgt_overlap', 'correspondences'):
            assert torch.equal(full[k][b], one[k][0]), (b, k)


def test_range_bound():
    bound = ops.overlap_coord_bound(R)
    assert 140 < bound < 170
    for scale, bad in ((0.999, False), (1.001, True)):
        far = np.array([[bound * scale, 0.0, 0.0], [0.0, 0.0, 0.0]])
        prep = A.TrainingPrep(cfg())
        prep(batch_of([(far, far, np.eye(3, 4))]), augment=False)
        if bad:
            with pytest.raises(ValueError, match='beyond'):
                prep.check()
        else:
            prep.check()


def lattice(n, shift=0.0):
    i = np.arange(n)
    return np.stack([i % 100, (i // 100) % 100, i // 10000], axis=1) * 0.01 + shift


def decode(x, shift=0.0):
    k = np.rint((np.asarray(x, np.float64) - shift) * 100).astype(np.int64)
    return k[:, 0] + 100 * k[:, 1] + 10000 * k[:, 2]


SHIFT = 0.003


def recovered_perms(out, B, shifts=(0.0, SHIFT)):
    """Input-side permutations (src, tgt) of every pair from a perturb-'none', noise-0 run on lattice clouds."""
    perms = []
    for b in range(B):
        sw = bool(out['aug']['swap'][b])
        s, t = out['src_xyz'][b].cpu().numpy(), out['tgt_xyz'][b].cpu().numpy()
        if sw:
            s, t = t, s
        perms.append((decode(s, shifts[0]), decode(t, shifts[1])))
    return perms


def test_shuffle_is_a_truncated_bijection_and_masks_follow():
    sizes = [1, 2, 29999, 30000, 30001, 45000]
    pairs = [(lattice(n), lattice(min(n, 500), SHIFT), np.eye(3, 4)) for n in sizes]
    prep = A.TrainingPrep(cfg(mode='none', noise=0.0), seed=5)
    out = prep(batch_of(pairs))
    for b, (sp, tp) in enumerate(recovered_perms(out, len(sizes))):
        n = sizes[b]
        assert len(sp) == min(n, 30000) and len(np.unique(sp)) == len(sp) and sp.min() >= 0 and sp.max() < n
        s, t, p = pairs[b]
        sm, tm, corr, _, _ = O.overlap(s, t, p, R)
        ref = O.shuffle_points(dict(src_xyz=s, tgt_xyz=t, src_overlap=sm, tgt_overlap=tm, correspondences=corr),
                               sp, tp)
        ref = O.random_swap(ref, bool(out['aug']['swap'][b]))
        for k in ('src_overlap', 'tgt_overlap'):
            assert np.array_equal(out[k][b].cpu().numpy(), ref[k]), (b, k)
        assert np.array_equal(out['correspondences'][b].cpu().numpy().reshape(2, -1), ref['correspondences']), b
    # position against index over many steps: uniform
    n, B = 32, 8
    counts = np.zeros((n, n))
    pairs = [(lattice(n), lattice(n, SHIFT), np.eye(3, 4))] * B
    batch = batch_of(pairs)
    for _ in range(200):
        for sp, tp in recovered_perms(prep(batch), B):
            counts[np.arange(n), sp] += 1
            counts[np.arange(n), tp] += 1
    chi2 = ((counts - counts.mean()) ** 2 / counts.mean()).sum()
    assert stats.chi2.sf(chi2, (n - 1) ** 2) > 1e-4, chi2


@pytest.mark.parametrize('mode', ['small', 'large', 'none'])
def test_perturb_and_swap_vs_oracle(mode):
    B = 4
    pairs = [(lattice(3000 + 700 * b, -0.2), lattice(2500 + 300 * b, SHIFT - 0.2), np.eye(3, 4)) for b in range(B)]
    batch = batch_of(pairs)
    plain = A.TrainingPrep(cfg(mode='none', noise=0.0), seed=9)
    prep = A.TrainingPrep(cfg(mode=mode, noise=0.0), seed=9)
    swaps = set()
    for _ in range(3):
        ref_out, out = plain(batch), prep(batch)
        perms = recovered_perms(ref_out, B, (-0.2, SHIFT - 0.2))
        aug = out['aug']
        for b in range(B):
            s, t, p = pairs[b]
            d = dict(src_xyz=s, tgt_xyz=t, pose=p)
            if mode != 'none':
                d = O.rigid_perturb(d, aug['perturb'][b], bool(aug['perturb_source'][b]), centre=mode == 'small')
            d = O.random_swap(O.shuffle_points(d, *perms[b]), bool(aug['swap'][b]))
            swaps.add(bool(aug['swap'][b]))
            for k in ('src_xyz', 'tgt_xyz'):
                got = out[k][b].cpu().numpy().astype(np.float64)
                assert np.abs(got - d[k]).max() <= 4e-7 * np.abs(d[k]).max(), (mode, b, k)
            assert np.abs(out['pose'][b].cpu().numpy() - d['pose']).max() <= 1e-6, (mode, b)
    assert swaps == {False, True}


def test_jitter_statistics():
    B, n = 8, 30000
    pairs = [synth(300 + b, 15000)[:2] + (np.eye(3, 4),) for b in range(B)]
    pairs = [(np.resize(s, (n, 3)), np.resize(t, (n, 3)), p) for s, t, p in pairs]
    batch = batch_of(pairs)
    noisy, clean = A.TrainingPrep(cfg(mode='none'), seed=3), A.TrainingPrep(cfg(mode='none', noise=0.0), seed=3)
    diffs = []
    for _ in range(3):
        a, b = noisy(batch), clean(batch)
        for k in ('src_xyz', 'tgt_xyz'):
            diffs += [(x.double() - y.double()).cpu().numpy() for x, y in zip(a[k], b[k])]
    d = np.concatenate(diffs)
    assert d.size >= 3e6
    m, s = d.mean(axis=0), d.std(axis=0)
    assert np.all(np.abs(m) < 5 * 0.005 / np.sqrt(d.shape[0])), m
    assert np.all(np.abs(s / 0.005 - 1) < 5 / np.sqrt(2 * d.shape[0])), s
    for a in range(3):          # per axis: the three values of a point come from shared Box-Muller pairs
        assert stats.kstest(d[:, a], stats.norm(0, 0.005).cdf).pvalue > 1e-3, a


def test_determinism_sync_and_launches():
    pairs = [synth(400 + b, 8000) for b in range(3)]
    batch = batch_of(pairs)
    keys = ('src_xyz', 'tgt_xyz', 'src_overlap', 'tgt_overlap', 'correspondences')
    a, b = A.TrainingPrep(cfg(), seed=1)(batch), A.TrainingPrep(cfg(), seed=1)(batch)
    for k in keys:
        assert all(torch.equal(x, y) for x, y in zip(a[k], b[k])), k
    assert torch.equal(a['pose'], b['pose'])
    prep = A.TrainingPrep(cfg(), seed=1)
    prep(batch)
    c = prep(batch)
    assert not torch.equal(a['src_xyz'][0][:100], c['src_xyz'][0][:100])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        prep(batch)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    counts = []
    for B in (1, 8):
        bb = batch_of([synth(500 + i, 4000) for i in range(B)])
        n0 = ops.LAUNCHES
        prep(bb)
        counts.append(ops.LAUNCHES - n0)
    assert counts[0] == counts[1] > 0, counts
    prep.check()


def _write_real(root):
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    for s, t, p, row in O.real_pairs(GOLDEN):
        for rel, x in ((row['src'], s), (row['tgt'], t)):
            os.makedirs(root / os.path.dirname(rel), exist_ok=True)
            torch.save(x, root / rel)
        infos['rot'].append(p[:, :3]); infos['trans'].append(p[:, 3:])
        infos['src'].append(row['src']); infos['tgt'].append(row['tgt']); infos['overlap'].append(row['overlap'])
    with open(root / 'info.pkl', 'wb') as f:
        pickle.dump(infos, f)
    return str(root), str(root / 'info.pkl')


def test_end_to_end_training_step_on_real_pairs(tmp_path):
    from regtr_b200 import optim
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.weights import random_state_dict
    root, info = _write_real(tmp_path)
    mcfg = get_config('3dmatch')
    ds = D.ThreeDMatchPairs(root, info, pin=True, float64=True)

    def run():
        model = RegTR(mcfg).cuda()
        model.load_state_dict(random_state_dict(mcfg, 11), strict=True)
        opt = optim.AdamW(model.parameters(), lr=1e-4, weight_decay=1e-4)
        prep = A.TrainingPrep(mcfg, seed=21)
        losses = []
        for batch in D.PairStream(ds, [[0, 1]], workers=2):
            b = prep(batch)
            pred = model.forward_train(b, train_encoder=True)
            loss = model.compute_loss(pred, b)
            assert all(bool(torch.isfinite(v).all()) for v in loss.values())
            assert torch.equal(b['overlap_pyr']['pyr_0'].bool(), torch.cat(b['src_overlap'] + b['tgt_overlap']))
            opt.zero_grad(set_to_none=True)
            loss['total'].backward()
            optim.clip_grad_norm_(model.parameters(), 0.1)
            opt.step()
            losses.append({k: v.detach().cpu() for k, v in loss.items()})
        prep.check()
        return losses
    l1, l2 = run(), run()
    assert all(torch.equal(a[k], b[k]) for a, b in zip(l1, l2) for k in a)
    # the val phase equals the CPU loader's overlap
    ref = D.ThreeDMatchPairs(root, info, overlap_radius=R)
    out = A.TrainingPrep(mcfg)(D.collate_pair([ds[0], ds[1]]), augment=False)
    for b in range(2):
        it = ref[b]
        for k in ('src_overlap', 'tgt_overlap', 'correspondences'):
            assert np.array_equal(out[k][b].cpu().numpy(), it[k].numpy()), (b, k)
