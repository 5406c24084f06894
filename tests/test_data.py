"""CPU tests of the input pipeline (SURVEY.md 8f N2, regtr_b200/data.py): file formats of the reference's
3DMatch loader, collate layout, size bucketing, read-ahead stream.  What the reference's own functions return
on the same inputs is stored in tests/golden/data.npz (tests/golden/make_golden.py)."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden
from regtr_b200 import data as D

COLLATE_ITEMS = (4, 0, 7)


def _make_dataset(tmp_path, n_pairs=11, seed=0):
    rng = np.random.default_rng(seed)
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    os.makedirs(tmp_path / 'test' / 'scene', exist_ok=True)
    for i in range(n_pairs + 1):
        pts = rng.normal(size=(int(rng.integers(50, 400)), 3))                      # float64, like the real files
        torch.save(pts, tmp_path / 'test' / 'scene' / f'cloud_bin_{i}.pth')
    for i in range(n_pairs):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        infos['rot'].append(q); infos['trans'].append(rng.normal(size=(3, 1)))
        infos['src'].append(f'test/scene/cloud_bin_{i + 1}.pth'); infos['tgt'].append(f'test/scene/cloud_bin_{i}.pth')
        infos['overlap'].append(float(rng.uniform(0.1, 0.9)))
    with open(tmp_path / 'info.pkl', 'wb') as f:
        pickle.dump(infos, f)
    return D.ThreeDMatchPairs(str(tmp_path), str(tmp_path / 'info.pkl')), infos


def test_dataset_items_and_collate(tmp_path):
    ds, infos = _make_dataset(tmp_path)
    assert len(ds) == 11
    it = ds[3]
    assert it['src_xyz'].dtype == torch.float32 and it['src_xyz'].shape[1] == 3
    assert it['pose'].shape == (3, 4) and it['idx'] == 3 and it['src_path'].endswith('cloud_bin_4.pth')
    np.testing.assert_allclose(it['pose'][:, :3].numpy(), infos['rot'][3], atol=1e-6)
    np.testing.assert_allclose(it['pose'][:, 3:].numpy(), infos['trans'][3], atol=1e-6)
    b = D.collate_pair([ds[0], ds[1], ds[2]])
    assert isinstance(b['src_xyz'], list) and len(b['tgt_xyz']) == 3 and b['pose'].shape == (3, 3, 4)
    assert b['overlap_p'].shape == (3,) and b['idx'] == [0, 1, 2]


def encode_collate(batch):
    """A collated batch as flat arrays: 'collate/<key>' for a tensor, 'collate/<key>/<i>' for list entries, plus
    the key list and which keys are lists."""
    fx = {'collate/__keys__': np.array(sorted(batch)),
          'collate/__lists__': np.array(sorted(k for k, v in batch.items() if isinstance(v, list)))}
    for k, v in batch.items():
        for name, x in ([(f'collate/{k}', v)] if torch.is_tensor(v) else
                        [(f'collate/{k}/{i}', x) for i, x in enumerate(v)]):
            fx[name] = x.numpy() if torch.is_tensor(x) else np.array(x)
    return fx


def seq_inputs():
    rng = np.random.default_rng(2)
    seqs = [torch.from_numpy(rng.normal(size=(n, 5)).astype(np.float32)) for n in (7, 3, 11, 1)]
    six = torch.from_numpy(rng.normal(size=(6, 11, 4, 5)).astype(np.float32))
    return seqs, six


def encode_seq(S, seqs, six):
    """Outputs of pad_sequence / unpad_sequences / split_src_tgt of module S on the inputs above, as flat arrays."""
    fx = {}
    lens = [len(x) for x in seqs]
    for name, kw in (('plain', dict()), ('mask_lens', dict(require_padding_mask=True, require_lens=True))):
        padded, mask, plens = S.pad_sequence(seqs, **kw)
        fx[f'seq/pad_{name}'] = padded.numpy()
        fx[f'seq/pad_{name}_mask'] = np.zeros(0, bool) if mask is None else mask.numpy()
        fx[f'seq/pad_{name}_lens'] = np.array(-1 if plens is None else plens)
    for b, x in enumerate(S.unpad_sequences(six, lens)):
        fx[f'seq/unpad_{b}'] = x.numpy()
    src, tgt = S.split_src_tgt(torch.cat(seqs), lens)
    for side, xs in (('src', src), ('tgt', tgt)):
        for i, x in enumerate(xs):
            fx[f'seq/split_{side}_{i}'] = x.numpy()
    return fx


def assert_same_arrays(got, want, prefix):
    want = {k: v for k, v in want.items() if k.startswith(prefix)}
    assert set(got) == set(want)
    for k, v in want.items():
        assert got[k].dtype == v.dtype and got[k].shape == v.shape and np.array_equal(got[k], v), k


def test_collate_matches_reference_function(tmp_path):
    """collate_pair vs what the reference's collate_functions.collate_pair returned on the same items."""
    ds, _ = _make_dataset(tmp_path)
    got = encode_collate(D.collate_pair([ds[i] for i in COLLATE_ITEMS]))
    assert_same_arrays(got, load_golden('data'), 'collate/')


def test_reads_the_reference_sample_pairs(tmp_path):
    """The reference's two shipped 3DMatch benchmark pairs (data/indoor, demo.py) through a benchmark pickle with
    their real rows, the clouds stored as the dataset stores them (float64 .pth under test/<scene>/)."""
    rows = json.load(open(os.path.join(GOLDEN, 'real', 'test_3DMatch_info_rows.json')))
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    raws = {}
    for r in rows:
        inp = np.load(os.path.join(GOLDEN, 'real', r['fixture'] + '_input.npz'))
        for rel in (r['src'], r['tgt']):
            which = 'src_xyz' if os.path.basename(rel) == os.path.basename(str(inp['src_file'])) else 'tgt_xyz'
            os.makedirs(tmp_path / 'indoor' / os.path.dirname(rel), exist_ok=True)
            raws[rel] = inp[which].astype(np.float64)
            torch.save(raws[rel], tmp_path / 'indoor' / rel)
        for k in ('rot', 'trans'):
            infos[k].append(np.array(r[k]))
        for k in ('src', 'tgt', 'overlap'):
            infos[k].append(r[k])
    with open(tmp_path / 'info.pkl', 'wb') as f:
        pickle.dump(infos, f)
    root = str(tmp_path / 'indoor')
    ds = D.ThreeDMatchPairs(root, str(tmp_path / 'info.pkl'))
    assert len(ds) == len(rows) == 2
    for i, r in enumerate(rows):
        it = ds[i]
        raw = torch.load(os.path.join(root, it['src_path']), weights_only=False)
        assert raw.dtype == np.float64 and np.array_equal(raw, raws[r['src']])
        assert torch.equal(it['src_xyz'], torch.from_numpy(raw).float())
        assert 5000 < it['src_xyz'].shape[0] < 60000 and it['pose'].shape == (3, 4)
        np.testing.assert_allclose(it['pose'][:, :3].numpy(), np.array(r['rot']), atol=1e-6)
        np.testing.assert_allclose(it['pose'][:, 3:].numpy(), np.array(r['trans']), atol=1e-6)


def test_bucket_order_is_a_partition_grouped_by_capacity():
    rng = np.random.default_rng(1)
    sizes = rng.integers(20000, 60000, size=200).tolist()
    batches = D.bucket_order(sizes, batch_size=4, bucket=8192, window=64)
    flat = [i for b in batches for i in b]
    assert sorted(flat) == list(range(200))
    assert all(len(b) <= 4 for b in batches)
    assert max(flat[:64]) < 64 and min(flat[64:128]) >= 64                   # windows keep the dataset order
    cap = lambda i: -(-sizes[i] // 8192)
    assert all(cap(a) <= cap(b) for a, b in zip(flat[:63], flat[1:64]))       # grouped by bucket inside a window
    changes = sum(cap(a) != cap(b) for a, b in zip(flat, flat[1:]))
    naive = sum(cap(a) != cap(b) for a, b in zip(range(199), range(1, 200)))
    assert changes < naive / 3                                                # far fewer graph switches


def test_pair_stream_order_and_errors(tmp_path):
    ds, _ = _make_dataset(tmp_path, n_pairs=23)
    batches = D.bucket_order(ds.sizes(), batch_size=3, bucket=256, window=8)
    got = [b['idx'] for b in D.PairStream(ds, batches, workers=3, depth=2)]
    assert got == [list(b) for b in batches]
    os.remove(tmp_path / 'test' / 'scene' / 'cloud_bin_5.pth')
    with pytest.raises(Exception):
        list(D.PairStream(ds, batches, workers=2, depth=2))


def test_sequence_helpers_match_reference():
    """regtr_b200.seq vs what utils/seq_manipulation.py returned on the same inputs, plus a padded round trip."""
    from regtr_b200 import seq as S
    seqs, six = seq_inputs()
    padded, mask, lens = S.pad_sequence(seqs, require_padding_mask=True, require_lens=True)
    assert padded.shape == (11, 4, 5) and mask.shape == (4, 11) and lens == [7, 3, 11, 1]
    assert mask[1, 3:].all() and not mask[1, :3].any() and not mask[2].any()
    back = S.unpad_sequences(padded, lens)
    assert all(torch.equal(a, b) for a, b in zip(back, seqs))
    stacked = torch.cat(seqs)
    src, tgt = S.split_src_tgt(stacked, torch.tensor(lens))
    assert len(src) == 2 and torch.equal(tgt[1], seqs[3])
    assert_same_arrays(encode_seq(S, seqs, six), load_golden('data'), 'seq/')


def test_compute_overlap_properties(tmp_path):
    rng = np.random.default_rng(4)
    tgt = rng.uniform(0, 1, size=(400, 3))
    src = np.concatenate([tgt[:250] + rng.normal(scale=0.002, size=(250, 3)), rng.uniform(2, 3, size=(80, 3))])
    sm, tm, corr = D.compute_overlap(src, tgt, 0.02)
    assert sm[:250].all() and not sm[250:].any()                 # the shifted copies overlap, the far blob does not
    assert tm[:250].all() and tm[250:].sum() < 40
    s_idx, t_idx = corr
    assert (np.linalg.norm(src[s_idx] - tgt[t_idx], axis=1) < 0.02).all()
    assert (s_idx[t_idx == s_idx] > 0).all() and len(s_idx) > 200     # mutual matches, index 0 excluded (reference quirk)
    # brute-force nearest neighbour agrees
    d = np.linalg.norm(src[:, None] - tgt[None], axis=-1)
    assert np.array_equal(sm, d.min(1) < 0.02)
    ds, infos = _make_dataset(tmp_path)
    ds.overlap_radius = 0.5
    it = ds[2]
    assert it['src_overlap'].dtype == torch.bool and it['src_overlap'].shape[0] == it['src_xyz'].shape[0]
    assert it['correspondences'].shape[0] == 2
    b = D.collate_pair([ds[0], ds[1]])
    assert isinstance(b['correspondences'], list) and len(b['src_overlap']) == 2
