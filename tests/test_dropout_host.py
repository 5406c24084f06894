"""Host tests of the cross-encoder dropout: construction and checkpoint layout at p > 0, and the statistics and
stream separation of the keep rule (tests/dropout_rule.py, the restatement of regtr_b200/csrc/philox.cuh)."""
import os
import zlib

import numpy as np
import pytest
import torch

import dropout_rule as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.mark.parametrize('p', [0.1, 0.5])
def test_dropout_models_build_and_keep_the_checkpoint_layout(p):
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.transformer import TransformerCrossEncoderLayer
    from regtr_b200.weights import random_state_dict
    for name in ('modelnet', '3dmatch'):
        m0, m = RegTR(get_config(name)), RegTR(get_config(name, dropout=p))
        assert m.transformer_encoder.dropout_p == p
        sd0 = m0.state_dict()
        assert list(m.state_dict()) == list(sd0)                            # no state: same keys, same order
        ref = random_state_dict(get_config(name, dropout=p), 0)             # the project's checkpoint spec
        assert set(ref) == set(sd0)
        m.load_state_dict(ref, strict=True)
        m0.load_state_dict(m.state_dict(), strict=True)
    assert TransformerCrossEncoderLayer(256, 8, 1024, p, normalize_before=True).dropout_p == p


@pytest.mark.parametrize('p', [-0.1, 1.0, 1.5, float('nan')])
def test_dropout_outside_unit_interval_raises(p):
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.transformer import TransformerCrossEncoderLayer
    with pytest.raises(ValueError):
        TransformerCrossEncoderLayer(256, 8, 1024, p)
    with pytest.raises(ValueError):
        RegTR(get_config('modelnet', dropout=p))


def test_threshold_and_scale():
    for p in (0.1, 0.25, 0.5, 1e-6, 0.999):
        assert abs(R.threshold(p) / 65536 - p) <= 2 ** -16
        assert R.scale(p) == np.float32(1.0 / (1.0 - p))
    from regtr_b200 import ops
    assert ops.dropout_threshold(0.1) == R.threshold(0.1) == 6554
    assert ops.dropout_scale(0.1) == float(R.scale(0.1))


def test_philox_known_answer():
    """Philox4x32-10 known-answer vectors of the Random123 distribution (counter, key -> output)."""
    got = R.philox((0, 0, 0, 0), 0, 0)
    assert [int(v) for v in got] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    got = R.philox((0xFFFFFFFF,) * 4, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(v) for v in got] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_keep_rate_within_5_sigma():
    for p in (0.1, 0.5):
        m = R.keep_mask(p, seed=1234, step=7, cloud=3, layer=2, site=1, head=5, rows=1024, cols=1024)
        n = m.size
        q = 1 - R.threshold(p) / 65536
        assert abs(m.mean() - q) <= 5 * np.sqrt(q * (1 - q) / n), (p, m.mean())


def test_masks_uncorrelated_across_every_key_field():
    """Pearson correlation of two masks that differ in one field (layer, site, head, step, pair, side, seed) or are
    the same mask shifted by one row / column: within 5 sigma of 0."""
    p, rows, cols = 0.1, 512, 512
    base = dict(seed=99, step=3, cloud=2 * 5 + 0, layer=1, site=3, head=2)
    a = R.keep_mask(p, rows=rows, cols=cols, **base).astype(np.float64)
    variants = {'layer': dict(layer=2), 'site': dict(site=4), 'head': dict(head=3), 'step': dict(step=4),
                'pair': dict(cloud=2 * 6 + 0), 'side': dict(cloud=2 * 5 + 1), 'seed': dict(seed=100)}
    bound = 5 / np.sqrt(rows * cols)
    for name, over in variants.items():
        b = R.keep_mask(p, rows=rows, cols=cols, **dict(base, **over)).astype(np.float64)
        assert (a != b).any(), name
        r = np.corrcoef(a.ravel(), b.ravel())[0, 1]
        assert abs(r) <= bound, (name, r)
    for name, (x, y) in {'row': (a[1:], a[:-1]), 'row+8': (a[8:], a[:-8]), 'col': (a[:, 1:], a[:, :-1])}.items():
        r = np.corrcoef(x.ravel(), y.ravel())[0, 1]
        assert abs(r) <= 5 / np.sqrt(x.size), (name, r)


def test_rank_invariance_of_the_mask_key():
    """A pair's masks depend on its global index only: pair 3 alone (pair_base 3, B 1) or inside a batch of 4
    starting at pair 1 (local clouds 2 and 6)."""
    kw = dict(p=0.1, seed=5, step=11, layer=0, site=1, head=0, rows=40, cols=33)
    for side in (0, 1):
        alone = R.local_keep_mask(pair_base=3, n_pairs=1, local=side, **kw)
        inside = R.local_keep_mask(pair_base=1, n_pairs=4, local=2 + 4 * side, **kw)
        assert np.array_equal(alone, inside)
    assert not np.array_equal(R.local_keep_mask(pair_base=3, n_pairs=1, local=0, **kw),
                              R.local_keep_mask(pair_base=3, n_pairs=1, local=1, **kw))


def test_dropout_streams_disjoint_from_augmentation_streams():
    """Under the same Philox key (seed) and counter words 2..3 (step), the augmentation draws use counter word 1 =
    2 pair + side (< 2^31 for any pair below 2^30; csrc/traindata.cu, csrc/modelnet.cu, make_perm) and the dropout
    draws set bit 31 of it: the two counter sets never meet, so no Philox block is shared."""
    for cloud in (0, 1, 2 * 1000 + 1, (1 << 20) - 1):
        for layer in range(16):
            for site in R.SITES:
                for head in (0, 7, 15):
                    w = R.word1(cloud, layer, site, head)
                    assert w >> 31 == 1 and w < 1 << 32
    aug = {2 * pair + side for pair in range(4096) for side in (0, 1)}
    assert max(aug) < 1 << 31
    # fields do not overlap: word 1 and word 0 are injective in (cloud, layer, site, head) and (row group, col)
    words = {R.word1(c, l, s, h) for c in range(64) for l in range(16) for s in R.SITES for h in range(16)}
    assert len(words) == 64 * 16 * 6 * 16


def test_dropout_key_refuses_fields_outside_the_layout():
    from regtr_b200 import ops
    with pytest.raises(ValueError):
        ops.DropoutKey(0.0, 0, 0, 0, 1)
    with pytest.raises(ValueError):
        ops.DropoutKey(0.1, 0, 0, 0, 1, max_len=1 << 16)
    k = ops.DropoutKey(0.1, 2 ** 64 - 1, 2 ** 40, 3, 2)
    a = k.args(5, 6)
    assert (a.seed, a.step, a.pair_base, a.n_pairs, a.layer, a.site) == (2 ** 64 - 1, 2 ** 40, 3, 2, 5, 6)
    assert a.threshold == R.threshold(0.1) and np.float32(a.scale) == R.scale(0.1)


def test_forward_train_signature_keeps_its_defaults():
    import inspect
    from regtr_b200.regtr import RegTR
    sig = inspect.signature(RegTR.forward_train)
    assert sig.parameters['train_encoder'].default is False
    assert sig.parameters['dropout_key'].kind is inspect.Parameter.KEYWORD_ONLY
    assert sig.parameters['dropout_key'].default is None


def test_state_dict_keys_match_the_reference_at_dropout():
    """The unmodified reference RegTR built with the same dropout has exactly our keys (checkpoints load both ways)."""
    from oracle import ref_bridge
    if not ref_bridge.available():
        pytest.skip('the reference sources are not present')
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    for name in ('modelnet', '3dmatch'):
        cfg = get_config(name, dropout=0.1)
        ref = ref_bridge.build_reference_model(cfg)
        ours = RegTR(cfg)
        assert set(ref.state_dict()) == set(ours.state_dict())
        ours.load_state_dict(ref.state_dict(), strict=True)
        ref.load_state_dict(ours.state_dict(), strict=True)


# forward_pre's order of the 12 dropout calls of one layer: (site, side)
LAYER_ORDER = [(1, 0), (2, 0), (1, 1), (2, 1), (3, 0), (3, 1), (4, 0), (4, 1), (5, 0), (6, 0), (5, 1), (6, 1)]


@pytest.mark.parametrize('case', ['fwd_modelnet_b1', 'fwd_3dmatch_small_b2'])
def test_dropout_fixture_served_the_keep_rule(case):
    """dropout.npz is self-consistent: every mask its generator served to the reference, in forward_pre's order for
    all 6 layers, is the keep rule's mask at the stored key (kept count and CRC32 regenerated here)."""
    fx = np.load(os.path.join(GOLDEN, 'dropout.npz'))
    seed, step, pair_base = (int(v) for v in fx[f'{case}|key'])
    p = float(fx[f'{case}|p'])
    log = fx[f'{case}|mask_log']
    n_pairs = int(log[:, 3].max()) + 1
    order = []
    for layer, site, side, b, head, rows, cols, kept, crc in log.tolist():
        if not order or order[-1][:3] != (layer, site, side):
            order.append((layer, site, side))
        m = R.local_keep_mask(p, seed, step, pair_base, n_pairs, b + side * n_pairs, layer, site, head, rows, cols)
        assert int(m.sum()) == kept and zlib.crc32(np.packbits(m).tobytes()) == crc, (layer, site, side, b, head)
        if site in (1, 3):
            assert cols == (rows if site == 1 else int(log[(log[:, 0] == layer) & (log[:, 1] == 2) &
                                                          (log[:, 2] == 1 - side) & (log[:, 3] == b)][0, 5]))
        else:
            assert cols == (1024 if site == 5 else 256)
    assert order == [(layer, site, side) for layer in range(6) for site, side in LAYER_ORDER]
    kept = log[:, 7].sum() / (log[:, 5] * log[:, 6]).sum()
    assert abs(kept - (1 - p)) < 0.01
    assert np.isfinite(float(fx[f'{case}|loss_total']))
