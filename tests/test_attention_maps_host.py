"""CPU tests of the attention-map feature (`TransformerCrossEncoder.get_attentions()`):
  * the attention-map oracle (tests/attention_map_oracle.py) against the unmodified reference's maps
    (tests/golden/attention.npz, tests/golden/make_attention_golden.py), at the tolerance the oracle meets for the
    forward fixtures' features (tests/test_oracle_golden.py: 2e-5 of the largest value);
  * the host-side output tables (`attention_map_layout`) that place every problem's block in the padded layout."""
import numpy as np
import pytest
import torch

from attention_map_oracle import attention_maps
from conftest import load_golden, make_case
from regtr_b200.transformer import attention_map_layout

MAPS = ('src_satt', 'tgt_satt', 'src_xatt', 'tgt_xatt')
FEAT_RTOL = 2e-5          # the oracle's feature tolerance against the forward fixtures


@pytest.fixture(scope='module')
def golden():
    return load_golden('attention')


def check_maps_against_golden(maps, lens, fx, case, rtol):
    """Shared by the GPU test: maps = ((src_satt, tgt_satt), (src_xatt, tgt_xatt)) as numpy-convertible stacks."""
    npy = lambda t: t.detach().cpu().double().numpy() if hasattr(t, 'detach') else np.asarray(t, np.float64)
    assert list(lens) == fx[f'{case}|lens'].tolist()
    (ss, ts), (sx, tx) = maps
    for name, m in zip(MAPS, (ss, ts, sx, tx)):
        a = npy(m)
        assert a.shape == tuple(fx[f'{case}|{name}|shape']), (name, a.shape)
        want = fx[f'{case}|{name}|rows'].astype(np.float64)
        scale = np.abs(want).max()
        err = np.abs(a.reshape(-1)[::int(fx[f'{case}|{name}|step'])] - want).max()
        assert err <= rtol * scale, (case, name, err, rtol * scale)
        assert abs(a.sum() - float(fx[f'{case}|{name}|sum'])) <= rtol * scale * a.size ** 0.5 * 4, (case, name)
        np.testing.assert_allclose(a.sum(-1), fx[f'{case}|{name}|rowsum'], rtol=0, atol=1e-5)


@pytest.mark.parametrize('case', ['fwd_modelnet_b1', 'fwd_3dmatch_small_b2', 'var_modelnet_postnorm_b1'])
def test_oracle_maps_match_reference(case, golden):
    cfg, sd, src, tgt = make_case(case)
    maps, lens = attention_maps(sd, cfg, src, tgt)
    check_maps_against_golden(maps, lens, golden, case, FEAT_RTOL)


def _fill(lens, lay):
    """Write each problem's block through the tables (value = problem id + 1) -> the four padded maps."""
    B = len(lens) // 2
    buf = np.zeros(lay['numel'], np.float64)
    for kind, partner in (('self', lambda c: c), ('cross', lambda c: c + B if c < B else c - B)):
        for c in range(2 * B):
            ql, kl = lens[c], lens[partner(c)]
            off, pitch = lay[f'{kind}_offset'][c], lay[f'{kind}_pitch'][c]
            for r in range(ql):
                assert off + r * pitch + kl <= lay['numel']
                assert np.all(buf[off + r * pitch:off + r * pitch + kl] == 0), 'blocks overlap'
                buf[off + r * pitch:off + r * pitch + kl] = c + 1
    return [buf[b:b + int(np.prod(sh))].reshape(sh) for b, sh in zip(lay['bases'], lay['shapes'])]


@pytest.mark.parametrize('lens', [[7, 5], [5, 9, 4, 4], [3, 0, 0, 6], [0, 0], [0, 4]])
def test_map_layout_tables(lens):
    """B = 1, B = 2 uneven, empty clouds: every problem's block lands at [b, :len_q, :len_k] of its padded map and
    nothing else is written."""
    B = len(lens) // 2
    lay = attention_map_layout(lens)
    s, t = lens[:B], lens[B:]
    Ns, Nt = max(s), max(t)
    assert (lay['Ns'], lay['Nt']) == (Ns, Nt)
    assert lay['shapes'] == [(B, Ns, Ns), (B, Nt, Nt), (B, Ns, Nt), (B, Nt, Ns)]
    assert lay['numel'] == B * (Ns * Ns + Nt * Nt + 2 * Ns * Nt)
    maps = _fill(lens, lay)
    q_of = [s, t, s, t]
    k_of = [s, t, t, s]
    for j, m in enumerate(maps):
        for b in range(B):
            want = np.zeros(m.shape[1:])
            owner = b + 1 if j in (0, 2) else B + b + 1
            want[:q_of[j][b], :k_of[j][b]] = owner
            assert np.array_equal(m[b], want), (lens, j, b)


def test_map_layout_padded_sizes():
    """The padded adaptor records in the caller's padded sizes, which may exceed the longest cloud."""
    lay = attention_map_layout([3, 2, 4, 1], Ns=5, Nt=6)
    assert lay['shapes'] == [(2, 5, 5), (2, 6, 6), (2, 5, 6), (2, 6, 5)]
    assert lay['self_pitch'] == [5, 5, 6, 6] and lay['cross_pitch'] == [6, 6, 5, 5]
    _fill([3, 2, 4, 1], lay)
    with pytest.raises(ValueError):
        attention_map_layout([3, 2, 4, 1], Ns=2, Nt=6)


def test_get_attentions_before_recording_raises():
    from regtr_b200.transformer import TransformerCrossEncoder, TransformerCrossEncoderLayer
    layer = TransformerCrossEncoderLayer(64, 2, 128, 0.0, normalize_before=True)
    enc = TransformerCrossEncoder(layer, 2, torch.nn.LayerNorm(64), return_intermediate=True)
    assert all(lay.satt_weights is None and not lay.record_attentions for lay in enc.layers)
    with pytest.raises(RuntimeError, match='no attention maps recorded'):
        enc.get_attentions()
    enc.record_attentions = True
    assert all(lay.record_attentions for lay in enc.layers)
    with pytest.raises(RuntimeError, match='no attention maps recorded'):
        enc.get_attentions()
    assert set(enc.state_dict()) == set(TransformerCrossEncoder(layer, 2, torch.nn.LayerNorm(64), True).state_dict())
