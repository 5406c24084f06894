"""The training-loss checks are sharp: on the numpy model of the loss kernels' fp32 arithmetic (tests/loss_oracle.py)
the shipped design meets the geometry rule, the fp32 yardstick and the sum d tgt invariant, and every emulated
wrong kernel fails at least one of the checks tests/test_gpu_loss_domain.py makes.  The configs' and the real
fixtures' shapes lie inside that file's grid.  CPU only."""
import os

import numpy as np
import pytest
import torch

import loss_oracle as lo
from grad_yardstick import Yardstick

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _infonce_checks(case, variant=None):
    """The checks of the GPU file on term feature_1 of the InfoNCE model -> (names of the failed checks, report)."""
    layer, key = case['feature_on'][0], f'feature_{case["feature_on"][0]}'
    gk = float(case['g'][case['keys'].index(key)])
    v64, g64 = lo.reference(case, torch.float64)
    v32, g32 = lo.reference(case, torch.float32)
    m = lo.model_infonce(case, case['cond'][layer], case['W'], variant=variant, g=gk)
    geo, mg = case['geo'], m['geo']
    failed = set()
    if not (np.array_equal(mg['anchor'], geo['anchor']) and np.array_equal(mg['n_anchor'], geo['n_anchor'])
            and np.array_equal(mg['pos'], geo['pos'])):
        failed.add('geometry')
    n_src = geo['offs'][geo['B']]
    ys = Yardstick(f'InfoNCE model {variant or "shipped"}, lens {case["lens"]}, {case["family"]}')
    j = case['keys'].index(key)
    if not np.isfinite(m['value']) or not ys.add('value', torch.tensor(float(m['value'])), v32[j], v64[j]):
        failed.add('value')
    d = torch.from_numpy(m['dfeat'])
    ref = g64['cond'][layer]
    if not ys.add('d src', d[:n_src], g32['cond'][layer][:n_src], ref[:n_src]):
        failed.add('d src')
    if not ys.add('d tgt', d[n_src:], g32['cond'][layer][n_src:], ref[n_src:]):
        failed.add('d tgt')
    got = dict(cond=torch.zeros_like(g32['cond']), both_un=g32['both_un'])
    got['cond'][layer] = d
    inv_case = dict(case, g=np.where(np.arange(len(case['keys'])) == j, case['g'], 0).astype(np.float32))
    if lo.invariant_failures(lo.invariant_rows(inv_case, got, g32, g64)):
        failed.add('invariant')
    ys.report()
    return failed


INFONCE_VARIANTS = ('anchor_le', 'ignore_positive', 'mean_all_rows', 'tail_dropped', 'lse_fp32')


@pytest.mark.parametrize('family,lens', [('edges', [90, 40, 65, 33]), ('model', [40, 33, 65, 97]),
                                         ('peaked', [300, 257, 650, 33]), ('flat', [64, 31, 257, 33])])
def test_infonce_model_meets_the_checks(family, lens):
    case = lo.make_case(lens, family, 3)
    assert not _infonce_checks(case)


@pytest.mark.parametrize('variant,family,lens', [
    ('anchor_le', 'edges', [90, 40, 65, 33]),
    ('ignore_positive', 'model', [40, 33, 65, 97]),
    ('mean_all_rows', 'model', [40, 33, 65, 97]),
    ('tail_dropped', 'flat', [40, 33, 63, 50]),
    ('lse_fp32', 'peaked', [300, 257, 650, 33]),
])
def test_infonce_wrong_kernels_fail(variant, family, lens):
    case = lo.make_case(lens, family, 3)
    if variant == 'anchor_le':                            # the family puts key points exactly at r_p
        g2 = case['geo']['g2']
        assert any((np.min(g, 1) == case['geo']['rp2']).any() for g in g2 if g.size)
    if variant == 'mean_all_rows':
        assert (case['geo']['n_anchor'] < np.array(lens[:2])).all()
    failed = _infonce_checks(case, variant)
    print(f'{variant} on {family}: fails {sorted(failed)}')
    assert failed


@pytest.mark.parametrize('variant', [None, 'circle_skip_zero'])
def test_circle_model_and_entries_left_out_of_the_lse(variant):
    """The circle model's value meets the yardstick; leaving the entries outside the positive / negative sets out of
    the log-sum-exps (instead of exp(0) = 1 each) fails it."""
    case = lo.make_case([64, 33, 65, 40], 'margins', 4, loss='circle')
    key = 'feature_1'
    j = case['keys'].index(key)
    v64 = lo.reference(case, torch.float64, grad=False)[0][j]
    v32 = lo.reference(case, torch.float32, grad=False)[0][j]
    _, value = lo.model_circle(case, case['cond'][1], variant)
    ys = Yardstick(f'circle model {variant or "shipped"}')
    ok = ys.add('value', torch.tensor(float(value)), v32, v64)
    ys.report()
    assert ok == (variant is None)


@pytest.mark.parametrize('variant', [None, 'bce_src_norm'])
def test_bce_model_and_the_source_count_normaliser(variant):
    case = lo.make_case([64, 33, 65, 40], 'pointwise', 5)
    (v64, g64), (v32, g32) = lo.reference(case, torch.float64), lo.reference(case, torch.float32)
    value, d = lo.model_bce(case, 1, variant)
    gk = float(case['g'][0])
    ys = Yardstick(f'BCE model {variant or "shipped"}')
    ok = ys.add('value', torch.tensor(float(value)), v32[0], v64[0])
    ok &= ys.add('d logit', torch.from_numpy(d) * gk, g32['logit'][1, :, 0], g64['logit'][1, :, 0])
    ys.report()
    assert ok == (variant is None)


@pytest.mark.parametrize('variant', [None, 'pyr_div_k'])
@pytest.mark.parametrize('K', [1, 40, 50])
def test_pyramid_model_and_division_by_k(K, variant):
    """The pyramid criterion of the GPU file (within 1e-6 of float64, NaN where it is NaN) holds for the model and
    fails when it divides by K (at K = 1 through the row of only shadow slots, which must stay NaN)."""
    pyr0, pools, n_prev = lo.pyramid_case(K)
    got = lo.model_pyramid(pyr0, pools, n_prev, variant)
    want = lo.pyramid(pyr0, pools, n_prev, torch.float64)
    ok = True
    for g, w in zip(got, want):
        g = torch.from_numpy(g).double()
        nan = torch.isnan(w)
        ok &= torch.equal(torch.isnan(g), nan) and float((g - w)[~nan].abs().max()) <= 1e-6
    assert ok == (variant is None)


def test_every_variant_is_exercised():
    assert set(INFONCE_VARIANTS) | {'circle_skip_zero', 'bce_src_norm', 'pyr_div_k'} == set(lo.VARIANTS)


def test_reference_matches_the_torch_restatement_away_from_thresholds():
    """With no distance near r_p / r_n and no tied nearest target, the references equal losses.infonce_loss and
    losses.circle_loss (which decide by torch.cdist) in float64."""
    from regtr_b200 import losses as LS
    for loss in ('infonce', 'circle'):
        case = lo.make_case([60, 45, 70, 50], 'margins' if loss == 'circle' else 'model', 8, loss=loss)
        geo = case['geo']
        for g2 in geo['g2']:
            d = np.sqrt(g2)
            assert np.abs(d / case['r_p'] - 1).min() > 1e-6 and np.abs(d / case['r_n'] - 1).min() > 1e-6
        B, offs = geo['B'], geo['offs']
        f = torch.from_numpy(case['cond'][1]).double()
        xs = torch.from_numpy(case['xyz']).double()
        gt = torch.from_numpy(geo['gt']).double()
        src = [f[offs[b]:offs[b + 1]] for b in range(B)]
        tgt = [f[offs[B + b]:offs[B + b + 1]] for b in range(B)]
        sxyz = [gt[offs[b]:offs[b + 1]] for b in range(B)]
        txyz = [xs[offs[B + b]:offs[B + b + 1]] for b in range(B)]
        if loss == 'infonce':
            want = LS.infonce_loss(torch.from_numpy(case['W']).double(), src, tgt, sxyz, txyz, case['r_p'], case['r_n'])
            got = torch.stack(lo.infonce_pairs(f, lo.sym(torch.from_numpy(case['W']).double()), geo)).mean()
        else:
            want = LS.circle_loss(src, tgt, sxyz, txyz, case['r_p'], case['r_n'])
            got = torch.stack(lo.circle_pairs(f, geo)).mean()
        np.testing.assert_allclose(float(got), float(want), rtol=1e-12)


def test_geometry_rule_at_exact_thresholds_and_ties():
    """The numpy rule on hand-placed points: a nearest target at exactly r_p is no anchor, equidistant targets give
    the lower index, a target at exactly r_n is not ignored, duplicates tie to the first."""
    xyz = np.array([[0, 0, 0], [10, 0, 0], [20, 0, 0],
                    [-0.5, 0, 0], [0.5, 0, 0], [10.25, 0, 0], [9.75, 0, 0], [20.375, 0, 0], [20.375, 0, 0],
                    [21.0, 0, 0]], np.float32)
    pose = np.zeros((1, 3, 4), np.float32)
    pose[0, :, :3] = np.eye(3)
    geo = lo.geometry(xyz, [3, 7], pose, 0.5, 1.0)
    assert geo['pos'][:3].tolist() == [3, 5, 7]
    assert geo['anchor'][:3].tolist() == [0, 1, 1]
    assert geo['ignore'][0][2].tolist() == [False] * 4 + [False, True, False]     # 21.0 is exactly r_n away


def test_domain_covers_the_configs_and_the_real_fixtures():
    """The 3DMatch and ModelNet configs' layer counts, loss layers and batch sizes, the real fixtures' coarse cloud
    sizes and the forward fixtures' lie inside the GPU file's grid."""
    from conftest import REAL_CASES
    from regtr_b200.config import get_config
    cases = lo.domain_cases()
    lens = [n for _, _, kw in cases for n in kw['lens']]
    layers = {kw.get('n_layers', 2) for _, _, kw in cases}
    Bs = {len(kw['lens']) // 2 for _, _, kw in cases}
    assert set(lo.EDGE_LENS) <= set(lens)
    assert {1, 2, 4, 8, 16} <= Bs and {1, 6, 8} <= layers
    assert max(sum(kw['lens']) for _, _, kw in cases) >= 49 * lo.PW
    assert any(len(kw.get('feature_on', ())) + 1 == 8 for _, _, kw in cases)
    for name in ('3dmatch', 'modelnet'):
        cfg = get_config(name)
        assert cfg.num_encoder_layers in layers and cfg.train_batch_size in Bs
        six = [kw for _, _, kw in cases if kw.get('n_layers') == cfg.num_encoder_layers]
        assert any(list(kw['feature_on']) == list(cfg.feature_loss_on) for kw in six)
    sizes = []
    for name in list(REAL_CASES) + ['fwd_modelnet_b1', 'fwd_3dmatch_small_b2']:
        z = np.load(os.path.join(GOLDEN, name + '.npz'))
        last = max(int(k.rsplit('_', 1)[1]) for k in z if k.startswith('stack_lengths_'))
        sizes += [int(v) for v in z[f'stack_lengths_{last}']]
    print('coarse cloud sizes of the fixtures:', sorted(sizes))
    assert min(lens) <= min(sizes) and max(sizes) <= max(lens)
    for lo_, hi in ((325, 430), (520, 660)):                # the 3DMatch and ModelNet coarse ranges
        assert any(lo_ <= n <= hi for n in lens)
