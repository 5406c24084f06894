"""CPU tests of the circle feature loss (`feature_loss_type: circle`) against the unmodified reference
(tests/golden/circle.npz, written by tests/golden/make_circle_golden.py): the torch restatement `losses.circle_loss`
against `CircleLossFull` on seeded feature sets that take every branch of the loss, `losses.compute_loss` and the
oracle's autograd against `RegTR.compute_loss` and its backward, and the circle model's state_dict."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import make_case

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402
from oracle import regtr_oracle as O  # noqa: E402
from regtr_b200 import losses as LS  # noqa: E402
from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'circle.npz')
LOSS_SETS = ('single', 'uneven', 'one_token', 'nan')
MODEL_CASES = ('fwd_modelnet_b1', 'fwd_3dmatch_small_b2')
PAIRS = {'fwd_modelnet_b1': lambda: [make_modelnet_pair(1000)],
         'fwd_3dmatch_small_b2': lambda: [make_3dmatch_pair(2001, 2500), make_3dmatch_pair(2002, 4000)]}


@pytest.fixture(scope='module')
def fx():
    return dict(np.load(GOLDEN))


def loss_set(fx, name, dtype=torch.float64):
    """(source features, target features, source xyz, target xyz) lists, the radii, the packed lengths."""
    lens = [int(v) for v in fx[f'{name}|lens']]
    B = len(lens) // 2
    f = torch.split(torch.from_numpy(fx[f'{name}|feat']).to(dtype), lens)
    x = torch.split(torch.from_numpy(fx[f'{name}|xyz']).to(dtype), lens)
    r_p, r_n = (float(v) for v in fx[f'{name}|radii'])
    return list(f[:B]), list(f[B:]), list(x[:B]), list(x[B:]), r_p, r_n, lens


@pytest.mark.parametrize('name', LOSS_SETS)
def test_restatement_matches_the_reference_circle_loss(fx, name):
    """Value and both feature gradients of `losses.circle_loss` in float64 against CircleLossFull in float64; NaN
    exactly where the reference's value is NaN, with finite gradients."""
    sf, tf, sx, tx, r_p, r_n, lens = loss_set(fx, name)
    leaves = [t.clone().requires_grad_(True) for t in sf + tf]
    B = len(sf)
    val = LS.circle_loss(leaves[:B], leaves[B:], sx, tx, r_p, r_n)
    val.backward()
    want = float(fx[f'{name}|value'])
    assert np.isnan(want) == bool(torch.isnan(val)), (name, want, float(val))
    if not np.isnan(want):
        np.testing.assert_allclose(float(val.detach()), want, rtol=1e-12)
    grad = torch.cat([t.grad for t in leaves]).numpy()
    ref = fx[f'{name}|grad'].astype(np.float64)
    assert np.isfinite(ref).all() and np.isfinite(grad).all()
    assert np.abs(grad - ref).max() <= 1e-6 * np.abs(ref).max()
    if name == 'nan':
        assert float(np.abs(ref).max()) > 0          # the NaN pair takes no gradient; the other pair does


def test_loss_sets_take_every_branch(fx):
    """The fixture's inputs hit both margins, both softplus branches and the degenerate selections."""
    counts = dict(pos_lo=0, pos_hi=0, neg_lo=0, neg_hi=0, lin=0, log=0, no_pos=0)
    for name in LOSS_SETS:
        sf, tf, sx, tx, r_p, r_n, _ = loss_set(fx, name)
        for a, p, ax, px in zip(sf, tf, sx, tx):
            g = torch.cdist(ax, px)
            d = torch.sqrt(((a[:, None] - p[None]) ** 2).sum(-1) + 1e-12)
            pm, nm = g < r_p, g > r_n
            counts['pos_lo'] += int((pm & (d < 0.1)).sum()); counts['pos_hi'] += int((pm & (d > 0.1)).sum())
            counts['neg_lo'] += int((nm & (d < 1.4)).sum()); counts['neg_hi'] += int((nm & (d > 1.4)).sum())
            zp = torch.where(pm, 10 * (d - 0.1) * (d - 0.1).clamp_min(0), 0.0)
            zn = torch.where(nm, 10 * (1.4 - d) * (1.4 - d).clamp_min(0), 0.0)
            x = (zp.logsumexp(-1) + zn.logsumexp(-1))[(pm.sum(-1) > 0) & (nm.sum(-1) > 0)]
            counts['lin'] += int((x > 20).sum()); counts['log'] += int((x <= 20).sum())
            counts['no_pos'] += int(((pm.sum(-1) == 0) & (nm.sum(-1) > 0)).sum())
    assert all(v > 0 for v in counts.values()), counts
    assert min(int(v) for v in fx['one_token|lens']) == 1
    assert np.isnan(fx['nan|value']) and np.isnan(fx['one_token|value'])
    assert np.isfinite(fx['single|value']) and np.isfinite(fx['uneven|value'])


def _oracle_case(case, grad=False):
    cfg, sd, src, tgt = make_case(case)
    cfg['feature_loss_type'] = 'circle'
    sd = {k: v for k, v in sd.items() if not k.startswith('feature_criterion')}
    if grad:
        sd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    pred = O.forward(sd, cfg, src, tgt)
    meta = pred['kpconv_meta']
    batch = {'kpconv_meta': {k: [torch.as_tensor(np.asarray(v)) for v in meta[k]]
                             for k in ('points', 'pools', 'stack_lengths')}}
    batch.update(ei.loss_inputs(PAIRS[case](), [len(s) for s in src], [len(t) for t in tgt]))
    return cfg, sd, pred, batch


@pytest.mark.parametrize('case', MODEL_CASES)
def test_compute_loss_matches_the_reference_model_losses(fx, case):
    """`losses.compute_loss` on the oracle's forward with feature_loss_type='circle' equals the reference's
    RegTR.compute_loss: every value to 2e-4 (as test_losses.py), no W needed."""
    cfg, _, pred, batch = _oracle_case(case)
    losses = LS.compute_loss(types.SimpleNamespace(cfg=cfg), pred, batch)
    want = {k.split('|loss_')[1]: float(v) for k, v in fx.items() if k.startswith(f'{case}|loss_')}
    assert list(losses) == ['overlap_5', 'feature_5', 'feature_un', 'corr_5', 'total'] and set(losses) == set(want)
    for k, v in losses.items():
        np.testing.assert_allclose(float(v), want[k], rtol=2e-4, err_msg=k)


def test_oracle_gradients_match_the_reference_backward(fx):
    """The oracle's autograd through `losses.compute_loss` (circle) against the reference's backward on
    fwd_modelnet_b1, with test_oracle_grad.py's criteria: norm within 1e-3, sampled entries within 5e-3 of the rms."""
    case = 'fwd_modelnet_b1'
    cfg, sd, pred, batch = _oracle_case(case, grad=True)
    total = LS.compute_loss(types.SimpleNamespace(cfg=cfg), pred, batch)['total']
    np.testing.assert_allclose(float(total.detach()), float(fx[f'{case}|loss_total']), rtol=2e-5)
    total.backward()
    names = [k.split('|g|')[1] for k in fx if k.startswith(f'{case}|g|')]
    assert len(names) >= 140
    worst = 0.0
    for name in names:
        g = sd[name].grad
        assert g is not None, name
        g = g.detach().double().reshape(-1)
        want = fx[f'{case}|g|{name}']
        idx = ei.grad_sample_index(name, g.numel())
        scale = max(want[0] / np.sqrt(g.numel()), 1e-12)
        assert abs(float(g.norm()) - want[0]) <= 1e-3 * want[0] + 1e-9, (name, float(g.norm()), want[0])
        err = np.abs(g[torch.from_numpy(idx)].numpy() - want[2:]).max() / scale
        worst = max(worst, err)
        assert err <= 5e-3, (name, err)
    print('worst sampled-entry error / rms', worst)


@pytest.mark.parametrize('case,n_keys', [('fwd_modelnet_b1', 144), ('fwd_3dmatch_small_b2', 166)])
def test_circle_state_dict_has_no_loss_parameters_and_loads_strictly(case, n_keys):
    """RegTR(cfg) with the circle loss has the reference's module tree: no feature_criterion*.W, and the seeded
    state_dict (the reference's key set) loads with strict=True."""
    from regtr_b200.regtr import RegTR
    from regtr_b200.weights import random_state_dict
    cfg, _, _, _ = make_case(case)
    cfg['feature_loss_type'] = 'circle'
    model = RegTR(cfg)
    keys = list(model.state_dict())
    assert len(keys) == n_keys and not any(k.startswith('feature_criterion') for k in keys)
    sd = random_state_dict(cfg, 0)
    assert set(sd) == set(keys)
    model.load_state_dict(sd, strict=True)
    cfg_nce, _, _, _ = make_case(case)
    assert len(RegTR(cfg_nce).state_dict()) == n_keys + 2


def test_compute_loss_rejects_other_feature_losses():
    """A feature_loss_type other than 'infonce' and 'circle' raises."""
    cfg, _, _, _ = make_case('fwd_modelnet_b1')
    cfg['feature_loss_type'] = 'triplet'
    with pytest.raises(NotImplementedError, match='triplet'):
        LS.compute_loss(types.SimpleNamespace(cfg=cfg), {}, {})
