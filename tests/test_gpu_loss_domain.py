"""The training-loss kernels (csrc/loss.cu through ops.loss_forward / ops.loss_backward) over every batch shape they
accept, for both feature losses: clouds of 0 to 1500 tokens on every 32-row tile edge and the 256-token chunk edge,
source and target clouds of very different sizes, B from 1 to 16 (N up to about 50 pointwise chunks), 1, 2, 6 and 8
layers (all 8 term slots), the feature_un term live and off, on the input families of tests/loss_oracle.py.  Per case
the geometry (positives, anchors, circle counts) equals the numpy rule bit for bit; every loss value and every
gradient is a row of the fp32 yardstick (tests/grad_yardstick.py) against float64; the sum of d feat over a pair's
tokens meets its invariant; reruns are bit-identical and each pair's loss is the same alone as in the batch.  Also:
the overlap pyramid alone, the data-parallel normalisers on two slices, the 9-layer / 9-term refusals, and that
the checks are sharp on the GPU's own outputs.  tests/test_loss_sharpness.py shows on a model of the kernels that
these checks catch each of a set of subtly wrong kernels."""
import functools

import numpy as np
import pytest
import torch

import loss_oracle as lo
from grad_yardstick import Yardstick

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
GRADS = ('both_un', 'cond', 'corr', 'logit', 'W', 'W_un')
_WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _worst_ratios():
    """After the module: the largest GPU / fp32-oracle error ratio of each part (over both measures)."""
    yield
    if _WORST:
        print('\nworst GPU / fp32-oracle error ratio per part')
        for part, (r, where) in sorted(_WORST.items()):
            print(f'  {part:28s} {r:8.2f}  ({where})')


def _note(part, where, eg, ef):
    r = max([a / b for a, b in zip(eg, ef) if b > 0], default=0.0)
    if r > _WORST.get(part, (-1.0, None))[0]:
        _WORST[part] = (r, where)


def _part(case, key):
    kind = 'InfoNCE' if case['loss'] == 'infonce' else 'circle'
    if key.startswith('overlap') or key == 'd logit':
        return 'BCE ' + ('value' if key.startswith('overlap') else 'd logit')
    if key.startswith('corr') or key == 'd corr':
        return 'L1 ' + ('value' if key.startswith('corr') else 'd corr')
    return f'{kind} ' + ('value' if key.startswith('feature') else key)


def _dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _geometry(case, norm=None):
    from regtr_b200 import ops
    return ops.LossGeometry(_dev(case['xyz']), _dev(lo.offsets(case['lens']), torch.int32), case['lens'],
                            _dev(case['pose']), _dev(case['w']), case['overlap_on'], case['feature_on'],
                            case['corr_on'], case['r_p'], case['r_n'], norm=norm, feature_loss=case['loss'])


def _run(case, norm=None, lse_scale=None):
    """ops.loss_forward then ops.loss_backward for the upstream gradient case['g'] -> (state, grads on the CPU).
    lse_scale: multiply the stored InfoNCE log-sum-exps by it between the two (a sharpness check)."""
    from regtr_b200 import ops
    infonce = case['loss'] == 'infonce'
    st = ops.loss_forward(_dev(case['both_un']), _dev(case['cond']), _dev(case['corr']), _dev(case['logit']),
                          _dev(case['W']) if infonce else None, _dev(case['W_un']) if infonce else None,
                          _geometry(case, norm))
    if lse_scale is not None:
        st['lse'].mul_(lse_scale)
    d = ops.loss_backward(st, _dev(case['g']))
    torch.cuda.synchronize()
    return st, {k: (None if t is None else t.cpu()) for k, t in zip(GRADS, d)}


@functools.lru_cache(maxsize=None)
def _case(cid):
    loss, kw = {c[0]: c[1:] for c in lo.domain_cases()}[cid]
    case = lo.make_case(loss=loss, **kw)
    return case, _run(case), lo.reference(case, torch.float64), lo.reference(case, torch.float32)


def _rows(title, case, vals, grads, r64, r32, part=True):
    """The yardstick rows of every value and gradient -> Yardstick; NaN values and all-zero gradients are checked
    for being exactly that on the GPU instead."""
    (v64, g64), (v32, g32) = r64, r32
    vals = vals.cpu()
    ys = Yardstick(title)
    for j, k in enumerate(case['keys']):
        if bool(torch.isnan(v64[j])):
            assert bool(torch.isnan(vals[j])), (k, float(vals[j]))
            continue
        ys.add(k, vals[j], v32[j], v64[j])
    for k in GRADS:
        if k not in g64:
            assert grads.get(k) is None, k
            continue
        assert grads[k].shape == g64[k].shape, k
        if float(g64[k].abs().max()) == 0.0:
            assert int(torch.count_nonzero(grads[k])) == 0, k
            continue
        ys.add('d ' + k, grads[k], g32[k], g64[k])
    if part:
        for name, eg, ef, _ in ys.rows:
            _note(_part(case, name), f'{title}: {name}', eg, ef)
    return ys


def _check_geometry(case, st):
    geo = case['geo']
    n_src = geo['offs'][geo['B']]
    if case['loss'] == 'infonce':
        assert np.array_equal(st['pos'].cpu().numpy()[:n_src], geo['pos'][:n_src])
        assert np.array_equal(st['anchor'].cpu().numpy()[:n_src], geo['anchor'][:n_src])
        assert np.array_equal(st['n_anchor'].cpu().numpy(), geo['n_anchor'])
    else:
        for k in ('n_pos', 'n_neg', 'n_sel'):
            assert np.array_equal(st[k].cpu().numpy(), geo[k]), k


def _check_invariant(title, case, grads, r64, r32):
    rows = lo.invariant_rows(case, grads, r32[1], r64[1])
    for key, b, dg, df, bound in rows:
        r = dg / max(bound, 1e-300)
        if r > _WORST.get('invariant (dev / bound)', (-1.0, None))[0]:
            _WORST['invariant (dev / bound)'] = (r, f'{title}: {key} pair {b}')
    return lo.invariant_failures(rows)


# ------------------------------------------------------------------------------------------------------ the grid

CASE_IDS = [c[0] for c in lo.domain_cases()]


@pytest.mark.parametrize('cid', CASE_IDS)
def test_loss_domain(cid):
    """Geometry bit-exact; every value and gradient under the yardstick; the d feat invariant per pair and term;
    a rerun bit-identical; an anchor row whose only unmasked target is its positive has a row loss of exactly 0."""
    case, (st, grads), r64, r32 = _case(cid)
    title = f'loss {cid}: lens {case["lens"]}, {case["family"]}, L={case["cond"].shape[0]}'
    _check_geometry(case, st)
    ys = _rows(title, case, st['vals'], grads, r64, r32)
    ys.report()
    assert not ys.failures(), ys.failures()
    inv = _check_invariant(title, case, grads, r64, r32)
    assert not inv, inv
    st2, grads2 = _run(case)
    assert torch.equal(st['vals'].nan_to_num(7.0), st2['vals'].nan_to_num(7.0))
    for k in GRADS:
        assert (grads[k] is None and grads2[k] is None) or torch.equal(grads[k], grads2[k]), k
    if case['loss'] == 'infonce':
        geo, row_loss = case['geo'], st['row_loss'].cpu()
        n_only = 0
        for b in range(geo['B']):
            s0, s1 = geo['offs'][b], geo['offs'][b + 1]
            ig = geo['ignore'][b]
            only = (geo['anchor'][s0:s1] == 1) & (ig.sum(1) == ig.shape[1] - 1) & (ig.shape[1] > 1)
            idx = torch.from_numpy(np.nonzero(only)[0] + s0)
            n_only += len(idx)
            assert int(torch.count_nonzero(row_loss[:, idx])) == 0
        if cid.endswith('8layers-b2'):
            assert n_only > 0


BATCHED = [c for c in CASE_IDS if c.endswith(('-b2', '-b4', '-b8', '-empty'))]


@pytest.mark.parametrize('cid', BATCHED)
def test_pair_loss_alone_and_in_the_batch(cid):
    """Each pair's per-pair loss run alone equals its entry in the batch: bit for bit for the circle loss (no GEMM),
    within 1e-6 relative for InfoNCE, whose source rows pass through a GEMM whose split depends on the row count."""
    case, (st, _), _, _ = _case(cid)
    B = case['geo']['B']
    for b in range(B):
        alone, _ = _run(lo.subset(case, [b]))
        a, w = alone['pair_loss'][:, 0].cpu(), st['pair_loss'][:, b].cpu()
        assert torch.equal(torch.isnan(a), torch.isnan(w)), b
        a, w = a.nan_to_num(0.0), w.nan_to_num(0.0)
        if case['loss'] == 'circle':
            assert torch.equal(a, w), b
        else:
            assert float((a - w).abs().max()) <= 1e-6 * float(w.abs().max()) + 1e-30, (b, a, w)


# ---------------------------------------------------------------------------------------------------- normalisers

@pytest.mark.parametrize('loss', ['infonce', 'circle'])
def test_slices_with_the_summed_norms_add_up_to_the_batch(loss):
    """Two slices of a 4-pair batch, each given the summed loss_norms: their values add up to the whole batch's
    float64 values and their gradient rows are the whole batch's for the same tokens, under the yardstick."""
    from regtr_b200 import ops
    case = lo.make_case([90, 257, 33, 140, 64, 31, 300, 120], 'model' if loss == 'infonce' else 'margins', 30,
                        loss=loss, wt_un=1.0)
    assert (case['geo']['n_anchor'] > 0).all() and (case['geo']['n_sel'] > 0).all()
    r64, r32 = lo.reference(case, torch.float64), lo.reference(case, torch.float32)
    parts = [lo.subset(case, [0, 1]), lo.subset(case, [2, 3])]
    total = sum(ops.loss_norms(_geometry(p)) for p in parts)
    np.testing.assert_allclose(total.cpu().numpy(), lo.norms_of(case, case['geo']), rtol=1e-12)
    vals = torch.zeros(len(case['keys']), dtype=torch.float64)
    grads = {k: torch.zeros_like(r64[1][k], dtype=torch.float32) for k in r64[1]}
    for p in parts:
        st, g = _run(p, norm=total.clone())
        vals += st['vals'].cpu().double()
        rows = torch.from_numpy(p['rows'])
        grads['both_un'][rows] = g['both_un']
        grads['cond'][:, rows], grads['corr'][:, rows], grads['logit'][:, rows] = g['cond'], g['corr'], g['logit']
        for k in ('W', 'W_un'):
            if k in grads:
                grads[k] += g[k]
        ref_p = lo.reference(p, torch.float64, norm=lo.norms_of(case, case['geo']), grad=False)[0]
        np.testing.assert_allclose(st['vals'].cpu().double().numpy(), ref_p.numpy(), rtol=1e-4)
    ys = _rows(f'{loss}: two slices with the summed normalisers', case, vals, grads, r64, r32, part=False)
    ys.report()
    assert not ys.failures(), ys.failures()


# ------------------------------------------------------------------------------------------------------- pyramid

@pytest.mark.parametrize('K', [1, 40, 50])
def test_overlap_pyramid(K):
    """ops.overlap_pyramid on pools of width K with shadow slots and rows of only shadow slots (NaN, as
    compute_overlaps), the level sizes read from capacity-sized offset rows: within 1e-6 of float64, NaN where it is
    NaN, levels 0 and 1 bit-equal to losses.compute_overlaps."""
    from regtr_b200 import losses as LS
    from regtr_b200 import ops
    pyr0, pools, n_prev = lo.pyramid_case(K)
    offs = [_dev(np.array([0, n // 2, n, 10 ** 6, -5, 3, 7, 99], np.int32)) for n in n_prev]
    got = [t.cpu() for t in ops.overlap_pyramid(_dev(pyr0), [_dev(p) for p in pools], offs, 2)]
    want = lo.pyramid(pyr0, pools, n_prev, torch.float64)
    meta = dict(points=[None] * (len(pools) + 1), pools=[torch.from_numpy(p.astype(np.int64)) for p in pools],
                stack_lengths=[torch.tensor([n]) for n in n_prev] + [torch.tensor([len(pools[-1])])])
    route = LS.compute_overlaps(dict(kpconv_meta=meta, src_overlap=[torch.from_numpy(pyr0)], tgt_overlap=[]))
    worst = 0.0
    for lvl, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == torch.float32 and g.shape == w.shape
        nan = torch.isnan(w)
        assert torch.equal(torch.isnan(g), nan), lvl
        if lvl:
            assert bool(nan[-1]), 'a row of only shadow slots'
        err = float((g.double() - w)[~nan].abs().max())
        worst = max(worst, err)
        assert err <= 1e-6, (lvl, err)
        if lvl <= 1:
            assert torch.equal(g.nan_to_num(-1.0), route[f'pyr_{lvl}'].nan_to_num(-1.0)), lvl
    print(f'\noverlap pyramid K={K}: levels {[len(g) for g in got]}, max error {worst:.2e} (bound 1e-6)')
    if worst / 1e-6 > _WORST.get('pyramid (error / 1e-6)', (-1.0, None))[0]:
        _WORST['pyramid (error / 1e-6)'] = (worst / 1e-6, f'K={K}')


# ------------------------------------------------------------------------------------------------------ refusals

def test_nine_layers_or_nine_terms_are_refused():
    """ops.loss_forward refuses 9 layers and 8 feature layers (9 terms with feature_un); the C entry points refuse
    L = 9 and 9 terms before they launch anything."""
    from regtr_b200 import lib as _lib
    from regtr_b200 import ops
    L = _lib.load()
    case = lo.make_case([40, 33], 'model', 40)
    base = dict(case)
    with pytest.raises(ValueError, match='9 layers'):
        _run(dict(base, cond=np.repeat(case['cond'][:1], 9, 0), corr=np.repeat(case['corr'][:1], 9, 0),
                  logit=np.repeat(case['logit'][:1], 9, 0)))
    eight = dict(base, cond=np.repeat(case['cond'][:1], 8, 0), corr=np.repeat(case['corr'][:1], 8, 0),
                 logit=np.repeat(case['logit'][:1], 8, 0), feature_on=list(range(8)))
    with pytest.raises(ValueError, match='8 layers'):
        _run(eight)
    offs = _dev(np.array([0, 40, 73], np.int32))
    for field, n in (('L', 9), ('n_terms', 9)):
        a = np.zeros((), ops.LOSS_ARGS)
        a['offs'], a['N'], a['B'], a['L'], a['n_terms'], a['max_src'], a['max_tgt'] = offs.data_ptr(), 73, 1, 1, 1, 40, 33
        a[field] = n
        for fn in ('regtr_loss_pointwise', 'regtr_infonce_fwd', 'regtr_loss_finalize'):
            args = (a.ctypes.data, None, None) if fn != 'regtr_infonce_fwd' else (a.ctypes.data, None)
            assert getattr(L, fn)(*args) != 0, (fn, field)


# ----------------------------------------------------------------------------------------------------- sharpness

@pytest.mark.parametrize('loss', ['infonce', 'circle'])
def test_checks_are_sharp(loss):
    """The GPU's own values and gradients times (1 + 1e-5) fail their rows (on families whose fp32 error leaves
    room: near-uniform softmax rows for InfoNCE, the margin family for the circle loss)."""
    fam = 'flat' if loss == 'infonce' else 'margins'
    case = lo.make_case([96, 65, 80, 33], fam, 50, loss=loss)
    st, grads = _run(case)
    r64, r32 = lo.reference(case, torch.float64), lo.reference(case, torch.float32)
    ok = _rows(f'{loss} {fam}, as computed', case, st['vals'], grads, r64, r32, part=False)
    ok.report()
    assert not ok.failures(), ok.failures()
    s = 1 + 1e-5
    bad = _rows(f'{loss} {fam}, scaled by 1 + 1e-5', case, st['vals'] * s,
                {k: (None if v is None else v * s) for k, v in grads.items()}, r64, r32, part=False)
    bad.report()
    assert set(bad.failures()) == {r[0] for r in bad.rows}, bad.failures()


@pytest.mark.parametrize('family', ['model', 'flat', 'shared'])
def test_invariant_catches_a_raised_lse(family):
    """The stored InfoNCE log-sum-exps raised by 1e-5 of themselves before the backward (softmax rows summing to
    less than 1) fail the sum d tgt invariant, while the unchanged run meets it."""
    case = lo.make_case([120, 90, 100, 70], family, 60)
    r64, r32 = lo.reference(case, torch.float64), lo.reference(case, torch.float32)
    _, grads = _run(case)
    assert not _check_invariant(f'{family}, as computed', case, grads, r64, r32)
    _, raised = _run(case, lse_scale=1 + 1e-5)
    rows = lo.invariant_rows(case, raised, r32[1], r64[1])
    print(f'\n{family}: lse x (1 + 1e-5): worst deviation / bound '
          f'{max(r[2] / r[4] for r in rows):.3g} over {len(rows)} (pair, term) rows')
    assert len(lo.invariant_failures(rows)) == len(rows) > 0
