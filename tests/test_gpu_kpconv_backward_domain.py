"""The KPConv-encoder backward (csrc/kpconv_bwd.cu) over every shape the forward accepts: KPConv dx and dW at each
Cin path (1, the small-Cin widths 4 to 16, 32 to 256) and K from 1 to 128 (both sides of the aggregation's K = 64
switch, up to the edge kernel's largest shared-memory layout), with and without the forward's row flags; the
neighbour-list transpose at in-degrees from 0 to 4096; the max-pool backward at K up to its 255 limit.  Every dx
and dW goes through the fp32 yardstick (tests/grad_yardstick.py) on three output-gradient families; reruns, and a
cloud alone or stacked after another, are bit-identical.  tests/test_kpconv_bwd_sharpness.py shows on a model of
the kernels that these checks catch each of a set of subtly wrong kernels."""
import functools

import numpy as np
import pytest
import torch

import kpconv_bwd_oracle as kb
from grad_yardstick import Yardstick
from test_gpu_forward_ops import _kp_inputs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
NQ, COUT = 61, 64
_WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _worst_ratios():
    """After the module: the largest GPU / fp32-oracle error ratio of each part (over both measures)."""
    yield
    if _WORST:
        print('\nworst GPU / fp32-oracle error ratio per part')
        for part, (r, where) in sorted(_WORST.items()):
            print(f'  {part:28s} {r:6.2f}  ({where})')


def _note(part, title, row):
    name, eg, ef, _ = row
    r = max([a / b for a, b in zip(eg, ef) if b > 0], default=0.0)
    if r > _WORST.get(part, (-1.0, None))[0]:
        _WORST[part] = (r, f'{title}: {name}')


def _dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _weights(cin, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((15, cin, COUT)) / np.sqrt(15 * cin)).astype(np.float32)


def _gpu_grads(c, W, gouts, mode):
    """[(dx, dW or None)] of ops.kpconv's backward for each output gradient, each computed twice (bit-identical)."""
    from regtr_b200 import ops
    xs = _dev(c['x']).requires_grad_(True)
    ws = _dev(W).requires_grad_(mode != 'x_only')
    flags = _dev((c['x'].astype(np.float64).sum(1) > 0).astype(np.uint8)) if mode == 'flags' else None
    out = ops.kpconv(_dev(c['q']), _dev(c['s']), _dev(c['idx'], torch.int32), xs, ws, _dev(c['kp']), c['extent'],
                     row_flags=flags)
    wrt = [xs, ws] if mode != 'x_only' else [xs]
    res = []
    for g in gouts:
        a = torch.autograd.grad(out, wrt, _dev(g), retain_graph=True)
        b = torch.autograd.grad(out, wrt, _dev(g), retain_graph=True)
        assert all(torch.equal(u, v) for u, v in zip(a, b)), 'two backward passes differ'
        res.append((a[0].cpu(), a[1].cpu() if mode != 'x_only' else None))
    return res


def _kp_rows(title, c, W, gouts, got, mode, names=kb.FAMILIES, part='KPConv'):
    need_w = mode != 'x_only'
    r64 = kb.kpconv_grads(c, W, gouts, torch.float64, need_w)
    r32 = kb.kpconv_grads(c, W, gouts, torch.float32, need_w)
    ys = Yardstick(title)
    for name, (dx, dw), (dx64, dw64), (dx32, dw32) in zip(names, got, r64, r32):
        ys.add(f'dx, gout {name}', dx, dx32, dx64)
        if need_w:
            ys.add(f'dW, gout {name}', dw, dw32, dw64)
    ys.report()
    if part:
        for row in ys.rows:
            _note(f'{part} {row[0].split(",")[0]}', title, row)
    return ys, r64, r32


@functools.lru_cache(maxsize=None)
def _kp_case(cin, K, mode):
    c = _kp_inputs(cin, K, NQ)
    W = _weights(cin, 10 * cin + K)
    gouts = [kb.gout_family(f, NQ, COUT, cin * 1000 + K) for f in kb.FAMILIES]
    return c, W, gouts, _gpu_grads(c, W, gouts, mode)


# ------------------------------------------------------------------------------------------------------ KPConv grid

@pytest.mark.parametrize('cin,K,mode', kb.kpconv_cases(), ids=[f'cin{c}-K{k}-{m}' for c, k, m in kb.kpconv_cases()])
def test_kpconv_backward_domain(cin, K, mode):
    """dx and dW against float64 autograd of oracle.regtr_oracle.kpconv under the fp32 yardstick, on
    test_gpu_forward_ops._kp_inputs (supports at a kernel point's extent and just either side of it, rows summing to
    exactly 0 and negative rows, a query with no valid and one with no counted neighbour, shadow slots between real
    ones) for zero-mean, offset and zero-row output gradients.  mode: the forward's row flags passed in | computed by
    the aggregation | dx alone (the count recomputed from x inside the edge kernel)."""
    c, W, gouts, got = _kp_case(cin, K, mode)
    ys, _, _ = _kp_rows(f'KPConv backward Cin={cin} K={K} Nq={NQ} Ns={c["Ns"]} {mode}', c, W, gouts, got, mode)
    assert not ys.failures(), ys.failures()


@pytest.mark.parametrize('cin', [4, 64, 256])
def test_kpconv_backward_checks_are_sharp(cin):
    """The GPU's own dx or dW times (1 + 1e-5) fails its row."""
    c, W, gouts, got = _kp_case(cin, 40, 'flags')
    ys, r64, r32 = _kp_rows(f'KPConv backward Cin={cin} K=40, scaled by 1 + 1e-5', c, W, gouts[:1],
                            [(got[0][0] * (1 + 1e-5), got[0][1] * (1 + 1e-5))], 'flags', names=['zero_mean'],
                            part=None)
    assert set(ys.failures()) == {'dx, gout zero_mean', 'dW, gout zero_mean'}, ys.failures()


# ---------------------------------------------------------------------------------- transpose at degree extremes

DEGREE_CASES = [('hub', 4096, 1, 3, 4), ('skewed', 2048, 2, 64, 64), ('uniform', 16, 40, 5000, 256)]


@pytest.mark.parametrize('degrees,Nq,K,Ns,cin', DEGREE_CASES, ids=[d[0] for d in DEGREE_CASES])
def test_transpose_and_dx_at_degree_extremes(degrees, Nq, K, Ns, cin):
    """One support referenced by all 4096 queries of a 4096 x 1 list; in-degrees from 0 to about 2000 with Nq > Ns;
    Ns > Nq with most supports unreferenced.  row_start and edges equal the numpy inverse; dx and dW meet the
    yardstick at those degrees."""
    from regtr_b200 import ops
    c = kb.dense_case(Nq, K, Ns, cin, seed=Nq + K, degrees=degrees)
    t = _dev(c['idx'], torch.int32)
    rs, ed = ops.neighbor_csr(t, Ns)
    want_rs, want_ed = kb.csr_numpy(c['idx'], Ns)
    deg = np.diff(want_rs)
    print(f'\n{degrees}: Nq={Nq} K={K} Ns={Ns}, in-degree {deg.min()}..{deg.max()}')
    assert deg.max() <= 4096
    assert np.array_equal(rs.cpu().numpy(), want_rs)
    assert np.array_equal(ed.cpu().numpy()[:want_rs[-1]], want_ed)
    W = _weights(cin, Nq)
    gouts = [kb.gout_family('zero_mean', Nq, COUT, Ns)]
    got = _gpu_grads(c, W, gouts, 'noflags')
    ys, _, _ = _kp_rows(f'KPConv backward, {degrees} in-degrees, Cin={cin}', c, W, gouts, got, 'noflags',
                        names=['zero_mean'], part='degree extremes')
    assert not ys.failures(), ys.failures()


# ------------------------------------------------------------------------------------------ invariance and cache

def _stack(b, a):
    """Cloud b then cloud a as one batch: supports, features and queries concatenated, a's ids shifted past b's,
    every shadow slot moved to the stacked support count."""
    nb, ns = b['Ns'], b['Ns'] + a['Ns']
    ib = np.where((b['idx'] >= 0) & (b['idx'] < nb), b['idx'], ns)
    ia = np.where((a['idx'] >= 0) & (a['idx'] < a['Ns']), a['idx'] + nb, ns)
    return dict(q=np.r_[b['q'], a['q']], s=np.r_[b['s'], a['s']], x=np.r_[b['x'], a['x']], idx=np.r_[ib, ia],
                kp=a['kp'], extent=a['extent'], Ns=ns)


@pytest.mark.parametrize('cin', [4, 64])
def test_kpconv_backward_is_batch_invariant(cin):
    """dx of a cloud is bit-identical alone and stacked after another cloud: the edge rows are per query and each
    support's CSR row keeps its edges' order.  (dW sums over every query of the batch, so stacking changes it.)"""
    a = _kp_inputs(cin, 40, NQ)
    b = _kp_inputs(cin, 40, 47)
    b = dict(b, q=b['q'] + np.float32(0.5), s=b['s'] + np.float32(0.5))
    W = _weights(cin, 5)
    ga = kb.gout_family('offset', NQ, COUT, 1)
    gb = kb.gout_family('zero_mean', 47, COUT, 2)
    (dxa, _), = _gpu_grads(a, W, [ga], 'noflags')
    (dxs, _), = _gpu_grads(_stack(b, a), W, [np.r_[gb, ga]], 'noflags')
    assert torch.equal(dxs[b['Ns']:], dxa)


def test_neighbor_csr_cache_follows_in_place_changes():
    """The same index tensor changed with copy_ (a version bump) gets a fresh transpose, and the KPConv backward
    through it equals that of a new tensor holding the same list."""
    from regtr_b200 import ops
    c = _kp_inputs(16, 40, NQ)
    Ns = c['Ns']
    idx2 = c['idx'][::-1].copy()
    t = _dev(c['idx'], torch.int32)
    rs1, _ = ops.neighbor_csr(t, Ns)
    W = _weights(16, 3)
    g = [kb.gout_family('zero_mean', NQ, COUT, 4)]

    def dx_of(idx_t):
        xs = _dev(c['x']).requires_grad_(True)
        out = ops.kpconv(_dev(c['q']), _dev(c['s']), idx_t, xs, _dev(W), _dev(c['kp']), c['extent'])
        out.backward(_dev(g[0]))
        return xs.grad
    dx1 = dx_of(t)
    t.copy_(_dev(idx2, torch.int32))
    rs2, ed2 = ops.neighbor_csr(t, Ns)
    want_rs, want_ed = kb.csr_numpy(idx2, Ns)
    assert rs2 is not rs1
    assert np.array_equal(rs2.cpu().numpy(), want_rs) and np.array_equal(ed2.cpu().numpy()[:want_rs[-1]], want_ed)
    dx2 = dx_of(t)
    dx_fresh = dx_of(_dev(idx2, torch.int32))
    assert torch.equal(dx2, dx_fresh) and not torch.equal(dx1, dx2)


# -------------------------------------------------------------------------------------------------------- max-pool

@pytest.mark.parametrize('K', kb.POOL_K)
@pytest.mark.parametrize('C', kb.POOL_C)
def test_max_pool_backward_domain(C, K):
    """Ties, all-negative columns, all-shadow rows and rows equal across all K slots (kb.max_pool_case): the forward
    equals float64 exactly, the entries that receive gradient are float64 autograd's and their values are within
    1e-6 max of it; two passes are bit-identical."""
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    x, idx, g = kb.max_pool_case(C, K, seed=C * 1000 + K)

    def run():
        xs = _dev(x).requires_grad_(True)
        y = ops.max_pool(xs, _dev(idx))
        y.backward(_dev(g))
        return y.detach().cpu(), xs.grad.cpu()
    y, dx = run()
    _, dx2 = run()
    assert torch.equal(dx, dx2)
    assert torch.equal(y.double(), O.max_pool(torch.from_numpy(x).double(), torch.from_numpy(idx).long()))
    want = kb.max_pool_dx(x, idx, g, torch.float64)
    err = float((dx.double() - want).abs().max() / want.abs().max())
    print(f'\nmax-pool backward C={C} K={K}: {int((want != 0).sum())} entries receive gradient, '
          f'max error {err:.2e} of max (bound 1e-6)')
    if err / 1e-6 > _WORST.get('max-pool dx (error / 1e-6)', (-1.0, None))[0]:
        _WORST['max-pool dx (error / 1e-6)'] = (err / 1e-6, f'C={C} K={K}')
    fails = kb.max_pool_failures(dx, want)
    assert not fails, fails


def test_max_pool_backward_refuses_more_than_255_neighbours():
    """The backward keeps each winner's slot in a byte: with grad on, K = 256 raises before the forward runs and
    names the limit; the forward alone takes any K; the C entry point refuses K = 256 as well."""
    from oracle import regtr_oracle as O
    from regtr_b200 import lib as _lib
    from regtr_b200 import ops
    x, idx, g = kb.max_pool_case(8, 256)
    with pytest.raises(ValueError, match='at most 255'):
        ops.max_pool(_dev(x).requires_grad_(True), _dev(idx))
    with torch.no_grad():
        y = ops.max_pool(_dev(x), _dev(idx))
    assert torch.equal(y.cpu().double(), O.max_pool(torch.from_numpy(x).double(), torch.from_numpy(idx).long()))
    t = _dev(idx)
    with pytest.raises(_lib.RegtrLibError):
        ops.max_pool_bwd(_dev(x), t, _dev(g), ops.neighbor_csr(t, x.shape[0]))
