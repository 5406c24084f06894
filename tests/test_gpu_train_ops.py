"""GPU tests of the training step's op-level kernels under the fp32 yardstick (tests/grad_yardstick.py): the LayerNorm
backward (`k_layernorm_bwd` + `k_colsum`), the per-cloud InstanceNorm backward (`k_inb_partial` / `k_inb_finalize` /
`k_inb_apply`, alone and behind both InstanceNorm forwards), the dense-layer backward (`regtr_relu_bwd`, the dX GEMM,
`regtr_linear_wgrad`), and one Adam / AdamW step from loaded states.  Each compares the kernel and the same math in
fp32 with float64, on the same inputs and with the GPU's branch decisions (LeakyReLU / ReLU masks read from the
forward's output).  `regtr_relu_bwd` and InfoNCE's `regtr_sym_weight` / `regtr_sym_weight_bwd` are held bit for bit
to a numpy restatement.

Every float case also reruns bit-identically and has sharpness companions: outputs that a subtly wrong kernel would
give (dx times (1 + f), the LayerNorm recomputed with eps x 10, the InstanceNorm with the unbiased variance or with its
LeakyReLU mask taken from x) must fail their rows.  The case builders and references live here;
tests/test_train_ops_host.py checks them on the CPU."""
import itertools
import math

import numpy as np
import pytest
import torch

from grad_yardstick import FACTOR, FLOOR, Yardstick, errors

DEV = 'cuda:0'
EPS = 1e-5


def _seed(*parts):
    s = 0
    for p in parts:
        s = (s * 1000003 + (p if isinstance(p, int) else sum(map(ord, str(p))))) % (2 ** 31)
    return s


def fails(mutated, fp32, ref):
    """True when `mutated` breaks the yardstick rule on (fp32, ref) in one of its two measures."""
    eg, ef = errors(mutated, ref), errors(fp32, ref)
    return not all(a <= FACTOR * b + FLOOR for a, b in zip(eg, ef))


def leaf(t, dtype):
    """A fresh CPU leaf in `dtype` (never the case's own tensor, whose .grad would accumulate across calls)."""
    return t.detach().to('cpu', dtype, copy=True).requires_grad_(True)


def add_row(ys, name, gpu, fp32, ref):
    """A yardstick row, or for a tensor that is exactly 0 in float64 (dgamma of constant rows), exact zeros."""
    ref = ref.detach().double().cpu()
    if ref.numel() == 0:
        return
    if not bool(ref.any()):
        assert not bool(gpu.detach().cpu().any()), f'{ys.title}: {name} must be exactly 0'
        return
    ys.add(name, gpu, fp32, ref)


# Scaling factors f for which `x * (1 + f)` must fail the row of x, on the GPU and in tests/test_train_ops_host.py,
# which prints the smallest failing factor of every case and checks that it is at most this one.  On the CPU the fp32
# oracle times (1 + f) first fails at f = 5e-6 on every dx / dX row except those of the `offset` families, whose rows
# sit 1e3 standard deviations from 0: fp32's own error there is up to 5e-5 (LayerNorm) and 1e-5 (InstanceNorm), so the
# rule cannot see a smaller error.  dgamma and dbeta are sums over up to 1503 rows and first fail at 5e-6 and 1e-5
# (dgamma at 1e-3 on the offset rows).  Away from the 5e-6 dx / dX rows the factor is twice the CPU's, so that the
# GPU's own error (up to 10x fp32's) cannot hide the scaling.
SHARP = {
    ('layernorm', 'dx'): 5e-6, ('layernorm', 'dx', 'offset'): 1e-3,
    ('layernorm', 'dgamma'): 1e-5, ('layernorm', 'dgamma', 'offset'): 2e-3,
    ('layernorm', 'dbeta'): 2e-5,
    ('instnorm', 'dx'): 5e-6, ('instnorm', 'dx', 'offset'): 2e-4,
    ('instats', 'dx'): 5e-6,
    ('linear', 'dX'): 5e-6,
}


def sharp_factor(kernel, tensor, family=None):
    return SHARP.get((kernel, tensor, family), SHARP[(kernel, tensor)])


# ---------------------------------------------------------------------------------------------------- LayerNorm

LN_E = (32, 64, 160, 256)
LN_N = (0, 1, 63, 64, 65, 1503)
LN_GRADS = ('dy', 'dy_pos', 'both', 'both_dres')
LN_FAMILIES = ('normal', 'small_std', 'constant', 'offset')
LN_CASES = list(itertools.product(LN_E, LN_N, LN_GRADS, LN_FAMILIES))


def ln_case(E, n, grads, family):
    """Rows: normal 2·N(0, 1) + 0.5; small_std 0.02 + 0.01·N(0, 1), whose variance is 10x eps; constant, on a 1/8 grid so
    that every row sum and mean is exact in fp32 (rstd = eps^-1/2, x-hat = 0); offset ±1e3 + N(0, 1)."""
    g = torch.Generator().manual_seed(_seed(E, n, grads, family))
    z = torch.randn(n, E, generator=g)
    if family == 'normal':
        x = z * 2 + 0.5
    elif family == 'small_std':
        x = z * 0.01 + 0.02
    elif family == 'constant':
        x = (torch.randint(-40, 41, (n, 1), generator=g).float() / 8).expand(n, E).contiguous()
    else:
        x = z + 1e3 * (torch.randint(0, 2, (n, 1), generator=g).float() * 2 - 1)
    c = dict(x=x, gamma=torch.randn(E, generator=g), beta=torch.randn(E, generator=g),
             pos=torch.randn(n, E, generator=g), dy=None, dyp=None, dres=None)
    if grads in ('dy', 'both', 'both_dres'):
        c['dy'] = torch.randn(n, E, generator=g)
    if grads in ('dy_pos', 'both', 'both_dres'):
        c['dyp'] = torch.randn(n, E, generator=g)
    if grads == 'both_dres':
        c['dres'] = torch.randn(n, E, generator=g)
    return c


def ln_reference(c, dtype, eps=EPS):
    """-> (dx, dgamma, dbeta): torch autograd of F.layer_norm (+ pos, + the residual x) in `dtype`."""
    E = c['x'].shape[1]
    x, gm, bt = (leaf(c[k], dtype) for k in ('x', 'gamma', 'beta'))
    y = torch.nn.functional.layer_norm(x, (E,), gm, bt, eps)
    loss = 0
    if c['dy'] is not None:
        loss = loss + (y * c['dy'].to(dtype)).sum()
    if c['dyp'] is not None:
        loss = loss + ((y + c['pos'].to(dtype)) * c['dyp'].to(dtype)).sum()
    if c['dres'] is not None:
        loss = loss + (x * c['dres'].to(dtype)).sum()
    loss.backward()
    return x.grad, gm.grad, bt.grad


def ln_float64(c, eps=EPS):
    """-> (dx, dgamma, dbeta) restated in float64: with g = dy + dy_pos, x-hat = (x - mean) rstd and g-hat = g gamma,
    dx = rstd (g-hat - mean(g-hat) - x-hat mean(g-hat x-hat)) + dres, dgamma = sum_rows g x-hat, dbeta = sum_rows g.
    (torch's own CPU LayerNorm does not find a constant row's mean exactly, so its dgamma there is 1e-12, not 0.)"""
    x = c['x'].double()
    E = x.shape[1]
    g = torch.zeros_like(x)
    for k in ('dy', 'dyp'):
        if c[k] is not None:
            g = g + c[k].double()
    mu = x.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(((x - mu) ** 2).sum(1, keepdim=True) / E + eps)
    xh = (x - mu) * rstd
    gh = g * c['gamma'].double()
    dx = rstd * (gh - gh.mean(1, keepdim=True) - xh * (gh * xh).mean(1, keepdim=True))
    if c['dres'] is not None:
        dx = dx + c['dres'].double()
    return dx, (g * xh).sum(0), g.sum(0)


@pytest.mark.gpu
@pytest.mark.parametrize('family', LN_FAMILIES)
@pytest.mark.parametrize('grads', LN_GRADS)
@pytest.mark.parametrize('n', LN_N)
@pytest.mark.parametrize('E', LN_E)
def test_layernorm_backward(E, n, grads, family):
    """ops.layernorm_bwd and ops.layernorm_pos autograd (the same bits) against float64, with the sharpness rows."""
    from regtr_b200 import ops
    c = ln_case(E, n, grads, family)
    G = lambda t: None if t is None else t.to(DEV).contiguous()
    args = [G(c[k]) for k in ('x', 'gamma', 'dy', 'dyp', 'dres')]
    dx, dg, db = ops.layernorm_bwd(*args, EPS)
    again = ops.layernorm_bwd(*args, EPS)
    assert all(torch.equal(a, b) for a, b in zip((dx, dg, db), again))
    xs, gs, bs = (G(c[k]).requires_grad_(True) for k in ('x', 'gamma', 'beta'))
    outs = ops.layernorm_pos(xs, gs, bs, G(c['pos']), EPS, want_plain=c['dy'] is not None,
                             want_pos=c['dyp'] is not None, skip=c['dres'] is not None)
    pairs = [(o, G(c[k])) for o, k in zip(outs, ('dy', 'dyp', 'dres')) if c[k] is not None]
    torch.autograd.backward([o for o, _ in pairs], [t for _, t in pairs])
    assert torch.equal(xs.grad, dx) and torch.equal(gs.grad, dg) and torch.equal(bs.grad, db)
    if n == 0:                                     # k_colsum over zero partial blocks
        assert dx.shape == (0, E) and not bool(dg.any()) and not bool(db.any())
        assert not bool(torch.signbit(dg).any()) and not bool(torch.signbit(db).any())
        return
    r64, r32 = ln_float64(c), ln_reference(c, torch.float32)
    ys = Yardstick(f'LayerNorm backward E={E} n={n} {grads} {family}')
    for name, got, w32, w64 in zip(('dx', 'dgamma', 'dbeta'), (dx, dg, db), r32, r64):
        add_row(ys, name, got, w32, w64)
    ys.report()
    assert not ys.failures(), ys.failures()
    for name, got, w32, w64 in zip(('dx', 'dgamma', 'dbeta'), (dx, dg, db), r32, r64):
        if bool(w64.any()):
            f = sharp_factor('layernorm', name, family)
            assert fails(got * (1 + f), w32, w64), (name, f)
    if family in ('small_std', 'constant'):        # eps matters on these rows: a wrong eps fails dx
        for bad in (EPS * 10, 0.0) if family == 'small_std' else (EPS * 10,):
            assert fails(ops.layernorm_bwd(*args, bad)[0], r32[0], r64[0]), bad


@pytest.mark.gpu
def test_layernorm_backward_rejections():
    from regtr_b200 import lib, ops
    for E, what in ((48, 'REGTR_ERR_ARG'), (288, 'REGTR_ERR_UNSUPPORTED')):
        x = torch.randn(5, E, device=DEV)
        with pytest.raises(lib.RegtrLibError, match=what):
            ops.layernorm_bwd(x, torch.ones(E, device=DEV), x, None, None, EPS)


# ------------------------------------------------------------------------------------------------- InstanceNorm

IN_C = (4, 36, 132, 256, 1028)
IN_LENS = (127, 0, 128, 1, 129, 257)              # across the 128-row chunks of k_inb_partial, and sizes 0 and 1
IN_SLOPES = (-1.0, 0.0, 0.1)
IN_FAMILIES = ('normal', 'special', 'offset')
IN_CASES = list(itertools.product(IN_C, IN_SLOPES, (False, True), IN_FAMILIES))
IN_PAD = 37                                       # rows past offs[n_clouds] in the capacity form


def _zero_sum_pattern(n):
    """n values in {-1, 0, 1} that sum to exactly 0, the first one 0."""
    p = np.zeros(n, np.float32)
    k = max(n - 1, 0) // 2 * 2
    p[1:1 + k] = np.tile([-1.0, 1.0], k // 2)
    return torch.from_numpy(p)


def in_case(C, with_res, family, lens=IN_LENS):
    """x (n, C), res or None, the upstream g.  normal: 3·N(0, 1) + 1.5.  special: channel 4j is constant within each
    cloud; channel 4j + 1 is m + 0.5·(0, -1, 1, -1, 1, ...) per cloud with m on a 1/8 grid, so its mean is m exactly and
    the rows where the pattern is 0 normalise to exactly 0 (res is 0 there, so the activation sees exactly 0); the
    other channels as normal.  offset: ±1e3 + N(0, 1) per channel and cloud."""
    n = sum(lens)
    g = torch.Generator().manual_seed(_seed(C, with_res, family, len(lens)))
    x = torch.randn(n, C, generator=g) * 3 + 1.5
    res = torch.randn(n, C, generator=g) if with_res else None
    if family == 'offset':
        x = torch.randn(n, C, generator=g)
    a = 0
    for m in lens:
        if family == 'special':
            lvl = torch.randint(-40, 41, (2, C), generator=g).float() / 8
            x[a:a + m, 0::4] = lvl[0, 0::4]
            x[a:a + m, 1::4] = lvl[1, 1::4] + 0.5 * _zero_sum_pattern(m)[:, None]
            if res is not None:
                res[a:a + m, 1::4] = 0.0
        elif family == 'offset':
            x[a:a + m] += 1e3 * (torch.randint(0, 2, (1, C), generator=g).float() * 2 - 1)
        a += m
    return dict(x=x, res=res, g=torch.randn(n, C, generator=g), lens=list(lens))


def instance_norm(x, lens, eps=EPS, unbiased=False):
    """oracle.regtr_oracle.instance_norm; unbiased=True divides the variance by n - 1 instead (a mutation)."""
    out = torch.empty_like(x)
    a = 0
    for n in map(int, lens):
        if n == 0:
            continue
        seg = x[a:a + n]
        mu = seg.mean(0, keepdim=True)
        var = seg.var(0, unbiased=unbiased and n > 1, keepdim=True)
        out[a:a + n] = (seg - mu) / torch.sqrt(var + eps)
        a += n
    return out


def act_weight(mask, slope, dtype):
    """The LeakyReLU's derivative with the given decisions (mask: pre-activation > 0); 1 without an activation."""
    if slope < 0:
        return torch.ones(mask.shape, dtype=dtype)
    return torch.where(mask, torch.ones((), dtype=dtype), torch.tensor(slope, dtype=dtype))


def in_reference(c, slope, mask, dtype, unbiased=False):
    """-> (dx, dres) of act(InstanceNorm_per_cloud(x) + res) in `dtype`, the activation's decisions given by `mask`."""
    x = leaf(c['x'], dtype)
    r = leaf(torch.zeros(x.shape) if c['res'] is None else c['res'], dtype)
    z = instance_norm(x, c['lens'], unbiased=unbiased) + r
    (z * act_weight(mask, slope, dtype) * c['g'].to(dtype)).sum().backward()
    return x.grad, r.grad


def _nan_rows(t, k):
    return torch.cat([t, torch.full((k, t.shape[1]), float('nan'), device=t.device)])


@pytest.mark.gpu
@pytest.mark.parametrize('family', IN_FAMILIES)
@pytest.mark.parametrize('with_res', [False, True])
@pytest.mark.parametrize('slope', IN_SLOPES)
@pytest.mark.parametrize('C', IN_C)
def test_instnorm_backward(C, slope, with_res, family):
    """ops.instnorm_bwd on instnorm_act's output, the same bits through instnorm_act autograd and in the capacity
    form (NaN padding rows get dx = dres = 0), one-point clouds dx = 0, and the sharpness rows."""
    from regtr_b200 import ops
    c = in_case(C, with_res, family)
    nc, n = len(c['lens']), sum(c['lens'])
    offs = ops.make_offsets(c['lens'], DEV)
    x, g = c['x'].to(DEV), c['g'].to(DEV)
    res = None if c['res'] is None else c['res'].to(DEV)
    out = ops.instnorm_act(x, offs, nc, res=res, slope=slope)
    dx, dres = ops.instnorm_bwd(g, x, out, offs, nc, slope, want_dres=True)
    dx2, dres2 = ops.instnorm_bwd(g, x, out, offs, nc, slope, want_dres=True)
    assert torch.equal(dx, dx2) and torch.equal(dres, dres2)
    xs = x.clone().requires_grad_(True)
    rs = None if res is None else res.clone().requires_grad_(True)
    y = ops.instnorm_act(xs, offs, nc, res=rs, slope=slope)
    y.backward(g)
    assert torch.equal(y.detach(), out) and torch.equal(xs.grad, dx) and (rs is None or torch.equal(rs.grad, dres))
    cx, cr = ops.instnorm_bwd(_nan_rows(g, IN_PAD), _nan_rows(x, IN_PAD), _nan_rows(out, IN_PAD), offs, nc, slope,
                              want_dres=True)
    assert torch.equal(cx[:n], dx) and torch.equal(cr[:n], dres)
    assert not bool(cx[n:].any()) and not bool(cr[n:].any()) and not bool(cx[n:].isnan().any())
    starts = np.concatenate([[0], np.cumsum(c['lens'])])
    single = [int(starts[i]) for i, m in enumerate(c['lens']) if m == 1]
    assert not bool(dx[single].any())                               # one-point clouds: dx = 0 exactly
    mask = out.cpu() > 0
    r64 = in_reference(c, slope, mask, torch.float64)
    r32 = in_reference(c, slope, mask, torch.float32)
    ys = Yardstick(f'InstanceNorm backward C={C} slope={slope:g} res={with_res} {family}')
    add_row(ys, 'dx', dx, r32[0], r64[0])
    if with_res:
        add_row(ys, 'dres', dres, r32[1], r64[1])
    ys.report()
    assert not ys.failures(), ys.failures()
    assert fails(dx * (1 + sharp_factor('instnorm', 'dx', family)), r32[0], r64[0])
    assert fails(in_reference(c, slope, mask, torch.float32, unbiased=True)[0], r32[0], r64[0])
    if slope >= 0:                                 # the kernel fed x in place of out takes its mask from x
        wrong = ops.instnorm_bwd(g, x, x, offs, nc, slope, want_dres=True)
        assert fails(wrong[0], r32[0], r64[0])
        if with_res:
            assert fails(wrong[1], r32[1], r64[1])


@pytest.mark.gpu
def test_instnorm_backward_rejects_channels_not_a_multiple_of_4():
    from regtr_b200 import lib, ops
    offs = ops.make_offsets([3, 2], DEV)
    x = torch.randn(5, 6, device=DEV)
    with pytest.raises(lib.RegtrLibError, match='REGTR_ERR_UNSUPPORTED'):
        ops.instnorm_bwd(x, x, None, offs, 2, -1.0)


INS_CASES = list(itertools.product((32, 160, 256), (-1.0, 0.1), (False, True), (False, True)))


def ins_case(N, with_res, skip):
    lens = IN_LENS
    n, K = sum(lens), 64
    g = torch.Generator().manual_seed(_seed(N, with_res, skip))
    return dict(x=torch.randn(n, K, generator=g), w=torch.randn(N, K, generator=g) / 8,
                res=torch.randn(n, N, generator=g) if with_res else None, g=torch.randn(n, N, generator=g),
                gs=torch.randn(n, K, generator=g) if skip else None, lens=list(lens))


def ins_reference(c, slope, mask, dtype):
    """-> (dx, dW, dres) of act(InstanceNorm(x W^T) + res), plus the shortcut's gradient on x when skip."""
    x, w = leaf(c['x'], dtype), leaf(c['w'], dtype)
    r = leaf(torch.zeros(x.shape[0], w.shape[0]) if c['res'] is None else c['res'], dtype)
    z = instance_norm(x @ w.t(), c['lens']) + r
    loss = (z * act_weight(mask, slope, dtype) * c['g'].to(dtype)).sum()
    if c['gs'] is not None:
        loss = loss + (x * c['gs'].to(dtype)).sum()
    loss.backward()
    return x.grad, w.grad, r.grad


def unary_block_case():
    """The model's UnaryBlock shape: clouds of 200, 1 and 333 points, 64 -> 128 channels, a residual, no shortcut."""
    lens = [200, 1, 333]
    n = sum(lens)
    g = torch.Generator().manual_seed(5)
    x, w = torch.randn(n, 64, generator=g), torch.randn(128, 64, generator=g) / 8
    res, gy = torch.randn(n, 128, generator=g), torch.randn(n, 128, generator=g)
    return dict(x=x, w=w, res=res, g=gy, gs=None, lens=lens)


def check_instats_backward(c, slope):
    """linear_instats (statistics from the GEMM epilogue; with c['gs'] the skip output hands x to the shortcut, whose
    gradient c['gs'] joins the dX GEMM's epilogue) -> instnorm_apply: dx, dW and dres under the yardstick, a
    bit-identical rerun, and dx * (1 + 5e-6) failing its row."""
    from regtr_b200 import ops
    skip, with_res = c['gs'] is not None, c['res'] is not None
    nc = len(c['lens'])
    offs = ops.make_offsets(c['lens'], DEV)

    def run():
        xs, ws = c['x'].to(DEV).requires_grad_(True), c['w'].to(DEV).requires_grad_(True)
        rs = None if c['res'] is None else c['res'].to(DEV).requires_grad_(True)
        r = ops.linear_instats(xs, ws, offs, nc, skip=skip)
        out = ops.instnorm_apply(r[0], offs, nc, r[1], res=rs, slope=slope)
        if skip:
            torch.autograd.backward([out, r[2]], [c['g'].to(DEV), c['gs'].to(DEV)])
        else:
            out.backward(c['g'].to(DEV))
        return out.detach(), xs.grad, ws.grad, (None if rs is None else rs.grad)

    out, dx, dw, dr = run()
    again = run()
    assert all(a is None and b is None or torch.equal(a, b) for a, b in zip((out, dx, dw, dr), again))
    mask = out.cpu() > 0
    r64, r32 = ins_reference(c, slope, mask, torch.float64), ins_reference(c, slope, mask, torch.float32)
    ys = Yardstick(f'linear_instats -> instnorm_apply backward lens={c["lens"]} N={c["w"].shape[0]} '
                   f'slope={slope:g} res={with_res} skip={skip}')
    add_row(ys, 'dx', dx, r32[0], r64[0])
    add_row(ys, 'dW', dw, r32[1], r64[1])
    if with_res:
        add_row(ys, 'dres', dr, r32[2], r64[2])
    ys.report()
    assert not ys.failures(), ys.failures()
    assert fails(dx * (1 + sharp_factor('instats', 'dx')), r32[0], r64[0])


@pytest.mark.gpu
@pytest.mark.parametrize('N,slope,with_res,skip', INS_CASES)
def test_instnorm_backward_through_linear_instats(N, slope, with_res, skip):
    """UnaryBlock's path on the chunk-boundary clouds, with and without the residual and the shortcut (skip=True).
    The model's own shape is tests/test_gpu_kpconv_backward.py::test_instnorm_backward_through_epilogue_statistics."""
    check_instats_backward(ins_case(N, with_res, skip), slope)


# ------------------------------------------------------------------------------------------------- dense layers

LIN_CONFIGS = [(256, 768, False, False), (256, 1024, True, False), (1024, 256, False, True), (256, 256, True, False),
               (256, 3, False, False), (256, 1, False, False), (256, 3, True, False), (256, 1, True, False)]
LIN_M = (1, 37, 1503)
LIN_CASES = [(M,) + cfg for M in LIN_M for cfg in LIN_CONFIGS]


def lin_case(M, K, N, relu, residual):
    g = torch.Generator().manual_seed(M * 7 + N + 1000 * relu)
    return dict(x=torch.randn(M, K, generator=g), w=torch.randn(N, K, generator=g) / math.sqrt(K),
                b=torch.randn(N, generator=g), r=torch.randn(M, N, generator=g) if residual else None,
                gy=torch.randn(M, N, generator=g))


def lin_reference(c, mask, dtype):
    """-> (dX, dW, db, dres) of act(x W^T + b + r) in `dtype`; mask: the ReLU's decisions (None: no ReLU)."""
    x, w, b = (leaf(c[k], dtype) for k in ('x', 'w', 'b'))
    r = None if c['r'] is None else leaf(c['r'], dtype)
    z = x @ w.t() + b + (0 if r is None else r)
    if mask is not None:
        z = z * mask.to(dtype)
    z.backward(c['gy'].to(dtype))
    return x.grad, w.grad, b.grad, (None if r is None else r.grad)


@pytest.mark.gpu
@pytest.mark.parametrize('M,K,N,relu,residual', LIN_CASES)
def test_linear_backward(M, K, N, relu, residual):
    """_LinearFn's backward (regtr_relu_bwd, the dX GEMM, regtr_linear_wgrad) through ops.linear autograd."""
    from regtr_b200 import ops
    c = lin_case(M, K, N, relu, residual)

    def run():
        xs, ws, bs = (c[k].to(DEV).requires_grad_(True) for k in ('x', 'w', 'b'))
        rs = None if c['r'] is None else c['r'].to(DEV).requires_grad_(True)
        y = ops.linear(xs, ws, bs, residual=rs, relu=relu)
        y.backward(c['gy'].to(DEV))
        return y.detach(), xs.grad, ws.grad, bs.grad, (None if rs is None else rs.grad)

    y, dx, dw, db, dr = run()
    again = run()
    assert all(a is None and b is None or torch.equal(a, b) for a, b in zip((y, dx, dw, db, dr), again))
    mask = (y.cpu() > 0) if relu else None
    r64, r32 = lin_reference(c, mask, torch.float64), lin_reference(c, mask, torch.float32)
    ys = Yardstick(f'dense backward M={M} K={K} N={N} relu={relu} residual={residual}')
    for name, got, w32, w64 in zip(('dX', 'dW', 'db', 'dres'), (dx, dw, db, dr), r32, r64):
        if w64 is not None:
            add_row(ys, name, got, w32, w64)
    ys.report()
    assert not ys.failures(), ys.failures()
    if bool(r64[0].any()):
        assert fails(dx * (1 + sharp_factor('linear', 'dX')), r32[0], r64[0])


# ------------------------------------------------------------------------------------------------ regtr_relu_bwd

def relu_bwd_inputs(n):
    """h and dh (fp32 numpy) with h = ±0, NaN, ±inf and ±subnormal, dh subnormal, ±0, NaN and near the overflow, in the
    first entries; entry 0 always has h > 0 and a subnormal dh (so dh·scale is subnormal and must not flush)."""
    rng = np.random.default_rng(n)
    h = rng.standard_normal(n).astype(np.float32)
    dh = rng.standard_normal(n).astype(np.float32)
    sub = np.float32(3e-39)
    hs = np.array([1.0, 0.0, -0.0, 1e-45, -1e-45, 1e-40, np.nan, np.inf, -np.inf, 2.0, 0.5, 3.0], np.float32)
    ds = np.array([sub, 1.0, 1.0, 1.0, 1.0, -2.0, 1.0, 1.0, 1.0, -1e-45, -0.0, 3.3e38], np.float32)
    k = min(n, len(hs))
    h[:k], dh[:k] = hs[:k], ds[:k]
    if n > 64:
        h[-40:] = np.abs(h[-40:])
        dh[-40:] = rng.standard_normal(40).astype(np.float32) * np.float32(1e-38)     # subnormal and normal tiny
    return h, dh


def relu_bwd_restated(h, dh, scale):
    with np.errstate(over='ignore', invalid='ignore'):
        prod = (dh * np.float32(scale)).astype(np.float32)
    return np.where(h > 0, prod, np.float32(0.0)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize('scale', ['1', 'dropout'])
@pytest.mark.parametrize('n', [1, 255, 257, 10 ** 6 + 3])
def test_relu_bwd_is_bit_exact(n, scale):
    """out = where(h > 0, fp32(dh · scale), +0), bit for bit (NaN where the product is NaN); the dropout's scale is
    1 / (1 - 0.1) in fp32.  A subnormal dh · scale survives: the build has no flush-to-zero."""
    from regtr_b200 import ops
    s = 1.0 if scale == '1' else ops.dropout_scale(0.1)
    h, dh = relu_bwd_inputs(n)
    out = ops.relu_bwd(torch.from_numpy(dh).to(DEV), torch.from_numpy(h).to(DEV), s).cpu().numpy()
    want = relu_bwd_restated(h, dh, s)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(out), nan)
    assert np.array_equal(out[~nan].view(np.uint32), want[~nan].view(np.uint32))
    assert out[0] != 0 and abs(out[0]) < np.finfo(np.float32).tiny          # subnormal, not flushed
    assert (out[(np.abs(want) < np.finfo(np.float32).tiny) & (want != 0)] != 0).all()


# ------------------------------------------------------------------------------------- InfoNCE's symmetric weight

def sym_inputs(seed=0, D=256):
    """W (D, D) fp32: N(0, 1) with TF32 rounding ties of both parities, one ulp either side of a tie, -0, subnormals
    and large magnitudes planted above, on and below the diagonal."""
    rng = np.random.default_rng(seed)
    W = rng.standard_normal((D, D)).astype(np.float32)
    u = W.view(np.uint32)
    idx = rng.choice(D * D, 3000, replace=False)
    low = np.array([0x1000, 0x0FFF, 0x1001, 0x3000, 0x2FFF, 0x0000, 0x1FFF], np.uint32)
    flat = u.reshape(-1)
    flat[idx] = (flat[idx] & np.uint32(0xFFFFC000)) | low[np.arange(len(idx)) % len(low)]
    for r, c in ((0, 0), (3, 7), (7, 3), (100, 100), (5, 200)):
        W[r, c] = -0.0
    for r, c in ((1, 1), (2, 9), (9, 2), (40, 41)):
        W[r, c] = np.float32(2.5e-40)
    W[10, 10], W[11, 12], W[12, 11] = np.float32(1e38), np.float32(-3e37), np.float32(3e37)
    return W


def sym_restated(W):
    """(v, hi, lo) of k_sym_weight in fp32: v = (c >= r ? W[r, c] : 0) + (r >= c ? W[c, r] : 0), hi = tf32_rne(v),
    lo = tf32_rne(v - hi)."""
    from gemm_oracle import tf32_rne
    r, c = np.indices(W.shape)
    z = np.float32(0.0)
    v = (np.where(c >= r, W, z) + np.where(r >= c, W.T, z)).astype(np.float32)
    hi = tf32_rne(v)
    return v, hi, tf32_rne((v - hi).astype(np.float32))


def sym_two_term_ok(hi, lo, W):
    """hi + lo against the float64 triu(W) + triu(W)^T: within TF32's two-term rounding, 2^-22 |S| (plus 2^-136, the
    TF32 spacing among subnormals)."""
    S = np.triu(W.astype(np.float64)) + np.triu(W.astype(np.float64)).T
    err = np.abs(hi.astype(np.float64) + lo.astype(np.float64) - S)
    return bool((err <= 2.0 ** -22 * np.abs(S) + 2.0 ** -136).all())


@pytest.mark.gpu
def test_sym_weight_is_bit_exact():
    from regtr_b200 import lib, ops
    W = sym_inputs()
    hi, lo = (t.cpu().numpy() for t in ops.sym_weight(torch.from_numpy(W).to(DEV)))
    v, want_hi, want_lo = sym_restated(W)
    assert np.array_equal(hi.view(np.uint32), want_hi.view(np.uint32))
    assert np.array_equal(lo.view(np.uint32), want_lo.view(np.uint32))
    d = np.arange(W.shape[0])
    assert np.array_equal(v[d, d], (2 * W[d, d]).astype(np.float32))              # the diagonal is 2 W, exactly
    assert sym_two_term_ok(hi, lo, W)
    with pytest.raises(lib.RegtrLibError):
        ops.sym_weight(torch.zeros(128, 128, device=DEV))


@pytest.mark.gpu
def test_sym_weight_bwd_is_bit_exact():
    """dW += dWs + dWs^T on and above the diagonal, the sum of the pair rounded first; below it dW keeps its bits."""
    from regtr_b200 import ops
    rng = np.random.default_rng(1)
    dWs = rng.standard_normal((256, 256)).astype(np.float32)
    dW0 = rng.standard_normal((256, 256)).astype(np.float32)
    dW0[5, 2], dW0[2, 5] = np.float32(-0.0), np.float32(np.nan)
    dW = torch.from_numpy(dW0).to(DEV)
    ops.sym_weight_bwd(torch.from_numpy(dWs).to(DEV), dW)
    got = dW.cpu().numpy()
    r, c = np.indices(dWs.shape)
    want = np.where(c >= r, (dW0 + (dWs + dWs.T).astype(np.float32)).astype(np.float32), dW0)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


# ------------------------------------------------------------------------------------------------ Adam / AdamW

ADAM_SHAPES = [(256, 256), (1000,), (33, 7), (4097,), (5,)]
ADAM_GROUPS = [0, 0, 1, 1, 0]
ADAM_HP = [(1e-3, 1e-2), (3e-4, 0.1)]                 # (lr, weight decay) per group
ADAM_STEPS = (0, 1, 2, 1000, 100000)                  # the loaded state's step count; 0: no state (the fresh path)
# Share of p / m / v entries equal bit for bit to torch's foreach=False step on the same state, at least this on every
# case.  Measured on an H100 80GB HBM3: 1.0 from the states at steps 1, 1000 and 100000; from a fresh state 0.99908
# (Adam) and 0.99927 (AdamW), from step 2 0.99956 and 0.99958.  m and v are always identical; the differing entries
# are p's last bit, and the dp rows above hold them to float64.
ADAM_SAME_AS_TORCH = 0.999


def adam_case(step, decoupled):
    g = torch.Generator().manual_seed(_seed(step, decoupled))
    p = [torch.randn(s, generator=g) for s in ADAM_SHAPES]
    gr = [torch.randn(s, generator=g) * 0.1 for s in ADAM_SHAPES]
    m = [torch.randn(s, generator=g) * 0.03 for s in ADAM_SHAPES]
    v = [(torch.randn(s, generator=g) * 0.1) ** 2 + 1e-6 for s in ADAM_SHAPES]
    return dict(p=p, g=gr, m=m, v=v)


def adam_restated(c, step, decoupled, b1=0.9, b2=0.999, eps=1e-8):
    """One step in float64 from the fp32 state (step 0: m = v = 0): -> (increment p_new - p, m_new, v_new) per tensor."""
    t = step + 1
    out = []
    for i in range(len(ADAM_SHAPES)):
        lr, wd = ADAM_HP[ADAM_GROUPS[i]]
        p, g = c['p'][i].double(), c['g'][i].double()
        m, v = (c['m'][i].double(), c['v'][i].double()) if step else (torch.zeros_like(p), torch.zeros_like(p))
        q = p * (1 - lr * wd) if decoupled else p
        if not decoupled:
            g = g + wd * p
        m = m + (1 - b1) * (g - m)
        v = b2 * v + (1 - b2) * g * g
        q = q - lr / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)
        out.append((q - p, m, v))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('step', ADAM_STEPS)
@pytest.mark.parametrize('decoupled', [True, False], ids=['AdamW', 'Adam'])
def test_adam_increment_matches_float64(decoupled, step):
    """One library step from a state loaded through load_state_dict against torch's foreach=False step on the same
    state (the fp32 reference) and a float64 restatement: the increment p_new - p, m and v per tensor."""
    from regtr_b200 import optim
    c = adam_case(step, decoupled)
    LibC, RefC = (optim.AdamW, torch.optim.AdamW) if decoupled else (optim.Adam, torch.optim.Adam)

    def make(cls, **kw):
        ps = [torch.nn.Parameter(t.to(DEV)) for t in c['p']]
        groups = [dict(params=[q for q, k in zip(ps, ADAM_GROUPS) if k == j], lr=lr, weight_decay=wd)
                  for j, (lr, wd) in enumerate(ADAM_HP)]
        opt = cls(groups, **kw)
        if step:
            order = [i for j in range(len(ADAM_HP)) for i, k in enumerate(ADAM_GROUPS) if k == j]
            sd = opt.state_dict()
            sd['state'] = {pos: {'step': torch.tensor(float(step)), 'exp_avg': c['m'][i].to(DEV),
                                 'exp_avg_sq': c['v'][i].to(DEV)} for pos, i in enumerate(order)}
            opt.load_state_dict(sd)
        for q, gr in zip(ps, c['g']):
            q.grad = gr.to(DEV)
        opt.step()
        return ps, opt

    lib_p, lib = make(LibC)
    ref_p, ref = make(RefC, foreach=False)
    torch.cuda.synchronize()
    want = adam_restated(c, step, decoupled)
    ys = Yardstick(f'{"AdamW" if decoupled else "Adam"} step {step + 1} (loaded state step {step})')
    same = total = 0
    differ = [0, 0, 0]
    for i, (p, q) in enumerate(zip(lib_p, ref_p)):
        sl, sr = lib.state[p], ref.state[q]
        assert float(sl['step']) == step + 1 and sl['step'].device.type == 'cpu'
        p0 = c['p'][i].double()
        ys.add(f'dp[{i}]', p.detach().double().cpu() - p0, q.detach().double().cpu() - p0, want[i][0])
        ys.add(f'm[{i}]', sl['exp_avg'], sr['exp_avg'], want[i][1])
        ys.add(f'v[{i}]', sl['exp_avg_sq'], sr['exp_avg_sq'], want[i][2])
        for k, (a, b) in enumerate(((p.detach(), q.detach()), (sl['exp_avg'], sr['exp_avg']),
                                    (sl['exp_avg_sq'], sr['exp_avg_sq']))):
            same += int((a == b).sum())
            total += a.numel()
            differ[k] += int((a != b).sum())
    ys.report()
    print(f'  {same / total:.6f} of p / m / v entries bit-identical to torch (differing: p {differ[0]}, m {differ[1]}, '
          f'v {differ[2]})')
    assert not ys.failures(), ys.failures()
    assert same / total >= ADAM_SAME_AS_TORCH, same / total
