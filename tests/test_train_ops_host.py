"""Host tests of the references that tests/test_gpu_train_ops.py holds the training kernels to.  CPU only.

The float64 references equal independent closed forms, and on every case of the GPU tests the fp32 rule is sharp:
the fp32 oracle scaled by (1 + f) fails the row, with f the factor the GPU test's sharpness check uses (5e-6 on the
dx / dX rows except where fp32's own error is larger; printed per case), and so do the LayerNorm with eps x 10 on the
rows where eps matters, the InstanceNorm with the unbiased variance and the InstanceNorm with its LeakyReLU mask taken
from x."""
import math
from collections import defaultdict

import numpy as np
import pytest
import torch

import test_gpu_train_ops as T
from grad_yardstick import errors

LADDER = (5e-6, 1e-5, 2e-5, 5e-5, 1e-4, 2e-4, 5e-4, 1e-3, 2e-3, 5e-3, 1e-2)


def _close(got, want, tol=1e-12):
    assert errors(got, want)[0] <= tol, errors(got, want)


def smallest_failing(fp32, ref):
    """The smallest factor f of LADDER for which fp32 * (1 + f) fails the rule on (fp32, ref); inf if none."""
    return next((f for f in LADDER if T.fails(fp32 * (1 + f), fp32, ref)), math.inf)


class Sharpness:
    """Smallest failing factor per (kernel, tensor, family): checked against test_gpu_train_ops.SHARP, printed."""

    def __init__(self, kernel):
        self.kernel, self.worst = kernel, defaultdict(float)

    def check(self, tensor, family, fp32, ref, case):
        assert T.fails(fp32, fp32, ref) is False
        if not bool(ref.any()):                    # exactly 0 in float64: the GPU test asserts exact zeros
            return
        f = smallest_failing(fp32, ref)
        want = T.sharp_factor(self.kernel, tensor, family)
        assert f <= want, (case, tensor, f, want)
        self.worst[(tensor, family)] = max(self.worst[(tensor, family)], f)

    def report(self):
        for (tensor, family), f in sorted(self.worst.items(), key=str):
            print(f'{self.kernel} {tensor} {family}: (1 + {f:g}) x fp32 fails on every case '
                  f'(factor used: {T.sharp_factor(self.kernel, tensor, family):g})')


# ---------------------------------------------------------------------------------------------------- LayerNorm

@pytest.mark.parametrize('family', T.LN_FAMILIES)
def test_layernorm_reference_and_sharpness(family):
    sh = Sharpness('layernorm')
    for E, n, grads, fam in T.LN_CASES:
        if fam != family or n == 0:
            continue
        c = T.ln_case(E, n, grads, family)
        r64, r32 = T.ln_float64(c), T.ln_reference(c, torch.float32)
        for got, want in zip(T.ln_reference(c, torch.float64), r64):
            if bool(want.any()):
                _close(got, want)
            else:                                   # constant rows' dgamma: torch's float64 is 1e-12 of dbeta
                assert float(got.abs().max()) <= 1e-12 * float(r64[2].abs().max())
        for name, w32, w64 in zip(('dx', 'dgamma', 'dbeta'), r32, r64):
            if bool(w64.any()):
                sh.check(name, family, w32, w64, (E, n, grads))
        if family in ('small_std', 'constant'):
            assert T.fails(T.ln_reference(c, torch.float32, eps=10 * T.EPS)[0], r32[0], r64[0]), (E, n, grads)
    sh.report()


def test_layernorm_constant_rows_are_exact():
    """The constant family's rows sum exactly in fp32: x-hat = 0, so the restated dgamma is exactly 0 and the GPU's
    must be too."""
    for E in T.LN_E:
        c = T.ln_case(E, 65, 'both', 'constant')
        x = c['x']
        assert torch.equal(x.sum(1) / E, x[:, 0]) and not bool(T.ln_float64(c)[1].any())


# ------------------------------------------------------------------------------------------------- InstanceNorm

def in_closed_form(c, slope, mask, eps=T.EPS):
    x = c['x'].double()
    gp = c['g'].double() * T.act_weight(mask, slope, torch.float64)
    dx = torch.zeros_like(x)
    a = 0
    for n in c['lens']:
        if n:
            s, g = x[a:a + n], gp[a:a + n]
            mu = s.mean(0)
            rstd = 1 / torch.sqrt(((s - mu) ** 2).mean(0) + eps)
            xh = (s - mu) * rstd
            dx[a:a + n] = rstd * (g - g.mean(0) - xh * (g * xh).mean(0))
        a += n
    return dx, gp


def _forward_mask(c, dtype=torch.float64):
    z = T.instance_norm(c['x'].to(dtype), c['lens'])
    if c['res'] is not None:
        z = z + c['res'].to(dtype)
    return z > 0


def test_instance_norm_restatement_is_the_oracle():
    from oracle import regtr_oracle as O
    c = T.in_case(36, False, 'normal')
    x = c['x'].double()
    assert torch.equal(T.instance_norm(x, c['lens']), O.instance_norm(x, c['lens']))


@pytest.mark.parametrize('family', T.IN_FAMILIES)
def test_instnorm_reference_and_sharpness(family):
    sh = Sharpness('instnorm')
    for C, slope, with_res, fam in T.IN_CASES:
        if fam != family:
            continue
        case = (C, slope, with_res)
        c = T.in_case(C, with_res, family)
        mask = _forward_mask(c)
        r64 = T.in_reference(c, slope, mask, torch.float64)
        want = in_closed_form(c, slope, mask)
        _close(r64[0], want[0])
        assert torch.equal(r64[1], want[1])
        mask = _forward_mask(c, torch.float32)                  # the decisions an fp32 forward takes
        r64, r32 = T.in_reference(c, slope, mask, torch.float64), T.in_reference(c, slope, mask, torch.float32)
        sh.check('dx', family, r32[0], r64[0], case)
        assert T.fails(T.in_reference(c, slope, mask, torch.float32, unbiased=True)[0], r32[0], r64[0]), case
        if slope >= 0:
            wrong = T.in_reference(c, slope, c['x'] > 0, torch.float32)
            assert T.fails(wrong[0], r32[0], r64[0]), case
            if with_res:
                assert T.fails(wrong[1], r32[1], r64[1]), case
        if family == 'special':                                 # exact zeros reach the activation
            z = T.instance_norm(c['x'], c['lens']) + (0 if c['res'] is None else c['res'])
            assert int((z[:, 1::4] == 0).sum()) >= C // 4 * 4
    sh.report()


def test_instnorm_through_statistics_reference_and_sharpness():
    sh = Sharpness('instats')
    cases = [(T.ins_case(N, with_res, skip), slope) for N, slope, with_res, skip in T.INS_CASES]
    for c, slope in cases + [(T.unary_block_case(), 0.1)]:
        with_res, skip = c['res'] is not None, c['gs'] is not None
        y = c['x'].double() @ c['w'].double().t()
        z = T.instance_norm(y, c['lens']) + (0 if c['res'] is None else c['res'].double())
        r64 = T.ins_reference(c, slope, z > 0, torch.float64)
        cf = dict(x=y, g=c['g'], lens=c['lens'])
        dy, dres = in_closed_form(cf, slope, z > 0)
        want_dx = dy @ c['w'].double() + (0 if c['gs'] is None else c['gs'].double())
        _close(r64[0], want_dx)
        _close(r64[1], dy.t() @ c['x'].double())
        _close(r64[2], dres)
        y32 = c['x'] @ c['w'].t()
        mask = T.instance_norm(y32, c['lens']) + (0 if c['res'] is None else c['res']) > 0
        r64, r32 = T.ins_reference(c, slope, mask, torch.float64), T.ins_reference(c, slope, mask, torch.float32)
        sh.check('dx', None, r32[0], r64[0], (c['w'].shape[0], slope, with_res, skip))
    sh.report()


# ------------------------------------------------------------------------------------------------- dense layers

def test_linear_reference_and_sharpness():
    sh = Sharpness('linear')
    for M, K, N, relu, residual in T.LIN_CASES:
        c = T.lin_case(M, K, N, relu, residual)
        x, w, b = c['x'].double(), c['w'].double(), c['b'].double()
        z = x @ w.t() + b + (0 if c['r'] is None else c['r'].double())
        mask = (z > 0) if relu else None
        gz = c['gy'].double() * (mask.double() if relu else 1)
        r64 = T.lin_reference(c, mask, torch.float64)
        for got, want in zip(r64, (gz @ w, gz.t() @ x, gz.sum(0), gz if residual else None)):
            if want is not None:
                _close(got, want)
        y32 = c['x'] @ c['w'].t() + c['b'] + (0 if c['r'] is None else c['r'])
        mask = (y32 > 0) if relu else None
        r64, r32 = T.lin_reference(c, mask, torch.float64), T.lin_reference(c, mask, torch.float32)
        sh.check('dX', None, r32[0], r64[0], (M, K, N, relu, residual))
    sh.report()


# --------------------------------------------------------------------------------------- relu_bwd, sym_weight

@pytest.mark.parametrize('n', [1, 255, 257, 10 ** 6 + 3])
def test_relu_bwd_inputs_reach_the_subnormal_range(n):
    tiny = np.finfo(np.float32).tiny
    for s in (1.0, float(np.float32(1 / (1 - 0.1)))):
        h, dh = T.relu_bwd_inputs(n)
        want = T.relu_bwd_restated(h, dh, s)
        assert want[0] != 0 and abs(want[0]) < tiny
        assert want[0] == np.float32(np.float64(dh[0]) * np.float32(s))       # exact product, rounded once
        if n > 1:
            assert (h[:12] == 0).any() and np.signbit(h[(h == 0)]).any() and np.isnan(h).any()


def test_sym_restatement_matches_triu_and_two_terms():
    W = T.sym_inputs()
    v, hi, lo = T.sym_restated(W)
    Wt = torch.from_numpy(W).double()
    S = (torch.triu(Wt) + torch.triu(Wt).t()).numpy()
    assert np.array_equal(v.astype(np.float64), S)
    d = np.arange(W.shape[0])
    assert np.array_equal(v[d, d], 2 * W[d, d])
    assert T.sym_two_term_ok(hi, lo, W)
    assert not T.sym_two_term_ok(hi, np.zeros_like(lo), W)             # one TF32 term is not enough
    bits = W.view(np.uint32) & np.uint32(0x1FFF)
    assert (bits == 0x1000).sum() > 100                                # ties are planted


# ------------------------------------------------------------------------------------------------ Adam / AdamW

@pytest.mark.parametrize('step', T.ADAM_STEPS)
@pytest.mark.parametrize('decoupled', [True, False], ids=['AdamW', 'Adam'])
def test_adam_restatement_matches_torch_in_float64(decoupled, step):
    """adam_restated equals torch's own foreach=False step run in float64 on the same state."""
    c = T.adam_case(step, decoupled)
    ps = [torch.nn.Parameter(t.double()) for t in c['p']]
    cls = torch.optim.AdamW if decoupled else torch.optim.Adam
    groups = [dict(params=[q for q, k in zip(ps, T.ADAM_GROUPS) if k == j], lr=lr, weight_decay=wd)
              for j, (lr, wd) in enumerate(T.ADAM_HP)]
    opt = cls(groups, foreach=False)
    if step:
        order = [i for j in range(len(T.ADAM_HP)) for i, k in enumerate(T.ADAM_GROUPS) if k == j]
        sd = opt.state_dict()
        sd['state'] = {pos: {'step': torch.tensor(float(step)), 'exp_avg': c['m'][i].double(),
                             'exp_avg_sq': c['v'][i].double()} for pos, i in enumerate(order)}
        opt.load_state_dict(sd)
    for q, g in zip(ps, c['g']):
        q.grad = g.double()
    opt.step()
    for i, (inc, m, v) in enumerate(T.adam_restated(c, step, decoupled)):
        _close(ps[i].detach() - c['p'][i].double(), inc, 1e-9)
        _close(opt.state[ps[i]]['exp_avg'], m)
        _close(opt.state[ps[i]]['exp_avg_sq'], v)
