"""GPU tests of the attention core's backward (regtr_mha_varlen_bwd) on inputs shaped like the model's.

The kernel's dQ, dK and dV are compared, each as its own row, with float64 autograd under the fp32 yardstick
(tests/grad_yardstick.py), and the invariants of tests/attention_oracle.py are checked per problem and head.  Each
input family targets one way this kernel can go wrong:
  zero_mean   q, k, v ~ 1.5 N(0, 1): the easy case;
  bias        q and k carry a per-head offset 3x their spread (the in-projection bias): an error in sum_j dS_ij
              reaches dQ / dK multiplied by the offset.  (An offset on v as well would leave the fp32 reference's own
              dQ about 1e-5 off float64, too loose a yardstick to flag a 1e-5 error; the flat family has one);
  flat        tiny q, so P is near uniform, and v with a shared offset, so dP - delta cancels almost entirely;
  peaked      base-2 scores up to 60: P is nearly one-hot;
  shared_do   dO with a per-head shared component 10x its spread: delta is large against dP - delta.
Shapes: self problems of 1, 17, 64, 65, 731 and 1500 tokens (the coarse level of a 35k-point 3DMatch-config cloud
holds about 500), then cross problems over four clouds of 40, 130, 77 and 0 tokens (q_len != k_len, an empty key range
and an empty query range), all in one launch.
"""
import pytest
import torch

import attention_oracle as ao
from grad_yardstick import Yardstick

pytestmark = pytest.mark.gpu

H = 8
FAMILIES = ao.FAMILIES


def _gpu(q, k, v, d_o, problems, o=None, lse=None):
    return ao.run_kernel(q, k, v, d_o, problems, H, o, lse)


_CASES = {}


def _case(family):
    """Inputs and CPU references of a family (computed once per session): the float64 and fp32 references with keys
    k and with keys k + c."""
    if family not in _CASES:
        self_p, cross_p, n = ao.layout()
        problems = self_p + cross_p
        q, k, v, d_o = ao.family(family, n, problems, H)
        ks = k + ao.key_shift(k, problems, H)
        ref = {(dt, sh): ao.reference(q, kk, v, d_o, problems, H, dt)
               for dt in (torch.float64, torch.float32) for sh, kk in ((False, k), (True, ks))}
        _CASES[family] = dict(self_p=self_p, cross_p=cross_p, problems=problems, x=(q, k, v, d_o), ks=ks, ref=ref)
    return _CASES[family]


def _check(title, c, got, got_shift):
    """Yardstick rows (self / cross x dq / dk / dv) and invariants; prints both tables -> (row failures, invariant
    failures)."""
    ref, d_o = c['ref'], c['x'][3]
    r64, r32, s64, s32 = (ref[torch.float64, False], ref[torch.float32, False], ref[torch.float64, True],
                          ref[torch.float32, True])
    ys = Yardstick(title)
    ao.add_rows(ys, 'self ', c['self_p'], got, r32, r64)
    ao.add_rows(ys, 'cross ', c['cross_p'], got, r32, r64)
    ys.report()
    inv = ao.invariants(c['problems'], H, d_o, got, r32, r64, got_shift, s32, s64)
    ao.report_invariants(title, inv)
    return ys.failures(), ao.failed(inv)


@pytest.mark.parametrize('family', FAMILIES)
def test_attention_backward_split_rows_and_invariants(family):
    """The training path: the kernel's forward gives O and lse, then the backward.  dq, dk and dv meet the
    yardstick separately, for the self and for the cross problems, and the invariants hold per problem and head.
    Empty ranges give exact zeros, and a second backward is bit-identical."""
    c = _case(family)
    q, k, v, d_o = c['x']
    got = _gpu(q, k, v, d_o, c['problems'])
    got_shift = _gpu(q, c['ks'], v, d_o, c['problems'])
    rows, inv = _check(f'attention backward, {family} inputs, O and lse from the forward kernel', c, got, got_shift)
    e = c['cross_p'][2]                                  # empty key range -> dQ = 0; no queries -> dK = dV = 0
    assert float(got['dq'][e[0]:e[0] + e[1]].abs().max()) == 0.0
    assert float(got['dk'][e[0]:e[0] + e[1]].abs().max()) == 0.0 and float(got['dv'][e[0]:e[0] + e[1]].abs().max()) == 0.0
    again = _gpu(q, k, v, d_o, c['problems'])
    assert all(torch.equal(got[t], again[t]) for t in got)
    assert not rows, rows
    assert not inv, inv[:8]


@pytest.mark.parametrize('family', FAMILIES)
def test_attention_backward_arithmetic_given_float64_softmax(family):
    """The backward alone: O and lse of the float64 reference, rounded to fp32, in place of the forward kernel's.
    This separates the backward's own arithmetic from any inconsistency between the forward's softmax and the one
    the backward recomputes."""
    c = _case(family)
    q, k, v, d_o = c['x']
    r64, s64 = c['ref'][torch.float64, False], c['ref'][torch.float64, True]
    got = _gpu(q, k, v, d_o, c['problems'], r64['o'].float(), r64['lse'].float())
    got_shift = _gpu(q, c['ks'], v, d_o, c['problems'], s64['o'].float(), s64['lse'].float())
    rows, inv = _check(f'attention backward, {family} inputs, O and lse from float64', c, got, got_shift)
    assert not rows, rows
    assert not inv, inv[:8]


def test_attention_backward_checks_are_sharp():
    """On the bias family: a dQ, dK or dV scaled by (1 + 1e-5) fails its yardstick row for both the self and the
    cross problems, and a delta raised by 1e-5 of itself (changing dQ and dK as ao.reference describes) fails the
    sum dK and dQ(k + c) invariants.  The changes are applied to the kernel's outputs here, not to the kernel."""
    c = _case('bias')
    q, k, v, d_o = c['x']
    got = _gpu(q, k, v, d_o, c['problems'])
    got_shift = _gpu(q, c['ks'], v, d_o, c['problems'])
    for t in ('dq', 'dk', 'dv'):
        bad = dict(got, **{t: got[t] * (1 + 1e-5)})
        rows, _ = _check(f'bias inputs, {t} x (1 + 1e-5)', c, bad, got_shift)
        assert f'self {t}' in rows and f'cross {t}' in rows, (t, rows)
    r64, s64 = c['ref'][torch.float64, False], c['ref'][torch.float64, True]
    bad = dict(got, dk=got['dk'].double() - 1e-5 * r64['ddk'])
    bad_shift = dict(got_shift, dq=got_shift['dq'].double() - 1e-5 * s64['ddq'])
    _, inv = _check('bias inputs, delta x (1 + 1e-5)', c, bad, bad_shift)
    assert {r[0] for r in inv} >= {'sum dK = 0', 'dQ(k + c)'}, {r[0] for r in inv}
