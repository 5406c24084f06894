"""GPU tests of the bf16 wgmma attention core (`regtr_mha_bf16_tc_fwd`, csrc/attention_tc.cu), the `bf16_tc` fast
mode, against a float64 restatement of its own rounding (attention_oracle.bf16_forward_reference).

The core is called through `lib` on bf16 QK / Vt built on the host, so it is tested apart from the in-projection GEMM
(tests/test_gpu_gemm.py holds that GEMM's bf16 epilogue to bf16 RNE).  O is checked under the fp32 yardstick
(tests/grad_yardstick.py): the restatement run in fp32, with the same bf16 rounding of p, says how far an fp32
computation of the operation may be from float64.

Near ties.  A p within a few fp32 ulps of a bf16 rounding midpoint may round to either neighbour in fp32 (a flip),
and one flip moves a row of O by up to 2^-8 p_j / l of a value, far more than fp32 arithmetic does.  On the families
layout the fp32 run flips 171 (flat) to 3745 (peaked) of 22.8M p; on the model's activations often none in a call,
while the kernel flips other entries.  The plain yardstick then fails a correct kernel (a model of one, fp32 scores
and exp2 with bf16 p, is 10 to 400 times off the fp32 run per problem and head; on an H100 the kernel was about 500 times
off it on layer 2's self attention of fwd_3dmatch_small_b2, where the fp32 run flipped no p) and, where the fp32 run
flips many, passes O x (1 + 1e-4).  So the restatement also marks the p whose exact value lies within an fp32
computation's error of a midpoint (`ties`: 0.05% to 15% of the p) and how far flipping all of them could move each
output; both the kernel's and the fp32 run's deviations are shrunk by that before the yardstick compares them
(attention_oracle.beyond_ties).  Every flip of the fp32 run lies among the marked p
(tests/test_attention_bf16_host.py), and what is left is fp32 arithmetic: O x (1 + 1e-5) fails every row.

Layouts, each key range with its purpose:
  * 'families': ATT_SELF_LENS self problems and the cross problems of attention_oracle.layout, among them an empty
    key range (77 queries, 0 keys) and an empty query range;
  * 'edges': EDGE below: k_start at every residue mod 8 (0 to 7 masked leading keys in the first tile), 1 to 5 key
    tiles and 21 and 24 (pass 2 starting on stage 1 and stage 0, the ring phase wrapping 10 and 12 times), query
    ranges of one, two and many 128-query CTAs (a 1-row last tile, last tiles whose rows all belong to the first
    warpgroup), an empty key and an empty query range, and a last problem whose Q and K tiles run past the end of
    the token array.
Every launch uses ld_qk > 2E, an ld_vt above the minimum with a large finite value in Vt's padding columns, and
ldo > E into a sentinel-filled output; rows and columns outside the problems' query rows must keep the sentinel.
"""
import math

import numpy as np
import pytest
import torch

import attention_oracle as ao
from grad_yardstick import Yardstick

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
H = 8
E = H * ao.HD
ATT_SELF_LENS = ao.SELF_LENS + [127, 128, 129]
FAMILIES = ['zero_mean', 'bias', 'flat', 'peaked']
QK_PAD, VT_PAD, O_PAD = 24, 72, 12            # ld_qk = 2E + 24, ld_vt = n rounded up to 8 + 72, ldo = E + 12
OUT_SENT = float(np.float32(-1.2345e30))
PAD_SENT = 2.0 ** 100                         # large finite bf16 in the padding columns of QK and Vt
POISON = 4096.0                               # large finite bf16 for the tokens a problem must not see
OK, UNSUPPORTED = 0, -3

# (query length, k_start mod 8, key length, purpose); key tiles n_kt = ceil((k_start % 8 + k_len) / 64)
EDGE = [
    (1, 0, 64, 'one query; one full key tile'),
    (2, 1, 100, 'two queries; 2 tiles'),
    (64, 2, 150, 'first warpgroup only; 3 tiles'),
    (65, 3, 190, 'both warpgroups, one row in the second; 4 tiles, 1 key in the last'),
    (128, 4, 300, 'one full CTA; 5 tiles'),
    (129, 5, 1, 'two CTAs, a 1-row last tile; a single key'),
    (192, 6, 58, 'two CTAs, the last one first warpgroup only; 6 masked + 58 keys = exactly one tile'),
    (200, 7, 58, 'two CTAs; 7 masked leading keys, 2 tiles with 1 key in the second'),
    (257, 3, 1300, 'three CTAs, a 1-row last tile; 21 tiles: pass 2 starts on stage 1'),
    (700, 6, 1500, 'six CTAs; 24 tiles: pass 2 starts on stage 0'),
    (300, 0, 0, 'empty key range: zero rows'),
    (0, 2, 77, 'empty query range: writes nothing'),
    (40, 1, 70, 'last: key range ends at the last token, Q and K tiles run past it'),
]


def _lib():
    from regtr_b200 import lib
    return lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def edge_layout():
    """(problems, n) of EDGE.  Before each key range a gap of 8 to 15 tokens that no problem uses (the first tile's
    masked leading keys are gap tokens, or the previous problem's queries); keys, then the problem's own queries.  The
    last problem puts its queries first and its keys at the very end."""
    problems, r = [], 0
    for ql, res, kl, _ in EDGE[:-1]:
        r += (res - r) % 8 + 8
        problems.append((r + kl, ql, r, kl))
        r += kl + ql
    ql, res, kl, _ = EDGE[-1]
    qs = r
    r += ql
    r += (res - r) % 8
    problems.append((qs, ql, r, kl))
    return problems, r + kl


def _layout(name):
    """(problems, n, groups [(row name, problems)])."""
    if name == 'families':
        self_p, cross_p, n = ao.layout(ATT_SELF_LENS)
        return self_p + cross_p, n, [('self', self_p), ('cross', cross_p)]
    problems, n = edge_layout()
    return problems, n, [('few tiles', [p for p in problems if p[3] < 1000]),
                         ('many tiles', [p for p in problems if p[3] >= 1000])]


def _tables(problems):
    return [torch.tensor(c, dtype=torch.int32, device=DEV) for c in zip(*problems)]


def _host_bf16(q, k, v):
    """The bf16 QK [n, 2E + QK_PAD] and Vt [E, ld_vt] the core reads (CPU), padding columns PAD_SENT."""
    n = q.shape[0]
    qk = torch.full((n, 2 * E + QK_PAD), PAD_SENT, dtype=torch.bfloat16)
    qk[:, :E], qk[:, E:2 * E] = q.to(torch.bfloat16), k.to(torch.bfloat16)
    vt = torch.full((E, (n + 7) // 8 * 8 + VT_PAD), PAD_SENT, dtype=torch.bfloat16)
    vt[:, :n] = v.t().to(torch.bfloat16)
    return qk, vt


def _launch(qk, vt, tb, n_problems, max_q, out, ldo, n_tokens, head_dim=ao.HD, ld_qk=None, ld_vt=None, qk_ptr=None,
            vt_ptr=None, n_heads=H):
    return _lib().regtr_mha_bf16_tc_fwd(qk.data_ptr() if qk_ptr is None else qk_ptr,
                                        qk.stride(0) if ld_qk is None else ld_qk,
                                        vt.data_ptr() if vt_ptr is None else vt_ptr,
                                        vt.stride(0) if ld_vt is None else ld_vt, n_tokens, out.data_ptr(), ldo,
                                        *(t.data_ptr() for t in tb), n_problems, max_q, n_heads, head_dim,
                                        1.0 / math.sqrt(ao.HD), _stream())


def run_core(qk, vt, problems, n):
    """The core on host bf16 QK / Vt -> O [n, E] (CPU fp32).  Writes into an [n + 1, E + O_PAD] sentinel buffer:
    everything outside the query rows of the problems (columns [0, E)) must keep the sentinel."""
    qk_d, vt_d = qk.to(DEV), vt.to(DEV)
    out = torch.full((n + 1, E + O_PAD), OUT_SENT, device=DEV)
    tb = _tables(problems)
    rc = _launch(qk_d, vt_d, tb, len(problems), max(p[1] for p in problems), out, E + O_PAD, n)
    assert rc == OK, rc
    out = out.cpu()
    written = torch.zeros(n + 1, E + O_PAD, dtype=torch.bool)
    for qs, ql, _, _ in problems:
        written[qs:qs + ql, :E] = True
    assert bool((out[~written] == OUT_SENT).all()), 'the core wrote outside the query rows of its problems'
    return out[:n, :E].clone()


# --------------------------------------------------------------------------------------- core against float64

_CASES = {}


def _case(layout, family):
    """Kernel outputs and references of a layout and input family: O, O(k + c), O(v + c), each with the float64 and
    fp32 restatements on the same (shifted, re-rounded) bf16 inputs."""
    key = (layout, family)
    if key in _CASES:
        return _CASES[key]
    problems, n, groups = _layout(layout)
    q, k, v, _ = ao.family(family, n, problems, H, seed=3 if layout == 'edges' else 0)
    ck, cv = ao.key_shift(k, problems, H, 0), ao.key_shift(v, problems, H, 1)
    c = dict(problems=problems, n=n, groups=groups, inputs={})
    for name, (a, b, d) in {'O': (q, k, v), 'O(k + c)': (q, k + ck, v), 'O(v + c)': (q, k, v + cv)}.items():
        qk, vt = _host_bf16(a, b, d)
        r64 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float64)
        r32 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float32)
        c[name] = dict(got=run_core(qk, vt, problems, n), r64=r64['o'], r32=r32['o'], flips=ao.p_flips(r64, r32),
                       l=r64['l'], l_exact=r64['l_exact'], allow=r64['ties']['allow'], ties=r64['ties']['count'])
        if name == 'O':
            c['inputs'] = dict(qk=qk, vt=vt)
    _CASES[key] = c
    return c


def _rows(title, c, override=None):
    """Yardstick rows per group: O, O(k + c), O(v + c); `override` replaces the kernel's O (sharpness) and then only
    the O rows are added -> Yardstick."""
    ys = Yardstick(title)
    for g, probs in c['groups']:
        rows = ao.rows_of([p for p in probs if p[1] and p[3]], 'q')
        for name in ('O',) if override is not None else ('O', 'O(k + c)', 'O(v + c)'):
            r = c[name]
            got = r['got'] if override is None else override
            ref, allow = r['r64'][rows], r['allow'][rows]
            ys.add(f'{g} {name}', ao.beyond_ties(got[rows], ref, allow), ao.beyond_ties(r['r32'][rows], ref, allow), ref)
    ys.report()
    return ys


@pytest.mark.parametrize('family', FAMILIES)
@pytest.mark.parametrize('layout', ['families', 'edges'])
def test_bf16_core_vs_float64(layout, family):
    """O, O(k + c) and O(v + c) under the yardstick per group of problems, against the restatement on the bf16
    inputs the core read (the shifted runs on k + c, v + c re-rounded to bf16); rows of an empty key range are exact
    zeros."""
    c = _case(layout, family)
    ys = _rows(f'bf16 attention core, {layout} layout, {family} inputs', c)
    print('  p entries rounded differently by the fp32 and the float64 restatement / near ties: ' +
          ', '.join(f'{name} {c[name]["flips"][0]} / {c[name]["ties"]} of {c[name]["flips"][1]}'
                    for name in ('O', 'O(k + c)', 'O(v + c)')))
    empty = [p for p in c['problems'] if p[1] and not p[3]]
    assert empty
    for name in ('O', 'O(k + c)', 'O(v + c)'):
        rows = ao.rows_of(empty, 'q')
        assert bool((c[name]['got'][rows] == 0).all()), f'{name}: rows without keys are not 0'
        assert torch.isfinite(c[name]['got']).all(), name
    assert not ys.failures(), ys.failures()


def test_bf16_core_checks_are_sharp():
    """Each planted error fails both O rows (self and cross problems) of the families layout on every family: O x
    (1 + 1e-4); the kernel's O rescaled to an l summed from the unrounded p (O l / l_exact); the kernel run with
    k_len - 1, and separately with k_start + 1."""
    fails = {}
    for family in FAMILIES:
        c = _case('families', family)
        o, r = c['O']['got'], c['O']
        probs, n = c['problems'], c['n']
        qk, vt = c['inputs']['qk'], c['inputs']['vt']
        planted = {
            'O x (1 + 1e-4)': o.double() * (1 + 1e-4),
            'l from unrounded p': (o.double().view(n, H, ao.HD) * (r['l'] / r['l_exact']).unsqueeze(-1)).view(n, E),
            'k_len - 1': run_core(qk, vt, [(a, b, s, max(l - 1, 0)) for a, b, s, l in probs], n),
            'k_start + 1': run_core(qk, vt, [(a, b, s + 1, l) for a, b, s, l in probs], n),
        }
        for what, got in planted.items():
            fails[family, what] = set(_rows(f'bf16 core, {family} inputs, {what}', c, override=got).failures())
    missed = {key: f for key, f in fails.items() if not {'self O', 'cross O'} <= f}
    assert not missed, missed


# --------------------------------------------------------------------------------- masking and determinism

@pytest.mark.parametrize('layout', ['families', 'edges'])
def test_bf16_core_masking_and_determinism(layout):
    """A rerun of the batch is bit-identical.  Each problem run alone gives its rows of the batch bit for bit, and so
    it does with every token outside its own query and key ranges set to POISON in q, k and v (the tokens its
    unaligned first key tile, its last key tile and its over-long Q tile read besides its own), with PAD_SENT in Vt's
    padding columns."""
    c = _case(layout, 'zero_mean')
    probs, n = c['problems'], c['n']
    qk, vt = c['inputs']['qk'], c['inputs']['vt']
    batch = c['O']['got']
    assert torch.equal(run_core(qk, vt, probs, n), batch), 'a rerun of the batch differs'
    for p in probs:
        qs, ql, ks, kl = p
        if ql == 0:
            continue
        alone = run_core(qk, vt, [p], n)
        assert torch.equal(alone[qs:qs + ql], batch[qs:qs + ql]), f'problem {p} alone differs from the batch'
        other = torch.ones(n, dtype=torch.bool)
        other[qs:qs + ql] = False
        other[ks:ks + kl] = False
        pq, pv = qk.clone(), vt.clone()
        pq[other, :2 * E] = POISON
        pv[:, :n][:, other] = -POISON
        poisoned = run_core(pq, pv, [p], n)
        assert torch.equal(poisoned[qs:qs + ql], batch[qs:qs + ql]), f'problem {p}: O depends on tokens outside it'


# ------------------------------------------------------------------------------------------------ rejections

def test_bf16_core_rejections():
    """Unsupported arguments return REGTR_ERR_UNSUPPORTED and leave the output untouched: head_dim != 32, ld_qk or
    ld_vt not a multiple of 8, ldo not a multiple of 4, QK or Vt not 16-byte aligned, n_problems > 65535.  Zero
    problems, queries or tokens return OK without a launch."""
    problems, n, _ = _layout('families')
    q, k, v, _ = ao.family('zero_mean', n, problems, H)
    qk, vt = (t.to(DEV) for t in _host_bf16(q, k, v))
    tb = _tables(problems)
    mq = max(p[1] for p in problems)
    out = torch.full((n, E + O_PAD), OUT_SENT, device=DEV)
    flat_qk = torch.zeros(qk.numel() + 8, dtype=torch.bfloat16, device=DEV)
    flat_vt = torch.zeros(vt.numel() + 8, dtype=torch.bfloat16, device=DEV)
    big = [torch.zeros(65536, dtype=torch.int32, device=DEV) for _ in range(4)]
    ldo = E + O_PAD
    cases = {
        'head_dim 16': dict(head_dim=16),
        'head_dim 64': dict(head_dim=64),
        'ld_qk % 8 = 4': dict(ld_qk=2 * E + 4),
        'ld_vt % 8 = 4': dict(ld_vt=vt.stride(0) - 4),
        'ldo % 4 = 2': dict(ldo=E + 2),
        'QK 2 bytes off 16': dict(qk_ptr=flat_qk.data_ptr() + 2),
        'Vt 8 bytes off 16': dict(vt_ptr=flat_vt.data_ptr() + 8),
        'n_problems 65536': dict(tb=big, n_problems=65536),
    }
    for what, kw in cases.items():
        a = dict(tb=tb, n_problems=len(problems), ldo=ldo) | kw
        rc = _launch(qk, vt, a.pop('tb'), a.pop('n_problems'), mq, out, a.pop('ldo'), n, **a)
        assert rc == UNSUPPORTED, (what, rc)
    torch.cuda.synchronize()
    assert bool((out == OUT_SENT).all()), 'a rejected call wrote its output'

    # no launch: with no problems or no queries a launch would have a zero grid dimension, which the entry point's
    # launch check returns as a CUDA error, not OK; with no tokens the real tables would make a launch write rows
    zero = {'no problems': (0, mq, n), 'no queries': (len(problems), 0, n), 'no tokens': (len(problems), mq, 0)}
    for what, (np_, mq_, n_) in zero.items():
        assert _launch(qk, vt, tb, np_, mq_, out, ldo, n_) == OK, what
    torch.cuda.synchronize()
    assert bool((out == OUT_SENT).all()), 'a call without work wrote its output'
    assert _launch(qk, vt, tb, len(problems), mq, out, ldo, n) == OK
    torch.cuda.synchronize()
    assert not bool((out[:, :E] == OUT_SENT).all()), 'the sentinel check cannot see a launch'


# ------------------------------------------------------------------------------ ops.mha_bf16_tc and the model

def by_hand(x, w, b, q_start, q_len, k_start, k_len, max_q_len, n_heads, m_dev=None):
    """ops.mha_bf16_tc's two launches run by hand: regtr_gemm_tf32x3_qkv_bf16 into qk / vt, then the core -> (qk,
    vt, O) on the device."""
    from regtr_b200 import ops
    L = _lib()
    N, E_ = x.shape
    hi, lo = ops.split_weight(w)
    ld_vt = (N + 63) // 64 * 64 + 64
    qk = torch.zeros((N, 2 * E_), dtype=torch.bfloat16, device=DEV)
    vt = torch.zeros((E_, ld_vt), dtype=torch.bfloat16, device=DEV)
    rc = L.regtr_gemm_tf32x3_qkv_bf16(x.data_ptr(), x.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0),
                                      b.data_ptr(), N, 3 * E_, E_, 2 * E_, qk.data_ptr(), 2 * E_, vt.data_ptr(), ld_vt,
                                      None if m_dev is None else m_dev.data_ptr(), _stream())
    assert rc == OK, rc
    out = torch.zeros((N, E_), dtype=torch.float32, device=DEV)
    rc = _launch(qk, vt, (q_start, q_len, k_start, k_len), q_start.numel(), int(max_q_len), out, E_, N,
                 head_dim=E_ // n_heads, n_heads=n_heads)
    assert rc == OK, rc
    return qk, vt, out


def test_mha_bf16_tc_is_gemm_then_core():
    """ops.mha_bf16_tc equals its GEMM and core launched by hand on the same buffers, bit for bit, on self and cross
    problems of ragged clouds (with the GEMM test of the bf16 epilogue, this covers the whole op)."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    g = torch.Generator().manual_seed(4)
    for lens in ([410, 339], [130, 7, 300, 129]):
        N = sum(lens)
        x = torch.randn(N, E, generator=g).to(DEV)
        w = (torch.randn(3 * E, E, generator=g) / E ** 0.5).to(DEV)
        b = (torch.randn(3 * E, generator=g) * 0.1).to(DEV)
        plan = AttentionPlan(lens, DEV)
        for ks, kl in ((plan.q_start, plan.q_len), (plan.xk_start, plan.xk_len)):
            got = ops.mha_bf16_tc(x, w, b, plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
            _, _, want = by_hand(x, w, b, plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
            torch.cuda.synchronize()
            assert torch.equal(got, want), lens


MODEL_CASES = ['fwd_3dmatch_small_b2', 'fwd_modelnet_b1', 'real_3dmatch_redkitchen_0_5']


@pytest.mark.parametrize('case', MODEL_CASES)
def test_bf16_core_on_model_activations(case):
    """An inference forward with attention_impl='bf16_tc', every ops.mha_bf16_tc call recorded.  Per cross-encoder
    layer and kind (self, cross): the GEMM rerun by hand gives the exact bf16 q | k and v^T the core read; the core's
    recorded O is checked under the yardstick against the restatement on them, and a rerun of the call is bit-identical
    to it.  These are the scores the fast mode sees: LayerNorm'd, position-encoded and more peaked than the families."""
    from conftest import REAL_CASES, make_case, make_real_case
    from regtr_b200 import ops
    from regtr_b200.regtr import RegTR
    cfg, sd, src, tgt = make_real_case(case) if case in REAL_CASES else make_case(case)
    src, tgt = ([src], [tgt]) if case in REAL_CASES else (src, tgt)
    cfg.attention_impl = 'bf16_tc'
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    batch = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    calls, orig = [], ops.mha_bf16_tc

    def recording(x, in_w, in_b, q_start, q_len, k_start, k_len, max_q_len, n_heads, m_dev=None):
        o = orig(x, in_w, in_b, q_start, q_len, k_start, k_len, max_q_len, n_heads, m_dev=m_dev)
        calls.append(dict(args=(x.detach().clone(), in_w, in_b.detach().clone(), q_start.clone(), q_len.clone(),
                                k_start.clone(), k_len.clone(), max_q_len, n_heads),
                          m_dev=None if m_dev is None else m_dev.clone(), o=o.detach().clone()))
        return o
    with torch.no_grad(), pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, 'mha_bf16_tc', recording)
        model(batch)
    torch.cuda.synchronize()
    assert len(calls) == 2 * cfg.num_encoder_layers, len(calls)
    ys = Yardstick(f'bf16 attention core on the activations of {case}')
    flips = []
    for i, c in enumerate(calls):
        a = c['args']
        kind = 'self' if torch.equal(a[3], a[5]) and torch.equal(a[4], a[6]) else 'cross'
        assert kind == ('self', 'cross')[i % 2], (i, kind)
        with torch.no_grad():
            qk, vt, o = by_hand(*a, m_dev=c['m_dev'])
        torch.cuda.synchronize()
        assert torch.equal(o, c['o']), f'layer {i // 2} {kind}: a rerun differs from the recorded call'
        problems = ao.problems_of(*a[3:7])
        qk, vt = qk.cpu(), vt.cpu()
        r64 = ao.bf16_forward_reference(qk, vt, problems, a[8], torch.float64)
        r32 = ao.bf16_forward_reference(qk, vt, problems, a[8], torch.float32)
        rows = ao.rows_of([p for p in problems if p[1] and p[3]], 'q')
        ref, allow = r64['o'][rows], r64['ties']['allow'][rows]
        ys.add(f'layer {i // 2} {kind} O', ao.beyond_ties(c['o'].cpu()[rows], ref, allow),
               ao.beyond_ties(r32['o'][rows], ref, allow), ref)
        f, tot = ao.p_flips(r64, r32)
        flips.append(f'layer {i // 2} {kind} {f} / {r64["ties"]["count"]} of {tot}')
    ys.report()
    print('  p entries rounded differently by the fp32 and the float64 restatement / near ties: ' + ', '.join(flips))
    assert not ys.failures(), ys.failures()
