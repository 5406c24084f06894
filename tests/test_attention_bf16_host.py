"""Host tests of the float64 restatement of the bf16 attention core (attention_oracle.bf16_forward_reference) that
tests/test_gpu_attention_bf16.py holds the kernel to.  CPU only."""
import numpy as np
import torch

import attention_oracle as ao
import gemm_oracle as go

H = 8
E = H * ao.HD


def _bf16_inputs(family='zero_mean', self_lens=(1, 17, 64, 65, 300), cross_lens=(40, 130, 77, 0), seed=0):
    self_p, cross_p, n = ao.layout(list(self_lens), list(cross_lens))
    problems = self_p + cross_p
    q, k, v, _ = ao.family(family, n, problems, H, seed)
    qk = torch.cat([q, k], 1).to(torch.bfloat16)
    vt = v.t().contiguous().to(torch.bfloat16)
    return qk, vt, problems, n


def _bits16(x):
    return x.view(torch.int16).numpy().view(np.uint16)


def test_bf16_rne_matches_torch():
    """gemm_oracle.bf16_rne equals torch's fp32 -> bfloat16 conversion on exact ties (both parities), one bit either
    side of a tie, signs, zeros, subnormals (ties among them) and normal magnitudes from 1e-38 to 1e38."""
    rng = np.random.default_rng(3)
    low = np.array([0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF], dtype=np.uint32)
    n = 20000
    normal = (rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)) | \
             (rng.integers(1, 254, n, dtype=np.uint32) << np.uint32(23)) | \
             (rng.integers(0, 1 << 7, n, dtype=np.uint32) << np.uint32(16)) | rng.choice(low, n)
    sub = (rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)) | \
          (rng.integers(0, 1 << 7, n, dtype=np.uint32) << np.uint32(16)) | rng.choice(low, n)
    x = np.concatenate([normal, sub, np.array([0, 0x80000000, 0x00008000, 0x00018000, 0x00007FFF, 0x007F8000],
                                              dtype=np.uint32)]).view(np.float32)
    assert (np.abs(x[n:2 * n]) < np.float32(2.0 ** -126)).all()
    want = _bits16(torch.from_numpy(x).to(torch.bfloat16))
    assert np.array_equal(go.bf16_rne(x), want)
    # the float64 path of round_bf16 rounds a float32-exact value as bf16_rne does
    got64 = ao.round_bf16(torch.from_numpy(x).double()).float().to(torch.bfloat16)
    assert np.array_equal(_bits16(got64), want)
    got32 = ao.round_bf16(torch.from_numpy(x))
    assert np.array_equal(_bits16(got32.to(torch.bfloat16)), want)
    assert torch.equal(got32, got32.to(torch.bfloat16).float())


def test_round_bf16_float64_rounds_once():
    """A float64 value just above a bf16 midpoint but below it after rounding to fp32 goes up from float64 (one
    rounding), where the fp32 value, a tie, goes to even."""
    mid = 1.0 + 2.0 ** -8                                       # midpoint of 1 and 1 + 2^-7: a tie, to even -> 1
    x = torch.tensor([mid, mid + 2.0 ** -40, mid - 2.0 ** -40, 2.0 ** -130 * 1.5, 2.0 ** -133 * 2.5],
                     dtype=torch.float64)
    assert float(np.float32(mid + 2.0 ** -40)) == mid
    got = ao.round_bf16(x).tolist()
    assert got == [1.0, 1.0 + 2.0 ** -7, 1.0, 2.0 ** -130 * 1.5, 2.0 ** -133 * 2], got
    assert ao.round_bf16(x.float()).tolist()[:3] == [1.0, 1.0, 1.0]


def test_unrounded_restatement_is_the_softmax_reference():
    """round_p=False: the restatement is softmax(q k^T / sqrt(32)) v of forward_reference, to 1e-12, on the bf16
    values of every family; rows of the empty key range and of no problem are 0."""
    for family in ('zero_mean', 'bias', 'flat', 'peaked'):
        qk, vt, problems, n = _bf16_inputs(family)
        got = ao.bf16_forward_reference(qk, vt, problems, H, torch.float64, round_p=False)
        want, _ = ao.forward_reference(qk[:, :E], qk[:, E:], vt.t(), problems, H, torch.float64)
        assert float((got['o'] - want).abs().max()) <= 1e-12 * float(want.abs().max()), family
        assert torch.allclose(got['l'], got['l_exact'], rtol=0, atol=0)
    e = [p for p in problems if p[1] and not p[3]][0]
    assert float(got['o'][e[0]:e[0] + e[1]].abs().max()) == 0.0


def test_rounded_restatement_follows_its_rounding():
    """round_p=True: every p is a bf16 value and the row's largest p is exactly 1; l is the sum of those p; the
    rounding moves l away from the unrounded sum."""
    qk, vt, problems, n = _bf16_inputs('bias')
    r = ao.bf16_forward_reference(qk, vt, problems, H, torch.float64)
    P = [p for p in problems if p[1] and p[3]]
    for (qs, ql, ks, kl), p in zip(P, r['p']):
        pd = p.double()
        assert torch.equal(pd.amax(-1), torch.ones(H, ql, dtype=torch.float64))
        assert torch.allclose(pd.sum(-1).t(), r['l'][qs:qs + ql], rtol=1e-15, atol=0)
    rows = ao.rows_of(P, 'q')
    assert float((r['l'][rows] / r['l_exact'][rows] - 1).abs().max()) > 1e-4


def test_fp32_restatement_is_within_fp32_distance():
    """The fp32 run against the float64 run.  Unrounded: within 1e-5 of max|O| (fp32 arithmetic alone).  Rounded:
    the two runs round some p to neighbouring bf16 values (the flips p_flips counts); each row of O is within what
    its flips can move it, sum_j |p32_j - p64_j| max|v - O| / l, plus the same 1e-5."""
    qk, vt, problems, n = _bf16_inputs('zero_mean', self_lens=(1, 17, 64, 65, 300, 1500))
    f64 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float64, round_p=False)
    f32 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float32, round_p=False)
    scale = float(f64['o'].abs().max())
    assert float((f32['o'].double() - f64['o']).abs().max()) <= 1e-5 * scale
    r64 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float64)
    r32 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float32)
    flips, total = ao.p_flips(r64, r32)
    assert 0 < flips < 1e-3 * total, (flips, total)
    v = vt.t().double()
    P = [p for p in problems if p[1] and p[3]]
    for (qs, ql, ks, kl), a, b in zip(P, r64['p'], r32['p']):
        dp = (a.double() - b.double()).abs().sum(-1)                                    # [H, ql]
        vh = ao._heads(v, ks, kl, H)                                                    # [H, kl, 32]
        o = ao._heads(r64['o'], qs, ql, H)                                              # [H, ql, 32]
        spread = (vh.abs().amax(1, keepdim=True) + o.abs()).amax(-1)                    # >= max_j |v_j - O_i|
        allow = dp * spread / r64['l'][qs:qs + ql].t() + 1e-5 * scale
        err = (ao._heads(r32['o'].double(), qs, ql, H) - o).abs().amax(-1)
        assert bool((err <= allow).all()), (qs, ql, float((err - allow).max()))


def test_fp32_flips_are_near_ties():
    """Every p the fp32 run rounds differently from float64 is one of the float64 run's near ties, on every family and
    with the keys shifted by 4x their spread (larger scores, larger fp32 errors); the ties are a small part of the p."""
    for family in ('zero_mean', 'bias', 'flat', 'peaked'):
        for shift in (False, True):
            qk, vt, problems, n = _bf16_inputs(family, self_lens=(1, 17, 64, 65, 300, 700))
            if shift:
                k = qk[:, E:].float() + ao.key_shift(qk[:, E:].float(), problems, H, 2)
                qk = torch.cat([qk[:, :E], k.to(torch.bfloat16)], 1)
            r64 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float64)
            r32 = ao.bf16_forward_reference(qk, vt, problems, H, torch.float32)
            flips, total = ao.p_flips(r64, r32)
            outside = sum(int(((a != b) & ~m).sum()) for a, b, m in zip(r64['p'], r32['p'], r64['ties']['masks']))
            assert flips > 0 and outside == 0, (family, shift, flips, outside)
            assert r64["ties"]["count"] <= 0.2 * total, (family, shift, r64['ties']['count'], total)
            o = ao.beyond_ties(r32['o'], r64['o'], r64['ties']['allow'])
            assert float((o - r64['o']).abs().max()) <= 1e-5 * float(r64['o'].abs().max()), (family, shift)
