"""Float64 reference of the attention core (softmax(q k^T / sqrt(32)) v per head over (query range, key range)
problems) and the checks of its backward that tests/test_gpu_attention_backward.py and tests/test_gpu_grad_stages.py
share.

A problem is (q_start, q_len, k_start, k_len): rows of the packed [n, E] q / dO / O matrices and of the packed k / v
matrices, E = n_heads * 32.  Every key row lies in the key range of at most one problem.

Besides the yardstick rows (tests/grad_yardstick.py), three invariants of exact arithmetic are checked per problem
and head, each against the fp32 reference's deviation from it:
  * sum_j dK_j = 0: softmax does not change when one vector is added to every key;
  * sum_j dV_j = sum_i dO_i: every row of P sums to 1;
  * dQ with every key shifted by one vector c equals the float64 dQ: the same invariance, seen from the query side.
A kernel whose sum_j dS_ij is off by e gets dQ off by e * (the part the keys share) and dK off by e * (the part the
queries share), so these catch errors that zero-mean inputs hide.
"""
import math

import numpy as np
import torch

from grad_yardstick import FACTOR, FLOOR

HD = 32
SCALE = 1.0 / math.sqrt(HD)
SELF_LENS = [1, 17, 64, 65, 731, 1500]
CROSS_LENS = [40, 130, 77, 0]
FAMILIES = ['zero_mean', 'bias', 'flat', 'peaked', 'shared_do']
PEAK = 60.0                      # largest |base-2 score| of the peaked family


def layout(self_lens=SELF_LENS, cross_lens=CROSS_LENS):
    """(self problems, cross problems, rows): every key row in exactly one problem's key range.  The cross problems
    pair clouds 0 <-> 1 and 2 <-> 3 of `cross_lens`."""
    self_p, r = [], 0
    for n in self_lens:
        self_p.append((r, n, r, n))
        r += n
    c = []
    for n in cross_lens:
        c.append(r)
        r += n
    L = cross_lens
    cross_p = [(c[0], L[0], c[1], L[1]), (c[1], L[1], c[0], L[0]), (c[2], L[2], c[3], L[3]), (c[3], L[3], c[2], L[2])]
    return self_p, cross_p, r


def family(name, n, problems, n_heads, seed=0):
    """q, k, v, dO [n, n_heads * HD] fp32 (CPU) of an input family (tests/test_gpu_attention_backward.py describes
    them)."""
    E = n_heads * HD
    g = torch.Generator().manual_seed(seed)
    r = lambda s=1.0: torch.randn(n, E, generator=g) * s
    head = lambda s: torch.randn(1, E, generator=g) * s             # one vector per head, shared by every row
    q, k, v, d_o = r(1.5), r(1.5), r(1.5), r()
    if name == 'bias':
        q, k = r(0.5) + head(1.5), r(0.5) + head(1.5)
    elif name == 'flat':
        q, v = r(0.02), r(0.3) + head(1.0)
    elif name == 'peaked':
        smax = max(float((_heads(q, qs, ql, n_heads) @ _heads(k, ks, kl, n_heads).transpose(1, 2)).abs().max())
                   for qs, ql, ks, kl in problems if ql and kl) * SCALE * 1.4426950408889634
        q = q * (PEAK / smax)
    elif name == 'shared_do':
        d_o = r() + head(10.0)
    return q, k, v, d_o


def problems_of(q_start, q_len, k_start, k_len):
    """Problem tuples from the (device) tables."""
    return list(zip(*(t.tolist() for t in (q_start, q_len, k_start, k_len))))


def _heads(x, start, length, n_heads):
    return x[start:start + length].view(length, n_heads, HD).transpose(0, 1)


def reference(q, k, v, d_o, problems, n_heads, dtype=torch.float64):
    """Autograd of the core in `dtype` on the CPU.  -> dict of [n, E] CPU tensors o, dq, dk, dv (0 on rows outside
    every problem), lse [n, n_heads] (base 2, -inf for a query without keys) and, in float64, ddq / ddk: how much
    dQ and dK fall when delta_i = sum_j P_ij dP_ij is raised by the fraction 1 (dS_ij = P_ij (dP_ij - delta_i), so
    dQ_i falls by scale * delta_i * sum_j P_ij k_j and dK_j by scale * sum_i P_ij delta_i q_i)."""
    n, E = q.shape
    x = [t.detach().cpu().to(dtype).requires_grad_(True) for t in (q, k, v)]
    g = d_o.detach().cpu().to(dtype)
    o = torch.zeros(n, E, dtype=dtype)
    lse = torch.full((n, n_heads), -math.inf, dtype=dtype)
    ddq, ddk = torch.zeros(n, E, dtype=torch.float64), torch.zeros(n, E, dtype=torch.float64)
    outs, gouts = [], []
    for qs, ql, ks, kl in problems:
        if ql == 0 or kl == 0:
            continue
        Q, K, V = _heads(x[0], qs, ql, n_heads), _heads(x[1], ks, kl, n_heads), _heads(x[2], ks, kl, n_heads)
        s = Q @ K.transpose(1, 2) * SCALE
        p = torch.softmax(s, -1)
        out = p @ V
        go = _heads(g, qs, ql, n_heads)
        outs.append(out)
        gouts.append(go)
        o[qs:qs + ql] = out.detach().transpose(0, 1).reshape(ql, E)
        lse[qs:qs + ql] = (torch.logsumexp(s.detach(), -1) / math.log(2)).transpose(0, 1)
        if dtype == torch.float64:
            with torch.no_grad():
                P, Qd, Kd = p.detach(), Q.detach(), K.detach()
                delta = (go * out.detach()).sum(-1, keepdim=True)
                ddq[qs:qs + ql] = (SCALE * delta * (P @ Kd)).transpose(0, 1).reshape(ql, E)
                ddk[ks:ks + kl] += (SCALE * P.transpose(1, 2) @ (delta * Qd)).transpose(0, 1).reshape(kl, E)
    grads = torch.autograd.grad(outs, x, gouts, allow_unused=True) if outs else (None,) * 3
    dq, dk, dv = (gr if gr is not None else torch.zeros(n, E, dtype=dtype) for gr in grads)
    return dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv, ddq=ddq, ddk=ddk)


def key_shift(k, problems, n_heads, seed=0):
    """[1, E] fp32: per head a vector of 4x the rms spread of that head's keys (about their mean), in a seeded random
    direction.  Added to every key it changes neither the softmax nor dQ."""
    rows = torch.cat([torch.arange(ks, ks + kl) for _, _, ks, kl in problems if kl > 0])
    kh = k.detach().cpu().double()[rows].view(-1, n_heads, HD)
    spread = (kh - kh.mean(0)).pow(2).sum(-1).mean(0).sqrt()                      # [n_heads]
    u = torch.randn(n_heads, HD, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    return (4 * spread[:, None] * u / u.norm(dim=1, keepdim=True)).reshape(1, -1).float()


def run_kernel(q, k, v, d_o, problems, n_heads, o=None, lse=None):
    """The CUDA backward (after the training forward, unless O and lse are given) on CUDA or CPU fp32 q, k, v, dO
    packed as one [n, 3E] matrix, as the model packs them -> dict of CPU dq, dk, dv."""
    from regtr_b200 import ops
    dev = 'cuda:0'
    E = q.shape[1]
    tb = [torch.tensor(c, dtype=torch.int32, device=dev) for c in zip(*problems)]
    mq, mk = max(p[1] for p in problems), max(p[3] for p in problems)
    qkv = torch.cat([t.to(dev) for t in (q, k, v)], 1)
    qd, kd, vd = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    if o is None:
        o, lse = ops.mha_varlen_lse(qd, kd, vd, *tb, mq, n_heads)
    d = torch.zeros_like(qkv)
    ops.mha_varlen_bwd(qd, kd, vd, o.to(dev), lse.to(dev), d_o.to(dev).contiguous(), d[:, :E], d[:, E:2 * E],
                       d[:, 2 * E:], *tb, mq, mk, n_heads)
    torch.cuda.synchronize()
    d = d.cpu()
    return dict(dq=d[:, :E], dk=d[:, E:2 * E], dv=d[:, 2 * E:])


def rows_of(problems, which):
    """Concatenated query ('q') or key ('k') rows of the problems."""
    i = 0 if which == 'q' else 2
    parts = [torch.arange(p[i], p[i] + p[i + 1]) for p in problems]
    return torch.cat(parts) if parts else torch.zeros(0, dtype=torch.long)


def add_rows(ys, prefix, problems, got, fp32, ref):
    """One yardstick row each for dq (query rows), dk and dv (key rows) of the problems."""
    qr, kr = rows_of(problems, 'q'), rows_of(problems, 'k')
    for name, rows in (('dq', qr), ('dk', kr), ('dv', kr)):
        ys.add(f'{prefix}{name}', got[name][rows], fp32[name][rows], ref[name][rows])


def invariants(problems, n_heads, d_o, got, fp32, ref, got_shift, fp32_shift, ref_shift):
    """The three invariants per problem with queries and keys, and head.  got / fp32 / ref: dicts with dk, dv (the
    kernel's, the fp32 reference's, the float64 reference's); *_shift: the same runs with keys k + c (dq is read).
    -> [(check, (q_len, k_len), head, kernel deviation, fp32 deviation, bound)]; the kernel passes a row when its
    deviation <= FACTOR * fp32 deviation + FLOOR * max|float64 gradient over the problem|."""
    g = d_o.detach().cpu().double()
    out = []

    def dev_sum(t, s, length, target=None):
        x = t.detach().double()[s:s + length].view(length, n_heads, HD).sum(0)
        return (x if target is None else x - target).abs().amax(-1)                  # [n_heads]

    for qs, ql, ks, kl in problems:
        if ql == 0 or kl == 0:
            continue
        sum_do = g[qs:qs + ql].view(ql, n_heads, HD).sum(0)
        checks = (
            ('sum dK = 0', [dev_sum(t['dk'], ks, kl) for t in (got, fp32)], ref['dk'][ks:ks + kl]),
            ('sum dV = sum dO', [dev_sum(t['dv'], ks, kl, sum_do) for t in (got, fp32)], ref['dv'][ks:ks + kl]),
            ('dQ(k + c)', [(t['dq'].detach().double()[qs:qs + ql] - ref_shift['dq'][qs:qs + ql]).view(ql, n_heads, HD)
                           .abs().amax(-1).amax(0) for t in (got_shift, fp32_shift)], ref_shift['dq'][qs:qs + ql]),
        )
        for name, (dg, df), r in checks:
            if kl == 1 and name != 'sum dV = sum dO':
                continue            # one key: dQ = dK = 0 exactly, no scale for an absolute bound (rows check them)
            bound = FACTOR * df + FLOOR * float(r.abs().max())
            for h in range(n_heads):
                out.append((name, (ql, kl), h, float(dg[h]), float(df[h]), float(bound[h])))
    return out


def failed(rows):
    return [r for r in rows if not r[3] <= r[5]]


def report_invariants(title, rows):
    """Per check: the worst (kernel deviation / bound) over problems and heads, and how many rows fail."""
    print(f'\n{title}\n  invariants per problem and head; pass: kernel deviation <= {FACTOR:g} x fp32 deviation + '
          f'{FLOOR:g} x max|float64 gradient over the problem|')
    wn = max([len(r[0]) for r in rows] + [16])
    print(f'  {"check":{wn}s} {"worst ratio":>11s}  {"at (q_len, k_len, head)":>24s} {"kernel":>9s} {"fp32":>9s}  failing')
    for name in dict.fromkeys(r[0] for r in rows):
        rs = [r for r in rows if r[0] == name]
        w = max(rs, key=lambda r: r[3] / max(r[5], 1e-300))
        at = f'({w[1][0]}, {w[1][1]}, {w[2]})'
        print(f'  {name:{wn}s} {w[3] / max(w[5], 1e-300):11.3g}  {at:>24s} {w[3]:9.2e} {w[4]:9.2e}  '
              f'{len(failed(rs))}/{len(rs)}')


def forward_reference(q, k, v, problems, n_heads, dtype):
    """softmax(q k^T / sqrt(32)) v per head and problem in `dtype` on the CPU -> (O [n, E], base-2 lse [n, n_heads]);
    rows outside every problem stay 0 / -inf."""
    n, E = q.shape
    q, k, v = (t.detach().cpu().to(dtype) for t in (q, k, v))
    o = torch.zeros(n, E, dtype=dtype)
    lse = torch.full((n, n_heads), -math.inf, dtype=dtype)
    for qs, ql, ks, kl in problems:
        if ql == 0 or kl == 0:
            continue
        s = _heads(q, qs, ql, n_heads) @ _heads(k, ks, kl, n_heads).transpose(1, 2) * SCALE
        o[qs:qs + ql] = (torch.softmax(s, -1) @ _heads(v, ks, kl, n_heads)).transpose(0, 1).reshape(ql, E)
        lse[qs:qs + ql] = (torch.logsumexp(s, -1) / math.log(2)).transpose(0, 1)
    return o, lse


LOG2E = 1.4426950408889634


def round_bf16(x):
    """x rounded to the nearest bfloat16 value, ties to even, kept in x's dtype.  float32 goes through
    gemm_oracle.bf16_rne, the rounding of the kernels' fp32 -> bf16 conversions.  float64 is rounded once, from the
    float64 value itself: x / ulp is exact, so torch.round (half to even) rounds it.  bf16 has fp32's exponent range,
    so below 2^-126 the ulp stays 2^-133 (subnormals)."""
    if x.dtype == torch.float32:
        import gemm_oracle as go
        u = torch.from_numpy(go.bf16_rne(x.detach().contiguous().numpy()).astype(np.int32)) << 16
        return u.view(torch.float32).view(x.shape)
    _, e = torch.frexp(x)                                                   # |x| in [2^(e-1), 2^e)
    ulp = torch.pow(2.0, (e.clamp_min(-125) - 8).to(x.dtype))
    return torch.round(x / ulp) * ulp


def bf16_forward_reference(qk, vt, problems, n_heads, dtype, round_p=True):
    """The bf16 wgmma core's operation (csrc/attention_tc.cu) in `dtype` on the CPU, on the bf16 tensors it reads:
    qk [n, >= 2E] (q | k columns) and vt [E, >= n] (v transposed).  Per problem with queries and keys, and head:
    s = q k^T, m = max_j s over the problem's keys, p = bf16(exp2((s - m) * scale * log2 e)), l = sum_j p of the rounded
    p, O = (sum_j p_j v_j) / l.  round_p=False leaves p unrounded (then this is softmax(q k^T * scale) v).
    -> dict: o [n, E] (0 on rows outside every problem, as on the rows of a problem without keys), l [n, n_heads] (sum
    of the p used), l_exact [n, n_heads] (sum of the unrounded p), p: per such problem the p used, [n_heads, q_len,
    k_len] bfloat16 when rounded (every value is a bf16 one), and in float64 with rounding the near ties (`ties`)."""
    E = n_heads * HD
    n = qk.shape[0]
    q, k = qk[:, :E].to(dtype), qk[:, E:2 * E].to(dtype)
    v = vt[:, :n].t().to(dtype)
    c = SCALE * LOG2E
    o = torch.zeros(n, E, dtype=dtype)
    l, l_exact = torch.zeros(n, n_heads, dtype=dtype), torch.zeros(n, n_heads, dtype=dtype)
    tie = dtype == torch.float64 and round_p
    allow, n_ties, tie_masks = torch.zeros(n, E, dtype=dtype), 0, []
    ps = []
    for qs, ql, ks, kl in problems:
        if ql == 0 or kl == 0:
            continue
        Q, K, V = _heads(q, qs, ql, n_heads), _heads(k, ks, kl, n_heads), _heads(v, ks, kl, n_heads)
        s = Q @ K.transpose(1, 2)
        pe = torch.exp2((s - s.amax(-1, keepdim=True)) * c)
        p = round_bf16(pe) if round_p else pe
        l_exact[qs:qs + ql] = pe.sum(-1).t()
        lp = p.sum(-1, keepdim=True)
        l[qs:qs + ql] = lp[..., 0].t()
        out = p @ V / lp
        o[qs:qs + ql] = out.transpose(0, 1).reshape(ql, E)
        if tie:
            # the p an fp32 computation may round to the other neighbour: within its error of a rounding midpoint.
            # Error of the exponent: s and m summed from 32 products in fp32 (at most 2^-19 sum_d |q_d k_d| each),
            # the products with c and their difference (2^-22 (|s| + |m|) c); exp2 and the rest: 2^-21 of p.
            a = Q.abs() @ K.abs().transpose(1, 2)
            m_abs = s.abs().amax(-1, keepdim=True)
            tau = (2.0 ** -19 * (a + a.amax(-1, keepdim=True)) + 2.0 ** -22 * (s.abs() + m_abs)) * c * math.log(2) \
                + 2.0 ** -21
            del a
            _, e = torch.frexp(pe)
            ulp = torch.pow(2.0, (e.clamp_min(-125) - 8).to(dtype))
            near = (ulp / 2 - (pe - p).abs()) <= tau * pe
            w = torch.where(near, ulp, torch.zeros_like(ulp)) / lp                # one flip moves O_i by w_ij (v_j - O_i)
            allow[qs:qs + ql] = (w @ V.abs() + w.sum(-1, keepdim=True) * out.abs()).transpose(0, 1).reshape(ql, E)
            n_ties += int(near.sum())
            tie_masks.append(near)
        del s, pe
        ps.append(p.to(torch.bfloat16) if round_p else p)
    r = dict(o=o, l=l, l_exact=l_exact, p=ps)
    if tie:
        r['ties'] = dict(allow=allow, count=n_ties, masks=tie_masks)
    return r


def beyond_ties(got, ref, allow):
    """got with its deviation from ref shrunk by `allow` (bf16_forward_reference's ties['allow']): what is left is the
    part no set of near-tie roundings can explain."""
    d = got.detach().double() - ref.double()
    return ref.double() + d.sign() * (d.abs() - allow.double()).clamp_min(0)


def p_flips(a, b):
    """(entries of p that differ, entries) between two runs of bf16_forward_reference."""
    return sum(int((x != y).sum()) for x, y in zip(a['p'], b['p'])), sum(x.numel() for x in a['p'])


def per_problem(name, problems, n_heads, hd, got, fp32, ref):
    """Invariant rows (name, (q_len, k_len), head, kernel deviation, fp32 deviation, bound) of the [n, n_heads * hd]
    tensors got / fp32 against ref over each problem's query rows; bound as in `invariants`."""
    out = []
    for qs, ql, ks, kl in problems:
        if ql == 0 or kl == 0:
            continue
        r = ref[qs:qs + ql].double()
        dg, df = ((t[qs:qs + ql].double() - r).view(ql, n_heads, hd).abs().amax(-1).amax(0) for t in (got, fp32))
        bound = FACTOR * df + FLOOR * float(r.abs().max())
        out += [(name, (ql, kl), h, float(dg[h]), float(df[h]), float(bound[h])) for h in range(n_heads)]
    return out
