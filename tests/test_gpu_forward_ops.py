"""GPU tests of the inference forward's ops on inputs shaped like the model's, against float64.

Every CUDA result is compared with the same operation evaluated in float64 on the kernel's own inputs, and so is the
fp32 restatement of that operation; the kernel passes a row when its error is within the fp32 yardstick
(tests/grad_yardstick.py).  Invariants of exact arithmetic are checked per problem with the bound rule of
tests/attention_oracle.py.  The inputs target the places where these kernels go wrong:
  * InstanceNorm statistics (`gemm_instats` -> `instnorm_apply`, and `instnorm_act`): channels whose mean is 0, 3, 30
    and 300 times their spread, clouds of 1, 31, 32, 33, 700 and 4000 rows whose boundaries fall inside the GEMM
    epilogue's 32-row groups, and a split-K shape;
  * attention forward cores (`mha_varlen`, the lse of `mha_varlen_lse`, `mha_tf32_tc`): the
    input families of tests/attention_oracle.py, self problems around the 64- and 128-query tiles, O(k + c) = O and
    O(v + c) = O + c per problem and head;
  * `corr_decode`: six layers, key clouds of 1, 31, 32 and 33 points around the 32-key chunk, a peaked softmax,
    coordinates 2.5 m from the origin, corr(xyz + t) = corr(xyz) + t and invariance to a vector added to every key;
  * the pose solve (`se3.compute_rigid_transform`, `ops.pose_from_corr`): world offsets, rotations at and near 180
    degrees, coplanar points, a reflection as the best unconstrained fit, logits of +-30, 1 to 33 points, zero
    total weight.
Each check is shown to be sharp: an output changed by 1e-5 of itself fails it.
"""
import math

import numpy as np
import pytest
import torch

import attention_oracle as ao
from grad_yardstick import Yardstick

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


def _dev_tables(problems):
    return [torch.tensor(c, dtype=torch.int32, device=DEV) for c in zip(*problems)]


# ------------------------------------------------------------------------------------ InstanceNorm statistics

IN_LENS = [1, 31, 32, 33, 700, 4000]
IN_LENS_SPLIT = [1, 31, 32, 33, 700]
RATIOS = (0, 3, 30, 300)                     # |mean| / std of each group of 32 channels
IN_CH = 32 * len(RATIOS)
_IN = {}


def _in_stats(x, lens, dtype):
    """Per-cloud mean and 1 / sqrt(var + eps) with oracle.regtr_oracle.instance_norm's operations."""
    means, rstds, a = [], [], 0
    for n in lens:
        seg = x[a:a + n].to(dtype)
        means.append(seg.mean(0))
        rstds.append(1.0 / torch.sqrt(seg.var(0, unbiased=False) + 1e-5))
        a += n
    return torch.stack(means), torch.stack(rstds)


def _gemm_instats_case(split):
    """C = A W^T with channel c of mean RATIOS[c // 32] * (+-1) and spread 1 (A's last column is 1), through
    gemm_instats (capacity-shaped, garbage padding rows, device row count) and instnorm_apply; K = 1024 takes the
    split-K path, whose statistics read every row from C."""
    if split in _IN:
        return _IN[split]
    from regtr_b200 import lib, ops
    lens = IN_LENS_SPLIT if split else IN_LENS
    K = 1024 if split else 64
    rng = np.random.default_rng(7 + split)
    M = sum(lens)
    # the GEMM needs a split-K workspace exactly when it splits: the case must take the path it is named after
    assert (lib.load().regtr_gemm_ws_bytes(M + 100, IN_CH, K) > 256) == split, 'split-K choice changed for this shape'
    a = np.full((M + 100, K), 1e3, dtype=np.float32)
    a[:M, :K - 1] = rng.normal(size=(M, K - 1))
    a[:M, K - 1] = 1.0
    w = np.empty((IN_CH, K), dtype=np.float32)
    w[:, :K - 1] = rng.normal(size=(IN_CH, K - 1)) / math.sqrt(K - 1)
    w[:, K - 1] = np.repeat(RATIOS, 32) * rng.choice([-1.0, 1.0], IN_CH)
    offs = ops.make_offsets(lens, DEV)
    m_dev = offs[len(lens):len(lens) + 1]
    hi, lo = ops.split_weight(torch.from_numpy(w).to(DEV))
    A = torch.from_numpy(a).to(DEV)
    c, stats = ops.gemm_instats(A, hi, lo, offs, len(lens), m_dev=m_dev)
    c2, stats2 = ops.gemm_instats(A, hi, lo, offs, len(lens), m_dev=m_dev)
    c = c[:M].contiguous()
    out = ops.instnorm_apply(c, offs, len(lens), stats)
    torch.cuda.synchronize()
    _IN[split] = dict(lens=lens, c=c.cpu(), stats=stats.cpu(), out=out.cpu(),
                      identical=torch.equal(stats, stats2) and torch.equal(c, c2[:M]))
    return _IN[split]


def _add_instats_rows(ys, r, mean, rstd, out):
    """mean, rstd and the normalised output per ratio group: the GPU's against float64 and fp32 on the GPU's C.  The
    statistics rows leave out one-row clouds: their rstd is 1 / sqrt(eps), about 300x every other cloud's, and would
    hide the others' errors; they are checked by `_check_one_row_clouds`."""
    from oracle import regtr_oracle as O
    lens, c = r['lens'], r['c']
    m64, s64 = _in_stats(c, lens, torch.float64)
    m32, s32 = _in_stats(c, lens, torch.float32)
    o64, o32 = O.instance_norm(c.double(), lens), O.instance_norm(c.float(), lens)
    multi = [i for i, n in enumerate(lens) if n > 1]
    for g, ratio in enumerate(RATIOS):
        ch = slice(32 * g, 32 * g + 32)
        ys.add(f'mean/std {ratio:3d}: mean', mean[multi, ch], m32[multi, ch], m64[multi, ch])
        ys.add(f'mean/std {ratio:3d}: rstd', rstd[multi, ch], s32[multi, ch], s64[multi, ch])
        ys.add(f'mean/std {ratio:3d}: out', out[:, ch], o32[:, ch], o64[:, ch])


def _check_one_row_clouds(r):
    """A one-row cloud: mean = its row exactly, rstd = 1 / sqrt(eps) (variance 0), output 0."""
    st = np.concatenate([[0], np.cumsum(r['lens'])])
    for i in [i for i, n in enumerate(r['lens']) if n == 1]:
        assert torch.equal(r['stats'][i, :, 0], r['c'][st[i]]), i
        assert float((r['stats'][i, :, 1].double() * math.sqrt(1e-5) - 1).abs().max()) <= 1e-7, i
        assert float(r['out'][st[i]].abs().max()) == 0.0, i


@pytest.mark.parametrize('split', [False, True], ids=['epilogue_partials', 'split_k'])
def test_gemm_instats_statistics_vs_float64(split):
    """gemm_instats -> instnorm_apply: per-cloud mean, rstd and normalised output under the yardstick, bit-identical
    across two calls."""
    r = _gemm_instats_case(split)
    ys = Yardstick(f'gemm_instats -> instnorm_apply, clouds {r["lens"]}{", split-K" if split else ""}')
    _add_instats_rows(ys, r, r['stats'][..., 0], r['stats'][..., 1], r['out'])
    ys.report()
    assert r['identical'], 'gemm_instats not bit-identical from call to call'
    _check_one_row_clouds(r)
    assert not ys.failures(), ys.failures()


def test_instnorm_act_vs_float64():
    """The stand-alone InstanceNorm (fp64 statistics in norm.cu) on the same channel families and clouds."""
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    rng = np.random.default_rng(5)
    M = sum(IN_LENS)
    x = (rng.normal(size=(M, IN_CH)) + np.repeat(RATIOS, 32) * rng.choice([-1.0, 1.0], IN_CH)).astype(np.float32)
    xt = torch.from_numpy(x)
    got = ops.instnorm_act(xt.to(DEV), ops.make_offsets(IN_LENS, DEV), len(IN_LENS)).cpu()
    o64, o32 = O.instance_norm(xt.double(), IN_LENS), O.instance_norm(xt, IN_LENS)
    ys = Yardstick(f'instnorm_act, clouds {IN_LENS}')
    for g, ratio in enumerate(RATIOS):
        ch = slice(32 * g, 32 * g + 32)
        ys.add(f'mean/std {ratio:3d}: out', got[:, ch], o32[:, ch], o64[:, ch])
    ys.report()
    assert not ys.failures(), ys.failures()


def test_instats_checks_are_sharp():
    """rstd raised by 1e-5 of itself fails the rstd row of every channel group, for both statistics paths."""
    for split in (False, True):
        r = _gemm_instats_case(split)
        ys = Yardstick(f'gemm_instats, rstd x (1 + 1e-5){", split-K" if split else ""}')
        _add_instats_rows(ys, r, r['stats'][..., 0], r['stats'][..., 1] * (1 + 1e-5), r['out'])
        ys.report()
        assert {f'mean/std {q:3d}: rstd' for q in RATIOS} <= set(ys.failures()), ys.failures()


# ------------------------------------------------------------------------------------ attention forward cores

H = 8
E = H * ao.HD
ATT_SELF_LENS = ao.SELF_LENS + [127, 128, 129]
FWD_FAMILIES = [f for f in ao.FAMILIES if f != 'shared_do']    # shared_do changes only dO: its q, k, v are zero_mean's


def _attn_ref(q, k, v, problems, dtype):
    return ao.forward_reference(q, k, v, problems, H, dtype)


def _head_shift(x, problems, seed):
    """[1, E]: per head a vector of 4x the rms spread of x's key rows, in a seeded random direction."""
    return ao.key_shift(x, problems, H, seed)


_ATT = {}


def _attn_case(family):
    """Problems, inputs (q, k, v as the varlen cores take them; x, W, b as mha_tf32_tc takes them) and the shifts c_k,
    c_v of a family."""
    if family in _ATT:
        return _ATT[family]
    self_p, cross_p, n = ao.layout(ATT_SELF_LENS)
    problems = self_p + cross_p
    q, k, v, _ = ao.family(family, n, problems, H)
    # the same family through the in-projection: x ~ N(0, 1), W = spread / sqrt(E), the per-head offsets in the bias
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, E, generator=g)
    spread = {'zero_mean': (1.5, 1.5, 1.5), 'bias': (0.5, 0.5, 1.5), 'flat': (0.02, 1.5, 0.3),
              'peaked': (1.5, 1.5, 1.5)}[family]
    w = torch.cat([torch.randn(E, E, generator=g) * (s / math.sqrt(E)) for s in spread])
    b = torch.zeros(3 * E)
    if family == 'bias':
        b[:2 * E] = torch.randn(2 * E, generator=g) * 1.5
    elif family == 'flat':
        b[2 * E:] = torch.randn(E, generator=g)
    elif family == 'peaked':
        qq, kk = (x.double() @ w[i * E:(i + 1) * E].double().t() for i in (0, 1))
        smax = max(float((ao._heads(qq, qs, ql, H) @ ao._heads(kk, ks, kl, H).transpose(1, 2)).abs().max())
                   for qs, ql, ks, kl in problems if ql and kl) * ao.SCALE * 1.4426950408889634
        w[:E] *= ao.PEAK / smax
    c = dict(problems=problems, qkv=(q, k, v), xwb=(x, w, b), ck=_head_shift(k, problems, 0),
             cv=_head_shift(v, problems, 1))
    _ATT[family] = c
    return c


def _proj(x, w, b, dtype):
    """q, k, v of the in-projection in `dtype` (oracle.regtr_oracle.mha's packed projection)."""
    y = x.to(dtype) @ w.to(dtype).t() + b.to(dtype)
    return y[:, :E], y[:, E:2 * E], y[:, 2 * E:]


def _run_core(core, c, dk=None, dv=None):
    """The core's O (and lse for 'lse') on the family's inputs with c added to every key (dk) / value (dv)."""
    from regtr_b200 import ops
    tb = _dev_tables(c['problems'])
    mq = max(p[1] for p in c['problems'])
    if core == 'tf32_tc':
        x, w, b = c['xwb']
        b = b.clone()
        if dk is not None:
            b[E:2 * E] += dk[0]
        if dv is not None:
            b[2 * E:] += dv[0]
        o = ops.mha_tf32_tc(x.to(DEV), w.to(DEV), b.to(DEV), *tb, mq, H)
        return o.cpu(), None
    q, k, v = c['qkv']
    k = k + dk if dk is not None else k
    v = v + dv if dv is not None else v
    qkv = torch.cat([q, k, v], 1).to(DEV)                 # column slices of one packed matrix, as the model has them
    args = (qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], *tb, mq, H)
    if core == 'lse':
        o, lse = ops.mha_varlen_lse(*args)
        return o.cpu(), lse.cpu()
    return ops.mha_varlen(*args).cpu(), None


def _refs(c, core, dk=None, dv=None):
    """(float64, fp32) O and lse of the core's operation on its inputs (for mha_tf32_tc the in-projection too)."""
    out = []
    for dt in (torch.float64, torch.float32):
        if core == 'tf32_tc':
            x, w, b = c['xwb']
            q, k, v = _proj(x, w, b, dt)
        else:
            q, k, v = (t.to(dt) for t in c['qkv'])
        k = k + dk.to(dt) if dk is not None else k
        v = v + dv.to(dt) if dv is not None else v
        out.append(_attn_ref(q, k, v, c['problems'], dt))
    return out


def _attn_results(core, family):
    c = _attn_case(family)
    res = dict(c=c)
    res['o'], res['lse'] = _run_core(core, c)
    res['o_k'], _ = _run_core(core, c, dk=c['ck'])
    res['o_v'], _ = _run_core(core, c, dv=c['cv'])
    (res['r64'], res['l64']), (res['r32'], res['l32']) = _refs(c, core)
    res['k32'] = _refs(c, core, dk=c['ck'])[1][0]
    res['v64'], res['v32'] = (r[0] for r in _refs(c, core, dv=c['cv']))
    return res


def _attn_checks(title, res, o=None, o_v=None):
    """Yardstick rows (O of the self and of the cross problems, lse) and the O(k + c), O(v + c) invariants; o / o_v
    replace the kernel's outputs (sharpness checks) -> (row failures, invariant failures)."""
    c = res['c']
    o = res['o'] if o is None else o
    o_v = res['o_v'] if o_v is None else o_v
    problems = c['problems']
    n_self = len(ATT_SELF_LENS)
    ys = Yardstick(title)
    for part, probs in (('self', problems[:n_self]), ('cross', problems[n_self:])):
        rows = ao.rows_of([p for p in probs if p[3] > 0], 'q')
        ys.add(f'{part} O', o[rows], res['r32'][rows], res['r64'][rows])
        if res['lse'] is not None:
            ys.add(f'{part} lse', res['lse'][rows], res['l32'][rows], res['l64'][rows])
    ys.report()
    cv = c['cv'].double()
    inv = ao.per_problem('O(k + c) = O', problems, H, ao.HD, res['o_k'], res['k32'], res['r64'])
    inv += ao.per_problem('O(v + c) = O + c', problems, H, ao.HD, o_v.double() - cv, res['v32'].double() - cv,
                        res['r64'])
    ao.report_invariants(title, inv)
    return ys.failures(), ao.failed(inv)


@pytest.mark.parametrize('family', FWD_FAMILIES)
@pytest.mark.parametrize('core', ['mma', 'lse', 'tf32_tc'])
def test_attention_forward_core_vs_float64(core, family):
    """O (and the lse of mha_varlen_lse) under the yardstick for the self and the cross problems; O(k + c) = O and
    O(v + c) = O + c per problem and head.  Cores: mha_varlen ('mma': the 3xTF32 mma.sync kernel), mha_varlen_lse
    ('lse') and mha_tf32_tc (in-projection included, the families built through its bias)."""
    res = _attn_results(core, family)
    rows, inv = _attn_checks(f'attention forward, core {core}, {family} inputs', res)
    e = res['c']['problems'][-2]                          # queries of the empty-key cross problem: not rows above
    assert e[3] == 0 and e[1] > 0
    assert not rows, rows
    assert not inv, inv[:8]


def test_attention_forward_checks_are_sharp():
    """On the bias family and the mha_varlen core: O x (1 + 1e-5) fails the self and cross O rows; O(v + c) + 1e-5 c,
    what a P whose rows sum to 1 + 1e-5 gives, fails the O(v + c) invariant."""
    res = _attn_results('mma', 'bias')
    rows, _ = _attn_checks('bias inputs, O x (1 + 1e-5)', res, o=res['o'] * (1 + 1e-5))
    assert {'self O', 'cross O'} <= set(rows), rows
    _, inv = _attn_checks('bias inputs, O(v + c) + 1e-5 c', res, o_v=res['o_v'].double() + 1e-5 * res['c']['cv'].double())
    assert 'O(v + c) = O + c' in {r[0] for r in inv}, inv[:4]


def test_mha_varlen_rejects_odd_ldo():
    """The core stores its output two floats at a time: an odd output leading dimension is refused, not written."""
    from regtr_b200 import lib, ops
    c = _attn_case('zero_mean')
    q, k, v = (t.to(DEV) for t in c['qkv'])
    out = torch.zeros((q.shape[0], E + 1), device=DEV)[:, :E]
    with pytest.raises(lib.RegtrLibError, match='REGTR_ERR_UNSUPPORTED'):
        ops.mha_varlen(q, k, v, *_dev_tables(c['problems']), max(p[1] for p in c['problems']), H, out=out)
    assert not out.any()


# ------------------------------------------------------------------------------------------------ corr_decode

CORR_LENS = [1, 31, 32, 33, 200, 77, 129, 40]   # pairs (c, c + 4): key clouds of 200, 77, 129, 40, 1, 31, 32, 33
CORR_L, CORR_D = 6, 256
XYZ_OFFSET = (2.5, -1.2, 2.4)
_CORR = {}


def _corr_problems():
    st = np.concatenate([[0], np.cumsum(CORR_LENS)])
    B = len(CORR_LENS) // 2
    return [(int(st[c]), CORR_LENS[c], int(st[(c + B) % (2 * B)]), CORR_LENS[(c + B) % (2 * B)])
            for c in range(2 * B)]


def _corr_ref(qp, kp, xyz, dtype):
    """softmax(qp kp^T / sqrt(D)) xyz per layer and problem in `dtype` (oracle.regtr_oracle.corr_decoder's
    attention) -> [L * n, 3]."""
    n = xyz.shape[0]
    q, k, x = (t.detach().cpu().to(dtype) for t in (qp, kp, xyz))
    q, k = q.view(CORR_L, n, CORR_D) / math.sqrt(CORR_D), k.view(CORR_L, n, CORR_D)
    out = torch.zeros(CORR_L, n, 3, dtype=dtype)
    for qs, ql, ks, kl in _corr_problems():
        out[:, qs:qs + ql] = torch.softmax(q[:, qs:qs + ql] @ k[:, ks:ks + kl].transpose(1, 2), -1) @ x[ks:ks + kl]
    return out.view(CORR_L * n, 3)


def _corr_case(family):
    """corr_decode on a family ('plain': N(0, 1) projections; 'peaked': scores up to 40) with xyz about 2.5 m from
    the origin, translated by t, and with a vector added to every kp row; and the references."""
    if family in _CORR:
        return _CORR[family]
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    g = torch.Generator().manual_seed(2)
    n = sum(CORR_LENS)
    qp, kp = torch.randn(CORR_L * n, CORR_D, generator=g), torch.randn(CORR_L * n, CORR_D, generator=g)
    xyz = torch.randn(n, 3, generator=g) * 0.5 + torch.tensor(XYZ_OFFSET)
    if family == 'peaked':
        q3, k3 = qp.view(CORR_L, n, CORR_D).double(), kp.view(CORR_L, n, CORR_D).double()
        smax = max(float((q3[:, qs:qs + ql] @ k3[:, ks:ks + kl].transpose(1, 2)).abs().max())
                   for qs, ql, ks, kl in _corr_problems()) / math.sqrt(CORR_D)
        qp *= 40.0 / smax
    t = torch.tensor([[3.0, -2.0, 1.5]])
    ck = torch.randn(1, CORR_D, generator=g)
    ck *= 4 * float((kp - kp.mean(0)).pow(2).sum(1).mean().sqrt()) / float(ck.norm())
    plan = AttentionPlan(CORR_LENS, DEV)

    def run(q, k, x):
        return ops.corr_decode(q.to(DEV), k.to(DEV), x.to(DEV), plan.q_start, plan.q_len, plan.xk_start, plan.xk_len,
                               plan.max_len, CORR_L).cpu()
    xt = (xyz + t).float()
    c = dict(got=run(qp, kp, xyz), got_t=run(qp, kp, xt), got_k=run(qp, kp + ck, xyz), t=t,
             r64=_corr_ref(qp, kp, xyz, torch.float64), r32=_corr_ref(qp, kp, xyz, torch.float32),
             t32=_corr_ref(qp, kp, xt, torch.float32), k32=_corr_ref(qp, kp + ck, xyz, torch.float32))
    _CORR[family] = c
    return c


def _corr_checks(title, c, got=None, got_t=None):
    got = c['got'] if got is None else got
    got_t = c['got_t'] if got_t is None else got_t
    n = sum(CORR_LENS)
    ys = Yardstick(title)
    ys.add('corr', got, c['r32'], c['r64'])
    ys.report()
    layered = [(l * n + qs, ql, l * n + ks, kl) for l in range(CORR_L) for qs, ql, ks, kl in _corr_problems()]
    t = c['t'].double()
    inv = ao.per_problem('corr(xyz + t) = corr + t', layered, 1, 3, got_t.double() - t, c['t32'].double() - t, c['r64'])
    inv += ao.per_problem('corr(kp + c) = corr', layered, 1, 3, c['got_k'], c['k32'], c['r64'])
    ao.report_invariants(title, inv)
    return ys.failures(), ao.failed(inv)


@pytest.mark.parametrize('family', ['plain', 'peaked'])
def test_corr_decode_vs_float64(family):
    """corr under the yardstick; translating xyz translates corr and a vector added to every kp row changes nothing,
    per layer and problem."""
    rows, inv = _corr_checks(f'corr_decode, {family} inputs, {CORR_L} layers, clouds {CORR_LENS}', _corr_case(family))
    assert not rows, rows
    assert not inv, inv[:8]


def test_corr_decode_checks_are_sharp():
    """corr x (1 + 1e-5) fails the corr row; corr(xyz + t) + 1e-5 t, what a softmax whose rows sum to 1 + 1e-5
    gives, fails the translation invariant."""
    c = _corr_case('plain')
    rows, _ = _corr_checks('corr_decode, corr x (1 + 1e-5)', c, got=c['got'] * (1 + 1e-5))
    assert 'corr' in rows, rows
    _, inv = _corr_checks('corr_decode, corr(xyz + t) + 1e-5 t', c, got_t=c['got_t'].double() + 1e-5 * c['t'].double())
    assert 'corr(xyz + t) = corr + t' in {r[0] for r in inv}, inv[:4]


# ------------------------------------------------------------------------------------------------- pose solve

def _kabsch64(a, b, w):
    """oracle.regtr_oracle.kabsch in float64 numpy: weighted centroids, covariance, SVD, and the reference's flip of
    V's last column when V U^T is not a rotation -> (R, t, singular values)."""
    a, b, w = (np.asarray(x, dtype=np.float64) for x in (a, b, w))
    wn = w[:, None] / max(w.sum(), 1e-6)
    ca, cb = (a * wn).sum(0), (b * wn).sum(0)
    cov = (a - ca).T @ ((b - cb) * wn)
    u, s, vh = np.linalg.svd(cov)
    v = vh.T
    R = v @ u.T
    if not np.linalg.det(R) > 0:
        v[:, 2] *= -1
        R = v @ u.T
    return R, cb - R @ ca, s


def _rot(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    axis /= np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def _residual(R, t, a, b, w):
    a, b, w = (np.asarray(x, dtype=np.float64) for x in (a, b, w))
    return float((w * ((a @ R.T + t - b) ** 2).sum(1)).sum() / max(w.sum(), 1e-6))


def _pose_problems():
    """(name, a, b, w, unique): fp32 point sets; `unique` when the constrained optimum is a single rotation."""
    rng = np.random.default_rng(9)
    off = np.array(XYZ_OFFSET)
    probs = []

    def add(name, a, R, t, noise=0.01, w=None, unique=True, mirror=False):
        n = len(a)
        src = a * np.array([1, 1, -1]) if mirror else a
        b = src @ R.T + t + rng.normal(size=(n, 3)) * noise
        w = rng.uniform(0.1, 1.0, n) if w is None else w
        probs.append((name, a.astype(np.float32), b.astype(np.float32), np.asarray(w, dtype=np.float32), unique))

    cloud = lambda n, s=(1.0, 0.6, 0.3): rng.normal(size=(n, 3)) * np.array(s) * 0.5 + off
    add('world offset', cloud(500), _rot(rng.normal(size=3), 0.7), np.array([0.4, -2.0, 1.1]))
    add('180 deg', cloud(300), _rot(rng.normal(size=3), math.pi), np.array([1.0, 0.5, -0.3]))
    add('180 deg - 1e-4', cloud(300), _rot(rng.normal(size=3), math.pi - 1e-4), np.array([-1.0, 0.2, 0.3]))
    plane = np.c_[rng.normal(size=(120, 2)) * 0.6, np.zeros(120)] @ _rot(rng.normal(size=3), 1.0).T + off
    add('coplanar', plane, _rot(rng.normal(size=3), 2.0), np.array([0.1, 0.2, 0.3]))
    add('reflection fits best', cloud(150), _rot(rng.normal(size=3), 1.3), np.array([0.3, 0.0, -0.5]), mirror=True)
    for n in (3, 31, 32, 33):
        add(f'{n} points', cloud(n), _rot(rng.normal(size=3), 2.5), np.array([0.2, -0.1, 0.05]))
    for n in (1, 2):
        add(f'{n} points', cloud(n), _rot(rng.normal(size=3), 0.5), np.zeros(3), unique=False)
    add('zero total weight', cloud(50), _rot(rng.normal(size=3), 0.5), np.zeros(3), w=np.zeros(50), unique=False)
    return probs


def _pose_check(name, T, a, b, w, unique, table, fails):
    """Unique problems: R and t against float64 Kabsch.  Others: finite, R^T R = I and det R = +1 to 1e-6, weighted
    mean square residual no larger than the float64 optimum's plus what moving every fitted point by d = 2e-7 x scale
    (fp32 rounding of R and t) can add: 2 d sqrt(optimum) + d^2."""
    R, t = T[:, :3].astype(np.float64), T[:, 3].astype(np.float64)
    R64, t64, s = _kabsch64(a, b, w)
    scale = 1.0 + float(np.abs(a).max()) + float(np.abs(b).max())
    if unique:
        eR, et = float(np.abs(R - R64).max()), float(np.abs(t - t64).max()) / scale
        table.append(f'  {name:28s} |R - R64| {eR:9.2e}  |t - t64| / scale {et:9.2e}  singular values {s[0]:.2e} '
                     f'{s[1]:.2e} {s[2]:.2e}')
        if not (eR <= 1e-6 and et <= 1e-6):
            fails.append(name)
        return
    ok = bool(np.isfinite(T).all())
    orth = float(np.abs(R.T @ R - np.eye(3)).max()) if ok else math.inf
    det = float(np.linalg.det(R)) if ok else math.nan
    res, res64 = (_residual(R, t, a, b, w) if ok else math.inf), _residual(R64, t64, a, b, w)
    d = 2e-7 * scale
    tol = 2 * d * math.sqrt(res64) + d * d
    table.append(f'  {name:28s} |R^T R - I| {orth:9.2e}  det - 1 {det - 1:9.2e}  residual {res:.3e} (float64 optimum '
                 f'{res64:.3e}, tolerance {tol:.1e})')
    if not (ok and orth <= 1e-6 and abs(det - 1) <= 1e-6 and res <= res64 + tol):
        fails.append(name)


def test_compute_rigid_transform_vs_float64():
    from regtr_b200 import se3
    table, fails = [], []
    for name, a, b, w, unique in _pose_problems():
        T = se3.compute_rigid_transform(torch.from_numpy(a)[None].to(DEV), torch.from_numpy(b)[None].to(DEV),
                                        torch.from_numpy(w)[None].to(DEV))[0].cpu().numpy()
        _pose_check(name, T, a, b, w, unique, table, fails)
    print('\nse3.compute_rigid_transform against float64 Kabsch (unique problems: bound 1e-6)\n' + '\n'.join(table))
    assert not fails, fails


def test_pose_from_corr_layers_and_pairs_vs_float64():
    """pose_from_corr with 6 layers and 3 pairs of unequal size: each (layer, pair) solved from its own rows --
    (kp, corr) of the source, (corr, kp) of the target, weights sigmoid(logit) with logits up to +-30 -- against
    float64 Kabsch, each with its own rotation (some at 180 degrees) and translation."""
    from regtr_b200 import ops
    rng = np.random.default_rng(4)
    L_, src_lens, tgt_lens = 6, [40, 7, 33], [25, 90, 3]
    B = len(src_lens)
    lens = src_lens + tgt_lens
    st = np.concatenate([[0], np.cumsum(lens)])
    n = int(st[-1])
    kp = (rng.normal(size=(n, 3)) * 0.5 + np.array(XYZ_OFFSET)).astype(np.float32)
    corr = np.empty((L_, n, 3), dtype=np.float32)
    logit = rng.uniform(-30, 30, size=(L_, n)).astype(np.float32)
    logit[:, ::5], logit[:, 1::7] = 30.0, -30.0
    for l in range(L_):
        for b in range(B):
            R = _rot(rng.normal(size=3), math.pi if (l + b) % 4 == 0 else rng.uniform(0, 3))
            t = rng.normal(size=3)
            s, tg = slice(st[b], st[b + 1]), slice(st[B + b], st[B + b + 1])
            corr[l, s] = kp[s] @ R.T + t + rng.normal(size=(src_lens[b], 3)) * 0.02
            corr[l, tg] = (kp[tg] - t) @ R + rng.normal(size=(tgt_lens[b], 3)) * 0.02
    pose = ops.pose_from_corr(torch.from_numpy(kp).to(DEV), torch.from_numpy(corr).to(DEV),
                              torch.from_numpy(logit).to(DEV), ops.make_offsets(lens, DEV), B).cpu().numpy()
    table, fails = [], []
    for l in range(L_):
        for b in range(B):
            s, tg = slice(st[b], st[b + 1]), slice(st[B + b], st[B + b + 1])
            a = np.concatenate([kp[s], corr[l, tg]])
            bb = np.concatenate([corr[l, s], kp[tg]])
            w = 1.0 / (1.0 + np.exp(-np.concatenate([logit[l, s], logit[l, tg]]).astype(np.float64)))
            _pose_check(f'layer {l} pair {b}', pose[l, b], a, bb, w, True, table, fails)
    print('\npose_from_corr against float64 Kabsch (bound 1e-6)\n' + '\n'.join(table))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------------ KPConv

KP_OFFSET = np.array(XYZ_OFFSET)
KP_NQ, KP_EXTENT, KP_RADIUS = 301, 0.05, 0.0625         # the 3DMatch config's first level
KP_PATHS = [(1, 'fused'), (1, 'aggregate'), (4, 'default')] + [(c, 'default') for c in (32, 64, 128, 256)]
_KPC = {}


def _kp_inputs(cin, K, nq=KP_NQ):
    """Model-like KPConv inputs: queries ~2.5 m from the origin, per query its own support rows -- three at a kernel
    point's extent (exactly, and 2 ulp inside / outside), the rest in the radius ball -- scattered over the K slots
    with shadow slots (id == Ns) between them.  Feature rows: every 5th sums to exactly 0, every 7th is negative (both
    uncounted: they move the divisor).  Query 7 has no valid neighbour, query 11 no counted one."""
    rng = np.random.default_rng(100 * cin + K)
    kp = np.zeros((15, 3))
    d = rng.normal(size=(14, 3))
    kp[1:] = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.25, 0.65, (14, 1)) * KP_RADIUS
    kp = kp.astype(np.float32)
    ext = float(np.float32(KP_EXTENT))
    q = (KP_OFFSET + rng.normal(size=(nq, 3)) * 0.4).astype(np.float32)
    s_rows, idx = [], np.empty((nq, K), dtype=np.int64)
    for i in range(nq):
        n = 0 if i == 7 else int(rng.integers(1, K + 1)) if i % 3 else K
        rel = rng.normal(size=(n, 3))
        rel = rel / np.linalg.norm(rel, axis=1, keepdims=True) * KP_RADIUS * rng.uniform(0, 1, (n, 1)) ** (1 / 3)
        for j, f in enumerate((1.0, 1 - 1e-5, 1 + 1e-5)[:n]):   # at, just inside, just outside kernel point j's extent
            u = rng.normal(size=3)
            rel[j] = kp[j + 3] + u / np.linalg.norm(u) * ext * f
        slots = np.sort(rng.choice(K, size=n, replace=False))
        idx[i] = -1
        idx[i, slots] = len(s_rows) + np.arange(n)
        s_rows.extend(q[i] + rel)
    Ns = len(s_rows)
    s = np.asarray(s_rows, dtype=np.float32)
    idx[idx < 0] = Ns                                                    # shadow slots, also between real ones
    x = (rng.normal(size=(Ns, cin)) * 0.8 + 0.3).astype(np.float32)
    x[::7] = -np.abs(x[::7]) - 0.1
    x[::5] = 0
    if cin > 1:
        c = rng.uniform(0.5, 2, size=len(x[::5])).astype(np.float32)
        x[::5, 0], x[::5, 1] = c, -c
    own = idx[11][idx[11] < Ns]
    x[own] = -np.abs(x[own]) - 0.1
    x[own[::2]] = 0
    W = (rng.normal(size=(15, cin, 32 if cin == 4 else 64 if cin == 1 else cin)) / math.sqrt(15 * cin)).astype(np.float32)
    return dict(q=q, s=s, idx=idx, x=x, W=W, kp=kp, extent=ext, Ns=Ns)


def _kp_ref(c, dtype):
    """(wf [Nq, 15 Cin], out [Nq, Cout]) of oracle.regtr_oracle.kpconv's operations in `dtype`, with the divisor of the
    exact row sums (no fp32 rounding decides a count); wf is the influence-weighted sum already divided, as the
    kernels store it."""
    from oracle import regtr_oracle as O
    q, s, x, W, kp = (torch.from_numpy(c[k]).to(dtype) for k in ('q', 's', 'x', 'W', 'kp'))
    idx = torch.from_numpy(c['idx'])
    count = O.kpconv_count(idx, torch.from_numpy(c['x']).double())
    nb = torch.cat([s, torch.full_like(s[:1], 1e6)])[idx] - q[:, None]
    d2 = ((nb[:, :, None] - kp) ** 2).sum(-1)
    infl = torch.clamp(1 - torch.sqrt(d2) / c['extent'], min=0.0).transpose(1, 2)
    wf = infl @ torch.cat([x, torch.zeros_like(x[:1])])[idx] / count[:, None, None].to(dtype)
    out = O.kpconv(q, s, idx, x, W, kp, c['extent'], count=count)
    return wf.reshape(len(q), -1), out


def _kp_case(cin, impl, K, nq=KP_NQ):
    """GPU results of one path on _kp_inputs, exact-shaped and capacity-shaped, and the float64 / fp32 references."""
    key = (cin, impl, K, nq)
    if key in _KPC:
        return _KPC[key]
    from regtr_b200 import ops
    c = _kp_inputs(cin, K, nq)
    G = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)
    q, s, idx, x, W, kp = G(c['q']), G(c['s']), G(c['idx'], torch.int32), G(c['x']), G(c['W']), G(c['kp'])
    r = dict(ref=c)
    if not (cin == 1 and impl == 'fused'):
        r['wf'] = ops.kpconv_aggregate(q, s, idx, x, kp, c['extent']).cpu()
        r['wf2'] = ops.kpconv_aggregate(q, s, idx, x, kp, c['extent']).cpu()
    if impl != 'aggregate':
        r['out'] = ops.kpconv(q, s, idx, x, W, kp, c['extent']).cpu()
        r['out2'] = ops.kpconv(q, s, idx, x, W, kp, c['extent']).cpu()
    if cin > 1 and impl != 'aggregate':            # the InstanceNorm-statistics GEMM epilogue, two clouds
        lens = [180, nq - 180]
        o, st = ops.kpconv(q, s, idx, x, W, kp, c['extent'], instats=(ops.make_offsets(lens, DEV), 2))
        r['instats'] = (lens, o.cpu(), st.cpu())
    # capacity form: garbage query / support / feature rows past nq_dev / ns_dev; the real rows' shadow id Ns is a
    # garbage row of the capacity buffer and must still count as the shadow
    g = np.random.default_rng(1)
    pq, ps = 100, 20
    qc = G(np.r_[c['q'], g.uniform(-1e3, 1e3, (pq, 3))].astype(np.float32))
    sc = G(np.r_[c['s'], g.uniform(-1e3, 1e3, (ps, 3))].astype(np.float32))
    xc = G(np.r_[c['x'], np.full((ps, cin), 1e3)].astype(np.float32))
    ic = G(np.r_[c['idx'], g.integers(0, c['Ns'] + ps, (pq, K))], torch.int32)
    nq_dev, ns_dev = (torch.tensor([v], dtype=torch.int32, device=DEV) for v in (nq, c['Ns']))
    if not (cin == 1 and impl == 'fused'):
        wf = torch.full((nq + pq, 15 * cin), math.nan, device=DEV)
        ops.kpconv_aggregate(qc, sc, ic, xc, kp, c['extent'], wf=wf, nq_dev=nq_dev, ns_dev=ns_dev)
        r['wf_cap'] = wf.cpu()
    if impl != 'aggregate':
        out = torch.full((nq + pq, W.shape[2]), math.nan, device=DEV)
        ops.kpconv(qc, sc, ic, xc, W, kp, c['extent'], out=out, nq_dev=nq_dev, ns_dev=ns_dev)
        r['out_cap'] = out.cpu()
    torch.cuda.synchronize()
    (r['wf64'], r['out64']), (r['wf32'], r['out32']) = _kp_ref(c, torch.float64), _kp_ref(c, torch.float32)
    _KPC[key] = r
    return r


def _kp_rows(title, r, wf=None, out=None):
    """Yardstick rows: wf (aggregation) and out, exact-shaped and capacity-shaped; mean / rstd / normalised output of
    the statistics epilogue per cloud.  wf / out replace the kernel's (sharpness checks) -> Yardstick."""
    from oracle import regtr_oracle as O
    ys = Yardstick(title)
    wf = r.get('wf') if wf is None else wf
    out = r.get('out') if out is None else out
    nq = len(r['ref']['q'])
    if wf is not None:
        ys.add('wf', wf, r['wf32'], r['wf64'])
        ys.add('wf, capacity form', r['wf_cap'][:nq], r['wf32'], r['wf64'])
    if out is not None:
        ys.add('out', out, r['out32'], r['out64'])
        ys.add('out, capacity form', r['out_cap'][:nq], r['out32'], r['out64'])
    if 'instats' in r:
        lens, o, st = r['instats']
        ys.add('out, statistics epilogue', o, r['out32'], r['out64'])
        m64, s64 = _in_stats(r['out64'], lens, torch.float64)
        m32, s32 = _in_stats(r['out32'], lens, torch.float32)
        ys.add('  mean', st[..., 0], m32, m64)
        ys.add('  rstd', st[..., 1], s32, s64)
    ys.report()
    return ys


def _kp_check(cin, impl, K, nq=KP_NQ):
    """One path under the yardstick against float64; two calls are bit-identical; the capacity form's real rows equal
    the exact-shaped call's aggregation bit for bit, and its padding rows up to the consumer GEMM's 128-row tile are 0."""
    r = _kp_case(cin, impl, K, nq)
    ys = _kp_rows(f'kpconv Cin={cin} {impl}, K={K}, Nq={nq}', r)
    for a, b in (('wf', 'wf2'), ('out', 'out2')):
        if a in r:
            assert torch.equal(r[a], r[b]), f'{a} not bit-identical from call to call'
    band = (nq + 127) // 128 * 128
    if 'wf' in r:
        assert torch.equal(r['wf_cap'][:nq], r['wf']), 'capacity-form aggregation differs from the exact-shaped one'
        assert torch.equal(r['wf_cap'][nq:band], torch.zeros_like(r['wf_cap'][nq:band])), 'padding rows not 0'
    if 'out' in r and cin == 1:
        assert torch.equal(r['out_cap'][nq:band], torch.zeros_like(r['out_cap'][nq:band])), 'padding rows not 0'
    empty = r.get('out', r.get('wf'))[7]
    assert float(empty.abs().max()) == 0.0, 'a query without valid neighbours must give 0'
    assert not ys.failures(), ys.failures()


@pytest.mark.parametrize('K', [40, 50, 72])
@pytest.mark.parametrize('cin,impl', KP_PATHS, ids=[f'{c}-{i}' for c, i in KP_PATHS])
def test_kpconv_vs_float64(cin, impl, K):
    """Every KPConv dispatch path -- Cin = 1 fused (regtr_kpconv_fwd) and aggregate-only, the small-Cin kernel, Cin 32
    to 256 through the pipelined kernel (K <= 64) and the staged tensor-core kernel (K = 72, one 32-channel group per
    warp at this query count), and the statistics GEMM epilogue -- at K = 40 and 50 (the configs' limits) and 72."""
    _kp_check(cin, impl, K)


@pytest.mark.parametrize('K', [72, 128])
def test_kpconv_channel_groups_vs_float64(K):
    """The staged tensor-core kernel at Cin = 256 with 2048 queries, enough warps for two 32-channel groups per warp:
    at K = 72 it takes two; at K = 128 two groups' staged rows exceed the shared memory, and it takes one."""
    _kp_check(256, 'default', K, 2048)


def test_kpconv_checks_are_sharp():
    """wf or out multiplied by (1 + 1e-5) fails its row, on the fused Cin = 1 path and the default Cin = 64 path."""
    for cin, impl in ((1, 'aggregate'), (1, 'fused'), (64, 'default')):
        r = _kp_case(cin, impl, 40)
        if 'wf' in r:
            assert 'wf' in _kp_rows(f'kpconv Cin={cin} {impl}, wf x (1 + 1e-5)', r, wf=r['wf'] * (1 + 1e-5)).failures()
        if 'out' in r:
            assert 'out' in _kp_rows(f'kpconv Cin={cin} {impl}, out x (1 + 1e-5)', r, out=r['out'] * (1 + 1e-5)).failures()


# ---------------------------------------------------------------------------------------------------- max_pool

@pytest.mark.parametrize('C', [128, 6], ids=['vector', 'scalar'])
def test_max_pool_bit_exact(C):
    """max_pool equals oracle.regtr_oracle.max_pool bit for bit: C % 4 != 0 takes the scalar kernel; queries whose
    real neighbours are all negative take the zero shadow row when they have a shadow slot and their largest
    negative value when they have none; a query of shadows only gives 0; the capacity form (ns_dev, the shadow id
    pointing at a garbage row of the buffer) gives the same result."""
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    rng = np.random.default_rng(C)
    Nq, Ns, K = 500, 900, 40
    x = rng.normal(size=(Ns, C)).astype(np.float32)
    x[::3] = -np.abs(x[::3]) - 1e-3                                      # all-negative rows
    idx = rng.integers(0, Ns, size=(Nq, K))
    idx[:, 5:K:4] = np.where(rng.random((Nq, len(range(5, K, 4)))) < 0.5, Ns, idx[:, 5:K:4])   # shadows mid-row
    neg = np.arange(0, Ns, 3)
    idx[10:20] = rng.choice(neg, size=(10, K))                           # all negative, no shadow slot
    idx[20:30] = rng.choice(neg, size=(10, K))
    idx[20:30, 17] = Ns                                                  # all negative, one shadow slot
    idx[30] = Ns
    want = O.max_pool(torch.from_numpy(x), torch.from_numpy(idx))
    assert float(want[10:20].max()) < 0 and float(want[20:31].abs().max()) == 0
    G = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)
    got = ops.max_pool(G(x), G(idx, torch.int32)).cpu()
    xc = G(np.r_[x, np.full((50, C), 1e3, dtype=np.float32)])
    got_cap = ops.max_pool(xc, G(idx, torch.int32), ns_dev=torch.tensor([Ns], dtype=torch.int32, device=DEV)).cpu()
    assert torch.equal(got, want), int((got != want).sum())
    assert torch.equal(got_cap, want), int((got_cap != want).sum())


# ----------------------------------------------------------------------------------------------- layernorm_pos

LN_E, LN_N = 256, 400


def _ln_case():
    """Rows of mean / std 0, 3, 30 and 300 (row r: RATIOS[r % 4]) with std from 1e-2 to 10, model-like gamma, beta
    and position embedding."""
    rng = np.random.default_rng(12)
    sd = 10 ** rng.uniform(-2, 1, size=(LN_N, 1))
    ratio = np.array(RATIOS)[np.arange(LN_N) % len(RATIOS)][:, None]
    x = (rng.normal(size=(LN_N, LN_E)) + ratio * rng.choice([-1.0, 1.0], size=(LN_N, 1))) * sd
    gamma = 1 + 0.2 * rng.normal(size=LN_E)
    beta = 0.2 * rng.normal(size=LN_E)
    pos = rng.uniform(-1, 1, size=(LN_N, LN_E))
    return [torch.from_numpy(a.astype(np.float32)) for a in (x, gamma, beta, pos)]


def _ln_rows(title, got, got_pos, x, gamma, beta, pos):
    """Plain and +pos outputs per mean / std family, GPU against float64 and fp32 F.layer_norm."""
    ys = Yardstick(title)
    refs = {dt: torch.nn.functional.layer_norm(x.to(dt), (LN_E,), gamma.to(dt), beta.to(dt), 1e-5)
            for dt in (torch.float64, torch.float32)}
    fam = torch.arange(LN_N) % len(RATIOS)
    for g, ratio in enumerate(RATIOS):
        rows = torch.nonzero(fam == g).squeeze(1)
        ys.add(f'mean/std {ratio:3d}: LN(x)', got[rows], refs[torch.float32][rows], refs[torch.float64][rows])
        ys.add(f'mean/std {ratio:3d}: LN(x) + pos', got_pos[rows], refs[torch.float32][rows] + pos[rows],
               refs[torch.float64][rows] + pos[rows].double())
    ys.report()
    return ys


def test_layernorm_pos_vs_float64():
    """layernorm_pos under the yardstick, plain and +pos, per mean / std family; the capacity form (n_dev, garbage
    rows past it) gives the exact-shaped call's rows bit for bit."""
    from regtr_b200 import ops
    x, gamma, beta, pos = _ln_case()
    D = lambda t: t.to(DEV)
    y, yp = ops.layernorm_pos(D(x), D(gamma), D(beta), D(pos))
    y, yp = y.cpu(), yp.cpu()
    ys = _ln_rows(f'layernorm_pos, E = {LN_E}', y, yp, x, gamma, beta, pos)
    xc = D(torch.cat([x, torch.full((60, LN_E), 1e3)]))
    pc = D(torch.cat([pos, torch.full((60, LN_E), 1e3)]))
    yc, ypc = ops.layernorm_pos(xc, D(gamma), D(beta), pc, n_dev=torch.tensor([LN_N], dtype=torch.int32, device=DEV))
    assert torch.equal(yc[:LN_N].cpu(), y) and torch.equal(ypc[:LN_N].cpu(), yp), 'capacity form differs'
    assert not ys.failures(), ys.failures()


def test_layernorm_pos_checks_are_sharp():
    """Outputs x (1 + 1e-5) fail the rows of mean / std 0 and 3.  At 30 and 300 the fp32 oracle itself is about 1.5e-6
    and 1.2e-5 off float64 (the rounding of a mean 30 or 300 std from zero, carried into every output), so the
    yardstick cannot tell a 1e-5 error from fp32 rounding there."""
    from regtr_b200 import ops
    x, gamma, beta, pos = _ln_case()
    D = lambda t: t.to(DEV)
    y, yp = (t.cpu() for t in ops.layernorm_pos(D(x), D(gamma), D(beta), D(pos)))
    fails = set(_ln_rows('layernorm_pos, outputs x (1 + 1e-5)', y * (1 + 1e-5), yp * (1 + 1e-5), x, gamma, beta,
                         pos).failures())
    assert {f'mean/std {q:3d}: LN(x){p}' for q in RATIOS[:2] for p in ('', ' + pos')} <= fails, fails


# ---------------------------------------------------------------------------------------------- pos_embed_sine

def _pe_rows(title, got, xyz):
    """The sine and the cosine columns against float64 of the same operation on the same fp32 coordinates and the
    same fp32 frequency table (oracle.regtr_oracle.pos_embed_sine), and the fp32 oracle."""
    from oracle import regtr_oracle as O
    r64, r32 = O.pos_embed_sine(xyz.double()), O.pos_embed_sine(xyz)
    ys = Yardstick(title)
    n_freq = 256 // 3 // 2 * 2
    cols = torch.arange(3 * n_freq)
    for name, sel in (('sin', cols[(cols % n_freq) % 2 == 0]), ('cos', cols[(cols % n_freq) % 2 == 1])):
        ys.add(name, got[:, sel], r32[:, sel], r64[:, sel])
    ys.add('zero padding', got[:, 3 * n_freq:], r32[:, 3 * n_freq:], r64[:, 3 * n_freq:])
    ys.report()
    return ys


def _pe_inputs(span):
    rng = np.random.default_rng(int(span))
    xyz = rng.uniform(-span, span, size=(3000, 3))
    xyz[:8] = np.array([[span, -span, 0.0], [-span, span, 1e-7], [0, 0, 0], [span / 2, span / 3, -span / 7]] * 2)
    return torch.from_numpy(xyz.astype(np.float32))


@pytest.mark.parametrize('span', [5.0, 1.0], ids=['world_5m', 'modelnet_unit'])
def test_pos_embed_sine_vs_float64(span):
    """Coordinates up to +-5 m (arguments up to 10 pi) and the ModelNet unit range."""
    from regtr_b200 import ops
    xyz = _pe_inputs(span)
    got = ops.pos_embed_sine(xyz.to(DEV)).cpu()
    ys = _pe_rows(f'pos_embed_sine, coordinates in [-{span:g}, {span:g}]', got, xyz)
    assert float(got[:, 3 * (256 // 3 // 2 * 2):].abs().max()) == 0.0
    assert not ys.failures(), ys.failures()


def test_pos_embed_sine_checks_are_sharp():
    from regtr_b200 import ops
    xyz = _pe_inputs(5.0)
    got = ops.pos_embed_sine(xyz.to(DEV)).cpu()
    fails = _pe_rows('pos_embed_sine, output x (1 + 1e-5)', got * (1 + 1e-5), xyz).failures()
    assert {'sin', 'cos'} <= set(fails), fails
