"""References and a kernel model for the KPConv-encoder backward (csrc/kpconv_bwd.cu).  CPU only.

References: dx and dW of oracle.regtr_oracle.kpconv by autograd with the divisor fixed by O.kpconv_count, in
float64 (the truth) and fp32 (the yardstick, tests/grad_yardstick.py); dx of O.max_pool by autograd.

Model: the shipped kernels' arithmetic restated in numpy fp32.  Per valid edge (query q, slot k, support s) phase (a)
computes the influence h_p = max(0, fma(-|rel - kp_p|, 1 / extent, 1)) of each of the 15 kernel points and the edge
row E = (fma chain over p = 0..14 ascending of h_p dwf[q, p]) * (1 / max(count, 1)), the count taken from the row
flags or, without flags, recomputed from x as the fp64 row sum > 0; phase (b) sums each support's incoming rows in
fp32, in ascending edge id.  The max-pool backward gives each (query, channel) to the first slot holding the maximum
(shadow slots take part with value 0 and pass nothing on) and sums the same way.  The kernels' sqrt.approx and
rcp.approx are modelled by correctly rounded fp32 sqrt and division: both are within an ulp of those, which moves
the model's error by far less than the yardstick's factor.  dwf = dOut W^T comes from the 3xTF32 GEMM, which is as
accurate as fp32; the model takes it rounded to fp32 from float64.

Emulated wrong kernels (`variant`), each one small change to the model:
  valid_divisor   the divisor counts every valid neighbour instead of those whose feature row sums to > 0
  phantom_kp      the padded 16th kernel-point lane is not zeroed: the chain takes a 16th term, the influence of a
                  kernel point at the origin, against kernel point 0's gradient row
  tail_dropped    the last channel pass of the edge kernel is dropped when it is partial (Cin not a multiple of
                  32 NV, NV = 1 / 2 / 4 channels per lane for Cin <= 32 / 64 / more)
  shadow_to_last  shadow slots are clamped to support Ns - 1 instead of skipped, in the edge pass and the transpose
  fill_order      each support's incoming rows summed in a scheduling-dependent order (seeded) instead of ascending
                  edge id: within the yardstick, caught only by the bit-exactness assertions
Max-pool variants (`mp_variant`):
  ties_last       a tie goes to the last slot holding the maximum instead of the first
  shadow_leak     a shadow winner's gradient reaches a real row (support Ns - 1)
"""
import numpy as np
import torch

KP = 15
VARIANTS = ('shipped', 'valid_divisor', 'phantom_kp', 'tail_dropped', 'shadow_to_last', 'fill_order')
MP_VARIANTS = ('shipped', 'ties_last', 'shadow_leak')
FAMILIES = ('zero_mean', 'offset', 'zero_rows')

# The domain tests/test_gpu_kpconv_backward_domain.py runs (the model's own shapes must lie inside it).
KPCONV_CIN = (1, 4, 8, 12, 16, 32, 64, 128, 256)
KPCONV_K = (1, 7, 33, 40, 50, 64, 65, 72, 128)
CONFIG_K = (40, 50)                                 # the 3DMatch and ModelNet neighbourhood limits
SWEEP_CIN = (16, 64, 256)                           # every K at these
CORNERS = [(c, k) for c in (1, 256) for k in (1, 128)]
MODES = ('flags', 'noflags', 'x_only')
POOL_C = (1, 3, 6, 33, 128, 256, 512, 1024)
POOL_K = (1, 40, 50, 254, 255)


def kpconv_cases():
    """The covering set of (Cin, K, mode): every Cin at the configs' K, every K at SWEEP_CIN, every mode at the
    corners; the other cases rotate through the modes."""
    pairs = sorted({(c, k) for c in KPCONV_CIN for k in CONFIG_K} | {(c, k) for c in SWEEP_CIN for k in KPCONV_K}
                   | set(CORNERS))
    cases = []
    for i, (c, k) in enumerate(pairs):
        for m in (MODES if (c, k) in CORNERS else (MODES[i % 3],)):
            cases.append((c, k, m))
    return cases


def gout_family(name, Nq, C, seed):
    """Output gradients: zero-mean | a per-channel offset 10x the spread | every third row zero."""
    g = np.random.default_rng(seed).standard_normal((Nq, C))
    if name == 'zero_mean':
        g -= g.mean(0, keepdims=True)
    elif name == 'offset':
        g += 10.0 * np.random.default_rng(seed + 1).choice([-1.0, 1.0], size=C)
    elif name == 'zero_rows':
        g[::3] = 0
    else:
        raise ValueError(name)
    return g.astype(np.float32)


# ------------------------------------------------------------------------------------------------- references

def kpconv_grads(c, W, gouts, dtype, need_w=True):
    """[(dx, dW or None)] of oracle.regtr_oracle.kpconv in `dtype` for each output gradient in `gouts`, on a case of
    test_gpu_forward_ops._kp_inputs (q, s, idx, x, kp, extent), the divisor fixed from float64 row sums."""
    from oracle import regtr_oracle as O
    q, s, x, kp = (torch.from_numpy(np.asarray(c[k])).to(dtype) for k in ('q', 's', 'x', 'kp'))
    idx = torch.from_numpy(np.asarray(c['idx'], np.int64))
    count = O.kpconv_count(idx, torch.from_numpy(np.asarray(c['x'])).double())
    xr = x.requires_grad_(True)
    wr = torch.from_numpy(np.asarray(W)).to(dtype).requires_grad_(need_w)
    y = O.kpconv(q, s, idx, xr, wr, kp, c['extent'], count=count)
    res = []
    for g in gouts:
        gr = torch.autograd.grad(y, [xr, wr] if need_w else [xr], torch.from_numpy(np.asarray(g)).to(dtype),
                                 retain_graph=True)
        res.append((gr[0], gr[1] if need_w else None))
    return res


def max_pool_dx(x, idx, gout, dtype):
    """dx of oracle.regtr_oracle.max_pool by autograd in `dtype`."""
    from oracle import regtr_oracle as O
    xr = torch.from_numpy(np.asarray(x)).to(dtype).requires_grad_(True)
    y = O.max_pool(xr, torch.from_numpy(np.asarray(idx, np.int64)))
    y.backward(torch.from_numpy(np.asarray(gout)).to(dtype))
    return xr.grad


def max_pool_failures(got, want):
    """The max-pool backward's criteria: the entries that receive gradient are float64 autograd's, and every value is
    within 1e-6 max|want| of it.  -> list of the criteria broken."""
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    fails = []
    if not torch.equal(got != 0, want != 0):
        fails.append(f'support set: {int(((got != 0) != (want != 0)).sum())} entries differ')
    if got.numel() and float((got - want).abs().max()) > 1e-6 * float(want.abs().max()):
        fails.append('values beyond 1e-6 max')
    return fails


def csr_numpy(idx, Ns):
    """The incoming-edge CSR of a neighbour list: (row_start (Ns + 1), edges) with each row in ascending edge id."""
    flat = np.asarray(idx).reshape(-1)
    e = np.nonzero((flat >= 0) & (flat < Ns))[0]
    order = np.argsort(flat[e], kind='stable')                  # stable: ascending edge id within a row
    row_start = np.zeros(Ns + 1, np.int64)
    np.cumsum(np.bincount(flat[e], minlength=Ns), out=row_start[1:])
    return row_start.astype(np.int32), e[order].astype(np.int32)


# ------------------------------------------------------------------------------------------------- kernel model

def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32)


def _fma(a, b, c):
    """fmaf(a, b, c) on fp32 operands: the exact product and sum, rounded once (via float64)."""
    return _f32(a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64))


def _influence(rel, kp, inv_extent):
    """(E, 3) relative positions, (P, 3) kernel points -> (E, P) influences, the kernels' fp32 steps."""
    d = rel[:, None, :] - kp[None]
    d2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]
    return np.maximum(np.float32(0), _fma(-np.sqrt(d2), np.full_like(d2, inv_extent), np.ones_like(d2)))


def _rowsum(rows, Ns, idx_flat, seed=None):
    """dx[s] = fp32 sum of rows[e] over the edges e with idx_flat[e] == s, ascending e (or a seeded order)."""
    e = np.nonzero((idx_flat >= 0) & (idx_flat < Ns))[0]
    if seed is not None:
        e = np.random.default_rng(seed).permutation(e)
    e = e[np.argsort(idx_flat[e], kind='stable')]
    sup = idx_flat[e]
    first = np.searchsorted(sup, sup)                           # rank of each edge within its support's row
    rank = np.arange(len(e)) - first
    out = np.zeros((Ns, rows.shape[1]), np.float32)
    for r in range(int(rank.max(initial=-1)) + 1):
        m = rank == r
        out[sup[m]] = out[sup[m]] + rows[e[m]]
    return out


def model_dx(c, dwf, flags=None, variant='shipped', seed=1):
    """dx (Ns, Cin) of the edge kernel + CSR row sum on a _kp_inputs case; dwf (Nq, 15 Cin) fp32."""
    q, s, x, kp = (np.asarray(c[k], np.float32) for k in ('q', 's', 'x', 'kp'))
    idx = np.asarray(c['idx'], np.int64)
    Nq, K = idx.shape
    Ns, Cin = x.shape
    valid = (idx >= 0) & (idx < Ns)
    if variant == 'shadow_to_last':
        idx = np.where(valid, idx, Ns - 1)
    live = (idx >= 0) & (idx < Ns)
    qe, ke = np.nonzero(live)
    se = idx[qe, ke]
    inv_extent = np.float32(1) / np.float32(c['extent'])
    h = _influence(s[se] - q[qe], kp, inv_extent)
    pos = x.astype(np.float64).sum(1) > 0 if flags is None else np.asarray(flags).astype(bool)
    if variant == 'valid_divisor':
        pos = np.ones(Ns, bool)
    cnt = np.where(valid, pos[np.where(valid, idx, 0)], False).sum(1)
    inv = np.float32(1) / np.maximum(cnt, 1).astype(np.float32)
    d = np.asarray(dwf, np.float32).reshape(Nq, KP, Cin)
    acc = np.zeros((len(qe), Cin), np.float32)
    for p in range(KP):
        acc = _fma(np.repeat(h[:, p:p + 1], Cin, 1), d[qe, p], acc)
    if variant == 'phantom_kp':
        h0 = _influence(s[se] - q[qe], np.zeros((1, 3), np.float32), inv_extent)
        acc = _fma(np.repeat(h0, Cin, 1), d[qe, 0], acc)
    E = np.zeros((Nq * K, Cin), np.float32)
    E[qe * K + ke] = acc * inv[qe, None]
    if variant == 'tail_dropped':
        nv = 1 if Cin <= 32 else 2 if Cin <= 64 else 4
        if Cin % (32 * nv):
            E[:, Cin // (32 * nv) * 32 * nv:] = 0
    return _rowsum(E, Ns, idx.reshape(-1), seed if variant == 'fill_order' else None)


def model_max_pool_dx(x, idx, gout, mp_variant='shipped'):
    """dx (Ns, C) of the max-pool backward: winner slot per (query, channel), then the CSR row sum."""
    x, gout = np.asarray(x, np.float32), np.asarray(gout, np.float32)
    idx = np.asarray(idx, np.int64)
    Nq, K = idx.shape
    Ns, C = x.shape
    valid = (idx >= 0) & (idx < Ns)
    vals = np.where(valid[..., None], x[np.where(valid, idx, 0)], np.float32(0))          # (Nq, K, C)
    if mp_variant == 'ties_last':
        arg = K - 1 - np.argmax(vals[:, ::-1], axis=1)
    else:
        arg = np.argmax(vals, axis=1)                                                       # first maximum
    if mp_variant == 'shadow_leak':
        idx = np.where(valid, idx, Ns - 1)
    rows = np.where(np.arange(K)[None, :, None] == arg[:, None, :], gout[:, None, :], np.float32(0))
    return _rowsum(rows.reshape(Nq * K, C), Ns, idx.reshape(-1))


def max_pool_case(C, K, Nq=64, Ns=300, seed=0):
    """Max-pool inputs: values on a coarse grid (ties), every fourth column negative (the zero shadow wins where a
    query has a shadow slot), shadow slots (id Ns and -1) between real ones, an all-shadow row (query 0), a row whose
    K slots hold one support (query 1) and one whose K slots hold supports with equal rows (query 2).
    -> (x (Ns, C) fp32, idx (Nq, K) int32, gout (Nq, C) fp32 without zeros)."""
    rng = np.random.default_rng(seed)
    x = (rng.integers(-4, 5, size=(Ns, C)) * 0.5).astype(np.float32)
    x[:, ::4] = -np.abs(x[:, ::4]) - 0.5
    idx = rng.integers(0, Ns, size=(Nq, K))
    idx[rng.random((Nq, K)) < 0.2] = Ns
    idx[rng.random((Nq, K)) < 0.05] = -1
    idx[0] = Ns
    idx[1] = rng.integers(0, Ns)
    same = rng.choice(Ns, size=min(K, 16), replace=False)
    x[same] = x[same[0]]
    idx[2] = np.resize(same, K)
    gout = rng.standard_normal((Nq, C)).astype(np.float32)
    gout[gout == 0] = 1
    return x, idx.astype(np.int32), gout


def dense_case(Nq, K, Ns, cin, seed, degrees='uniform'):
    """KPConv inputs with shared supports: queries and supports in one ball of 0.4 radius, so that most influences are
    non-zero.  degrees: 'uniform' (slots drawn from every support, 10 % shadow) | 'hub' (every slot holds support 0) |
    'skewed' (slots drawn from the lower half of the supports with weights 1 / (j + 1)^1.5: at Nq K = 4096 edges
    the in-degrees run from about 1900 down to 0, the upper half unreferenced).  -> the dict of test_gpu_forward_ops._kp_inputs."""
    rng = np.random.default_rng(seed)
    radius, ext = 0.0625, float(np.float32(0.05))
    kp = np.zeros((15, 3))
    d = rng.normal(size=(14, 3))
    kp[1:] = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.25, 0.65, (14, 1)) * radius
    centre = np.array([2.0, -1.5, 0.5])

    def ball(n):
        u = rng.normal(size=(n, 3))
        return (centre + u / np.linalg.norm(u, axis=1, keepdims=True) * 0.4 * radius
                * rng.uniform(0, 1, (n, 1)) ** (1 / 3)).astype(np.float32)
    q, s = ball(Nq), ball(Ns)
    if degrees == 'hub':
        idx = np.zeros((Nq, K), np.int64)
    elif degrees == 'skewed':
        w = 1.0 / np.arange(1, max(Ns // 2, 1) + 1) ** 1.5
        idx = rng.choice(len(w), size=(Nq, K), p=w / w.sum())
    else:
        idx = rng.integers(0, Ns, size=(Nq, K))
        idx[rng.random((Nq, K)) < 0.1] = Ns
    x = (rng.normal(size=(Ns, cin)) * 0.8 + 0.3).astype(np.float32)
    x[::7] = -np.abs(x[::7]) - 0.1
    return dict(q=q, s=s, idx=idx, x=x, kp=kp.astype(np.float32), extent=ext, Ns=Ns)
