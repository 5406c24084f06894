"""GPU tests of every 3xTF32 GEMM entry point against float64, on each dispatch path, under the fp32 yardstick.

Each case's reference is the float64 product (plus bias, residual and ReLU) of the operands the kernel multiplies, and
its fp32 restatement is the same expression in torch CPU float32 (tests/grad_yardstick.py; tests/gemm_oracle.py holds
the families, the restated dispatch rules and the TF32 roundings; tests/test_gemm_sharpness.py shows on a model of the
kernel that the rule fails a kernel that is subtly wrong).  Every case asserts the path it is named after: BN from N,
the split count read back from `regtr_gemm_ws_bytes`.  Every launch writes into a sentinel-filled buffer wider and
taller than C: rows at or past the device row count and columns at or past N must keep the sentinel, and a second
launch must give the same buffer bit for bit.
"""
import numpy as np
import pytest
import torch

import gemm_oracle as go
from grad_yardstick import Yardstick

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SENT = float(np.float32(-1.2345e30))
GARBAGE = 1e3


def _lib():
    from regtr_b200 import lib
    return lib.load()


def _g(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _padded(x, pad, fill, offset=False):
    """x (rows, cols) on the device as a view of a (rows, cols + pad) buffer whose other entries are `fill`;
    offset: the view's base is 4 bytes past a 16-byte boundary."""
    rows, cols = x.shape
    ld = cols + pad
    flat = torch.full((rows * ld + 4,), fill, dtype=torch.float32, device=DEV)
    v = flat[int(offset):int(offset) + rows * ld].view(rows, ld)[:, :cols]
    v.copy_(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)))
    return v


def _out_buffer(rows, N, pad, offset):
    """Sentinel-filled flat buffer and the (rows, N) view with pitch N + pad that the GEMM writes."""
    ld = N + pad
    flat = torch.full(((rows + 2) * ld + 4,), SENT, dtype=torch.float32, device=DEV)
    return flat, flat[int(offset):int(offset) + rows * ld].view(rows, ld)[:, :N]


def _check_sentinel(flat, view, rows_written, N):
    """Everything in `flat` outside view[:rows_written, :N] still holds the sentinel."""
    keep = torch.ones_like(flat, dtype=torch.bool)
    if rows_written:
        idx = torch.arange(flat.numel(), device=DEV)
        base = view.storage_offset() - flat.storage_offset()
        rel = idx - base
        r, c = torch.div(rel, view.stride(0), rounding_mode='floor'), rel % view.stride(0)
        keep &= ~((rel >= 0) & (r < rows_written) & (c < N))
    assert bool((flat[keep] == SENT).all()), 'the GEMM wrote outside C[:m, :N]'


def _run(fn, rows, N, pad, offset, m):
    """Two launches into fresh sentinel buffers: bit-identical, sentinel kept outside C[:m, :N]; -> C[:m] (CPU)."""
    outs = []
    for _ in range(2):
        flat, view = _out_buffer(rows, N, pad, offset)
        fn(view)
        outs.append((flat, view))
    torch.cuda.synchronize()
    (f1, v1), (f2, _) = outs
    assert torch.equal(f1.view(torch.int32), f2.view(torch.int32)), 'two launches differ'
    _check_sentinel(f1, v1, m, N)
    return v1[:m].cpu()


def gemm_case(ys, family, M, N, K, bias=True, res=False, relu=False, m=None, lda_pad=0, ldc_pad=4, ldr_pad=0,
              misalign=(), splits=None, seed=0):
    """regtr_gemm_tf32x3 through ops.gemm on one shape and family; adds its yardstick rows.  M is the launch's row
    count (a capacity when m, the device row count, is given; rows past m hold garbage); splits: the split count the
    case is named after."""
    from regtr_b200 import ops
    bn, s, planes, per = go.gemm_path(M, N, K)
    assert bn == go.choose_bn(N)
    if splits is not None:
        assert s == splits, f'M={M} N={N} K={K}: {s} split-K planes, the case is named after {splits}'
    m = M if m is None else m
    rng = np.random.default_rng([seed, M, N, K])
    a = go.activations(family, M, K, rng)
    a[m:] = GARBAGE
    hi, lo = go.split_rne(go.weights(family, N, K, rng))
    B = hi + lo                                                         # exact in fp32: the operand multiplied
    c_scale = float(go.reference(a[:min(m, 512)], B).abs().max()) if m else 1.0
    bias = bias and family != 'row_scales'       # a bias of the output's size would hide the rows of 1e-3
    b = go.bias_for(N, rng, c_scale) if bias else None
    r = None
    if res:                                      # row_scales: each residual row of its own row's size
        rs = np.sqrt((a.astype(np.float64) ** 2).mean(1, keepdims=True)) if family == 'row_scales' else np.ones((M, 1))
        r = (rng.normal(size=(M, N)) * rs * (c_scale / rs[:max(m, 1)].max())).astype(np.float32)
    A = _padded(a, lda_pad, GARBAGE)
    Bh, Bl = _g(hi), _g(lo)
    Bias = (_padded(b[None], 0, 0.0, offset='bias' in misalign)[0]) if bias else None
    R = _padded(r, ldr_pad, GARBAGE, offset='res' in misalign) if res else None
    m_dev = torch.tensor([m], dtype=torch.int32, device=DEV) if m != M else None
    got = _run(lambda out: ops.gemm(A, Bh, Bl, bias=Bias, residual=R, relu=relu, m_dev=m_dev, out=out),
               M, N, ldc_pad, 'out' in misalign, m)
    flags = ''.join(t for t, on in (('+b', bias), ('+r', res), (' relu', relu)) if on)
    pads = ''.join(f' {k}+{p}' for k, p in (('lda', lda_pad), ('ldc', ldc_pad), ('ldr', ldr_pad)) if p and (
        k != 'ldc' or p != 4))
    name = (f'{family:10s} M{M}{f" m{m}" if m != M else ""} N{N} K{K} bn{bn} s{s}'
            f'{f" ({planes}x{per}kb)" if s > 1 else ""}{flags}{pads}{" misaligned " + "/".join(misalign) if misalign else ""}')
    if m == 0:
        assert got.numel() == 0
        return name
    rr = None if r is None else r[:m]
    go.add_rows(ys, name, got, go.reference(a[:m], B, b, rr, relu, torch.float32), go.reference(a[:m], B, b, rr, relu),
                family)
    return name


def _finish(ys):
    ys.report()
    assert not ys.failures(), ys.failures()


# ------------------------------------------------------------------------------------------ regtr_gemm_tf32x3

GEMM_N = [1, 3, 32, 33, 64, 65, 128, 129, 256, 260, 768]
GEMM_K = [4, 36, 64, 256, 1024, 3840]


@pytest.mark.parametrize('family', go.FAMILIES)
def test_gemm_shapes_vs_float64(family):
    """Every N (BN 32, 64 and 128 with partial tiles; N % 4 != 0 takes the scalar epilogue) at every K (K tails of 4
    and 36; K >= 512 at few tiles splits), M = 129."""
    ys = Yardstick(f'regtr_gemm_tf32x3, N x K at M = 129, {family}')
    for N in GEMM_N:
        for K in GEMM_K:
            gemm_case(ys, family, 129, N, K)
    _finish(ys)


@pytest.mark.parametrize('family', go.FAMILIES)
def test_gemm_rows_vs_float64(family):
    """M = 1, 127, 128, 129 and 20000 (several waves: CTAs walk their tiles persistently), on one-plane and split
    shapes (N = 260 on the split path crosses a 128-wide tile)."""
    ys = Yardstick(f'regtr_gemm_tf32x3, row counts, {family}')
    for M in (1, 127, 128, 129, 20000):
        for N, K in ((64, 256), (260, 1024), (768, 256)):
            gemm_case(ys, family, M, N, K, res=True)
    _finish(ys)


@pytest.mark.parametrize('family', ['zero_mean', 'leaky'])
def test_gemm_epilogue_vs_float64(family):
    """Bias, residual and ReLU each on and off, on the one-plane epilogue and through k_splitk_reduce."""
    ys = Yardstick(f'regtr_gemm_tf32x3, epilogue flags, {family}')
    for (M, N, K), s in (((300, 128, 256), 1), ((300, 64, 2048), 8)):
        for bias in (False, True):
            for res in (False, True):
                for relu in (False, True):
                    gemm_case(ys, family, M, N, K, bias=bias, res=res, relu=relu, splits=s)
    _finish(ys)


SPLIT_CASES = [((128, 64, 512), 2), ((256, 128, 1024), 4), ((128, 256, 2048), 8),
               ((64, 128, 9000), 16),        # the cap: 16 planes of 18 k-blocks
               ((1000, 260, 3840), 8)]       # raised from 6 by the rule of at most 16 k-blocks per plane


@pytest.mark.parametrize('family', go.FAMILIES)
def test_gemm_split_counts_vs_float64(family):
    ys = Yardstick(f'regtr_gemm_tf32x3, split-K counts, {family}')
    for (M, N, K), s in SPLIT_CASES:
        gemm_case(ys, family, M, N, K, res=True, splits=s)
    _finish(ys)


@pytest.mark.parametrize('family', ['zero_mean', 'row_scales'])
def test_gemm_strides_vs_float64(family):
    """lda > K, ldc > N and ldr > N through views, pitches that are multiples of 4 (float4 epilogue) and not (scalar),
    one-plane and split."""
    ys = Yardstick(f'regtr_gemm_tf32x3, strided views, {family}')
    for (M, N, K), s in (((300, 128, 256), 1), ((300, 64, 2048), 8)):
        gemm_case(ys, family, M, N, K, res=True, relu=True, lda_pad=8, ldc_pad=8, ldr_pad=4, splits=s)
        gemm_case(ys, family, M, N, K, res=True, lda_pad=12, ldc_pad=1, ldr_pad=3, splits=s)
    _finish(ys)


def test_gemm_device_row_count_vs_float64():
    """m_dev of 0, at a tile boundary and inside a tile, on one-plane and split launches of 300 capacity rows whose
    rows past m_dev are garbage; those rows of C keep the sentinel."""
    ys = Yardstick('regtr_gemm_tf32x3, device row count (capacity 300)')
    for (N, K), s in (((128, 256), 1), ((64, 2048), 8)):
        for m in (0, 128, 200):
            gemm_case(ys, 'zero_mean', 300, N, K, res=True, m=m, splits=s)
    _finish(ys)


def test_gemm_misaligned_views_vs_float64():
    """C, residual and bias views whose bases sit 4 bytes past a 16-byte boundary take the scalar epilogue."""
    ys = Yardstick('regtr_gemm_tf32x3, C / residual / bias views 4 bytes off alignment')
    for (M, N, K), s in (((300, 128, 256), 1), ((300, 64, 2048), 8)):
        for mis in (('out',), ('res',), ('bias',), ('out', 'res', 'bias')):
            gemm_case(ys, 'zero_mean', M, N, K, res=True, relu=True, misalign=mis, splits=s)
    _finish(ys)


# ------------------------------------------------------------------------------------------ weight and input gradients

WGRAD_PAIRS = [(64, 15), (32, 480), (64, 960), (128, 1920), (256, 3840),      # KPConv: Cout x 15 Cin
               (64, 32), (32, 64), (256, 128),                                  # unary blocks
               (768, 256), (256, 256), (1024, 256), (256, 1024),                # transformer
               (1, 256), (3, 256)]                                              # heads
TOKENS = [1, 3, 1503, 9000]
BIG_TOKENS = 50000


def _grad_operands(family, M, C, rng, gradient):
    """Token-major (M, C): activations of `family`, or for the upstream gradient zero-mean (leaky family: with a
    shared positive part) rows, scaled per token in the row_scales family."""
    if not gradient:
        return go.activations(family, M, C, rng)
    g = rng.normal(size=(M, C)) + (0.5 if family == 'leaky' else 0.0)
    if family == 'row_scales':
        g = g * 10.0 ** rng.uniform(-3, 3, size=(M, 1))
    return g.astype(np.float32)


def _wgrad_case(ys, family, M, N, K):
    from regtr_b200 import ops
    Mp, Kp = (M + 3) // 4 * 4, (K + 4) // 4 * 4
    bn, s, planes, per = go.gemm_path(N, Kp, max(Mp, 4))      # dW^T-free product: (N, Kp) over the Mp tokens
    rng = np.random.default_rng([M, N, K])
    x = _grad_operands(family, M, K, rng, False)
    dy = _grad_operands(family, M, N, rng, True)
    X, DY = _g(x), _g(dy)
    dw, db = ops.linear_wgrad(X, DY, True)
    dw2, db2 = ops.linear_wgrad(X, DY, True)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2) and torch.equal(db, db2), 'linear_wgrad not bit-identical on a rerun'
    if M == 0:
        assert not dw.any() and not db.any()
        return
    name = f'{family:10s} tokens {M} N{N} K{K} bn{bn} s{s}'
    x64, dy64 = torch.from_numpy(x).double(), torch.from_numpy(dy).double()
    x32, dy32 = torch.from_numpy(x), torch.from_numpy(dy)
    ys.add(name + ' dW', dw, dy32.T @ x32, dy64.T @ x64)
    ys.add(name + ' db', db, dy32.sum(0), dy64.sum(0))


@pytest.mark.parametrize('family', go.FAMILIES)
def test_linear_wgrad_vs_float64(family):
    """dW = dY^T X and db = sum dY (separate rows) at the model's (N, K) pairs; the token reduction runs on the
    split-K path up to the cap of 16 planes (9000 and 50000 tokens).  No tokens: dW and db are zero."""
    ys = Yardstick(f'regtr_linear_wgrad, {family}')
    for N, K in WGRAD_PAIRS:
        for M in [0] + TOKENS + ([BIG_TOKENS] if N * K <= 64 * 960 else []):
            _wgrad_case(ys, family, M, N, K)
    _finish(ys)


DGRAD_PAIRS = [(1, 256), (3, 256), (64, 32), (32, 64), (256, 128), (768, 256), (256, 256), (1024, 256), (256, 1024)]


@pytest.mark.parametrize('family', go.FAMILIES)
def test_linear_dgrad_vs_float64(family):
    """dX = dY W (+ the skip residual), weights (N_out, K_in) of the model; N_out % 4 != 0 zero-pads dY and W^T."""
    from regtr_b200 import ops
    ys = Yardstick(f'linear_dgrad (regtr_gemm_tf32x3 on the transposed split weight), {family}')
    for n_out, k_in in DGRAD_PAIRS:
        for M in TOKENS + ([BIG_TOKENS] if n_out * k_in <= 256 * 256 else []):
            for res in (False, True):
                bn, s, _, _ = go.gemm_path(M, k_in, (n_out + 3) // 4 * 4)
                rng = np.random.default_rng([M, n_out, k_in, res])
                dy = _grad_operands(family, M, n_out, rng, True)
                w = go.weights(family, n_out, k_in, rng)
                r = rng.normal(size=(M, k_in)).astype(np.float32) * float(np.abs(dy).max()) if res else None
                W, DY, R = _g(w), _g(dy), (_g(r) if res else None)
                got = ops.linear_dgrad(DY, W, residual=R)
                again = ops.linear_dgrad(DY, W, residual=R)
                torch.cuda.synchronize()
                assert torch.equal(got, again), 'linear_dgrad not bit-identical on a rerun'
                d64 = torch.from_numpy(dy).double() @ torch.from_numpy(w).double()
                d32 = torch.from_numpy(dy) @ torch.from_numpy(w)
                if res:
                    d64, d32 = d64 + torch.from_numpy(r).double(), d32 + torch.from_numpy(r)
                name = f'{family:10s} tokens {M} N_out {n_out} K_in {k_in} bn{bn} s{s}{" +skip" if res else ""}'
                go.add_rows(ys, name, got, d32, d64, family)
    _finish(ys)


# ------------------------------------------------------------------------------------------ attention in-projection

def _u32(t):
    return t.contiguous().view(torch.int32).cpu().numpy().view(np.uint32)


def _inproj_operands(family, M, E, seed):
    rng = np.random.default_rng([seed, M, E])
    x = go.activations(family, M, E, rng)
    hi, lo = go.split_rne(go.weights(family, 3 * E, E, rng))
    B = hi + lo
    b = go.bias_for(3 * E, rng, float(go.reference(x, B).abs().max()))
    return x, hi, lo, B, b


def _plain_inproj(ys, name, x, hi, lo, B, b, family):
    """The in-projection through regtr_gemm_tf32x3: the qkv launches run the same BN = 128, one-plane mainloop and
    add the bias the same way, so this C is the fp32 value their epilogues round."""
    from regtr_b200 import ops
    M, E = x.shape
    assert go.gemm_path(M, 3 * E, E)[:2] == (128, 1)
    c = ops.gemm(_g(x), _g(hi), _g(lo), bias=_g(b))
    torch.cuda.synchronize()
    c = c.cpu()
    go.add_rows(ys, name + ' x W^T + b', c, go.reference(x, B, b, dtype=torch.float32), go.reference(x, B, b), family)
    return c.numpy()


def _check_split_halves(hi, lo, what):
    """Low 13 bits zero; hi = rna(hi + lo) except where hi + lo sits exactly on a rounding tie the value it came
    from was below (|lo| = half a TF32 ulp of hi, lo of hi's sign); |lo| <= half a TF32 ulp of hi."""
    for t, nm in ((hi, 'hi'), (lo, 'lo')):
        assert not (t.view(np.uint32) & np.uint32(0x1FFF)).any(), f'{what}: {nm} has low mantissa bits set'
    h64, l64 = hi.astype(np.float64), lo.astype(np.float64)
    half = np.where(hi != 0, go.half_ulp_tf32(hi), 0.0)
    assert (np.abs(l64) <= half).all(), f'{what}: |lo| above half a TF32 ulp of hi'
    tie = (np.abs(l64) == half) & (np.sign(l64) == np.sign(h64)) & (hi != 0)
    back = go.tf32_rna((h64 + l64).astype(np.float32))
    assert np.array_equal(back.view(np.uint32)[~tie], hi.view(np.uint32)[~tie]), f'{what}: hi != rna(hi + lo)'


@pytest.mark.parametrize('E', [32, 96, 256])
@pytest.mark.parametrize('family', ['zero_mean', 'leaky'])
def test_qkv_split_epilogue(family, E):
    """regtr_gemm_tf32x3_qkv_split: q * qscale and k as TF32 (hi, lo) halves in qk4, v transposed with hi rows then
    lo rows in vt2 (ld_vt > M): the halves equal rna / rna of the plain GEMM's fp32 value bit for bit, hi + lo meets
    the yardstick against float64 (x W^T + b) * qscale for q and x W^T + b for k and v, and qk4's columns past 4E and
    vt2's past M keep the sentinel."""
    L = _lib()
    M, qscale = 300, float(np.float32(0.25 * 1.4426950408889634))
    ld4, ld_vt = 4 * E + 8, (M + 63) // 64 * 64 + 64
    x, hi, lo, B, b = _inproj_operands(family, M, E, 1)
    ys = Yardstick(f'regtr_gemm_tf32x3_qkv_split, E = {E}, {family}')
    c = _plain_inproj(ys, f'{family:10s} M{M} E{E}', x, hi, lo, B, b, family)
    X, Bh, Bl, Bias = _g(x), _g(hi), _g(lo), _g(b)
    outs = []
    for _ in range(2):
        qk4 = torch.full((M, ld4), SENT, dtype=torch.float32, device=DEV)
        vt2 = torch.full((2 * E, ld_vt), SENT, dtype=torch.float32, device=DEV)
        rc = L.regtr_gemm_tf32x3_qkv_split(X.data_ptr(), E, Bh.data_ptr(), Bl.data_ptr(), E, Bias.data_ptr(), M, 3 * E,
                                           E, E, qscale, qk4.data_ptr(), ld4, vt2.data_ptr(), ld_vt, None,
                                           torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc
        outs.append((qk4, vt2))
    torch.cuda.synchronize()
    assert all(torch.equal(p.view(torch.int32), q.view(torch.int32)) for p, q in zip(*outs)), 'two launches differ'
    qk4, vt2 = (_u32(t).view(np.float32) for t in outs[0])
    assert (qk4[:, 4 * E:] == np.float32(SENT)).all() and (vt2[:, M:] == np.float32(SENT)).all(), 'padding written'
    fq = c[:, :E] * np.float32(qscale)
    parts = {'q': (fq, qk4[:, :E], qk4[:, E:2 * E]), 'k': (c[:, E:2 * E], qk4[:, 2 * E:3 * E], qk4[:, 3 * E:4 * E]),
             'v': (c[:, 2 * E:], vt2[:E, :M].T, vt2[E:, :M].T)}
    B64, x64, b64 = torch.from_numpy(B).double(), torch.from_numpy(x).double(), torch.from_numpy(b).double()
    r64 = x64 @ B64.T + b64
    r32 = torch.from_numpy(x) @ torch.from_numpy(B).T + torch.from_numpy(b)
    for sec, (f, h, l) in parts.items():
        wh, wl = go.split_rna(f)
        assert np.array_equal(h.view(np.uint32), wh.view(np.uint32)), f'{sec}: hi is not rna of the fp32 value'
        assert np.array_equal(l.view(np.uint32), wl.view(np.uint32)), f'{sec}: lo is not rna of the remainder'
        _check_split_halves(np.ascontiguousarray(h), np.ascontiguousarray(l), sec)
        cols = slice({'q': 0, 'k': E, 'v': 2 * E}[sec], {'q': E, 'k': 2 * E, 'v': 3 * E}[sec])
        sc = qscale if sec == 'q' else 1.0
        ys.add(f'{family:10s} M{M} E{E} {sec} hi + lo', torch.from_numpy(h.astype(np.float64) + l.astype(np.float64)),
               r32[:, cols] * torch.tensor(sc, dtype=torch.float32), r64[:, cols] * sc)
    _finish(ys)


@pytest.mark.parametrize('E', [32, 96, 256])
def test_qkv_bf16_epilogue(E):
    """regtr_gemm_tf32x3_qkv_bf16: qk (ld_qk > 2E) and the transposed v (ld_vt > M) equal the bf16 RNE of the plain
    GEMM's fp32 value, which meets the yardstick; the padding keeps its sentinel."""
    L = _lib()
    M = 300
    ld_qk, ld_vt = 2 * E + 8, (M + 63) // 64 * 64 + 64
    x, hi, lo, B, b = _inproj_operands('zero_mean', M, E, 2)
    ys = Yardstick(f'regtr_gemm_tf32x3_qkv_bf16, E = {E}')
    c = _plain_inproj(ys, f'zero_mean  M{M} E{E}', x, hi, lo, B, b, 'zero_mean')
    X, Bh, Bl, Bias = _g(x), _g(hi), _g(lo), _g(b)
    sent16 = torch.tensor([SENT], dtype=torch.float32).to(torch.bfloat16)
    outs = []
    for _ in range(2):
        qk = torch.full((M, ld_qk), float(sent16), dtype=torch.bfloat16, device=DEV)
        vt = torch.full((E, ld_vt), float(sent16), dtype=torch.bfloat16, device=DEV)
        rc = L.regtr_gemm_tf32x3_qkv_bf16(X.data_ptr(), E, Bh.data_ptr(), Bl.data_ptr(), E, Bias.data_ptr(), M, 3 * E,
                                          E, 2 * E, qk.data_ptr(), ld_qk, vt.data_ptr(), ld_vt, None,
                                          torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc
        outs.append((qk, vt))
    torch.cuda.synchronize()
    assert all(torch.equal(p.view(torch.int16), q.view(torch.int16)) for p, q in zip(*outs)), 'two launches differ'
    qk, vt = (t.view(torch.int16).cpu().numpy().view(np.uint16) for t in outs[0])
    s16 = sent16.view(torch.int16).numpy().view(np.uint16)[0]
    assert (qk[:, 2 * E:] == s16).all() and (vt[:, M:] == s16).all(), 'padding written'
    assert np.array_equal(qk[:, :2 * E], go.bf16_rne(c[:, :2 * E])), 'q | k is not the bf16 RNE of the fp32 value'
    assert np.array_equal(vt[:, :M], go.bf16_rne(c[:, 2 * E:]).T), 'v^T is not the bf16 RNE of the fp32 value'
    _finish(ys)


def test_qkv_split_rejects_misaligned_bias():
    """The split epilogue reads the bias 16 bytes at a time: a bias view 4 bytes off alignment is refused."""
    L = _lib()
    M, E = 64, 32
    x, hi, lo, _, b = _inproj_operands('zero_mean', M, E, 3)
    X, Bh, Bl = _g(x), _g(hi), _g(lo)
    bias = _padded(b[None], 0, 0.0, offset=True)[0]
    qk4 = torch.zeros((M, 4 * E), dtype=torch.float32, device=DEV)
    vt2 = torch.zeros((2 * E, 128), dtype=torch.float32, device=DEV)
    rc = L.regtr_gemm_tf32x3_qkv_split(X.data_ptr(), E, Bh.data_ptr(), Bl.data_ptr(), E, bias.data_ptr(), M, 3 * E, E,
                                       E, 1.0, qk4.data_ptr(), 4 * E, vt2.data_ptr(), 128, None,
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == -3, rc                                                  # REGTR_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert not qk4.any() and not vt2.any()


# ------------------------------------------------------------------------------------------ regtr_split_tf32

def test_split_tf32_bit_exact():
    """regtr_split_tf32 equals hi = rne(x), lo = rne(x - hi) bit for bit on ties, near-ties, signs, zeros and
    magnitudes from 1e-30 to 1e30; hi + lo differs from x by at most half a TF32 ulp of x - hi (and does differ)."""
    L = _lib()
    rng = np.random.default_rng(11)
    low = np.array([0x0000, 0x0001, 0x0FFF, 0x1000, 0x1001, 0x17FF, 0x1800, 0x1FFF], dtype=np.uint32)
    n = 40000
    u = (rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)) | \
        (rng.integers(127 - 100, 127 + 100, n, dtype=np.uint32) << np.uint32(23)) | \
        (rng.integers(0, 1 << 10, n, dtype=np.uint32) << np.uint32(13)) | rng.choice(low, n)
    x = np.concatenate([u.view(np.float32), rng.normal(size=7001).astype(np.float32) * 10.0 ** rng.uniform(-30, 30, 7001),
                        np.array([0.0, -0.0, 1.0, -1.0, 2.0 ** -20, 3.0], dtype=np.float32)]).astype(np.float32)
    X = _g(x)
    hi, lo = torch.empty_like(X), torch.empty_like(X)
    rc = L.regtr_split_tf32(X.data_ptr(), x.size, hi.data_ptr(), lo.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    gh, gl = _u32(hi), _u32(lo)
    wh, wl = go.split_rne(x)
    assert np.array_equal(gh, wh.view(np.uint32)), 'hi differs from rne(x)'
    assert np.array_equal(gl, wl.view(np.uint32)), 'lo differs from rne(x - hi)'
    d = x.astype(np.float64) - (wh.astype(np.float64) + wl.astype(np.float64))
    rem = (x - wh).astype(np.float32)
    assert (np.abs(d) <= np.where(rem != 0, go.half_ulp_tf32(rem), 0.0)).all()
    assert (d != 0).any(), 'hi + lo = x everywhere: the cases do not exercise the rounding of lo'
