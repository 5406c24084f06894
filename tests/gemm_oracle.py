"""Shared pieces of the 3xTF32 GEMM tests: the library's dispatch rules restated, the TF32 roundings restated on fp32
bit patterns, the input families, and a numpy model of the kernel's arithmetic used to show that the fp32 yardstick
(tests/grad_yardstick.py) separates the shipped design from kernels that are subtly wrong.

The model of `k_gemm_tf32x3_wg` (csrc/gemm_tc.cu): A is split in registers, hi = rna(a), lo = rna(a - hi); B arrives as
the halves of `regtr_split_tf32` (rne).  Each 32-wide k-block is accumulated into a fresh block by 3 MMAs per k-step
of 8 (lo*hi, hi*lo, hi*hi: A half times B half).  An MMA forms its 8 products exactly and adds them to the block one
at a time, each sum truncated to fp32 (the tensor core's accumulation does not round to nearest); the block is then
added to the running sum with a round-to-nearest fp32 add.  A split-K launch runs
that per plane of k-blocks, and the reduction adds the planes in order, then bias, residual and ReLU, in fp32.
The model is a stand-in for the tensor core, not a bit-exact restatement of it.
"""
import numpy as np
import torch

from grad_yardstick import Yardstick

NUM_SMS, BM, BK = 132, 128, 32
MASK = np.uint32(0xFFFFE000)


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------ dispatch restated

def choose_bn(N):
    return 128 if N > 64 else (64 if N > 32 else 32)


def choose_splits(M, N, K):
    """`choose_splits` of csrc/gemm_tc.cu."""
    tiles = cdiv(M, BM) * cdiv(N, choose_bn(N))
    nkb = cdiv(K, BK)
    if tiles >= NUM_SMS // 2 or nkb < 16 or N % 4:
        return 1
    s = min(cdiv(NUM_SMS, tiles), nkb // 8, 8)
    s = min(max(s, cdiv(nkb, 16)), 16)
    return max(s, 1)


def ws_bytes(M, N, K, s):
    return (s * M * N * 4 + 255) // 256 * 256 if s > 1 else 256


def gemm_path(M, N, K):
    """(BN, split count, planes launched, k-blocks per plane) that `regtr_gemm_tf32x3` takes for this shape.  The split
    count is read back from `regtr_gemm_ws_bytes`, s * M * N floats rounded up to 256 bytes (256 bytes when it does not
    split), and must be the restated rule's.  (For M * N < 64 that size can name more than one count; the rule's must
    be among them.)"""
    from regtr_b200 import lib
    ws = int(lib.load().regtr_gemm_ws_bytes(M, N, K))
    read = [s for s in range(1, 17) if ws_bytes(M, N, K, s) == ws]
    s = choose_splits(M, N, K)
    assert s in read, f'M={M} N={N} K={K}: workspace of {ws} B is for {read} planes, the restated rule gives {s}'
    nkb = cdiv(K, BK)
    per = cdiv(nkb, s) if s > 1 else nkb
    return choose_bn(N), s, cdiv(nkb, per), per


# ------------------------------------------------------------------------------------------ TF32 roundings

def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def tf32_rne(x):
    """Round to TF32 (10 mantissa bits), nearest, ties to even: `regtr_tf32_rne` (regtr_split_tf32, weight splits)."""
    u = _bits(x)
    return ((u + np.uint32(0x0FFF) + ((u >> np.uint32(13)) & np.uint32(1))) & MASK).view(np.float32)


def tf32_rna(x):
    """Round to TF32, nearest, ties away from zero: `(bits + 0x1000) & mask`, the in-kernel split of A and the qkv
    epilogues."""
    return ((_bits(x) + np.uint32(0x1000)) & MASK).view(np.float32)


def tf32_trunc(x):
    """The low 13 bits dropped: what a TF32 MMA reads from an fp32 operand that was not split."""
    return (_bits(x) & MASK).view(np.float32)


def split_rne(x):
    x = np.asarray(x, dtype=np.float32)
    hi = tf32_rne(x)
    return hi, tf32_rne(x - hi)


def split_rna(x):
    x = np.asarray(x, dtype=np.float32)
    hi = tf32_rna(x)
    return hi, tf32_rna(x - hi)


def half_ulp_tf32(h):
    """Half a TF32 ulp of each (non-zero, finite) h: 2^(exponent - 11)."""
    e = (_bits(h) >> np.uint32(23)) & np.uint32(0xFF)
    return np.ldexp(1.0, e.astype(np.int64) - 127 - 11)


def bf16_rne(x):
    u = _bits(x).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return u.astype(np.uint16)


# ------------------------------------------------------------------------------------------ input families

FAMILIES = ('zero_mean', 'leaky', 'row_scales')
LEAKY_MU, LEAKY_SLOPE, SHARED_W = 0.35, 0.1, 0.25


def activations(family, M, K, rng):
    """A (M, K) fp32.  zero_mean: N(0, 1).  leaky: LeakyReLU(0.1) of N(0.35, 1), whose mean is 0.8 of its spread, as
    after the encoder's activations.  row_scales: N(0, 1) rows scaled by 10^u, u uniform on [-3, 3] (the first two
    rows exactly 1e-3 and 1e3)."""
    if family == 'leaky':
        z = rng.normal(LEAKY_MU, 1.0, size=(M, K))
        return np.where(z > 0, z, LEAKY_SLOPE * z).astype(np.float32)
    a = rng.normal(size=(M, K))
    if family == 'row_scales':
        s = 10.0 ** rng.uniform(-3, 3, size=M)
        s[:2] = [1e-3, 1e3][:M]
        a = a * s[:, None]
    return a.astype(np.float32)


def weights(family, N, K, rng):
    """W (N, K) fp32, scaled by 1 / sqrt(K); the leaky family's share a positive part, so that one-sided errors in
    the products add up coherently along K."""
    w = rng.normal(size=(N, K))
    if family == 'leaky':
        w = w + SHARED_W
    return (w / np.sqrt(K)).astype(np.float32)


def bias_for(N, rng, scale=1.0):
    return (rng.normal(size=N) * scale).astype(np.float32)


# ------------------------------------------------------------------------------------------ references

def reference(A, B, bias=None, R=None, relu=False, dtype=torch.float64):
    """act(A B^T + bias + R) in `dtype` on the CPU: float64 is the reference, float32 the fp32 restatement."""
    c = torch.as_tensor(np.asarray(A)).to(dtype) @ torch.as_tensor(np.asarray(B)).to(dtype).T
    if bias is not None:
        c = c + torch.as_tensor(np.asarray(bias)).to(dtype)
    if R is not None:
        c = c + torch.as_tensor(np.asarray(R)).to(dtype)
    return torch.relu(c) if relu else c


def row_normalised(*ts, ref):
    """Each row of each tensor divided by the float64 reference row's max |value|, so that rows of 1e-3 weigh as much
    as rows of 1e3 in the max-abs and Frobenius measures."""
    ref = torch.as_tensor(ref).detach().cpu().double()
    s = ref.abs().amax(1, keepdim=True).clamp_min(1e-300)
    return [torch.as_tensor(t).detach().cpu().double() / s for t in ts] + [ref / s]


def add_rows(ys, name, got, fp32, ref, family):
    """One yardstick row, and for the row_scales family a second, per-row-normalised row."""
    ok = ys.add(name, got, fp32, ref)
    if family == 'row_scales':
        g, f, r = row_normalised(got, fp32, ref=ref)
        ok = ys.add(name + ' per-row', g, f, r) and ok
    return ok


# ------------------------------------------------------------------------------------------ kernel model

def _trunc32(x):
    """float64 -> fp32 rounded toward zero."""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def _mma_step(c, prods):
    """c (M, N) fp32 plus the exact products (M, N, 8), one truncating fp32 add each."""
    for j in range(prods.shape[-1]):
        c = _trunc32(c.astype(np.float64) + prods[..., j])
    return c


VARIANTS = ('shipped', 'two_tf32', 'a_unsplit', 'one_chain', 'plane_dropped', 'plane_twice', 'bias_twice', 'scaled')


def emulate(A, B, bias=None, R=None, relu=False, splits=1, variant='shipped'):
    """The model of the kernel (module docstring) on fp32 A (M, K), B (N, K); `variant` names a wrong kernel:
      two_tf32       the lo(A) * hi(B) product dropped
      a_unsplit      A fed to the MMAs as fp32, which they read truncated to TF32, with no lo half
      one_chain      one truncating tensor-core chain over all of K (no per-k-block block, no round-to-nearest add,
                     no split-K)
      plane_dropped  one split-K plane left out of the reduction; plane_twice: one added twice
      bias_twice     the bias added twice
      scaled         the output times (1 + 1e-5)"""
    A = np.asarray(A, np.float32)
    M, K = A.shape
    Kp = cdiv(K, BK) * BK
    Ap = np.zeros((M, Kp), np.float32); Ap[:, :K] = A
    Bp = np.zeros((B.shape[0], Kp), np.float32); Bp[:, :K] = B
    ah, al = split_rna(Ap)
    if variant == 'a_unsplit':
        ah, al = tf32_trunc(Ap), np.zeros_like(Ap)
    bh, bl = split_rne(Bp)
    nks = Kp // 8
    terms = [(al, bh), (ah, bl), (ah, bh)]
    if variant == 'two_tf32':
        terms = terms[1:]
    terms = [(a.astype(np.float64).reshape(M, nks, 8), b.astype(np.float64).reshape(-1, nks, 8)) for a, b in terms]
    nkb = Kp // BK
    per = cdiv(nkb, splits) if splits > 1 and variant != 'one_chain' else nkb
    planes = []
    for k0 in range(0, nkb, per):
        acc = np.zeros((M, B.shape[0]), np.float32)
        blk = acc.copy()
        for kb in range(k0, min(k0 + per, nkb)):
            if variant != 'one_chain':
                blk = np.zeros_like(acc)
            for ks in range(4 * kb, 4 * kb + 4):
                for a, b in terms:
                    blk = _mma_step(blk, a[:, ks, None, :] * b[None, :, ks, :])
            if variant != 'one_chain':
                acc = (acc + blk).astype(np.float32)
        planes.append(blk if variant == 'one_chain' else acc)
    if variant == 'plane_dropped':
        planes.pop(len(planes) // 2)
    elif variant == 'plane_twice':
        planes.insert(len(planes) // 2, planes[len(planes) // 2])
    c = planes[0].copy()
    for p in planes[1:]:
        c = (c + p).astype(np.float32)
    if bias is not None:
        c = c + np.asarray(bias, np.float32)
        if variant == 'bias_twice':
            c = c + np.asarray(bias, np.float32)
    if R is not None:
        c = c + np.asarray(R, np.float32)
    if relu:
        c = np.maximum(c, np.float32(0))
    if variant == 'scaled':
        c = c * np.float32(1 + 1e-5)
    return c.astype(np.float32)


def sharpness_case(family, M, N, K, seed):
    """Operands of one sharpness case: A of `family`, W of `family` given as its TF32 halves' sum (the operand the
    kernel multiplies), a bias of the output's size."""
    rng = np.random.default_rng(seed)
    A = activations(family, M, K, rng)
    hi, lo = split_rne(weights(family, N, K, rng))
    B = hi + lo
    c = reference(A, B)
    bias = bias_for(N, rng, float(c.std()))
    return A, B, bias


def emulation_table(family, M, N, K, seed=0, variants=VARIANTS):
    """Yardstick rows of every emulated kernel on one case; -> the Yardstick."""
    A, B, bias = sharpness_case(family, M, N, K, seed)
    ref, f32 = reference(A, B, bias), reference(A, B, bias, dtype=torch.float32)
    s = choose_splits(M, N, K)
    ys = Yardstick(f'3xTF32 GEMM model, {family}, M={M} N={N} K={K}, {s} split-K planes')
    for v in variants:
        add_rows(ys, v, torch.from_numpy(emulate(A, B, bias, splits=s, variant=v)), f32, ref, family)
    return ys
