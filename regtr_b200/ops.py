"""Torch-tensor front end of the C ABI (one function per entry point of include/regtr_b200.h).

PyTorch is used for device memory and streams only; every operation below runs a
hand-written sm_90a kernel from libregtr_b200.so on the current CUDA stream.
Tensors must live on a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import contextlib
import ctypes
import inspect
import itertools
import math

import numpy as np
import torch

from . import lib as _lib

_ws_cache = {}

# Number of hand-written kernels (libregtr_b200.so, excluding CUB / cuBLAS) launched so far.
LAUNCHES = 0
# Optional profiler hooks (bench.py only): when KPCONV_TRACE is a list, ops.kpconv appends (cuda start event,
# end event, info dict) around every KPConv call; when TRACE is a list, the GEMM / attention-core / gather
# front ends append (kind, info dict, re-launch closure) so that the bench can re-time every launch of one
# forward on its own (L2 flushed) and build per-kernel-family rooflines from the real shapes.
KPCONV_TRACE = None
TRACE = None


def _count(n):
    global LAUNCHES
    LAUNCHES += n


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _chk(t, dtype, name, dims=None):
    if not t.is_cuda:
        raise _lib.RegtrLibError(f'{name}: expected a CUDA tensor (the product path has no CPU fallback)')
    if t.dtype != dtype:
        raise TypeError(f'{name}: expected {dtype}, got {t.dtype}')
    if not t.is_contiguous():
        raise ValueError(f'{name}: must be contiguous')
    if dims is not None and t.dim() != dims:
        raise ValueError(f'{name}: expected {dims}-d tensor, got shape {tuple(t.shape)}')
    return t


# Scratch buffers.  Eager calls share one set per (device, CUDA stream): stream order makes the reuse
# safe and two streams never alias each other's scratch (nor the self-resetting InstanceNorm counters).
# A CUDA-graph capture runs under its own NAMESPACE token (`scratch_namespace`): the raw pointers baked into
# that graph then belong to that graph alone; a buffer that has to grow inside a namespace keeps its
# predecessor alive (`_ws_retired`) because an already captured graph may still write to it, and everything
# is released together with `release_namespace` when the graph is dropped.
WS_NAMESPACE = None
_ws_retired = {}
_ns_counter = itertools.count(1)


def new_namespace():
    return ('graph', next(_ns_counter))


@contextlib.contextmanager
def scratch_namespace(ns):
    global WS_NAMESPACE
    prev, WS_NAMESPACE = WS_NAMESPACE, ns
    try:
        yield ns
    finally:
        WS_NAMESPACE = prev


def release_namespace(ns):
    """Drop every scratch buffer of a namespace (call when its captured graph is destroyed)."""
    for key in [k for k in _ws_cache if k[1] == ns]:
        del _ws_cache[key]
    _ws_retired.pop(ns, None)


def workspace(nbytes: int, device, slot: str = 'default', zero: bool = False) -> torch.Tensor:
    """Per-(device, namespace | stream, slot) grow-only scratch buffer (stream-ordered reuse).
    zero=True: allocated zero-filled (state that an op keeps zero between its own calls)."""
    dev = device.index if device.index is not None else torch.cuda.current_device()
    ns = WS_NAMESPACE if WS_NAMESPACE is not None else ('stream', torch.cuda.current_stream(device).cuda_stream)
    key = (dev, ns, slot)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None and WS_NAMESPACE is not None:
            _ws_retired.setdefault(ns, []).append(buf)      # a captured graph may hold this pointer
        n = max(int(nbytes * 1.25), 4096 if zero else 1 << 20)
        buf = (torch.zeros if zero else torch.empty)(n, dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def regtr_align_up(n, a=256):
    return (n + a - 1) // a * a


def make_offsets(lengths, device) -> torch.Tensor:
    """int32 prefix offsets (n_clouds+1) on `device` from a host list / tensor of lengths."""
    if torch.is_tensor(lengths):
        lengths = lengths.tolist()
    offs = [0]
    for v in lengths:
        offs.append(offs[-1] + int(v))
    return torch.tensor(offs, dtype=torch.int32, device=device)


def new_status(device) -> torch.Tensor:
    return torch.zeros(1, dtype=torch.int32, device=device)


# ---------------------------------------------------------------- pre-processing

def grid_subsample(xyz, offs, n_clouds: int, dl: float, status, out_cap=None, out_offs=None, dense: bool = True):
    """-> (out_xyz (out_cap,3) capacity buffer, out_offs (n_clouds+1) int32).  No host sync.
    out_cap defaults to the input capacity (always sufficient); a smaller value is memory-safe but
    raises REGTR_STATUS_CAPACITY in `status` when the sub-sampled level does not fit.
    dense=True: counting sort over a dense voxel grid (hand-written kernels; raises REGTR_STATUS_GRID in
    `status` when a cloud's bounding box exceeds the cell budget); dense=False: sort-based variant (any extent)."""
    L = _lib.load()
    _chk(xyz, torch.float32, 'xyz', 2); _chk(offs, torch.int32, 'offs', 1)
    n_cap = xyz.shape[0]
    out_cap = n_cap if out_cap is None else int(out_cap)
    out_xyz = torch.empty((out_cap, 3), dtype=torch.float32, device=xyz.device)
    out_offs = torch.empty(n_clouds + 1, dtype=torch.int32, device=xyz.device) if out_offs is None else out_offs
    if dense:
        ws = workspace(L.regtr_grid_subsample_ws_bytes(n_cap, n_clouds), xyz.device)
        state = workspace(L.regtr_grid_subsample_state_bytes(n_cap), xyz.device, 'subsample_state', zero=True)
        _lib.check(L.regtr_grid_subsample(_p(xyz), _p(offs), n_clouds, n_cap, float(dl), _p(out_xyz), out_cap,
                                          _p(out_offs), _p(status), _p(ws), ws.numel(), _p(state), state.numel(),
                                          _stream()), 'regtr_grid_subsample')
        _count(7)
    else:
        ws = workspace(L.regtr_grid_subsample_sorted_ws_bytes(n_cap), xyz.device)
        _lib.check(L.regtr_grid_subsample_sorted(_p(xyz), _p(offs), n_clouds, n_cap, float(dl), _p(out_xyz), out_cap,
                                                 _p(out_offs), _p(status), _p(ws), ws.numel(), _stream()),
                   'regtr_grid_subsample_sorted')
        _count(4)
    return out_xyz, out_offs


class CellGrid:
    """Opaque cell list over a stacked point set (+ the cell-sorted point order)."""

    def __init__(self, xyz, offs, n_clouds: int, cell: float, status):
        L = _lib.load()
        _chk(xyz, torch.float32, 'xyz', 2); _chk(offs, torch.int32, 'offs', 1)
        self.n_cap = xyz.shape[0]
        self.n_clouds = n_clouds
        self.cell = float(cell)
        self.buf = torch.empty(L.regtr_cellgrid_bytes(self.n_cap), dtype=torch.uint8, device=xyz.device)
        self.order = torch.empty(max(self.n_cap, 1), dtype=torch.int32, device=xyz.device)
        ws = workspace(L.regtr_cellgrid_ws_bytes(self.n_cap), xyz.device)
        state = workspace(L.regtr_cellgrid_state_bytes(self.n_cap), xyz.device, 'scan_state', zero=True)
        _lib.check(L.regtr_cellgrid_build(_p(xyz), _p(offs), n_clouds, self.n_cap, self.cell, _p(self.buf),
                                          _p(self.order), _p(status), _p(ws), ws.numel(), _p(state), state.numel(),
                                          _stream()), 'regtr_cellgrid_build')
        _count(4)


def ball_query(q, q_offs, s, s_offs, grid: CellGrid, K: int, radius: float, q_order=None,
               want32=True, want64=True):
    """First-K-in-index-order radius search.  -> (idx32 or None, idx64 or None), shape (nq_cap,K)."""
    L = _lib.load()
    _chk(q, torch.float32, 'q', 2); _chk(s, torch.float32, 's', 2)
    nq_cap = q.shape[0]
    if grid.n_cap != s.shape[0]:
        raise ValueError('grid was built over a different support capacity')
    if grid.cell < float(radius):
        raise ValueError('grid cell must be >= radius')
    i32 = torch.empty((nq_cap, K), dtype=torch.int32, device=q.device) if want32 else None
    i64 = torch.empty((nq_cap, K), dtype=torch.int64, device=q.device) if want64 else None
    _lib.check(L.regtr_ball_query(_p(q), _p(q_offs), _p(q_order), _p(s), _p(s_offs), _p(grid.buf), grid.n_clouds,
                                  nq_cap, s.shape[0], int(K), float(radius), _p(i32), _p(i64), _stream()),
               'regtr_ball_query')
    _count(1)
    return i32, i64


# ------------------------------------------------------------------------ encoder

def kpconv(q_pts, s_pts, idx32, x, weights, kernel_points, extent: float, out=None, nq_dev=None, ns_dev=None,
           row_flags=None, instats=None):
    """KPConv.forward (rigid / linear / sum).  idx32 (Nq,K) int32, x (Ns,Cin) -> (Nq,Cout).
    nq_dev / ns_dev: optional 1-element int32 device tensors with the actual counts when the
    leading dimensions are capacities.
    Differentiable with respect to x and weights (_KPConvFn) when grad mode is on and either requires grad (exact
    shapes only); kernel_points and the coordinates carry no gradient."""
    if _wants_grad(x, weights):
        if out is not None or nq_dev is not None or ns_dev is not None:
            raise ValueError('kpconv: the backward needs exact shapes (no out / nq_dev / ns_dev)')
        out, stats = _KPConvFn.apply(x, weights, q_pts, s_pts, idx32, kernel_points, float(extent), row_flags, instats)
        return out if instats is None else (out, stats)
    return _kpconv_fwd(q_pts, s_pts, idx32, x, weights, kernel_points, extent, out, nq_dev, ns_dev, row_flags, instats)


def _kpconv_fwd(q_pts, s_pts, idx32, x, weights, kernel_points, extent: float, out=None, nq_dev=None, ns_dev=None,
                row_flags=None, instats=None):
    L = _lib.load()
    _chk(q_pts, torch.float32, 'q_pts', 2); _chk(s_pts, torch.float32, 's_pts', 2)
    _chk(idx32, torch.int32, 'neighb_inds', 2); _chk(x, torch.float32, 'x', 2)
    _chk(weights, torch.float32, 'weights', 3); _chk(kernel_points, torch.float32, 'kernel_points', 2)
    Nq, K = idx32.shape
    Ns, Cin = x.shape
    P, Cin_w, Cout = weights.shape
    if P != 15 or kernel_points.shape != (15, 3) or Cin_w != Cin or q_pts.shape[0] != Nq or s_pts.shape[0] != Ns:
        raise ValueError('kpconv: inconsistent shapes')
    out = torch.empty((Nq, Cout), dtype=torch.float32, device=x.device) if out is None else out
    stats = None
    if instats is not None and (Cin == 1 or Cout % 32):
        raise ValueError('kpconv: the statistics epilogue needs Cin > 1 and Cout % 32 == 0')
    nb = L.regtr_kpconv_fwd_ws_bytes(Nq, Ns, Cin, Cout) if Cin == 1 else L.regtr_kpconv_ws_bytes(Nq, Ns, Cin)
    ws = workspace(nb, x.device, 'kpconv')
    trace = KPCONV_TRACE
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)] if trace is not None else None
    if ev:
        ev[0].record()
    if Cin == 1:
        # first block: gather + aggregation + the 15 x Cout contraction in one kernel (k_kpconv_c1)
        _lib.check(L.regtr_kpconv_fwd(_p(q_pts), _p(s_pts), _p(idx32), _p(x), _p(weights), _p(kernel_points), Nq, Ns,
                                      _p(nq_dev), _p(ns_dev), K, Cin, Cout, float(extent), _p(out), _p(ws),
                                      ws.numel(), _stream()), 'regtr_kpconv_fwd')
        _count(1)
    else:
        # gather/aggregate kernel, then the [Nq,15Cin] x [15Cin,Cout] contraction on the tensor cores
        if (15 * Cin) % 4:
            raise _lib.RegtrLibError(f'kpconv: Cin={Cin} breaks the 16-byte row pitch of the contraction (no fallback)')
        wf = ws[:Nq * 15 * Cin * 4].view(torch.float32).view(Nq, 15 * Cin)
        flags = row_flags if row_flags is not None else ws[regtr_align_up(Nq * 15 * Cin * 4):]
        _lib.check(L.regtr_kpconv_aggregate(_p(q_pts), _p(s_pts), _p(idx32), _p(x), _p(kernel_points), Nq, Ns,
                                            _p(nq_dev), _p(ns_dev), K, Cin, float(extent), _p(wf), _p(flags),
                                            1 if row_flags is not None else 0, _stream()), 'regtr_kpconv_aggregate')
        _count(1 if row_flags is not None else 2)
        hi, lo = split_weight(weights.view(15 * Cin, Cout), transpose=True)
        if ev:
            ev[1].record()
            ev.append(True)
        if instats is not None:                 # (offs, n_clouds): statistics of the output in the GEMM epilogue
            out, stats = gemm_instats(wf, hi, lo, instats[0], instats[1], m_dev=nq_dev, out=out)
        else:
            gemm(wf, hi, lo, m_dev=nq_dev, out=out)
    if ev:
        ev[2].record()
        trace.append((ev[0], ev[2], dict(Nq=Nq, Ns=Ns, K=K, Cin=Cin, Cout=Cout, idx=idx32,
                                         mid=ev[1] if len(ev) > 3 else None,
                                         args=(q_pts, s_pts, idx32, x, kernel_points, float(extent)),
                                         row_flags=row_flags)))
    return out if instats is None else (out, stats)


def kpconv_aggregate(q_pts, s_pts, idx32, x, kernel_points, extent: float, wf=None, nq_dev=None, ns_dev=None,
                     row_flags=None):
    """Gather + influence + aggregation only: -> wf (Nq, 15*Cin) (already / neighbour count)."""
    L = _lib.load()
    Nq, K = idx32.shape
    Ns, Cin = x.shape
    wf = torch.empty((Nq, 15 * Cin), dtype=torch.float32, device=x.device) if wf is None else wf
    flags = row_flags if row_flags is not None else workspace(max(Ns, 1), x.device, 'rowflags')
    _lib.check(L.regtr_kpconv_aggregate(_p(q_pts), _p(s_pts), _p(idx32), _p(x), _p(kernel_points), Nq, Ns,
                                        _p(nq_dev), _p(ns_dev), K, Cin, float(extent), _p(wf), _p(flags),
                                        1 if row_flags is not None else 0, _stream()), 'regtr_kpconv_aggregate')
    _count(1 if (row_flags is not None or Cin == 1) else 2)
    return wf


def max_pool(x, idx32, ns_dev=None):
    """max over the K gathered rows with a zero shadow row.  Differentiable (_MaxPoolFn) when grad mode is on and x
    requires grad (exact shapes only)."""
    if _wants_grad(x):
        if ns_dev is not None:
            raise ValueError('max_pool: the backward needs exact shapes (no ns_dev)')
        return _MaxPoolFn.apply(x, idx32)
    return _max_pool_fwd(x, idx32, ns_dev)


def _max_pool_fwd(x, idx32, ns_dev=None):
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2); _chk(idx32, torch.int32, 'inds', 2)
    Nq, K = idx32.shape
    out = torch.empty((Nq, x.shape[1]), dtype=torch.float32, device=x.device)
    _lib.check(L.regtr_max_pool(_p(x), _p(idx32), Nq, x.shape[0], _p(ns_dev), K, x.shape[1], _p(out), _stream()),
               'regtr_max_pool')
    _count(1)
    return out


def instnorm_act(x, offs, n_clouds: int, res=None, slope: float = -1.0, eps: float = 1e-5, out=None,
                 want_flags: bool = False):
    """out = act(InstanceNorm_per_cloud(x) + res); slope < 0 -> no activation.
    want_flags: also return the per-row `sum > 0` flags the consuming KPConv needs (uint8, n rows).
    Differentiable with respect to x and res (_InstNormFn) when grad mode is on and either requires grad."""
    if _wants_grad(x, res):
        if out is not None:
            raise ValueError('instnorm_act: no out= on the differentiable path')
        y, flags = _InstNormFn.apply(x, res, None, offs, n_clouds, float(slope), float(eps), bool(want_flags))
        return (y, flags) if want_flags else y
    return _instnorm_act_fwd(x, offs, n_clouds, res, slope, eps, out, want_flags)


def _instnorm_act_fwd(x, offs, n_clouds: int, res=None, slope: float = -1.0, eps: float = 1e-5, out=None,
                      want_flags: bool = False):
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2); _chk(offs, torch.int32, 'offs', 1)
    n, C = x.shape
    if res is not None:
        _chk(res, torch.float32, 'res', 2)
    out = torch.empty_like(x) if out is None else out
    nb = L.regtr_instnorm_ws_bytes(n, n_clouds, C)
    ws = workspace(nb, x.device, 'instnorm')
    flags = None
    if want_flags and C // 4 <= 32 and (C // 4) & (C // 4 - 1) == 0:
        flags = torch.empty(max(n, 1), dtype=torch.uint8, device=x.device)
    # self-resetting completion counters: the last statistics block of a (cloud, channel tile) finalises it
    cnt = workspace(L.regtr_instnorm_counter_bytes(n_clouds, C), x.device, 'instnorm_cnt', zero=True)
    _lib.check(L.regtr_instnorm_act(_p(x), _p(offs), n_clouds, n, C, float(eps), _p(res), float(slope), _p(out),
                                    _p(flags), _p(ws), ws.numel(), _p(cnt), _stream()), 'regtr_instnorm_act')
    _count(2)
    return (out, flags) if want_flags else out


def instnorm_apply(x, offs, n_clouds: int, stats, res=None, slope: float = -1.0, out=None, want_flags: bool = False,
                   eps: float = 1e-5):
    """Apply pass of the per-cloud InstanceNorm with statistics from `gemm_instats`:
    out = act((x - mean) * rstd + res).  Differentiable with respect to x and res (_InstNormFn) when grad mode is on
    and either requires grad: the statistics are functions of x, and the backward recomputes them from x (`eps` must
    be the one they were computed with)."""
    if _wants_grad(x, res):
        if out is not None:
            raise ValueError('instnorm_apply: no out= on the differentiable path')
        y, flags = _InstNormFn.apply(x, res, stats, offs, n_clouds, float(slope), float(eps), bool(want_flags))
        return (y, flags) if want_flags else y
    return _instnorm_apply_fwd(x, offs, n_clouds, stats, res, slope, out, want_flags)


def _instnorm_apply_fwd(x, offs, n_clouds: int, stats, res=None, slope: float = -1.0, out=None,
                        want_flags: bool = False):
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2); _chk(offs, torch.int32, 'offs', 1); _chk(stats, torch.float32, 'stats', 3)
    n, C = x.shape
    out = torch.empty_like(x) if out is None else out
    flags = None
    if want_flags and C // 4 <= 32 and (C // 4) & (C // 4 - 1) == 0:
        flags = torch.empty(max(n, 1), dtype=torch.uint8, device=x.device)
    _lib.check(L.regtr_instnorm_apply(_p(x), _p(offs), n_clouds, n, C, _p(stats), _p(res), float(slope), _p(out),
                                      _p(flags), _stream()), 'regtr_instnorm_apply')
    _count(1)
    return (out, flags) if want_flags else out


# -------------------------------------------------------------------- dense layers

def split_weight(w: torch.Tensor, transpose: bool = False):
    """(hi, lo) TF32 halves of a weight matrix [N,K] (or of its transpose).  Cached ON the owning
    parameter object (so the cache dies with the model and can never alias a recycled address),
    keyed by view geometry and the parameter's version counter: inference pays the split once."""
    L = _lib.load()
    owner = w._base if w._base is not None else w
    cache = owner.__dict__.setdefault('_regtr_split', {})
    key = (w.storage_offset(), tuple(w.shape), tuple(w.stride()), transpose, owner._version)
    hit = cache.get(key)
    if hit is not None:
        return hit
    src = (w.detach().t() if transpose else w.detach()).contiguous().to(torch.float32)
    hi, lo = torch.empty_like(src), torch.empty_like(src)
    _lib.check(L.regtr_split_tf32(_p(src), src.numel(), _p(hi), _p(lo), _stream()), 'regtr_split_tf32')
    _count(1)
    for k in [k for k in cache if k[-1] != owner._version]:
        del cache[k]
    cache[key] = (hi, lo)
    return hi, lo


def gemm(a, b_hi, b_lo, bias=None, residual=None, relu=False, m_dev=None, out=None):
    """act(a @ B^T + bias + residual) with B = b_hi + b_lo ([N,K] row-major), 3xTF32 wgmma kernel."""
    L = _lib.load()
    if not a.is_cuda or a.dtype != torch.float32 or a.dim() != 2 or a.stride(1) != 1:
        raise ValueError('gemm: A must be a CUDA fp32 matrix with unit column stride')
    M, K = a.shape
    N = b_hi.shape[0]
    out = torch.empty((M, N), dtype=torch.float32, device=a.device) if out is None else out
    nb = L.regtr_gemm_ws_bytes(M, N, K)
    ws = workspace(nb, a.device, 'gemm')
    if TRACE is not None:
        TRACE.append(('gemm', dict(M=M, N=N, K=K, split_k=nb > 256),
                      lambda: gemm(a, b_hi, b_lo, bias=bias, residual=residual, relu=relu, m_dev=m_dev, out=out)))
    _lib.check(L.regtr_gemm_tf32x3(_p(a), a.stride(0), _p(b_hi), _p(b_lo), b_hi.stride(0), _p(out), out.stride(0),
                                   _p(bias), _p(residual), residual.stride(0) if residual is not None else 0,
                                   M, N, K, _p(m_dev), 1 if relu else 0, _p(ws), ws.numel(), _stream()),
               'regtr_gemm_tf32x3')
    _count(2 if nb > 256 else 1)
    return out


def gemm_instats(a, b_hi, b_lo, offs, n_clouds: int, eps: float = 1e-5, m_dev=None, out=None):
    """a @ B^T plus the per-cloud InstanceNorm statistics of the result: 32-row partial sums from the GEMM
    epilogue + a small fixed-order finalisation (no atomics).  -> (out (M,N), stats (n_clouds, N, 2) = (mean, rstd))."""
    L = _lib.load()
    if not a.is_cuda or a.dtype != torch.float32 or a.dim() != 2 or a.stride(1) != 1:
        raise ValueError('gemm: A must be a CUDA fp32 matrix with unit column stride')
    M, K = a.shape
    N = b_hi.shape[0]
    out = torch.empty((M, N), dtype=torch.float32, device=a.device) if out is None else out
    stats = torch.empty((n_clouds, N, 2), dtype=torch.float32, device=a.device)
    nb = L.regtr_gemm_ws_bytes(M, N, K)
    ws = workspace(nb, a.device, 'gemm')
    acc = workspace(L.regtr_instnorm_part_bytes(M, N), a.device, 'instnorm_part')
    if TRACE is not None:
        TRACE.append(('gemm', dict(M=M, N=N, K=K, split_k=nb > 256, instats=True),
                      lambda: gemm_instats(a, b_hi, b_lo, offs, n_clouds, eps, m_dev=m_dev, out=out)))
    _lib.check(L.regtr_gemm_tf32x3_instats(_p(a), a.stride(0), _p(b_hi), _p(b_lo), b_hi.stride(0), _p(out), out.stride(0),
                                           M, N, K, _p(m_dev), _p(offs), n_clouds, float(eps), _p(acc), _p(stats),
                                           _p(ws), ws.numel(), _stream()), 'regtr_gemm_tf32x3_instats')
    _count(3 if nb > 256 else 2)
    return out, stats


def linear_instats(x, weight, offs, n_clouds: int, eps: float = 1e-5, m_dev=None, skip: bool = False):
    """nn.Linear(bias=False) followed by InstanceNorm statistics (UnaryBlock, kpconv_blocks.py:546-561).
    Differentiable with respect to x and weight (_LinearInstatsFn) when grad mode is on and either requires grad.
    skip=True also returns x itself as a third output, for the block's shortcut branch: its gradient then reaches the
    dX GEMM as a residual and is added in the epilogue, so x has one consumer in the autograd graph."""
    if _wants_grad(x, weight):
        if m_dev is not None:
            raise ValueError('linear_instats: the backward needs exact shapes (no m_dev)')
        y, stats, xs = _LinearInstatsFn.apply(x, weight, offs, n_clouds, float(eps), bool(skip))
        return (y, stats, xs) if skip else (y, stats)
    y, stats = _linear_instats_fwd(x, weight, offs, n_clouds, eps, m_dev)
    return (y, stats, x) if skip else (y, stats)


def _linear_instats_fwd(x, weight, offs, n_clouds: int, eps: float = 1e-5, m_dev=None):
    if x.shape[1] % 4 or x.stride(0) % 4 or x.data_ptr() % 16:
        raise _lib.RegtrLibError(f'linear: K={x.shape[1]}: rows must be 16-byte aligned multiples of 4 floats')
    hi, lo = split_weight(weight)
    return gemm_instats(x, hi, lo, offs, n_clouds, eps, m_dev=m_dev)


def _wants_grad(*ts):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def linear(x, weight, bias=None, residual=None, relu=False, m_dev=None, drop=None):
    """nn.Linear forward (x @ weight^T + bias) (+ residual, + ReLU) on the 3xTF32 wgmma GEMM of this
    library.  The TMA row pitch needs K % 4 == 0 and 16-byte aligned rows; anything else raises (callers
    with an odd K zero-pad it, see PositionEmbeddingLearned) -- there is no library fallback.
    Differentiable (_LinearFn) when grad mode is on and an input requires grad (exact shapes only).
    drop (a dropout site, training): dropout(relu(x W^T + b)) of the feed-forward block (site 5), the mask applied in
    place after the GEMM; it needs relu=True and no residual."""
    if drop is not None and (residual is not None or not relu):
        raise ValueError('linear: the feed-forward dropout follows a ReLU and takes no residual')
    if _wants_grad(x, weight, bias, residual):
        if m_dev is not None:
            raise ValueError('linear: the backward needs exact shapes (no m_dev)')
        return _LinearFn.apply(x, weight, bias, residual, bool(relu), drop)
    out = _linear_fwd(x, weight, bias, residual, relu, m_dev)
    return out if drop is None else dropout_rows_(out, drop)


def _linear_fwd(x, weight, bias=None, residual=None, relu=False, m_dev=None):
    if x.shape[1] % 4 or x.stride(0) % 4 or x.data_ptr() % 16:
        raise _lib.RegtrLibError(f'linear: K={x.shape[1]}, row stride {x.stride(0)}: rows must be 16-byte '
                                 'aligned multiples of 4 floats (zero-pad K); no cuBLAS fallback')
    hi, lo = split_weight(weight)
    return gemm(x, hi, lo, bias=bias, residual=residual, relu=relu, m_dev=m_dev)


# -------------------------------------------------------------------- transformer

_dim_t_cache = {}


def sine_dim_t(n_freq: int, temperature: float, device):
    """The reference's frequency table, computed with the same torch fp32 ops
    (position_embedding.py:39-40) and cached per device."""
    key = (n_freq, float(temperature), str(device))
    if key not in _dim_t_cache:
        d = torch.arange(n_freq, dtype=torch.float32)
        d = temperature ** (2 * torch.div(d, 2, rounding_mode='trunc') / n_freq)
        _dim_t_cache[key] = d.to(device)
    return _dim_t_cache[key]


def pos_embed_sine(xyz, d_model: int = 256, temperature: float = 10000.0, scale: float = 1.0):
    L = _lib.load()
    _chk(xyz, torch.float32, 'xyz', 2)
    n, n_dim = xyz.shape
    if n_dim != 3:
        raise ValueError('pos_embed_sine: only 3-D coordinates are on the hot path')
    n_freq = d_model // n_dim // 2 * 2
    out = torch.empty((n, d_model), dtype=torch.float32, device=xyz.device)
    s32 = torch.tensor(scale * 2 * math.pi, dtype=torch.float32).item()
    _lib.check(L.regtr_pos_embed_sine(_p(xyz), n, _p(sine_dim_t(n_freq, temperature, xyz.device)), n_freq, d_model,
                                      s32, _p(out), _stream()), 'regtr_pos_embed_sine')
    _count(1)
    return out


def layernorm_pos(x, gamma, beta, pos=None, eps: float = 1e-5, want_plain=True, want_pos=True, n_dev=None,
                  skip=False, z=None, drop=None):
    """-> (LN(x), LN(x)+pos); either may be skipped.  n_dev: device row count when x is capacity-shaped.
    Differentiable (_LayerNormPosFn) when grad mode is on and an input requires grad.  skip=True (training path)
    also returns x itself as a third output, for the residual connection that adds x back: its gradient then reaches
    the LayerNorm backward as `dres` and is added there, so x has one consumer in the autograd graph.
    z, drop (a dropout site, training): the residual dropout (site 2, 4 or 6) of a branch z (the out-projection or
    linear2 output, computed without residual=) fused into this LayerNorm: -> (LN(x'), LN(x')+pos, x') with
    x' = x + m * scale * z, one launch."""
    skip = bool(skip) or drop is not None
    if _wants_grad(x, gamma, beta, z):
        if n_dev is not None:
            raise ValueError('layernorm_pos: the backward needs exact shapes (no n_dev)')
        outs = _LayerNormPosFn.apply(x, gamma, beta, pos, float(eps), bool(want_plain), bool(want_pos), skip, z, drop)
        return outs if skip else outs[:2]
    outs = _layernorm_pos_fwd(x, gamma, beta, pos, eps, want_plain, want_pos, n_dev, z, drop)
    return outs if skip else outs[:2]


def _layernorm_pos_fwd(x, gamma, beta, pos=None, eps: float = 1e-5, want_plain=True, want_pos=True, n_dev=None,
                       z=None, drop=None):
    """-> (y, y_pos, x'), x' = x without a dropout site."""
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2)
    n, E = x.shape
    y = torch.empty_like(x) if want_plain else None
    yp = torch.empty_like(x) if want_pos else None
    offs = xo = dp = None
    if drop is not None:
        _chk(z, torch.float32, 'z', 2)
        if z.shape != x.shape:
            raise ValueError('layernorm_pos: x and z must have the same shape')
        offs, xo, dp = drop.key.offs, torch.empty_like(x), drop.ptr
    _lib.check(L.regtr_layernorm_pos(_p(x), _p(z), _p(gamma), _p(beta), _p(pos), n, _p(n_dev), _p(offs), E, float(eps),
                                     _p(y), _p(yp), _p(xo), dp, _stream()), 'regtr_layernorm_pos')
    _count(1)
    return y, yp, (x if xo is None else xo)


def attention_plan(offs, B: int):
    """Device-side (6, 2B + 1) int32 table: q_start, q_len, cross k_start, cross k_len, then the exclusive prefixes
    of the 64- and 128-query tile counts per problem (entry 2B = total).  No host sync."""
    L = _lib.load()
    _chk(offs, torch.int32, 'offs', 1)
    plan = torch.empty((6, 2 * B + 1), dtype=torch.int32, device=offs.device)
    _lib.check(L.regtr_attention_plan(_p(offs), B, _p(plan), _stream()), 'regtr_attention_plan')
    _count(1)
    return plan


def corr_decode(qp, kp, xyz, q_start, q_len, k_start, k_len, max_q_len: int, n_layers: int, out=None):
    """CorrespondenceDecoder.simple_attention for all decoder layers: qp/kp (n_layers*N, D) projected
    queries / keys, xyz (N,3) -> (n_layers*N, 3) attention-weighted key coordinates."""
    L = _lib.load()
    _chk(qp, torch.float32, 'qp', 2); _chk(kp, torch.float32, 'kp', 2); _chk(xyz, torch.float32, 'xyz', 2)
    rows, D = qp.shape
    N = xyz.shape[0]
    if kp.shape != qp.shape or rows != n_layers * N or qp.stride(0) != kp.stride(0) or qp.stride(1) != 1:
        raise ValueError('corr_decode: inconsistent shapes')
    out = torch.zeros((rows, 3), dtype=torch.float32, device=qp.device) if out is None else out
    _lib.check(L.regtr_corr_decode_fwd(_p(qp), _p(kp), qp.stride(0), _p(xyz.contiguous()), _p(out), _p(q_start),
                                       _p(q_len), _p(k_start), _p(k_len), int(q_start.numel()), int(max_q_len),
                                       int(n_layers), N, D, 1.0 / math.sqrt(D), _stream()), 'regtr_corr_decode_fwd')
    _count(1)
    return out


def mha_varlen(q, k, v, q_start, q_len, k_start, k_len, max_q_len: int, n_heads: int, out=None, tiles=None):
    """softmax(q k^T / sqrt(dh)) v per head over explicit (query range, key range) problems.
    q/k/v may be column slices of a wider row-major matrix (stride(0) is the leading dim)."""
    L = _lib.load()
    for t, nm in ((q, 'q'), (k, 'k'), (v, 'v')):
        if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
            raise ValueError(f'mha_varlen: {nm} must be a CUDA fp32 matrix with unit column stride')
    E = q.shape[1]
    dh = E // n_heads
    # rows outside every problem (capacity padding) stay uninitialised: every consumer is row-wise and skips them
    out = torch.empty((q.shape[0], E), dtype=torch.float32, device=q.device) if out is None else out
    if TRACE is not None:
        ql, kl = q_len.tolist(), k_len.tolist()
        TRACE.append(('mha', dict(pairs_qk=sum(a * b for a, b in zip(ql, kl)), E=E, tokens=sum(ql)),
                      lambda: mha_varlen(q, k, v, q_start, q_len, k_start, k_len, max_q_len, n_heads, out=out, tiles=tiles)))
    tb, mt = (tiles[0], int(tiles[1])) if tiles is not None else (None, 0)     # (device tile table, host bound)
    _lib.check(L.regtr_mha_varlen_fwd(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(out),
                                      out.stride(0), None, _p(q_start), _p(q_len), _p(k_start), _p(k_len),
                                      q_start.numel(), int(max_q_len), _p(tb), mt, n_heads, dh, 1.0 / math.sqrt(dh),
                                      None, _stream()), 'regtr_mha_varlen_fwd')
    _count(1)
    return out


def mha_probs_avg(q, k, out, p_offset, p_pitch, q_start, q_len, k_start, k_len, max_q_len: int, n_heads: int):
    """Head-averaged attention probabilities (1/H) sum_h softmax(q_h k_h^T / sqrt(dh)) of every (query range, key
    range) problem, written into `out` (flat fp32): problem p's block at p_offset[p] (int64) with row pitch p_pitch[p]
    (int32).  Elements outside every block are not written.  q / k may be column slices of a wider matrix."""
    L = _lib.load()
    for t, nm in ((q, 'q'), (k, 'k')):
        if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
            raise ValueError(f'mha_probs_avg: {nm} must be a CUDA fp32 matrix with unit column stride')
    _chk(out, torch.float32, 'out'); _chk(p_offset, torch.int64, 'p_offset', 1); _chk(p_pitch, torch.int32, 'p_pitch', 1)
    E = q.shape[1]
    dh = E // n_heads
    n_prob = q_start.numel()
    if p_offset.numel() != n_prob or p_pitch.numel() != n_prob:
        raise ValueError('mha_probs_avg: one output offset and pitch per problem')

    def launch():
        return L.regtr_mha_probs_avg(_p(q), q.stride(0), _p(k), k.stride(0), _p(out), _p(p_offset), _p(p_pitch),
                                     _p(q_start), _p(q_len), _p(k_start), _p(k_len), n_prob, int(max_q_len),
                                     n_heads, dh, 1.0 / math.sqrt(dh), _stream())
    if TRACE is not None:
        ql, kl = q_len.tolist(), k_len.tolist()
        TRACE.append(('mha_probs', dict(pairs_qk=sum(a * b for a, b in zip(ql, kl)), E=E, tokens=sum(ql)), launch))
    _lib.check(launch(), 'regtr_mha_probs_avg')
    _count(1)
    return out


def mha_bf16_tc(x, in_w, in_b, q_start, q_len, k_start, k_len, max_q_len: int, n_heads: int, m_dev=None):
    """Attention block core in the fast precision mode: packed in-projection (3xTF32 GEMM, bf16
    epilogue) + wgmma bf16 attention.  x (N,E) fp32 (already LN + pos); returns O (N,E) fp32."""
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2)
    N, E = x.shape
    dh = E // n_heads
    hi, lo = split_weight(in_w)
    ld_vt = (N + 63) // 64 * 64 + 64            # token pitch of the transposed V (TMA: 16-byte multiple)
    qk = torch.empty((N, 2 * E), dtype=torch.bfloat16, device=x.device)
    vt = torch.zeros((E, ld_vt), dtype=torch.bfloat16, device=x.device)
    _lib.check(L.regtr_gemm_tf32x3_qkv_bf16(_p(x), x.stride(0), _p(hi), _p(lo), hi.stride(0), _p(in_b), N, 3 * E, E,
                                            2 * E, _p(qk), 2 * E, _p(vt), ld_vt, _p(m_dev), _stream()),
               'regtr_gemm_tf32x3_qkv_bf16')
    out = torch.zeros((N, E), dtype=torch.float32, device=x.device)
    _lib.check(L.regtr_mha_bf16_tc_fwd(_p(qk), 2 * E, _p(vt), ld_vt, N, _p(out), E, _p(q_start), _p(q_len),
                                       _p(k_start), _p(k_len), q_start.numel(), int(max_q_len), n_heads, dh,
                                       1.0 / math.sqrt(dh), _stream()), 'regtr_mha_bf16_tc_fwd')
    _count(2)
    return out


def mha_tf32_tc(x, in_w, in_b, q_start, q_len, k_start, k_len, max_q_len: int, n_heads: int, m_dev=None, tiles=None):
    """Attention block core, fp32-accurate, on the Hopper tensor cores: packed in-projection (3xTF32 GEMM whose
    epilogue writes q / k / v^T as TF32 (hi, lo) halves) + the TMA-fed 3xTF32 attention kernel (P in registers).
    x (N,E) fp32 (already LN + pos); returns O (N,E) fp32."""
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2)
    N, E = x.shape
    dh = E // n_heads
    hi, lo = split_weight(in_w)
    ld_vt = (N + 63) // 64 * 64 + 64            # token pitch of the transposed V (16-byte multiple, tile over-read)
    qk4 = torch.empty((N, 4 * E), dtype=torch.float32, device=x.device)
    vt2 = torch.zeros((2 * E, ld_vt), dtype=torch.float32, device=x.device)     # padding tokens must stay finite
    qscale = (1.0 / math.sqrt(dh)) * 1.4426950408889634
    _lib.check(L.regtr_gemm_tf32x3_qkv_split(_p(x), x.stride(0), _p(hi), _p(lo), hi.stride(0), _p(in_b), N, 3 * E, E, E,
                                             float(qscale), _p(qk4), 4 * E, _p(vt2), ld_vt, _p(m_dev), _stream()),
               'regtr_gemm_tf32x3_qkv_split')
    out = torch.empty((N, E), dtype=torch.float32, device=x.device)
    tb, mt = (tiles[0], int(tiles[1])) if tiles is not None else (None, 0)
    if TRACE is not None:
        ql, kl = q_len.tolist(), k_len.tolist()
        TRACE.append(('gemm', dict(M=N, N=3 * E, K=E, split_k=False, qkv_split=True), lambda: L.regtr_gemm_tf32x3_qkv_split(
            _p(x), x.stride(0), _p(hi), _p(lo), hi.stride(0), _p(in_b), N, 3 * E, E, E, float(qscale), _p(qk4), 4 * E,
            _p(vt2), ld_vt, _p(m_dev), _stream())))
        TRACE.append(('mha', dict(pairs_qk=sum(a * b for a, b in zip(ql, kl)), E=E, tokens=sum(ql)),
                      lambda: L.regtr_mha_tf32_tc_fwd(_p(qk4), 4 * E, _p(vt2), ld_vt, N, _p(out), E, _p(q_start), _p(q_len),
                                                      _p(k_start), _p(k_len), q_start.numel(), int(max_q_len), _p(tb), mt,
                                                      n_heads, dh, _stream())))
    _lib.check(L.regtr_mha_tf32_tc_fwd(_p(qk4), 4 * E, _p(vt2), ld_vt, N, _p(out), E, _p(q_start), _p(q_len),
                                       _p(k_start), _p(k_len), q_start.numel(), int(max_q_len), _p(tb), mt, n_heads, dh,
                                       _stream()), 'regtr_mha_tf32_tc_fwd')
    _count(2)
    return out


def mha_varlen_lse(q, k, v, q_start, q_len, k_start, k_len, max_q_len: int, n_heads: int, drop=None):
    """Training forward of `mha_varlen` (the default 3xTF32 core): -> (O (N,E), lse (N, n_heads)), lse the base-2
    log-sum-exp of the scaled scores that `mha_varlen_bwd` recomputes the softmax from.  drop (a dropout site,
    site 1 or 3): the attention-probability dropout (problem c = local query cloud c)."""
    L = _lib.load()
    for t, nm in ((q, 'q'), (k, 'k'), (v, 'v')):
        if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
            raise ValueError(f'mha_varlen: {nm} must be a CUDA fp32 matrix with unit column stride')
    E = q.shape[1]
    dh = E // n_heads
    out = torch.empty((q.shape[0], E), dtype=torch.float32, device=q.device)
    lse = torch.empty((q.shape[0], n_heads), dtype=torch.float32, device=q.device)
    _lib.check(L.regtr_mha_varlen_fwd(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(out),
                                      out.stride(0), _p(lse), _p(q_start), _p(q_len), _p(k_start), _p(k_len),
                                      q_start.numel(), int(max_q_len), None, 0, n_heads, dh, 1.0 / math.sqrt(dh),
                                      None if drop is None else drop.ptr, _stream()), 'regtr_mha_varlen_fwd')
    _count(1)
    return out, lse


def mha_varlen_bwd(q, k, v, o, lse, d_o, dq, dk, dv, q_start, q_len, k_start, k_len, max_q_len: int, max_k_len: int,
                   n_heads: int, drop=None):
    """Backward of the attention core: writes dq / dk / dv (views of the caller's buffers, e.g. column slices of one
    packed [N, 3E] gradient).  Every key row must lie in the key range of exactly one problem.  drop: the forward's
    dropout site."""
    L = _lib.load()
    _chk(d_o, torch.float32, 'dO', 2)
    E = q.shape[1]
    dh = E // n_heads
    n_rows = q.shape[0]
    ws = workspace(L.regtr_mha_varlen_bwd_ws_bytes(n_rows, n_heads), q.device, 'mha_bwd')
    _lib.check(L.regtr_mha_varlen_bwd(_p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(o), o.stride(0),
                                      _p(d_o), d_o.stride(0), _p(lse), _p(dq), dq.stride(0), _p(dk), dk.stride(0),
                                      _p(dv), dv.stride(0), _p(q_start), _p(q_len), _p(k_start), _p(k_len),
                                      q_start.numel(), n_rows, int(max_q_len), int(max_k_len), n_heads, dh,
                                      1.0 / math.sqrt(dh), None if drop is None else drop.ptr, _p(ws), ws.numel(),
                                      _stream()), 'regtr_mha_varlen_bwd')
    _count(2)


def mha_packed(qkv, q_start, q_len, k_start, k_len, max_len: int, n_heads: int, drop=None):
    """Attention core over a packed in-projection output qkv (N, 3E) = [q | k | v]; differentiable with respect to
    qkv (one packed (N, 3E) gradient, written by the backward kernels directly) when grad mode is on.  drop (a dropout
    site, site 1 or 3): the attention-probability dropout, on the training core."""
    E = qkv.shape[1] // 3
    if drop is not None or _wants_grad(qkv):
        return _MHAPackedFn.apply(qkv, q_start, q_len, k_start, k_len, int(max_len), int(n_heads), drop)
    return mha_varlen(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], q_start, q_len, k_start, k_len, max_len, n_heads)


def layernorm_bwd(x, gamma, dy, dy_pos, dres, eps: float, drop=None):
    """-> (dx, dgamma, dbeta) of regtr_layernorm_pos; dy / dy_pos / dres may be None.  drop (the forward's dropout
    site; x = the forward's x'): -> (dx, dgamma, dbeta, dz), dz the gradient of the dropped branch z."""
    L = _lib.load()
    _chk(x, torch.float32, 'x', 2)
    n, E = x.shape
    for t, nm in ((dy, 'dy'), (dy_pos, 'dy_pos'), (dres, 'dres')):
        if t is not None:
            _chk(t, torch.float32, nm, 2)
    dx = torch.empty_like(x)
    dg = torch.empty_like(gamma)
    db = torch.empty_like(gamma)
    offs = dz = dp = None
    if drop is not None:
        offs, dz, dp = drop.key.offs, torch.empty_like(x), drop.ptr
    ws = workspace(L.regtr_layernorm_bwd_ws_bytes(n, E), x.device, 'ln_bwd')
    _lib.check(L.regtr_layernorm_bwd(_p(x), _p(gamma), _p(dy), _p(dy_pos), _p(dres), n, _p(offs), E, float(eps), _p(dx),
                                     _p(dz), _p(dg), _p(db), dp, _p(ws), ws.numel(), _stream()), 'regtr_layernorm_bwd')
    _count(2)
    return (dx, dg, db) if drop is None else (dx, dg, db, dz)


def relu_bwd(dh, h, scale: float = 1.0):
    """dh * scale where h > 0, else 0; h the ReLU's output, or with the feed-forward dropout the dropped ReLU output
    and scale the dropout's (h is positive exactly where both passed)."""
    L = _lib.load()
    out = torch.empty_like(dh)
    _lib.check(L.regtr_relu_bwd(_p(dh), _p(h), dh.numel(), float(scale), _p(out), _stream()), 'regtr_relu_bwd')
    _count(1)
    return out


def linear_dgrad(dy, weight, residual=None):
    """dX = dY @ W (+ residual, added in the epilogue) on the 3xTF32 GEMM with the transposed pre-split weight.  N_out % 4 != 0 (the 3- and 1-wide heads) zero-pads dY and W^T to the TMA row pitch."""
    N = weight.shape[0]
    hi, lo = split_weight(weight, transpose=True)            # (K, N)
    pad = (-N) % 4
    if pad:
        dy = torch.nn.functional.pad(dy, (0, pad))
        hi, lo = torch.nn.functional.pad(hi, (0, pad)), torch.nn.functional.pad(lo, (0, pad))
    return gemm(dy, hi, lo, residual=residual)


def linear_wgrad(x, dy, want_bias: bool):
    """-> (dW (N,K), db (N) or None): dW = dY^T X, db = sum_rows dY (regtr_linear_wgrad)."""
    L = _lib.load()
    M, K = x.shape
    N = dy.shape[1]
    dw = torch.empty((N, K), dtype=torch.float32, device=x.device)
    db = torch.empty(N, dtype=torch.float32, device=x.device) if want_bias else None
    ws = workspace(L.regtr_linear_wgrad_ws_bytes(M, N, K), x.device, 'wgrad')
    _lib.check(L.regtr_linear_wgrad(_p(x), x.stride(0), _p(dy), dy.stride(0), M, N, K, _p(dw), _p(db), _p(ws),
                                    ws.numel(), _stream()), 'regtr_linear_wgrad')
    _count(4 + (L.regtr_gemm_ws_bytes(N, (K + 4) // 4 * 4, (M + 3) // 4 * 4) > 256))
    return dw, db


class _LinearFn(torch.autograd.Function):
    """act(x W^T + b + residual), then the feed-forward dropout if a site is given; backward on regtr_relu_bwd (which
    also applies the dropout mask and scale), the 3xTF32 GEMM (dX) and regtr_linear_wgrad."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, relu, drop):
        out = _linear_fwd(x, weight, bias, residual, relu)
        if drop is not None:
            dropout_rows_(out, drop)
        ctx.save_for_backward(x, out if relu else None)
        ctx.weight, ctx.relu, ctx.has_bias = weight, relu, bias is not None   # the parameter itself: split cache
        ctx.scale = 1.0 if drop is None else drop.scale
        return out

    @staticmethod
    def backward(ctx, g):
        x, out = ctx.saved_tensors
        g = g.contiguous()
        if ctx.relu:
            g = relu_bwd(g, out, ctx.scale)
        need = ctx.needs_input_grad
        dx = linear_dgrad(g, ctx.weight) if need[0] else None
        dw = db = None
        if need[1] or need[2]:
            dw, db = linear_wgrad(x, g, ctx.has_bias and need[2])
        return dx, (dw if need[1] else None), db, (g if need[3] else None), None, None


class _LayerNormPosFn(torch.autograd.Function):
    """(LN(x), LN(x) + pos, x); with a dropout site x is first x + m * scale * z (a residual dropout, site 2, 4 or 6,
    fused into the LayerNorm that follows the residual add) and the third output is that x'."""

    @staticmethod
    def forward(ctx, x, gamma, beta, pos, eps, want_plain, want_pos, skip, z, drop):
        ctx.set_materialize_grads(False)
        y, yp, xo = _layernorm_pos_fwd(x, gamma, beta, pos, eps, want_plain, want_pos, None, z, drop)
        ctx.save_for_backward(xo, gamma)
        ctx.eps, ctx.drop = eps, drop
        return y, yp, (xo if skip else None)

    @staticmethod
    def backward(ctx, dy, dyp, dres):
        xo, gamma = ctx.saved_tensors
        c = lambda t: None if t is None else t.contiguous()
        grads = layernorm_bwd(xo, gamma, c(dy), c(dyp), c(dres), ctx.eps, ctx.drop)
        need = ctx.needs_input_grad
        dx, dg, db = (g if n else None for g, n in zip(grads[:3], need))
        return dx, dg, db, None, None, None, None, None, (grads[3] if need[8] else None), None


class _MHAPackedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, q_start, q_len, k_start, k_len, max_len, n_heads, drop):
        E = qkv.shape[1] // 3
        o, lse = mha_varlen_lse(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], q_start, q_len, k_start, k_len, max_len,
                                n_heads, drop)
        ctx.save_for_backward(qkv, o, lse, q_start, q_len, k_start, k_len)
        ctx.max_len, ctx.n_heads, ctx.drop = max_len, n_heads, drop
        return o

    @staticmethod
    def backward(ctx, g):
        qkv, o, lse, qs, ql, ks, kl = ctx.saved_tensors
        E = qkv.shape[1] // 3
        d = torch.zeros_like(qkv)            # rows outside every problem keep a zero gradient
        mha_varlen_bwd(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], o, lse, g.contiguous(), d[:, :E], d[:, E:2 * E],
                       d[:, 2 * E:], qs, ql, ks, kl, ctx.max_len, ctx.max_len, ctx.n_heads, ctx.drop)
        return d, None, None, None, None, None, None, None


# ------------------------------------------------------------------ transformer dropout (training)
# The six dropouts of TransformerCrossEncoderLayer.forward_pre (transformers.py:183-244), numbered as in
# include/regtr_b200.h: masks are regenerated from (seed, step, global cloud, layer, site, head, row, column), never
# stored (keep rule: csrc/philox.cuh).
SITE_SELF_ATTN, SITE_SELF_OUT, SITE_CROSS_ATTN, SITE_CROSS_OUT, SITE_FFN, SITE_FFN_OUT = 1, 2, 3, 4, 5, 6


class _DropoutArgs(ctypes.Structure):
    _fields_ = [('seed', ctypes.c_ulonglong), ('step', ctypes.c_ulonglong), ('pair_base', ctypes.c_int32),
                ('layer', ctypes.c_int32), ('site', ctypes.c_int32), ('threshold', ctypes.c_uint32),
                ('scale', ctypes.c_float), ('n_pairs', ctypes.c_int32)]


def dropout_threshold(p: float) -> int:
    """16-bit drop threshold: a value is dropped when its draw (0..65535) is below round(p * 65536)."""
    return int(round(float(p) * 65536.0))


def dropout_scale(p: float) -> float:
    """The fp32 value of 1 / (1 - p) that kept values are multiplied by."""
    return float(np.float32(1.0 / (1.0 - float(p))))


class DropoutKey:
    """The dropout masks of one training step of a (src x B, tgt x B) batch whose first pair is global pair
    `pair_base`: `args(layer, site)` is the C argument block of one site.  `offs` (2B + 1 int32, device) are the cloud
    offsets of the packed tokens and `max_len` a host bound of the cloud lengths (the elementwise sites need them)."""

    def __init__(self, p: float, seed: int, step: int, pair_base: int, n_pairs: int, offs=None, max_len: int = 0):
        if not 0.0 < float(p) < 1.0:
            raise ValueError(f'DropoutKey: p={p} outside (0, 1)')
        self.p, self.seed, self.step = float(p), int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1)
        self.pair_base, self.n_pairs = int(pair_base), int(n_pairs)
        self.threshold, self.scale = dropout_threshold(p), dropout_scale(p)
        self.offs, self.max_len = offs, int(max_len)
        if self.max_len >= 1 << 16:
            raise ValueError('dropout: clouds of 2^16 tokens or more are outside the mask counter layout')
        self._args = {}

    def args(self, layer: int, site: int) -> _DropoutArgs:
        a = self._args.get((layer, site))
        if a is None:
            a = self._args[(layer, site)] = _DropoutArgs(self.seed, self.step, self.pair_base, int(layer), int(site),
                                                         self.threshold, self.scale, self.n_pairs)
        return a

    def site(self, layer: int, site: int):
        return _DropSite(self, int(layer), int(site))


class _DropSite:
    """One (layer, site) of a DropoutKey: what the kernels of that site take."""

    def __init__(self, key: DropoutKey, layer: int, site: int):
        self.key, self.layer, self.site = key, layer, site
        self.scale = key.scale

    @property
    def ptr(self):
        return ctypes.addressof(self.key.args(self.layer, self.site))


def dropout_keep_mask(p: float, seed: int, step: int, pair_base: int, n_pairs: int, cloud: int, layer: int, site: int,
                      head: int, rows: int, cols: int, device=None):
    """(rows, cols) uint8 keep mask (1 = kept) of local cloud `cloud` (0..2B-1: src clouds, then tgt clouds) at one
    site, layer and head, from the same device function the kernels use (tests and analysis)."""
    L = _lib.load()
    key = DropoutKey(p, seed, step, pair_base, n_pairs)
    out = torch.empty((int(rows), int(cols)), dtype=torch.uint8, device=device or 'cuda')
    _lib.check(L.regtr_dropout_keep_mask(ctypes.addressof(key.args(layer, site)), int(cloud), int(head), int(rows),
                                         int(cols), _p(out), _stream()), 'regtr_dropout_keep_mask')
    _count(1)
    return out


def dropout_rows_(h, drop: _DropSite):
    """Feed-forward dropout (site 5) in place on the packed (N, F) rows of the batch's clouds."""
    L = _lib.load()
    _chk(h, torch.float32, 'h', 2)
    k = drop.key
    _lib.check(L.regtr_dropout_rows(_p(h), h.shape[0], h.shape[1], _p(k.offs), k.max_len, drop.ptr, _stream()),
               'regtr_dropout_rows')
    _count(1)
    return h


# ------------------------------------------------------------------ encoder backward

def neighbor_csr(idx32, Ns: int):
    """Incoming-edge CSR of a neighbour list (regtr_neighbor_csr) -> (row_start (Ns+1), edges (Nq*K)) int32.
    Cached on the index tensor itself, so the blocks that share a list in one training step (every block of a level
    shares its conv list; a strided block's KPConv and max-pool share its pool list) build it once."""
    L = _lib.load()
    _chk(idx32, torch.int32, 'neighb_inds', 2)
    cache = idx32.__dict__.setdefault('_regtr_csr', {})
    key = (int(Ns), idx32._version)
    hit = cache.get(key)
    if hit is not None:
        return hit
    Nq, K = idx32.shape
    row_start = torch.empty(Ns + 1, dtype=torch.int32, device=idx32.device)
    edges = torch.empty(max(Nq * K, 1), dtype=torch.int32, device=idx32.device)
    ws = workspace(L.regtr_neighbor_csr_ws_bytes(Ns), idx32.device, 'csr')
    _lib.check(L.regtr_neighbor_csr(_p(idx32), Nq, K, Ns, _p(row_start), _p(edges), _p(ws), ws.numel(), _stream()),
               'regtr_neighbor_csr')
    _count(5)
    cache.clear()
    cache[key] = (row_start, edges)
    return row_start, edges


def kpconv_bwd_input(q_pts, s_pts, idx32, x, flags, kernel_points, extent: float, dwf, csr):
    """dx (Ns, Cin) of the KPConv from dwf = dOut W^T (Nq, 15 Cin); flags: the forward's row flags or None."""
    L = _lib.load()
    Nq, K = idx32.shape
    Ns, Cin = x.shape
    _chk(dwf, torch.float32, 'dwf', 2)
    dx = torch.empty_like(x)
    ws = workspace(L.regtr_kpconv_bwd_input_ws_bytes(Nq, K, Cin), x.device, 'kpconv_bwd')
    _lib.check(L.regtr_kpconv_bwd_input(_p(q_pts), _p(s_pts), _p(idx32), _p(x), _p(flags), _p(kernel_points), Nq, Ns,
                                        K, Cin, float(extent), _p(dwf), _p(csr[0]), _p(csr[1]), _p(dx), _p(ws),
                                        ws.numel(), _stream()), 'regtr_kpconv_bwd_input')
    _count(2)
    return dx


def max_pool_bwd(x, idx32, dout, csr):
    L = _lib.load()
    Nq, K = idx32.shape
    Ns, C = x.shape
    _chk(dout, torch.float32, 'dout', 2)
    dx = torch.empty_like(x)
    ws = workspace(L.regtr_max_pool_bwd_ws_bytes(Nq, C), x.device, 'maxpool_bwd')
    _lib.check(L.regtr_max_pool_bwd(_p(x), _p(idx32), Nq, Ns, K, C, _p(dout), _p(csr[0]), _p(csr[1]), _p(dx), _p(ws),
                                    ws.numel(), _stream()), 'regtr_max_pool_bwd')
    _count(2)
    return dx


def instnorm_bwd(g, x, out, offs, n_clouds: int, slope: float, eps: float = 1e-5, want_dres: bool = False):
    """-> (dx, dres or None) of out = act(InstanceNorm_per_cloud(x) + res) (regtr_instnorm_bwd)."""
    L = _lib.load()
    _chk(g, torch.float32, 'g', 2); _chk(x, torch.float32, 'x', 2); _chk(offs, torch.int32, 'offs', 1)
    n, C = x.shape
    dx = torch.empty_like(x)
    dres = torch.empty_like(x) if want_dres else None
    ws = workspace(L.regtr_instnorm_bwd_ws_bytes(n, n_clouds, C), x.device, 'instnorm_bwd')
    _lib.check(L.regtr_instnorm_bwd(_p(g), _p(x), _p(out if slope >= 0 else None), _p(offs), n_clouds, n, C,
                                    float(eps), float(slope), _p(dx), _p(dres), _p(ws), ws.numel(), _stream()),
               'regtr_instnorm_bwd')
    _count(3)
    return dx, dres


def _kpconv_wf(q_pts, s_pts, idx32, x, kernel_points, extent: float, row_flags):
    """Recompute the forward's aggregated features wf (Nq, 15 Cin) for the weight gradient; -> (wf, row flags used by
    the count, or None for Cin = 1, whose aggregation counts from x itself)."""
    L = _lib.load()
    Nq, K = idx32.shape
    Ns, Cin = x.shape
    wf = torch.empty((Nq, 15 * Cin), dtype=torch.float32, device=x.device)
    flags = row_flags
    if flags is None:       # computed by the aggregation (Cin > 1); Cin = 1 never touches it
        flags = torch.empty(max(Ns, 1) if Cin > 1 else 1, dtype=torch.uint8, device=x.device)
    _lib.check(L.regtr_kpconv_aggregate(_p(q_pts), _p(s_pts), _p(idx32), _p(x), _p(kernel_points), Nq, Ns, None, None,
                                        K, Cin, float(extent), _p(wf), _p(flags), 1 if row_flags is not None else 0,
                                        _stream()), 'regtr_kpconv_aggregate')
    _count(1 if (row_flags is not None or Cin == 1) else 2)
    return wf, (flags if Cin > 1 else None)


class _KPConvFn(torch.autograd.Function):
    """KPConv forward (the fused C1 kernel, or the aggregation + contraction GEMM with optional statistics epilogue).
    Backward: wf recomputed by regtr_kpconv_aggregate, dW = wf^T dOut (regtr_linear_wgrad), dwf = dOut W^T (3xTF32
    GEMM), dx by regtr_kpconv_bwd_input through the list's CSR."""

    @staticmethod
    def forward(ctx, x, weights, q_pts, s_pts, idx32, kernel_points, extent, row_flags, instats):
        ctx.set_materialize_grads(False)
        r = _kpconv_fwd(q_pts, s_pts, idx32, x, weights, kernel_points, extent, row_flags=row_flags, instats=instats)
        out, stats = r if instats is not None else (r, None)
        ctx.save_for_backward(x, q_pts, s_pts, kernel_points, row_flags)
        ctx.idx, ctx.weights, ctx.extent = idx32, weights, extent     # idx: the CSR cache lives on this object
        if stats is not None:
            ctx.mark_non_differentiable(stats)
        return out, stats

    @staticmethod
    def backward(ctx, g, _gstats):
        x, q_pts, s_pts, kp, row_flags = ctx.saved_tensors
        need_x, need_w = ctx.needs_input_grad[:2]
        dx = dw = None
        if g is None:
            return (None,) * 9
        g = g.contiguous()
        Ns, Cin = x.shape
        Cout = ctx.weights.shape[2]
        flags = row_flags
        if need_w:
            wf, flags = _kpconv_wf(q_pts, s_pts, ctx.idx, x, kp, ctx.extent, row_flags)
            dw = linear_wgrad(g, wf, False)[0].view(15, Cin, Cout)       # (15 Cin, Cout) = wf^T dOut
        if need_x:
            hi, lo = split_weight(ctx.weights.view(15 * Cin, Cout))
            dwf = gemm(g, hi, lo)
            dx = kpconv_bwd_input(q_pts, s_pts, ctx.idx, x, flags, kp, ctx.extent, dwf, neighbor_csr(ctx.idx, Ns))
        return dx, dw, None, None, None, None, None, None, None


class _MaxPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, idx32):
        ctx.save_for_backward(x)
        ctx.idx = idx32
        return _max_pool_fwd(x, idx32)

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        return max_pool_bwd(x, ctx.idx, g.contiguous(), neighbor_csr(ctx.idx, x.shape[0])), None


class _InstNormFn(torch.autograd.Function):
    """act(InstanceNorm_per_cloud(x) + res); statistics from the producing GEMM's epilogue (stats) or computed here.
    Backward on regtr_instnorm_bwd (statistics recomputed from x)."""

    @staticmethod
    def forward(ctx, x, res, stats, offs, n_clouds, slope, eps, want_flags):
        ctx.set_materialize_grads(False)
        if stats is None:
            y, flags = _instnorm_act_fwd(x, offs, n_clouds, res=res, slope=slope, eps=eps, want_flags=True) \
                if want_flags else (_instnorm_act_fwd(x, offs, n_clouds, res=res, slope=slope, eps=eps), None)
        else:
            y, flags = _instnorm_apply_fwd(x, offs, n_clouds, stats, res=res, slope=slope, want_flags=True) \
                if want_flags else (_instnorm_apply_fwd(x, offs, n_clouds, stats, res=res, slope=slope), None)
        ctx.save_for_backward(x, y if slope >= 0 else None, offs)
        ctx.n_clouds, ctx.slope, ctx.eps = n_clouds, slope, eps
        if flags is not None:
            ctx.mark_non_differentiable(flags)
        return y, flags

    @staticmethod
    def backward(ctx, g, _gflags):
        if g is None:
            return (None,) * 8
        x, y, offs = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx, dres = instnorm_bwd(g.contiguous(), x, y, offs, ctx.n_clouds, ctx.slope, ctx.eps, want_dres=need[1])
        return (dx if need[0] else None), dres, None, None, None, None, None, None


class _LinearInstatsFn(torch.autograd.Function):
    """x W^T plus the per-cloud InstanceNorm statistics of the result (non-differentiable: _InstNormFn's backward
    differentiates through them).  Backward: dX on the 3xTF32 GEMM (+ the shortcut gradient of the skip output in its
    epilogue), dW on regtr_linear_wgrad."""

    @staticmethod
    def forward(ctx, x, weight, offs, n_clouds, eps, skip):
        ctx.set_materialize_grads(False)
        y, stats = _linear_instats_fwd(x, weight, offs, n_clouds, eps)
        ctx.save_for_backward(x)
        ctx.weight = weight
        ctx.mark_non_differentiable(stats)
        return y, stats, (x if skip else None)

    @staticmethod
    def backward(ctx, g, _gstats, gskip):
        x, = ctx.saved_tensors
        need = ctx.needs_input_grad
        if g is None:
            return gskip, None, None, None, None, None
        g = g.contiguous()
        dx = linear_dgrad(g, ctx.weight, residual=None if gskip is None else gskip.contiguous()) if need[0] else None
        dw = linear_wgrad(x, g, False)[0] if need[1] else None
        return dx, dw, None, None, None, None


# --------------------------------------------------------------------------- pose

def kabsch(a, b, w, offs):
    """Packed problems: rows [offs[i], offs[i+1]) -> T (n_problems,3,4)."""
    L = _lib.load()
    _chk(a, torch.float32, 'a', 2); _chk(b, torch.float32, 'b', 2); _chk(w, torch.float32, 'w', 1)
    n_prob = offs.numel() - 1
    T = torch.empty((n_prob, 3, 4), dtype=torch.float32, device=a.device)
    _lib.check(L.regtr_kabsch_fwd(_p(a), _p(b), _p(w), _p(offs), n_prob, _p(T), _stream()), 'regtr_kabsch_fwd')
    _count(1)
    return T


def pose_from_corr(kp, corr, logit, offs, B: int):
    """kp (n,3), corr (L,n,3), logit (L,n), offs (2B+1) -> pose (L,B,3,4)."""
    L_ = _lib.load()
    _chk(kp, torch.float32, 'kp', 2); _chk(corr, torch.float32, 'corr', 3); _chk(logit, torch.float32, 'logit', 2)
    nl, n = logit.shape
    pose = torch.empty((nl, B, 3, 4), dtype=torch.float32, device=kp.device)
    _lib.check(L_.regtr_pose_from_corr(_p(kp), _p(corr), _p(logit), _p(offs), n, B, nl, _p(pose), _stream()),
               'regtr_pose_from_corr')
    _count(1)
    return pose


# --------------------------------------------------------------------------- training data

PREP_PERTURB_SRC, PREP_CENTRE, PREP_SWAP, PREP_SHUFFLE = 1, 2, 4, 8     # REGTR_PREP_*
STATUS_RANGE = 8                                                         # REGTR_STATUS_RANGE


def overlap_cell(radius: float) -> float:
    """Cell size of the overlap search's cell list: radius * (1 + 1e-3), rounded to fp32."""
    return float(torch.tensor(radius * (1.0 + 1e-3), dtype=torch.float32))


def overlap_coord_bound(radius: float) -> float:
    """Largest |coordinate| (aligned clouds) for which the overlap search is exact (REGTR_STATUS_RANGE beyond)."""
    return float(_lib.load().regtr_overlap_coord_bound(float(radius), overlap_cell(radius)))


def overlap_nn(xyz, offs, B: int, pose, radius: float, status):
    """Nearest point of the partner cloud within `radius` (float64, strict, lowest index on ties) for every point of
    the stacked float64 clouds src_0..src_{B-1}, tgt_0..tgt_{B-1}; sources moved by `pose` (B,3,4) float64 first.
    -> nn (n,) int32: index inside the partner cloud or -1.  No host sync."""
    L = _lib.load()
    _chk(xyz, torch.float64, 'xyz', 2); _chk(offs, torch.int32, 'offs', 1); _chk(pose, torch.float64, 'pose', 3)
    n = xyz.shape[0]
    nn = torch.empty(max(n, 1), dtype=torch.int32, device=xyz.device)
    ws = workspace(L.regtr_overlap_ws_bytes(n), xyz.device)
    state = workspace(L.regtr_overlap_state_bytes(n), xyz.device, 'scan_state', zero=True)
    _lib.check(L.regtr_overlap_nn(_p(xyz), _p(offs), B, n, _p(pose), float(radius), overlap_cell(radius), _p(nn),
                                  _p(status), _p(ws), ws.numel(), _p(state), state.numel(), _stream()),
               'regtr_overlap_nn')
    _count(6 if n > 0 else 0)
    return nn[:n]



def registration_fit(src_list, tgt_list, pose, radius: float, status=None):
    """Fitness and inlier RMSE of B registered pairs (regtr_registration_fit on the matches of `overlap_nn`):
    src_list / tgt_list, B clouds (n,3) each (numpy or torch, any float dtype; stacked in float64 on the device),
    pose (B,3,4) source -> target.  -> (B,4) float64 device tensor (fitness_src, rmse_src, fitness_tgt, rmse_tgt).
    status: a device word (`new_status`) that the caller checks with `check_fit_status` where it syncs; this call does
    not read it.  status=None: a word of this call, read and checked before returning.  A coordinate of the moved source or the
    target beyond `overlap_coord_bound(radius)` raises RegtrLibError there."""
    L = _lib.load()
    B = len(src_list)
    if B == 0 or len(tgt_list) != B:
        raise ValueError('registration_fit: expected as many source as target clouds, at least one pair')
    dev = pose.device if torch.is_tensor(pose) and pose.is_cuda else torch.device('cuda', torch.cuda.current_device())
    clouds = [torch.as_tensor(c) for c in list(src_list) + list(tgt_list)]
    for c in clouds:
        if c.dim() != 2 or c.shape[1] != 3:
            raise ValueError(f'registration_fit: expected (n,3) clouds, got {tuple(c.shape)}')
    lens = [int(c.shape[0]) for c in clouds]
    n = sum(lens)
    xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
    a = 0
    for c, ln in zip(clouds, lens):
        xyz[a:a + ln].copy_(c.to(dev, torch.float64))
        a += ln
    pose64 = torch.as_tensor(pose).to(dev, torch.float64).reshape(B, 3, 4).contiguous()
    offs = make_offsets(lens, dev)
    own = status is None
    if own:
        status = new_status(dev)
    nn = overlap_nn(xyz, offs, B, pose64, radius, status)
    out = torch.empty((B, 4), dtype=torch.float64, device=dev)
    _lib.check(L.regtr_registration_fit(_p(xyz), _p(offs), B, n, _p(pose64), float(radius), _p(nn), _p(out),
                                        _p(status), _stream()), 'regtr_registration_fit')
    _count(1)
    if own:
        check_fit_status(status, radius)
    return out


def _stack_pairs(src_list, tgt_list, what: str, device=None):
    """src_0..src_{B-1}, tgt_0..tgt_{B-1} stacked in float64 on the device -> (xyz (n,3), offs (2B+1), lens)."""
    B = len(src_list)
    if B == 0 or len(tgt_list) != B:
        raise ValueError(f'{what}: expected as many source as target clouds, at least one pair')
    dev = device if device is not None else torch.device('cuda', torch.cuda.current_device())
    clouds = [torch.as_tensor(c) for c in list(src_list) + list(tgt_list)]
    for c in clouds:
        if c.dim() != 2 or c.shape[1] != 3:
            raise ValueError(f'{what}: expected (n,3) clouds, got {tuple(c.shape)}')
    lens = [int(c.shape[0]) for c in clouds]
    xyz = torch.empty((max(sum(lens), 1), 3), dtype=torch.float64, device=dev)
    a = 0
    for c, ln in zip(clouds, lens):
        xyz[a:a + ln].copy_(c.to(dev, torch.float64))
        a += ln
    return xyz, make_offsets(lens, dev), lens


def icp_launches(max_iteration: int) -> int:
    """Kernel launches of one `icp` call: the set-up, the targets' cell list (4), then 3 per round."""
    return 5 + 3 * (int(max_iteration) + 1)


ICP_METHODS = ('point_to_point', 'point_to_plane', 'generalized', 'colored')
ICP_LOSSES = ('l2', 'huber', 'cauchy', 'gm', 'tukey')      # REGTR_ICP_LOSS_L2 .. REGTR_ICP_LOSS_TUKEY


class IcpOptions(ctypes.Structure):
    """regtr_icp_options (include/regtr_b200.h)."""
    _fields_ = [('loss', ctypes.c_int), ('loss_k', ctypes.c_double), ('epsilon', ctypes.c_double),
                ('src_colors', ctypes.c_void_p), ('tgt_colors', ctypes.c_void_p),
                ('tgt_color_gradients', ctypes.c_void_p), ('lambda_geometric', ctypes.c_double)]


def _stack_normals(normals, lens, what, dev, kind='normals'):
    """B (n,3) normal (or `kind`) arrays aligned with clouds of `lens` points -> one (max(sum, 1), 3) float64 device
    tensor."""
    if normals is None or len(normals) != len(lens):
        raise ValueError(f'icp: {0 if normals is None else len(normals)} {what} {kind} arrays for {len(lens)} pairs')
    out = torch.empty((max(sum(lens), 1), 3), dtype=torch.float64, device=dev)
    a = 0
    for c, ln in zip(normals, lens):
        c = torch.as_tensor(c)
        if tuple(c.shape) != (ln, 3):
            raise ValueError(f'icp: {what} {kind} {tuple(c.shape)} for a {what} of {ln} points')
        out[a:a + ln].copy_(c.to(dev, torch.float64))
        a += ln
    return out


def icp(src_list, tgt_list, init, max_correspondence_distance: float, max_iteration: int = 30,
        relative_fitness: float = 1e-6, relative_rmse: float = 1e-6, status=None, method: str = 'point_to_point',
        tgt_normals=None, src_normals=None, epsilon: float = 1e-3, loss: str = 'l2', loss_k: float = None,
        src_colors=None, tgt_colors=None, tgt_color_gradients=None, lambda_geometric: float = 0.968):
    """ICP of B pairs (regtr_icp): Open3D's registration_icp with TransformationEstimationPointToPoint (no scaling) or,
    with method='point_to_plane', TransformationEstimationPointToPlane, or with method='generalized',
    registration_generalized_icp with TransformationEstimationForGeneralizedICP(epsilon), or with method='colored',
    registration_colored_icp with TransformationEstimationForColoredICP(lambda_geometric), and
    ICPConvergenceCriteria(relative_fitness, relative_rmse, max_iteration), on the device.
    src_list / tgt_list: B clouds (n,3) each (numpy or torch, any float dtype; stacked in float64 on the device);
    init (B,3,4) source -> target.  tgt_normals: with 'point_to_plane' and 'generalized', B (n,3) normals aligned with
    tgt_list (e.g. `estimate_normals(tgt_list, ...)`); a zero normal drops its correspondence out of the point-to-plane
    update.  src_normals: with 'generalized', B (n,3) normals aligned with src_list (a zero normal gives the identity
    covariance); epsilon in (0, 1] the covariances' epsilon.  'colored' takes tgt_normals, B (n,3) rgb arrays
    src_colors / tgt_colors aligned with the clouds, the targets' tgt_color_gradients (`color_gradients`) and
    lambda_geometric in [0, 1], the weight of the geometric residual.  loss: one of ICP_LOSSES, Open3D's robust kernel
    of the point-to-plane, generalized and colored estimations, with loss_k its parameter k > 0 ('l2', the default,
    takes none; the point-to-point estimation has no kernel).
    -> (pose (B,3,4) float64, result (B,4) float64 = fitness, inlier_rmse, n_corr, iterations), both device tensors.
    No host sync unless status is None: then a word of this call is read and a coordinate of a moved source or of a
    target beyond `overlap_coord_bound(max_correspondence_distance)` raises RegtrLibError; with the caller's word,
    `check_fit_status` does that where the caller syncs."""
    L = _lib.load()
    r = float(max_correspondence_distance)
    if not r > 0.0 or int(max_iteration) < 0 or not (relative_fitness >= 0.0 and relative_rmse >= 0.0):
        raise ValueError(f'icp: max_correspondence_distance {r} must be > 0, max_iteration {max_iteration} >= 0, '
                         f'relative_fitness / relative_rmse >= 0')
    if method not in ICP_METHODS:
        raise ValueError(f'icp: method {method!r} is not one of {ICP_METHODS}')
    if loss not in ICP_LOSSES:
        raise ValueError(f'icp: loss {loss!r} is not one of {ICP_LOSSES}')
    if loss != 'l2' and method == 'point_to_point':
        raise ValueError(f'icp: the point_to_point estimation takes no robust loss (got {loss!r})')
    if loss != 'l2' and not (loss_k is not None and math.isfinite(float(loss_k)) and float(loss_k) > 0.0):
        raise ValueError(f'icp: loss {loss!r} needs a finite loss_k > 0, got {loss_k!r}')
    gicp = method == 'generalized'
    if gicp and not (0.0 < float(epsilon) <= 1.0):
        raise ValueError(f'icp: epsilon {epsilon!r} must be in (0, 1]')
    if method != 'point_to_point' and tgt_normals is None:
        raise ValueError(f'icp: {method} needs the target normals (tgt_normals), e.g. from estimate_normals')
    if gicp and src_normals is None:
        raise ValueError('icp: generalized needs the source normals (src_normals), e.g. from estimate_normals')
    colored = method == 'colored'
    if colored:
        if not 0.0 <= float(lambda_geometric) <= 1.0:
            raise ValueError(f'icp: lambda_geometric {lambda_geometric!r} must be in [0, 1]')
        for name, v in (('src_colors', src_colors), ('tgt_colors', tgt_colors),
                        ('tgt_color_gradients', tgt_color_gradients)):
            if v is None:
                raise ValueError(f'icp: colored needs {name}')
    B = len(src_list)
    dev = init.device if torch.is_tensor(init) and init.is_cuda else None
    xyz, offs, lens = _stack_pairs(src_list, tgt_list, 'icp', dev)
    dev = xyz.device
    nrm = None if method == 'point_to_point' else _stack_normals(tgt_normals, lens[B:], 'target', dev)
    snrm = _stack_normals(src_normals, lens[:B], 'source', dev) if gicp else None
    opt = None
    if gicp or colored or loss != 'l2':
        opt = IcpOptions(ICP_LOSSES.index(loss), float(loss_k) if loss != 'l2' else 1.0, float(epsilon))
    if colored:
        scol = _stack_normals(src_colors, lens[:B], 'source', dev, 'colors')
        tcol = _stack_normals(tgt_colors, lens[B:], 'target', dev, 'colors')
        tgrd = _stack_normals(tgt_color_gradients, lens[B:], 'target', dev, 'color gradients')
        opt.src_colors, opt.tgt_colors, opt.tgt_color_gradients = _p(scol), _p(tcol), _p(tgrd)
        opt.lambda_geometric = float(lambda_geometric)
    init64 = torch.as_tensor(init).to(dev, torch.float64).reshape(B, 3, 4).contiguous()
    n = sum(lens)
    own = status is None
    if own:
        status = new_status(dev)
    pose = torch.empty((B, 3, 4), dtype=torch.float64, device=dev)
    out = torch.empty((B, 4), dtype=torch.float64, device=dev)
    ws = workspace(L.regtr_icp_ws_bytes(n, B), dev)
    state = workspace(L.regtr_icp_state_bytes(n), dev, 'scan_state', zero=True)
    _lib.check(L.regtr_icp(_p(xyz), _p(offs), B, n, _p(init64), r, overlap_cell(r), int(max_iteration),
                           float(relative_fitness), float(relative_rmse), _p(nrm), _p(snrm),
                           None if opt is None else ctypes.addressof(opt), _p(pose), _p(out), _p(status), _p(ws),
                           ws.numel(), _p(state), state.numel(), _stream()), 'regtr_icp')
    _count(icp_launches(max_iteration))
    if own:
        check_fit_status(status, r, 'icp')
    return pose, out


RANSAC_MAX_N = 16                   # REGTR_RANSAC_MAX_N
RANSAC_CHUNK_MAX = 8192             # REGTR_RANSAC_CHUNK_MAX


class RansacOptions(ctypes.Structure):
    """regtr_ransac_options (include/regtr_b200.h)."""
    _fields_ = [('max_iteration', ctypes.c_int), ('confidence', ctypes.c_double), ('ransac_n', ctypes.c_int),
                ('edge_length', ctypes.c_double), ('distance', ctypes.c_double), ('seed', ctypes.c_ulonglong),
                ('pair_base', ctypes.c_int), ('first_chunk', ctypes.c_int)]


def ransac_chunks(max_iteration: int, first_chunk: int = 256):
    """The hypothesis chunks of one `ransac` call: [(first hypothesis, count)], first_chunk * 2^c hypotheses each, at
    most RANSAC_CHUNK_MAX, the last one cut at max_iteration."""
    out, start, c = [], 0, 0
    while start < max_iteration:
        size = min(int(first_chunk) << min(c, 20), RANSAC_CHUNK_MAX, max_iteration - start)
        out.append((start, size))
        start += size
        c += 1
    return out


def _ransac_empty(max_correspondence_distance, ransac_n) -> bool:
    """Open3D's early return of every pair: ransac_n < 3 or a radius that is not positive."""
    return int(ransac_n) < 3 or not float(max_correspondence_distance) > 0.0


def ransac_launches(max_iteration: int, first_chunk: int = 256, ransac_n: int = 3,
                    max_correspondence_distance: float = 1.0) -> int:
    """Kernel launches of one `ransac` call: the set-up (2), the targets' cell list (4), then 3 per chunk; none when
    every pair returns Open3D's empty result for ransac_n < 3 or a radius that is not positive."""
    if _ransac_empty(max_correspondence_distance, ransac_n):
        return 0
    return 6 + 3 * len(ransac_chunks(int(max_iteration), first_chunk))


def _ransac_check(B, corr_src, corr_tgt, corr_mask, max_iteration, confidence, ransac_n, edge_length, distance, seed,
                  pair_base, first_chunk):
    """ValueError for every argument `ransac` rejects, before anything touches the device."""
    def real(v):
        return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool)
    if len(corr_src) != B or len(corr_tgt) != B:
        raise ValueError(f'ransac: {len(corr_src)} / {len(corr_tgt)} correspondence arrays for {B} pairs')
    if corr_mask is not None and len(corr_mask) != B:
        raise ValueError(f'ransac: {len(corr_mask)} correspondence masks for {B} pairs')
    for b in range(B):
        a, c = corr_src[b], corr_tgt[b]
        if len(a.shape) != 2 or a.shape[1] != 3 or tuple(a.shape) != tuple(c.shape):
            raise ValueError(f'ransac: pair {b}: correspondences {tuple(a.shape)} and {tuple(c.shape)}, expected two '
                             f'(m,3) arrays')
        if corr_mask is not None and tuple(corr_mask[b].shape) != (a.shape[0],):
            raise ValueError(f'ransac: pair {b}: mask {tuple(corr_mask[b].shape)} for {a.shape[0]} correspondences')
    if not (real(max_iteration) and int(max_iteration) == max_iteration and 0 <= max_iteration < 2 ** 31):
        raise ValueError(f'ransac: max_iteration {max_iteration!r} must be an integer in [0, 2^31)')
    if not (real(confidence) and 0.0 <= float(confidence) <= 1.0):
        raise ValueError(f'ransac: confidence {confidence!r} must be in [0, 1]')
    if not (real(ransac_n) and int(ransac_n) == ransac_n and int(ransac_n) <= RANSAC_MAX_N):
        raise ValueError(f'ransac: ransac_n {ransac_n!r} must be an integer <= {RANSAC_MAX_N}')
    for name, v in (('edge_length', edge_length), ('distance', distance)):
        if v is not None and not (real(v) and math.isfinite(float(v)) and float(v) >= 0.0):
            raise ValueError(f'ransac: {name} {v!r} must be None or a finite value >= 0 (0 or None: checker off)')
    if not (real(seed) and int(seed) == seed and 0 <= int(seed) < 2 ** 64):
        raise ValueError(f'ransac: seed {seed!r} must be an integer in [0, 2^64)')
    if not (real(pair_base) and int(pair_base) == pair_base and 0 <= int(pair_base) < 2 ** 31 - B):
        raise ValueError(f'ransac: pair_base {pair_base!r} must be an integer >= 0')
    if not (real(first_chunk) and int(first_chunk) == first_chunk and 1 <= int(first_chunk) <= RANSAC_CHUNK_MAX):
        raise ValueError(f'ransac: first_chunk {first_chunk!r} must be an integer in 1..{RANSAC_CHUNK_MAX}')


def ransac(src_list, tgt_list, corr_src, corr_tgt, max_correspondence_distance: float, max_iteration: int = 100000,
           confidence: float = 0.999, ransac_n: int = 3, edge_length: float = 0.9, distance: float = None,
           corr_mask=None, seed: int = 0, pair_base: int = 0, first_chunk: int = 256, status=None):
    """RANSAC over correspondences of B pairs (regtr_ransac): Open3D's registration_ransac_based_on_correspondence
    with TransformationEstimationPointToPoint(False), ransac_n, the checkers CorrespondenceCheckerBasedOnEdgeLength
    (edge_length) and CorrespondenceCheckerBasedOnDistance(distance) (0 or None: that checker is off) and
    RANSACConvergenceCriteria(max_iteration, confidence), with the library's deterministic sequential rule
    (include/regtr_b200.h, tests/ransac_oracle.py).
    src_list / tgt_list: B clouds (n,3) each, the validation clouds (numpy or torch, any float dtype; stacked in float64
    on the device).  corr_src / corr_tgt: B (m,3) arrays each, correspondence i of pair b being corr_src[b][i] ->
    corr_tgt[b][i] (Open3D's index form is src[corres[:,0]], tgt[corres[:,1]]); corr_mask: None or B (m,) boolean
    arrays, the correspondences that take part.  seed and pair_base + b key the draws, so a pair gets the same result
    alone or in a batch; first_chunk only sets the launch schedule, never the result.
    -> (pose (B,3,4) float64, result (B,5) float64 = fitness, inlier_rmse, hypotheses walked, hypotheses validated,
    index of the winning hypothesis or -1), both device tensors.  ransac_n < 3 or a radius that is not positive gives
    every pair Open3D's empty result (identity, zeros, -1) without a launch.
    No host sync unless status is None: then a word of this call is read and a coordinate of a moved source or of a
    target beyond `overlap_coord_bound(max_correspondence_distance)` raises RegtrLibError; with the caller's word,
    `check_fit_status` does that where the caller syncs."""
    B = len(src_list)
    if B == 0 or len(tgt_list) != B:
        raise ValueError('ransac: expected as many source as target clouds, at least one pair')
    corr_src = [torch.as_tensor(c) for c in corr_src]
    corr_tgt = [torch.as_tensor(c) for c in corr_tgt]
    corr_mask = None if corr_mask is None else [torch.as_tensor(m) for m in corr_mask]
    _ransac_check(B, corr_src, corr_tgt, corr_mask, max_iteration, confidence, ransac_n, edge_length, distance, seed,
                  pair_base, first_chunk)
    r = float(max_correspondence_distance)
    dev = next((c.device for c in corr_src if c.is_cuda), None)
    xyz, offs, lens = _stack_pairs(src_list, tgt_list, 'ransac', dev)
    dev = xyz.device
    pose = torch.zeros((B, 3, 4), dtype=torch.float64, device=dev)
    out = torch.zeros((B, 5), dtype=torch.float64, device=dev)
    if _ransac_empty(r, ransac_n):
        pose[:, 0, 0] = pose[:, 1, 1] = pose[:, 2, 2] = 1.0
        out[:, 4] = -1.0
        return pose, out
    L = _lib.load()
    ms = [int(c.shape[0]) for c in corr_src]
    m = sum(ms)
    ca = torch.empty((max(m, 1), 3), dtype=torch.float64, device=dev)
    cc = torch.empty((max(m, 1), 3), dtype=torch.float64, device=dev)
    mask = None if corr_mask is None else torch.empty(max(m, 1), dtype=torch.uint8, device=dev)
    a = 0
    for b, ln in enumerate(ms):
        ca[a:a + ln].copy_(corr_src[b].to(dev, torch.float64))
        cc[a:a + ln].copy_(corr_tgt[b].to(dev, torch.float64))
        if mask is not None:
            mask[a:a + ln].copy_(corr_mask[b].to(dev) != 0)
        a += ln
    coffs = make_offsets(ms, dev)
    opt = RansacOptions(int(max_iteration), float(confidence), int(ransac_n), float(edge_length or 0.0),
                        float(distance or 0.0), int(seed), int(pair_base), int(first_chunk))
    n = sum(lens)
    own = status is None
    if own:
        status = new_status(dev)
    ws = workspace(L.regtr_ransac_ws_bytes(n, m, B, int(max_iteration), int(first_chunk)), dev)
    state = workspace(L.regtr_icp_state_bytes(n), dev, 'scan_state', zero=True)
    _lib.check(L.regtr_ransac(_p(xyz), _p(offs), B, n, _p(ca), _p(cc), _p(coffs), _p(mask), m, r, overlap_cell(r),
                              ctypes.addressof(opt), _p(pose), _p(out), _p(status), _p(ws), ws.numel(), _p(state),
                              state.numel(), _stream()), 'regtr_ransac')
    _count(ransac_launches(max_iteration, first_chunk))
    if own:
        check_fit_status(status, r, 'ransac')
    return pose, out


def regtr_correspondences(pred, threshold: float = 0.5):
    """The two-way correspondence set of RegTR's weighted Kabsch, from a forward's output `pred`, per pair b:
    the final decoder layer's src_kp -> src_kp_warped followed by tgt_kp_warped -> tgt_kp, and the mask
    sigmoid(overlap) > threshold of the same rows.  -> (corr_src, corr_tgt, corr_mask), B device tensors each
    ((m,3) float32, (m,3) float32, (m,) bool), for `ransac`.  No host sync."""
    corr_src, corr_tgt, corr_mask = [], [], []
    for b in range(len(pred['src_kp'])):
        corr_src.append(torch.cat([pred['src_kp'][b], pred['tgt_kp_warped'][b][-1]], 0))
        corr_tgt.append(torch.cat([pred['src_kp_warped'][b][-1], pred['tgt_kp'][b]], 0))
        logit = torch.cat([pred['src_overlap'][b][-1][:, 0], pred['tgt_overlap'][b][-1][:, 0]], 0)
        corr_mask.append(torch.sigmoid(logit) > threshold)
    return corr_src, corr_tgt, corr_mask


NORMALS_MAX_NN = 64


def normals_launches() -> int:
    """Kernel launches of one `estimate_normals` call: the set-up, the cell list (4), the per-point solve."""
    return 6


def estimate_normals(clouds, radius: float, max_nn: int = 30, status=None, return_counts: bool = False):
    """Normals of C clouds (regtr_estimate_normals): Open3D's estimate_normals(KDTreeSearchParamHybrid(radius,
    max_nn)) oriented towards the origin, with the library's rules (the max_nn nearest points of the own cloud
    strictly within `radius`, the point itself included, ties to the lower index; a zero normal with fewer than 3).
    clouds: C (n,3) clouds (numpy or torch, any float dtype; stacked in float64 on the device).
    -> list of C (n,3) float64 device tensors; with return_counts also the list of (n,) int32 neighbour counts.
    No host sync unless status is None: then a word of this call is read and a coordinate beyond
    `overlap_coord_bound(radius)`, or not finite, raises RegtrLibError; with the caller's word, `check_fit_status`
    does that where the caller syncs."""
    L = _lib.load()
    r = float(radius)
    if not r > 0.0 or not 1 <= int(max_nn) <= NORMALS_MAX_NN:
        raise ValueError(f'estimate_normals: radius {r} must be > 0 and max_nn {max_nn} in 1..{NORMALS_MAX_NN}')
    C = len(clouds)
    if C == 0:
        raise ValueError('estimate_normals: expected at least one cloud')
    ts = [torch.as_tensor(c) for c in clouds]
    for c in ts:
        if c.dim() != 2 or c.shape[1] != 3:
            raise ValueError(f'estimate_normals: expected (n,3) clouds, got {tuple(c.shape)}')
    dev = next((c.device for c in ts if c.is_cuda), torch.device('cuda', torch.cuda.current_device()))
    lens = [int(c.shape[0]) for c in ts]
    n = sum(lens)
    xyz = torch.empty((max(n, 1), 3), dtype=torch.float64, device=dev)
    a = 0
    for c, ln in zip(ts, lens):
        xyz[a:a + ln].copy_(c.to(dev, torch.float64))
        a += ln
    offs = make_offsets(lens, dev)
    own = status is None
    if own:
        status = new_status(dev)
    normals = torch.empty((max(n, 1), 3), dtype=torch.float64, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev) if return_counts else None
    ws = workspace(L.regtr_estimate_normals_ws_bytes(n), dev)
    state = workspace(L.regtr_estimate_normals_state_bytes(n), dev, 'scan_state', zero=True)
    _lib.check(L.regtr_estimate_normals(_p(xyz), _p(offs), C, n, r, overlap_cell(r), int(max_nn), _p(normals),
                                        _p(counts), _p(status), _p(ws), ws.numel(),
                                        _p(state), state.numel(), _stream()), 'regtr_estimate_normals')
    _count(normals_launches())
    if own:
        check_fit_status(status, r, 'estimate_normals')
    bounds = [0]
    for ln in lens:
        bounds.append(bounds[-1] + ln)
    out = [normals[bounds[k]:bounds[k + 1]] for k in range(C)]
    if return_counts:
        return out, [counts[bounds[k]:bounds[k + 1]] for k in range(C)]
    return out


def color_gradients(clouds, normals, colors, radius: float, max_nn: int = 30, status=None):
    """Intensity gradients of C coloured clouds for colored ICP (regtr_color_gradients): Open3D's
    InitializePointCloudForColoredICP(KDTreeSearchParamHybrid(radius, max_nn)) with the library's rules (the
    neighbours of `estimate_normals`; a zero gradient with fewer than 4 neighbours, a zero normal or a failed solve).
    clouds / normals / colors: C (n,3) arrays each, normals from `estimate_normals`, colors rgb; numpy or torch, any
    float dtype, stacked in float64 on the device.  -> list of C (n,3) float64 device tensors.
    No host sync unless status is None: then a word of this call is read and a coordinate beyond
    `overlap_coord_bound(radius)`, or not finite, raises RegtrLibError; with the caller's word, `check_fit_status`
    does that where the caller syncs."""
    r = float(radius)
    if not r > 0.0 or not 1 <= int(max_nn) <= NORMALS_MAX_NN:
        raise ValueError(f'color_gradients: radius {r} must be > 0 and max_nn {max_nn} in 1..{NORMALS_MAX_NN}')
    C = len(clouds)
    if C == 0 or len(normals) != C or len(colors) != C:
        raise ValueError(f'color_gradients: {C} clouds, {len(normals)} normal and {len(colors)} colour arrays; '
                         f'expected as many, at least one')
    ts = [torch.as_tensor(c) for c in clouds]
    ns = [torch.as_tensor(c) for c in normals]
    cs = [torch.as_tensor(c) for c in colors]
    for c, m, k in zip(ts, ns, cs):
        if c.dim() != 2 or c.shape[1] != 3 or tuple(m.shape) != tuple(c.shape) or tuple(k.shape) != tuple(c.shape):
            raise ValueError(f'color_gradients: cloud {tuple(c.shape)}, normals {tuple(m.shape)} and colors '
                             f'{tuple(k.shape)}, expected three (n,3) arrays')
    L = _lib.load()
    dev = next((c.device for c in ts + ns + cs if c.is_cuda), torch.device('cuda', torch.cuda.current_device()))
    xyz, lens = _stack_clouds(ts, dev, 3, 'color_gradients')
    nrm, _ = _stack_clouds(ns, dev, 3, 'color_gradients')
    rgb, _ = _stack_clouds(cs, dev, 3, 'color_gradients')
    n = sum(lens)
    offs = make_offsets(lens, dev)
    own = status is None
    if own:
        status = new_status(dev)
    grad = torch.empty((max(n, 1), 3), dtype=torch.float64, device=dev)
    ws = workspace(L.regtr_color_gradients_ws_bytes(n), dev)
    state = workspace(L.regtr_color_gradients_state_bytes(n), dev, 'scan_state', zero=True)
    _lib.check(L.regtr_color_gradients(_p(xyz), _p(nrm), _p(rgb), _p(offs), C, n, r, overlap_cell(r), int(max_nn),
                                       _p(grad), _p(status), _p(ws), ws.numel(), _p(state), state.numel(), _stream()),
               'regtr_color_gradients')
    _count(normals_launches())
    if own:
        check_fit_status(status, r, 'color_gradients')
    return _split(grad, lens)


FPFH_DIM = 33                       # REGTR_FPFH_DIM
FPFH_MAX_NN = 128                   # REGTR_FPFH_MAX_NN


def fpfh_launches() -> int:
    """Kernel launches of one `fpfh` call: the set-up, the cell list (4), neighbour lists, SPFH and FPFH."""
    return 8


def feature_match_launches() -> int:
    """Kernel launches of one `feature_match` call: the distance sweep, the reduction of its partial minima and the
    mutual filter."""
    return 3


def _stack_clouds(ts, dev, width, what):
    """C (n,width) arrays stacked in float64 on the device -> (stacked (max(n,1),width), lens)."""
    lens = [int(c.shape[0]) for c in ts]
    out = torch.empty((max(sum(lens), 1), width), dtype=torch.float64, device=dev)
    a = 0
    for c, ln in zip(ts, lens):
        out[a:a + ln].copy_(c.to(dev, torch.float64))
        a += ln
    return out, lens


def _split(t, lens):
    bounds = np.concatenate([[0], np.cumsum(lens)]).astype(int)
    return [t[bounds[k]:bounds[k + 1]] for k in range(len(lens))]


def fpfh(clouds, normals, radius: float, max_nn: int = 100, status=None, return_counts: bool = False):
    """FPFH features of C clouds (regtr_fpfh): Open3D's compute_fpfh_feature(KDTreeSearchParamHybrid(radius, max_nn))
    with the library's rules (include/regtr_b200.h, tests/fpfh_oracle.py).
    clouds / normals: C (n,3) arrays each, normals aligned with their cloud (e.g. `estimate_normals`), numpy or torch,
    any float dtype; stacked in float64 on the device.
    -> list of C (n,33) float64 device tensors; with return_counts also the list of (n,) int32 neighbour counts.
    No host sync unless status is None: then a word of this call is read and a coordinate beyond
    `overlap_coord_bound(radius)`, or not finite, raises RegtrLibError; with the caller's word, `check_fit_status`
    does that where the caller syncs."""
    r = float(radius)
    if not r > 0.0 or not 1 <= int(max_nn) <= FPFH_MAX_NN:
        raise ValueError(f'fpfh: radius {r} must be > 0 and max_nn {max_nn} in 1..{FPFH_MAX_NN}')
    C = len(clouds)
    if C == 0 or len(normals) != C:
        raise ValueError(f'fpfh: {C} clouds and {len(normals)} normal arrays; expected as many, at least one')
    ts = [torch.as_tensor(c) for c in clouds]
    ns = [torch.as_tensor(c) for c in normals]
    for c, m in zip(ts, ns):
        if c.dim() != 2 or c.shape[1] != 3 or tuple(m.shape) != tuple(c.shape):
            raise ValueError(f'fpfh: cloud {tuple(c.shape)} and normals {tuple(m.shape)}, expected two (n,3) arrays')
    L = _lib.load()
    dev = next((c.device for c in ts + ns if c.is_cuda), torch.device('cuda', torch.cuda.current_device()))
    xyz, lens = _stack_clouds(ts, dev, 3, 'fpfh')
    nrm, _ = _stack_clouds(ns, dev, 3, 'fpfh')
    n = sum(lens)
    offs = make_offsets(lens, dev)
    own = status is None
    if own:
        status = new_status(dev)
    feat = torch.empty((max(n, 1), FPFH_DIM), dtype=torch.float64, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev) if return_counts else None
    ws = workspace(L.regtr_fpfh_ws_bytes(n, int(max_nn)), dev)
    state = workspace(L.regtr_fpfh_state_bytes(n), dev, 'scan_state', zero=True)
    _lib.check(L.regtr_fpfh(_p(xyz), _p(nrm), _p(offs), C, n, r, overlap_cell(r), int(max_nn), _p(feat), _p(counts),
                            _p(status), _p(ws), ws.numel(), _p(state), state.numel(), _stream()), 'regtr_fpfh')
    _count(fpfh_launches())
    if own:
        check_fit_status(status, r, 'fpfh')
    if return_counts:
        return _split(feat, lens), _split(counts, lens)
    return _split(feat, lens)


def feature_match(src_feat, tgt_feat, tgt_list, mutual_filter: bool = True, min_mutual: int = 9):
    """Feature-space matches of B pairs (regtr_feature_match): src_feat / tgt_feat B (n_s,33) / (n_t,33) arrays,
    tgt_list the B target clouds (n_t,3) (numpy or torch, any float dtype; stacked in float64 on the device).
    -> (nn, corr_tgt, mask, n_mutual): B (n_s,) int32 (the nearest target by (d2, index)), B (n_s,3) float64 (its
    point), B (n_s,) bool (mutual; every match without mutual_filter or below min_mutual mutual matches) and (B,)
    int32 mutual counts, all device tensors.  No host sync."""
    B = len(src_feat)
    if B == 0 or len(tgt_feat) != B or len(tgt_list) != B:
        raise ValueError(f'feature_match: {B} source, {len(tgt_feat)} target feature arrays and {len(tgt_list)} '
                         f'target clouds; expected as many, at least one pair')
    fs = [torch.as_tensor(f) for f in src_feat]
    ft = [torch.as_tensor(f) for f in tgt_feat]
    tx = [torch.as_tensor(c) for c in tgt_list]
    for b in range(B):
        for f in (fs[b], ft[b]):
            if f.dim() != 2 or f.shape[1] != FPFH_DIM:
                raise ValueError(f'feature_match: pair {b}: features {tuple(f.shape)}, expected (n,{FPFH_DIM})')
        if tuple(tx[b].shape) != (ft[b].shape[0], 3):
            raise ValueError(f'feature_match: pair {b}: target cloud {tuple(tx[b].shape)} for '
                             f'{ft[b].shape[0]} target features')
        if fs[b].shape[0] > 0 and ft[b].shape[0] == 0:
            raise ValueError(f'feature_match: pair {b}: a target without points')
    L = _lib.load()
    dev = next((c.device for c in fs + ft + tx if c.is_cuda), torch.device('cuda', torch.cuda.current_device()))
    sf, ls = _stack_clouds(fs, dev, FPFH_DIM, 'feature_match')
    tf, lt = _stack_clouds(ft, dev, FPFH_DIM, 'feature_match')
    txyz, _ = _stack_clouds(tx, dev, 3, 'feature_match')
    ns, nt = sum(ls), sum(lt)
    ns_max, nt_max = max(ls), max(lt)
    nn = torch.empty(max(ns, 1), dtype=torch.int32, device=dev)
    corr = torch.empty((max(ns, 1), 3), dtype=torch.float64, device=dev)
    mask = torch.empty(max(ns, 1), dtype=torch.uint8, device=dev)
    n_mutual = torch.empty(B, dtype=torch.int32, device=dev)
    ws = workspace(L.regtr_feature_match_ws_bytes(B, ns_max, nt_max, nt), dev)
    soffs, toffs = make_offsets(ls, dev), make_offsets(lt, dev)
    _lib.check(L.regtr_feature_match(_p(sf), _p(soffs), _p(tf), _p(txyz), _p(toffs), B, ns_max, nt_max, nt,
                                     int(bool(mutual_filter)), int(min_mutual), _p(nn), _p(corr), _p(mask), _p(n_mutual), _p(ws), ws.numel(), _stream()),
               'regtr_feature_match')
    _count(feature_match_launches())
    return _split(nn, ls), _split(corr, ls), _split(mask.bool(), ls), n_mutual


def feature_correspondences(src_list, tgt_list, src_feat, tgt_feat, mutual_filter: bool = True, ransac_n: int = 3):
    """The correspondences of Open3D's registration_ransac_based_on_feature_matching, in `ransac`'s layout: source
    point i -> its nearest target in feature space (`feature_match`); with mutual_filter only the mutual matches take
    part, unless fewer than 3 ransac_n are mutual (then all do, as in Open3D).
    -> (corr_src, corr_tgt, corr_mask, n_mutual): B (n_s,3) float64, B (n_s,3) float64, B (n_s,) bool device tensors
    and the (B,) int32 device tensor of mutual counts.  No host sync."""
    B = len(src_list)
    if B == 0 or len(tgt_list) != B or len(src_feat) != B or len(tgt_feat) != B:
        raise ValueError(f'feature_correspondences: {B} sources, {len(tgt_list)} targets, {len(src_feat)} / '
                         f'{len(tgt_feat)} feature arrays; expected as many, at least one pair')
    src = [torch.as_tensor(c) for c in src_list]
    for b in range(B):
        if src[b].dim() != 2 or src[b].shape[1] != 3 or src[b].shape[0] != torch.as_tensor(src_feat[b]).shape[0]:
            raise ValueError(f'feature_correspondences: pair {b}: source cloud {tuple(src[b].shape)} for '
                             f'{tuple(torch.as_tensor(src_feat[b]).shape)} source features')
    _, corr_tgt, corr_mask, n_mutual = feature_match(src_feat, tgt_feat, tgt_list, mutual_filter, 3 * int(ransac_n))
    dev = n_mutual.device
    return [c.to(dev, torch.float64) for c in src], corr_tgt, corr_mask, n_mutual


def ransac_feature_matching(src_list, tgt_list, src_feat, tgt_feat, mutual_filter: bool,
                            max_correspondence_distance: float, ransac_n: int = 3, **ransac_kwargs):
    """Open3D's registration_ransac_based_on_feature_matching for B pairs: `feature_correspondences`, then `ransac`
    over them (validated on src_list / tgt_list, the clouds the features describe) with max_correspondence_distance,
    ransac_n and ransac_kwargs (max_iteration, confidence, edge_length, distance, seed, ...).
    -> (pose (B,3,4), result (B,5), n_mutual (B,)): `ransac`'s outputs and the mutual counts.  Arguments `ransac`
    would reject raise ValueError before any launch."""
    a = inspect.signature(ransac).bind(src_list, tgt_list, src_list, src_list, max_correspondence_distance,
                                       ransac_n=ransac_n, **ransac_kwargs)
    a.apply_defaults()
    a = a.arguments
    src = [torch.as_tensor(c) for c in src_list]
    _ransac_check(len(src), src, src, None, a['max_iteration'], a['confidence'], a['ransac_n'], a['edge_length'],
                  a['distance'], a['seed'], a['pair_base'], a['first_chunk'])
    corr_src, corr_tgt, corr_mask, n_mutual = feature_correspondences(src_list, tgt_list, src_feat, tgt_feat,
                                                                      mutual_filter, ransac_n)
    pose, out = ransac(src_list, tgt_list, corr_src, corr_tgt, max_correspondence_distance, ransac_n=ransac_n,
                       corr_mask=corr_mask, **ransac_kwargs)
    return pose, out, n_mutual


FGR_MAX_CORR = 21474836             # REGTR_FGR_MAX_CORR
FGR_MAX_TUPLES = 1 << 20            # REGTR_FGR_MAX_TUPLES


class FgrOptions(ctypes.Structure):
    """regtr_fgr_options (include/regtr_b200.h)."""
    _fields_ = [('division_factor', ctypes.c_double), ('use_absolute_scale', ctypes.c_int),
                ('decrease_mu', ctypes.c_int), ('maximum_correspondence_distance', ctypes.c_double),
                ('iteration_number', ctypes.c_int), ('tuple_scale', ctypes.c_double),
                ('maximum_tuple_count', ctypes.c_int), ('tuple_test', ctypes.c_int), ('seed', ctypes.c_ulonglong),
                ('pair_base', ctypes.c_int)]


def fgr_launches() -> int:
    """Kernel launches of one `fgr` call: the preparation (means, scale, compaction, tuple test) and the solve."""
    return 2


def _fgr_check(B, corr_src, corr_tgt, corr_mask, maximum_correspondence_distance, iteration_number, division_factor,
               tuple_scale, maximum_tuple_count, seed, pair_base):
    """ValueError for every argument `fgr` rejects, before anything touches the device."""
    def real(v):
        return isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, bool)

    def integer(v):
        return real(v) and int(v) == v
    if len(corr_src) != B or len(corr_tgt) != B:
        raise ValueError(f'fgr: {len(corr_src)} / {len(corr_tgt)} correspondence arrays for {B} pairs')
    if corr_mask is not None and len(corr_mask) != B:
        raise ValueError(f'fgr: {len(corr_mask)} correspondence masks for {B} pairs')
    m = 0
    for b in range(B):
        a, c = corr_src[b], corr_tgt[b]
        if len(a.shape) != 2 or a.shape[1] != 3 or tuple(a.shape) != tuple(c.shape):
            raise ValueError(f'fgr: pair {b}: correspondences {tuple(a.shape)} and {tuple(c.shape)}, expected two '
                             f'(m,3) arrays')
        if corr_mask is not None and tuple(corr_mask[b].shape) != (a.shape[0],):
            raise ValueError(f'fgr: pair {b}: mask {tuple(corr_mask[b].shape)} for {a.shape[0]} correspondences')
        m += int(a.shape[0])
    if m > FGR_MAX_CORR:
        raise ValueError(f'fgr: {m} correspondences in all, at most {FGR_MAX_CORR}')
    for name, v in (('maximum_correspondence_distance', maximum_correspondence_distance),
                    ('division_factor', division_factor)):
        if not (real(v) and math.isfinite(float(v)) and float(v) > 0.0):
            raise ValueError(f'fgr: {name} {v!r} must be a finite value > 0')
    if not (integer(iteration_number) and 0 <= int(iteration_number) < 2 ** 31):
        raise ValueError(f'fgr: iteration_number {iteration_number!r} must be an integer >= 0')
    if not (real(tuple_scale) and 0.0 < float(tuple_scale) <= 1.0):
        raise ValueError(f'fgr: tuple_scale {tuple_scale!r} must be in (0, 1]')
    if not (integer(maximum_tuple_count) and 1 <= int(maximum_tuple_count) <= FGR_MAX_TUPLES):
        raise ValueError(f'fgr: maximum_tuple_count {maximum_tuple_count!r} must be an integer in 1..{FGR_MAX_TUPLES}')
    if not (integer(seed) and 0 <= int(seed) < 2 ** 64):
        raise ValueError(f'fgr: seed {seed!r} must be an integer in [0, 2^64)')
    if not (integer(pair_base) and 0 <= int(pair_base) <= 2 ** 31 - 1 - B):
        raise ValueError(f'fgr: pair_base {pair_base!r} must be an integer in [0, 2^31 - 1 - B]')


def fgr(src_list, tgt_list, corr_src, corr_tgt, corr_mask=None, *, maximum_correspondence_distance: float = 0.025,
        iteration_number: int = 64, division_factor: float = 1.4, decrease_mu: bool = True,
        use_absolute_scale: bool = False, tuple_test: bool = False, tuple_scale: float = 0.95,
        maximum_tuple_count: int = 1000, seed: int = 0, pair_base: int = 0):
    """Fast Global Registration of B pairs over correspondences (regtr_fgr): Open3D's
    registration_fgr_based_on_correspondence with FastGlobalRegistrationOption, with the library's deterministic rule
    (include/regtr_b200.h, tests/fgr_oracle.py).  Open3D runs no tuple test on given correspondences, hence
    tuple_test=False by default here.
    src_list / tgt_list: B clouds (n,3) each, whose means and scale normalise the problem (numpy or torch, any float
    dtype; stacked in float64 on the device).  corr_src / corr_tgt: B (m,3) arrays each, correspondence i of pair b
    being corr_src[b][i] -> corr_tgt[b][i]; corr_mask: None or B (m,) boolean arrays, the correspondences that take
    part.  seed and pair_base + b key the tuple draws, so a pair gets the same result alone or in a batch.
    -> (pose (B,3,4) float64 source -> target, result (B,4) float64 = correspondences entering the solve, tuples kept,
    trials walked, final par), both device tensors.  Fewer than 10 correspondences give the identity.  No host sync.
    Bad arguments raise ValueError before any launch."""
    B = len(src_list)
    if B == 0 or len(tgt_list) != B:
        raise ValueError('fgr: expected as many source as target clouds, at least one pair')
    corr_src = [torch.as_tensor(c) for c in corr_src]
    corr_tgt = [torch.as_tensor(c) for c in corr_tgt]
    corr_mask = None if corr_mask is None else [torch.as_tensor(m) for m in corr_mask]
    _fgr_check(B, corr_src, corr_tgt, corr_mask, maximum_correspondence_distance, iteration_number, division_factor,
               tuple_scale, maximum_tuple_count, seed, pair_base)
    L = _lib.load()
    dev = next((c.device for c in corr_src if c.is_cuda), None)
    xyz, offs, lens = _stack_pairs(src_list, tgt_list, 'fgr', dev)
    dev = xyz.device
    ca, ms = _stack_clouds(corr_src, dev, 3, 'fgr')
    cc, _ = _stack_clouds(corr_tgt, dev, 3, 'fgr')
    m = sum(ms)
    mask = None
    if corr_mask is not None:
        mask = torch.zeros(max(m, 1), dtype=torch.uint8, device=dev)
        a = 0
        for b, ln in enumerate(ms):
            mask[a:a + ln].copy_(corr_mask[b].to(dev) != 0)
            a += ln
    coffs = make_offsets(ms, dev)
    opt = FgrOptions(float(division_factor), int(bool(use_absolute_scale)), int(bool(decrease_mu)),
                     float(maximum_correspondence_distance), int(iteration_number), float(tuple_scale),
                     int(maximum_tuple_count), int(bool(tuple_test)), int(seed), int(pair_base))
    pose = torch.empty((B, 3, 4), dtype=torch.float64, device=dev)
    out = torch.empty((B, 4), dtype=torch.float64, device=dev)
    ws = workspace(L.regtr_fgr_ws_bytes(m, B, int(maximum_tuple_count)), dev)
    _lib.check(L.regtr_fgr(_p(xyz), _p(offs), B, sum(lens), _p(ca), _p(cc), _p(coffs), _p(mask), m,
                           ctypes.addressof(opt), _p(pose), _p(out), _p(ws), ws.numel(), _stream()), 'regtr_fgr')
    _count(fgr_launches())
    return pose, out


def fgr_feature_matching(src_list, tgt_list, src_feat, tgt_feat, **fgr_kwargs):
    """Open3D's registration_fgr_based_on_feature_matching for B pairs: the mutual matches of `feature_match` (its
    cross check; no fallback), source point i -> its nearest target in feature space, in source order, then `fgr` over
    them with fgr_kwargs (tuple_test defaults to True here, as in Open3D).
    -> (pose (B,3,4), result (B,4), n_mutual (B,)): `fgr`'s outputs and the mutual counts.  Arguments `fgr` would
    reject raise ValueError before any launch."""
    fgr_kwargs = dict(fgr_kwargs)
    fgr_kwargs.setdefault('tuple_test', True)
    B = len(src_list)
    if B == 0 or len(tgt_list) != B or len(src_feat) != B or len(tgt_feat) != B:
        raise ValueError(f'fgr_feature_matching: {B} sources, {len(tgt_list)} targets, {len(src_feat)} / '
                         f'{len(tgt_feat)} feature arrays; expected as many, at least one pair')
    a = inspect.signature(fgr).bind(src_list, tgt_list, src_list, src_list, **fgr_kwargs)
    a.apply_defaults()
    a = a.arguments
    src = [torch.as_tensor(c) for c in src_list]
    for b in range(B):
        if src[b].dim() != 2 or src[b].shape[1] != 3 or src[b].shape[0] != torch.as_tensor(src_feat[b]).shape[0]:
            raise ValueError(f'fgr_feature_matching: pair {b}: source cloud {tuple(src[b].shape)} for '
                             f'{tuple(torch.as_tensor(src_feat[b]).shape)} source features')
    _fgr_check(B, src, src, None, a['maximum_correspondence_distance'], a['iteration_number'],
               a['division_factor'], a['tuple_scale'], a['maximum_tuple_count'], a['seed'], a['pair_base'])
    _, corr_tgt, corr_mask, n_mutual = feature_match(src_feat, tgt_feat, tgt_list, True, 0)
    dev = n_mutual.device
    pose, out = fgr(src_list, tgt_list, [c.to(dev, torch.float64) for c in src], corr_tgt, corr_mask, **fgr_kwargs)
    return pose, out, n_mutual


def registration_information(src_list, tgt_list, pose, radius: float, status=None):
    """Fit and information matrices of B registered pairs from one `overlap_nn` (regtr_registration_fit and
    regtr_registration_information on the same matches): Open3D's evaluate_registration and
    get_information_matrix_from_point_clouds at `radius`.  Arguments as `registration_fit`.
    -> (fit (B,4) float64 = fitness_src, rmse_src, fitness_tgt, rmse_tgt; info (B,6,6) float64, info[:,5,5] the match
    count), both device tensors.  status: as in `registration_fit`."""
    L = _lib.load()
    B = len(src_list)
    dev = pose.device if torch.is_tensor(pose) and pose.is_cuda else None
    xyz, offs, lens = _stack_pairs(src_list, tgt_list, 'registration_information', dev)
    dev = xyz.device
    n = sum(lens)
    pose64 = torch.as_tensor(pose).to(dev, torch.float64).reshape(B, 3, 4).contiguous()
    own = status is None
    if own:
        status = new_status(dev)
    nn = overlap_nn(xyz[:n], offs, B, pose64, radius, status)
    fit = torch.empty((B, 4), dtype=torch.float64, device=dev)
    info = torch.empty((B, 6, 6), dtype=torch.float64, device=dev)
    _lib.check(L.regtr_registration_fit(_p(xyz), _p(offs), B, n, _p(pose64), float(radius), _p(nn), _p(fit),
                                        _p(status), _stream()), 'regtr_registration_fit')
    _lib.check(L.regtr_registration_information(_p(xyz), _p(offs), B, n, _p(pose64), float(radius), _p(nn), _p(info),
                                                _p(status), _stream()), 'regtr_registration_information')
    _count(2)
    if own:
        check_fit_status(status, radius, 'registration_information')
    return fit, info


def transform_clouds(clouds, poses):
    """C clouds (n,3) each moved by one (3,4) or (4,4) pose each, in float64 on the device (regtr_transform_clouds).
    -> ((n_total,3) float32 device tensor of the stacked moved clouds, offs (C+1) int32)."""
    L = _lib.load()
    C = len(clouds)
    if C == 0:
        raise ValueError('transform_clouds: expected at least one cloud')
    dev = torch.device('cuda', torch.cuda.current_device())
    ts = [torch.as_tensor(c) for c in clouds]
    lens = [int(c.shape[0]) for c in ts]
    xyz = torch.empty((max(sum(lens), 1), 3), dtype=torch.float64, device=dev)
    a = 0
    for c, ln in zip(ts, lens):
        xyz[a:a + ln].copy_(c.reshape(ln, 3).to(dev, torch.float64))
        a += ln
    offs = make_offsets(lens, dev)
    n = sum(lens)
    p = torch.as_tensor(poses).to(dev, torch.float64)[:, :3, :4].contiguous()
    if p.shape[0] != C:
        raise ValueError(f'transform_clouds: {p.shape[0]} poses for {C} clouds')
    out = torch.empty((max(n, 1), 3), dtype=torch.float32, device=dev)
    _lib.check(L.regtr_transform_clouds(_p(xyz), _p(offs), C, n, _p(p), _p(out), _stream()), 'regtr_transform_clouds')
    _count(1 if n > 0 else 0)
    return out[:n], offs


class PoseGraphOptions(ctypes.Structure):
    """regtr_pose_graph_options."""
    _fields_ = [('max_correspondence_distance', ctypes.c_double), ('edge_prune_threshold', ctypes.c_double),
                ('preference_loop_closure', ctypes.c_double), ('min_relative_increment', ctypes.c_double),
                ('min_relative_residual_increment', ctypes.c_double), ('min_right_term', ctypes.c_double),
                ('min_residual', ctypes.c_double), ('upper_scale_factor', ctypes.c_double),
                ('lower_scale_factor', ctypes.c_double), ('reference_node', ctypes.c_int32),
                ('max_iteration', ctypes.c_int32), ('max_iteration_lm', ctypes.c_int32)]


POSE_GRAPH_MAX_NODES = 256                                                  # REGTR_POSE_GRAPH_MAX_NODES


def pose_graph_optimize(poses, edges, transformation, information, uncertain, max_correspondence_distance: float,
                        edge_prune_threshold: float = 0.25, preference_loop_closure: float = 1.0,
                        reference_node: int = 0, max_iteration: int = 100, max_iteration_lm: int = 20,
                        min_relative_increment: float = 1e-6, min_relative_residual_increment: float = 1e-6,
                        min_right_term: float = 1e-6, min_residual: float = 1e-6,
                        upper_scale_factor: float = 2.0 / 3.0, lower_scale_factor: float = 1.0 / 3.0, status=None):
    """Robust optimisation of G pose graphs in one launch (regtr_pose_graph_optimize: Open3D's global_optimization with
    GlobalOptimizationLevenbergMarquardt and its two passes).  Lists of G entries each: poses (N_g,3,4) or (N_g,4,4)
    fragment -> world initial poses; edges (E_g,2) int (source, target) node indices; transformation (E_g,3,4) or
    (E_g,4,4) source -> target; information (E_g,6,6); uncertain (E_g,) bool (loop closures).
    -> (poses list of (N_g,3,4) float64, confidence list of (E_g,) float64, kept list of (E_g,) bool,
    result (G,4) float64 = pass-1 iterations, pass-2 iterations, final objective, edges kept), all device tensors.
    A graph above POSE_GRAPH_MAX_NODES nodes raises RegtrLibError (REGTR_ERR_UNSUPPORTED).  No host sync unless status
    is None: then a word of this call is read and a rejected graph (s = t, an index out of range, a non-finite input)
    raises RegtrLibError; with the caller's word the caller checks REGTR_STATUS_INPUT (`STATUS_INPUT`)."""
    L = _lib.load()
    G = len(poses)
    if G == 0 or not (len(edges) == len(transformation) == len(information) == len(uncertain) == G):
        raise ValueError('pose_graph_optimize: expected G >= 1 graphs with poses, edges, transformation, information '
                         'and uncertain each')
    dev = torch.device('cuda', torch.cuda.current_device())

    def cat(items, tail, dtype):
        ts = [torch.as_tensor(x).to(dev, dtype) for x in items]
        ts = [t.reshape((-1,) + t.shape[-len(tail):] if tail else (-1,)) for t in ts]
        ts = [t[(slice(None),) + tuple(slice(0, k) for k in tail)] for t in ts]       # (4,4) -> its (3,4) rows
        return torch.cat(ts).contiguous()

    n_nodes = [int(torch.as_tensor(p).shape[0]) for p in poses]
    n_edges = [int(torch.as_tensor(e).reshape(-1, 2).shape[0]) for e in edges]
    P = cat(poses, (3, 4), torch.float64)
    Ed = cat(edges, (2,), torch.int32)
    X = cat(transformation, (3, 4), torch.float64)
    I6 = cat(information, (6, 6), torch.float64)
    U = cat([torch.as_tensor(u).bool() for u in uncertain], (), torch.uint8)
    for name, t, want in (('transformation', X, n_edges), ('information', I6, n_edges), ('uncertain', U, n_edges)):
        if t.shape[0] != sum(want):
            raise ValueError(f'pose_graph_optimize: {name} has {t.shape[0]} rows for {sum(want)} edges')
    N, E = sum(n_nodes), sum(n_edges)
    max_nodes = max(n_nodes)
    node_offs, edge_offs = make_offsets(n_nodes, dev), make_offsets(n_edges, dev)
    opt = PoseGraphOptions(float(max_correspondence_distance), float(edge_prune_threshold),
                           float(preference_loop_closure), float(min_relative_increment),
                           float(min_relative_residual_increment), float(min_right_term), float(min_residual),
                           float(upper_scale_factor), float(lower_scale_factor), int(reference_node),
                           int(max_iteration), int(max_iteration_lm))
    conf = torch.empty(max(E, 1), dtype=torch.float64, device=dev)
    kept = torch.empty(max(E, 1), dtype=torch.uint8, device=dev)
    result = torch.empty((G, 4), dtype=torch.float64, device=dev)
    P = P if N > 0 else torch.empty((1, 3, 4), dtype=torch.float64, device=dev)
    own = status is None
    if own:
        status = new_status(dev)
    sq_nodes = sum(k * k for k in n_nodes) if max_nodes <= POSE_GRAPH_MAX_NODES else 0
    ws = workspace(max(L.regtr_pose_graph_ws_bytes(G, N, E, sq_nodes), 1), dev)
    _lib.check(L.regtr_pose_graph_optimize(_p(node_offs), _p(edge_offs), G, N, E, max_nodes, sq_nodes, _p(P), _p(Ed),
                                           _p(X), _p(I6), _p(U), ctypes.byref(opt), _p(conf), _p(kept), _p(result),
                                           _p(status), _p(ws), ws.numel(), _stream()), 'regtr_pose_graph_optimize')
    _count(1)
    if own and int(status.item()) & STATUS_INPUT:
        raise _lib.RegtrLibError('pose_graph_optimize: a graph was rejected (s = t, a node index or the reference node '
                                 'out of range, or a non-finite pose, transformation or information)')
    nb, eb = np.concatenate([[0], np.cumsum(n_nodes)]), np.concatenate([[0], np.cumsum(n_edges)])
    return ([P[nb[k]:nb[k + 1]] for k in range(G)], [conf[eb[k]:eb[k + 1]] for k in range(G)],
            [kept[eb[k]:eb[k + 1]].bool() for k in range(G)], result)


def check_fit_status(status, radius: float, what: str = 'registration_fit'):
    """Read the status word of `registration_fit` or `icp` (a host sync) and raise RegtrLibError if the result is not
    exact."""
    word = int(status.item())
    if word & (STATUS_RANGE | 1):             # REGTR_STATUS_RANGE | REGTR_STATUS_KEY_RANGE
        raise _lib.RegtrLibError(
            f'{what}: a coordinate of the moved source or of the target lies beyond +-'
            f'{overlap_coord_bound(radius):.3f} (overlap_coord_bound({radius})), the range in which the nearest-'
            f'neighbour search at this radius is exact, or is not finite (status {word:#x})')
    if word & STATUS_INPUT:                   # REGTR_STATUS_INPUT (defined below)
        raise _lib.RegtrLibError(f'{what}: a match the overlap search cannot have produced (status {word:#x})')


def train_augment(xyz, offs, B: int, n_src: int, pose, nn, pert, flags, seed: int, step: int, noise: float,
                  max_pts: int, out_offs, out_total: int, pair_base: int = 0):
    """The augmentations of regtr_train_augment on the clouds / overlap of `overlap_nn`; the device draws of pair b
    are keyed by pair_base + b.
    -> (out_xyz (out_total,3) f32, out_mask (out_total,) bool, out_pose (B,3,4) f32, corr (2, n_src) i32,
        corr_offs (B+1) i32).  No host sync."""
    L = _lib.load()
    _chk(xyz, torch.float64, 'xyz', 2); _chk(pose, torch.float64, 'pose', 3); _chk(pert, torch.float64, 'pert', 3)
    _chk(flags, torch.int32, 'flags', 1); _chk(out_offs, torch.int32, 'out_offs', 1); _chk(nn, torch.int32, 'nn', 1)
    dev = xyz.device
    out_xyz = torch.empty((out_total, 3), dtype=torch.float32, device=dev)
    out_mask = torch.empty(out_total, dtype=torch.bool, device=dev)
    out_pose = torch.empty((B, 3, 4), dtype=torch.float32, device=dev)
    corr = torch.empty((2, max(n_src, 1)), dtype=torch.int32, device=dev)
    corr_offs = torch.empty(B + 1, dtype=torch.int32, device=dev)
    ws = workspace(L.regtr_train_augment_ws_bytes(n_src, B), dev)
    state = workspace(L.regtr_train_augment_state_bytes(n_src), dev, 'scan_state', zero=True)
    _lib.check(L.regtr_train_augment(_p(xyz), _p(offs), B, n_src, _p(pose), _p(nn), _p(pert), _p(flags),
                                     int(seed) & (2**64 - 1), int(step) & (2**64 - 1), int(pair_base), float(noise),
                                     int(max_pts), _p(out_offs), out_total, _p(out_xyz), _p(out_mask), _p(out_pose),
                                     _p(corr), corr.shape[1], _p(corr_offs), _p(ws), ws.numel(), _p(state),
                                     state.numel(), _stream()), 'regtr_train_augment')
    _count(5 if out_total > 0 else 4)
    return out_xyz, out_mask, out_pose, corr, corr_offs


# --------------------------------------------------------------------------- training-loop bookkeeping

METER_MAX_KEYS, METER_MAX_BANKS = 16, 4                                   # REGTR_METER_MAX_*
METER_ARGS = np.dtype([('vals', '<u8', (METER_MAX_KEYS,)), ('banks', '<u8', (METER_MAX_BANKS,)), ('smooth', '<u8'),
                       ('log', '<u8'), ('step', '<i8'), ('n_keys', '<i4'), ('n_banks', '<i4'), ('total_key', '<i4'),
                       ('log_cap', '<i4')])
POSE_ERR_ARGS = np.dtype([('pred', '<u8'), ('gt', '<u8'), ('rot_hist', '<u8'), ('trans_hist', '<u8'), ('acc', '<u8'),
                          ('thresh_rot', '<f8'), ('thresh_trans', '<f8'), ('L', '<i4'), ('B', '<i4'),
                          ('offset', '<i4'), ('hist_cap', '<i4')])
assert (METER_ARGS.itemsize, POSE_ERR_ARGS.itemsize) == (200, 72)        # the C structs' sizes


def meter_update(vals, banks, step: int, total_key: int = -1, smooth=None, log=None):
    """One step's loss values into meter banks (regtr_meter_update): vals, a list of 0-d fp32 CUDA tensors (one per
    key, in the banks' key order); banks, (n_keys, 4) fp64 tensors (val, sum, sq_sum, count); smooth (2,) fp64 and
    log (1 + capacity,) int64 for the EMA of vals[total_key].  One launch, no host sync."""
    L = _lib.load()
    if not 1 <= len(vals) <= METER_MAX_KEYS or len(banks) > METER_MAX_BANKS:
        raise ValueError(f'meter_update: {len(vals)} keys, {len(banks)} banks (at most {METER_MAX_KEYS}, '
                         f'{METER_MAX_BANKS})')
    a = np.zeros((), METER_ARGS)
    for k, v in enumerate(vals):
        if v.numel() != 1:
            raise ValueError('meter_update: every value must be a single element')
        _chk(v, torch.float32, 'meter value')
        a['vals'][k] = v.data_ptr()
    for b, t in enumerate(banks):
        _chk(t, torch.float64, 'meter bank', 2)
        if tuple(t.shape) != (len(vals), 4):
            raise ValueError(f'meter bank: expected ({len(vals)}, 4), got {tuple(t.shape)}')
        a['banks'][b] = t.data_ptr()
    if smooth is not None:
        _chk(smooth, torch.float64, 'smooth', 1)
    if log is not None:
        _chk(log, torch.int64, 'log', 1)
    a['smooth'], a['log'] = _p(smooth) or 0, _p(log) or 0
    a['step'], a['n_keys'], a['n_banks'] = int(step), len(vals), len(banks)
    a['total_key'] = int(total_key) if smooth is not None else -1
    a['log_cap'] = log.numel() - 1 if log is not None else 0
    _lib.check(L.regtr_meter_update(a.ctypes.data, _stream()), 'regtr_meter_update')
    _count(1)


def pose_errors(pred, gt, rot_hist, trans_hist, acc, offset: int, thresh_rot: float, thresh_trans: float):
    """Pose errors of one validation batch (regtr_pose_errors): pred (L,B,3,4) and gt (B,3,4) fp32; writes
    rot_hist / trans_hist (L, cap) fp64 at columns [offset, offset + B) and accumulates acc (L, 4) fp64
    (sum rot, sum trans, n_success, n).  One launch, no host sync."""
    L_ = _lib.load()
    _chk(pred, torch.float32, 'pred', 4); _chk(gt, torch.float32, 'gt', 3)
    _chk(rot_hist, torch.float64, 'rot_hist', 2); _chk(trans_hist, torch.float64, 'trans_hist', 2)
    _chk(acc, torch.float64, 'acc', 2)
    nl, B = pred.shape[0], pred.shape[1]
    if tuple(pred.shape[2:]) != (3, 4) or tuple(gt.shape) != (B, 3, 4):
        raise ValueError(f'pose_errors: pred {tuple(pred.shape)}, gt {tuple(gt.shape)}')
    if tuple(acc.shape) != (nl, 4) or rot_hist.shape != trans_hist.shape or rot_hist.shape[0] != nl:
        raise ValueError('pose_errors: history / accumulator shapes do not match the layers')
    a = np.zeros((), POSE_ERR_ARGS)
    a['pred'], a['gt'], a['rot_hist'], a['trans_hist'], a['acc'] = (
        pred.data_ptr(), gt.data_ptr(), rot_hist.data_ptr(), trans_hist.data_ptr(), acc.data_ptr())
    a['thresh_rot'], a['thresh_trans'] = float(thresh_rot), float(thresh_trans)
    a['L'], a['B'], a['offset'], a['hist_cap'] = nl, B, int(offset), rot_hist.shape[1]
    _lib.check(L_.regtr_pose_errors(a.ctypes.data, _stream()), 'regtr_pose_errors')
    _count(1 if B else 0)


# --------------------------------------------------------------------------- training data (ModelNet40)

STATUS_INPUT, STATUS_CROP = 16, 32                                        # REGTR_STATUS_INPUT / _CROP
MODELNET_MAX_PTS, MODELNET_PARAMS = 2048, 18                              # REGTR_MODELNET_*
MODELNET_ARGS = np.dtype([('shapes', '<u8'), ('params', '<u8'), ('items', '<u8'), ('out_xyz', '<u8'),
                          ('out_mask', '<u8'), ('corr', '<u8'), ('corr_n', '<u8'), ('status', '<u8'), ('seed', '<u8'),
                          ('step', '<u8'), ('gamma', '<f8'), ('noise', '<f8'), ('clip', '<f8'), ('n_shapes', '<i4'),
                          ('n_pts', '<i4'), ('n_out', '<i4'), ('k', '<i4'), ('B', '<i4')], align=True)
assert MODELNET_ARGS.itemsize == 128                                      # the C struct's size


def modelnet_augment(shapes, params, items, seed: int, step: int, k: int, gamma: float, noise: float, clip: float,
                     n_out: int, status, pair_base: int = 0):
    """The ModelNet crop chain of B pairs (regtr_modelnet_augment): shapes (S, n_pts, 3) fp32; params
    (B, MODELNET_PARAMS) fp64 = crop direction of the source, of the target, the source's 3x4 transform; items (B)
    int32 shape indices.  -> (out_xyz (2B, n_out, 3) f32, out_mask (2B, n_out) bool, corr (B, 2, n_out) i32,
    corr_n (B,) i32).  The device draws of pair b are keyed by pair_base + b.  One launch, no host sync."""
    L = _lib.load()
    _chk(shapes, torch.float32, 'shapes', 3); _chk(params, torch.float64, 'params', 2); _chk(items, torch.int32, 'items', 1)
    _chk(status, torch.int32, 'status', 1)
    B = items.shape[0]
    if tuple(params.shape) != (B, MODELNET_PARAMS):
        raise ValueError(f'modelnet_augment: params {tuple(params.shape)}, expected ({B}, {MODELNET_PARAMS})')
    dev = shapes.device
    out_xyz = torch.empty((2 * B, n_out, 3), dtype=torch.float32, device=dev)
    out_mask = torch.empty((2 * B, n_out), dtype=torch.bool, device=dev)
    corr = torch.empty((B, 2, n_out), dtype=torch.int32, device=dev)
    corr_n = torch.empty(B, dtype=torch.int32, device=dev)
    a = np.zeros((), MODELNET_ARGS)
    for f, t in (('shapes', shapes), ('params', params), ('items', items), ('out_xyz', out_xyz), ('out_mask', out_mask),
                 ('corr', corr), ('corr_n', corr_n), ('status', status)):
        a[f] = t.data_ptr()
    a['seed'], a['step'] = int(seed) & (2**64 - 1), int(step) & (2**64 - 1)
    a['gamma'], a['noise'], a['clip'] = float(gamma), float(noise), float(clip)
    a['n_shapes'], a['n_pts'], a['n_out'], a['k'], a['B'] = shapes.shape[0], shapes.shape[1], int(n_out), int(k), B
    _lib.check(L.regtr_modelnet_augment(a.ctypes.data, int(pair_base), _stream()), 'regtr_modelnet_augment')
    _count(1)
    return out_xyz, out_mask, corr, corr_n


# --------------------------------------------------------------------------- training losses

LOSS_DIM, LOSS_MAX_LEVELS, LOSS_MAX_LAYERS, LOSS_MAX_TERMS = 256, 8, 8, 8              # REGTR_LOSS_*
OVERLAP_PYR_ARGS = np.dtype([('pyr', '<u8', (LOSS_MAX_LEVELS,)), ('pool', '<u8', (LOSS_MAX_LEVELS,)),
                             ('n_prev', '<u8', (LOSS_MAX_LEVELS,)), ('n', '<i4', (LOSS_MAX_LEVELS,)),
                             ('K', '<i4', (LOSS_MAX_LEVELS,)), ('n_levels', '<i4')], align=True)
LOSS_ARGS = np.dtype([('xyz', '<u8'), ('offs', '<u8'), ('pose', '<u8'), ('w', '<u8'), ('logit', '<u8'), ('corr', '<u8'),
                      ('dlogit', '<u8'), ('dcorr', '<u8'), ('dlogit_out', '<u8'), ('dcorr_out', '<u8'),
                      ('q', '<u8', (LOSS_MAX_TERMS,)), ('feat', '<u8', (LOSS_MAX_TERMS,)),
                      ('dq', '<u8', (LOSS_MAX_TERMS,)), ('dfeat', '<u8', (LOSS_MAX_TERMS,)), ('src_gt', '<u8'),
                      ('pos', '<u8'), ('anchor', '<u8'), ('lse', '<u8'), ('row_loss', '<u8'), ('pair_loss', '<u8'),
                      ('n_anchor', '<u8'), ('vals', '<u8'), ('g', '<u8'), ('ws', '<u8'), ('ws_bytes', '<u8'),
                      ('rp2', '<f8'), ('rn2', '<f8'), ('N', '<i4'), ('B', '<i4'), ('L', '<i4'), ('max_src', '<i4'),
                      ('max_tgt', '<i4'), ('n_terms', '<i4'), ('n_vals', '<i4'), ('ov_val', '<i4', (LOSS_MAX_LAYERS,)),
                      ('corr_val', '<i4', (LOSS_MAX_LAYERS,)), ('term_val', '<i4', (LOSS_MAX_TERMS,)), ('pad_', '<i4')],
                     align=True)
assert (OVERLAP_PYR_ARGS.itemsize, LOSS_ARGS.itemsize) == (264, 568)     # the C structs' sizes
CIRCLE_ARGS = np.dtype([('n_pos', '<u8'), ('n_neg', '<u8'), ('n_sel', '<u8'), ('lse_pos', '<u8'), ('lse_neg', '<u8')],
                       align=True)


def overlap_pyramid(pyr0, pools32, offs, n_clouds: int):
    """Ground-truth overlap of every pyramid level (regtr_overlap_pyramid): pyr0 (n_0) fp32 level-0 masks; pools32[p-1]
    the (n_p, K) int32 pooling table into level p; offs[p] the (n_clouds + 1) int32 device offsets of level p.
    -> [pyr_0, pyr_1, ...].  One launch per level, no host sync."""
    L = _lib.load()
    _chk(pyr0, torch.float32, 'pyr0', 1)
    n_levels = len(pools32) + 1
    if n_levels > LOSS_MAX_LEVELS or len(offs) < n_levels - 1:
        raise ValueError(f'overlap_pyramid: {n_levels} levels (at most {LOSS_MAX_LEVELS}), {len(offs)} offset rows')
    a = np.zeros((), OVERLAP_PYR_ARGS)
    out = [pyr0]
    a['pyr'][0], a['n'][0], a['n_levels'] = pyr0.data_ptr(), pyr0.shape[0], n_levels
    n_launch = 0
    for p in range(1, n_levels):
        pool = _chk(pools32[p - 1], torch.int32, 'pool', 2)
        _chk(offs[p - 1], torch.int32, 'offs', 1)
        lvl = torch.empty(pool.shape[0], dtype=torch.float32, device=pyr0.device)
        out.append(lvl)
        a['pyr'][p], a['pool'][p], a['n'][p], a['K'][p] = lvl.data_ptr(), pool.data_ptr(), pool.shape[0], pool.shape[1]
        a['n_prev'][p] = offs[p - 1].data_ptr() + 4 * n_clouds
        n_launch += int(pool.shape[0] > 0)
    _lib.check(L.regtr_overlap_pyramid(a.ctypes.data, _stream()), 'regtr_overlap_pyramid')
    _count(n_launch)
    return out


def sym_weight(W):
    """Ws = triu(W) + triu(W)^T of InfoNCELossFull's (256, 256) matrix, as the (hi, lo) TF32 halves `gemm` reads
    (regtr_sym_weight): Ws changes with every optimizer step, so it is split where it is built and never cached."""
    L = _lib.load()
    _chk(W, torch.float32, 'W', 2)
    if tuple(W.shape) != (LOSS_DIM, LOSS_DIM):
        raise _lib.RegtrLibError(f'sym_weight: W {tuple(W.shape)}; the InfoNCE kernels are built for d_embed = {LOSS_DIM}')
    hi, lo = torch.empty_like(W), torch.empty_like(W)
    _lib.check(L.regtr_sym_weight(_p(W), _p(hi), _p(lo), _stream()), 'regtr_sym_weight')
    _count(1)
    return hi, lo


def sym_weight_bwd(dWs, dW):
    """dW += triu(dWs + dWs^T) (regtr_sym_weight_bwd)."""
    L = _lib.load()
    _chk(dWs, torch.float32, 'dWs', 2); _chk(dW, torch.float32, 'dW', 2)
    _lib.check(L.regtr_sym_weight_bwd(_p(dWs), _p(dW), _stream()), 'regtr_sym_weight_bwd')
    _count(1)


class LossGeometry:
    """What the device loss reads besides the predictions: xyz (N, 3) coarse key points (source clouds, then target
    clouds), offs (2B + 1) int32 device offsets and lens, the same lengths on the host, pose (B, 3, 4) fp32 ground
    truth, w (N) coarsest ground-truth overlap, the layers each loss is applied to, and the feature loss's radii.
    norm: None, or the (4,) fp64 device normalisers of the whole batch (`loss_norms` summed over the ranks that each
    hold a slice of it): the values and gradients are then this slice's share of the batch's.
    feature_loss: 'infonce' (InfoNCELossFull, with its two W) or 'circle' (CircleLossFull(dist_type='euclidean'),
    no parameters)."""

    def __init__(self, xyz, offs, lens, pose, w, overlap_on, feature_on, corr_on, r_p: float, r_n: float, norm=None,
                 feature_loss: str = 'infonce'):
        if feature_loss not in ('infonce', 'circle'):
            raise ValueError(f'LossGeometry: feature_loss {feature_loss!r}')
        self.xyz, self.offs, self.lens, self.pose, self.w = xyz, offs, [int(v) for v in lens], pose, w
        self.norm = None if norm is None else _chk(norm, torch.float64, 'norm', 1)
        self.feature_loss = feature_loss
        self.B = len(self.lens) // 2
        self.overlap_on, self.feature_on, self.corr_on = list(overlap_on), list(feature_on), list(corr_on)
        self.r_p, self.r_n = float(r_p), float(r_n)

    def keys(self):
        """The loss names in the order of the values vector (the reference's insertion order)."""
        return [f'overlap_{i}' for i in self.overlap_on] + [f'feature_{i}' for i in self.feature_on] + \
            ['feature_un'] + [f'corr_{i}' for i in self.corr_on]


def loss_norms(geo: LossGeometry):
    """(4,) fp64 device vector of this batch's loss normalisers (regtr_loss_norms): token count, sum of the
    coarsest overlap over the source and over the target tokens, pair count.  One launch, no host sync."""
    L = _lib.load()
    w, offs = _chk(geo.w, torch.float32, 'w', 1), _chk(geo.offs, torch.int32, 'offs', 1)
    if sum(geo.lens) != w.shape[0] or offs.shape[0] != 2 * geo.B + 1 or geo.B < 1:
        raise ValueError('loss_norms: inconsistent shapes')
    out = torch.empty(4, dtype=torch.float64, device=w.device)
    a = np.zeros((), LOSS_ARGS)
    a['w'], a['offs'], a['N'], a['B'] = w.data_ptr(), offs.data_ptr(), w.shape[0], geo.B
    _lib.check(L.regtr_loss_norms(a.ctypes.data, out.data_ptr(), _stream()), 'regtr_loss_norms')
    _count(1)
    return out


def loss_forward(both_un, cond, corr, logit, W, W_un, geo: LossGeometry):
    """Loss values of packed predictions: both_un (N, 256), cond (L, N, 256), corr (L, N, 3), logit (L, N, 1), the two
    InfoNCE matrices.  -> state dict; 'vals' is the fp32 vector of geo.keys(), the rest feeds loss_backward
    ('pair_loss' (terms, B) fp64 and 'n_anchor' (B) are the per-pair InfoNCE results).  The number of launches does
    not depend on B; no host sync.  With geo.feature_loss == 'circle' the feature terms are the circle loss (W and W_un
    are None): 'pair_loss' holds its per-pair values, 'n_pos' / 'n_neg' (N) the geometric counts, 'n_sel' (2B) the
    selected tokens of each cloud and 'lse_pos' / 'lse_neg' (terms, N) the fp64 row and column log-sum-exps."""
    L = _lib.load()
    dev = both_un.device
    both_un, cond = _chk(both_un.detach().contiguous(), torch.float32, 'both_un', 2), \
        _chk(cond.detach().contiguous(), torch.float32, 'cond', 3)
    corr, logit = _chk(corr.detach().contiguous(), torch.float32, 'corr', 3), \
        _chk(logit.detach().contiguous(), torch.float32, 'logit', 3)
    xyz, pose, w = _chk(geo.xyz, torch.float32, 'xyz', 2), _chk(geo.pose, torch.float32, 'pose', 3), \
        _chk(geo.w, torch.float32, 'w', 1)
    offs = _chk(geo.offs, torch.int32, 'offs', 1)
    nl, N, B = cond.shape[0], cond.shape[1], geo.B
    keys = geo.keys()
    if both_un.shape != (N, LOSS_DIM) or cond.shape[2] != LOSS_DIM or corr.shape != (nl, N, 3) or \
            logit.shape != (nl, N, 1) or xyz.shape != (N, 3) or w.shape[0] != N or sum(geo.lens) != N or \
            tuple(pose.shape) != (B, 3, 4) or offs.shape[0] != 2 * B + 1 or B < 1:
        raise ValueError('loss_forward: inconsistent shapes')
    if nl > LOSS_MAX_LAYERS or len(geo.feature_on) + 1 > LOSS_MAX_TERMS or \
            any(not 0 <= i < nl for i in geo.overlap_on + geo.feature_on + geo.corr_on):
        raise ValueError(f'loss_forward: {nl} layers, loss layers {geo.overlap_on} {geo.feature_on} {geo.corr_on}')
    n_src = sum(geo.lens[:B])
    term_layers = list(geo.feature_on) + [-1]                    # -1: feature_un on both_un with W_un
    feats = [cond[l] if l >= 0 else both_un for l in term_layers]
    T = len(term_layers)
    circle = geo.feature_loss == 'circle'
    if circle:
        if W is not None or W_un is not None:
            raise ValueError('loss_forward: the circle loss has no W')
        Ws, q = None, None
    else:
        Ws = [sym_weight(W.detach()), sym_weight(W_un.detach())]
        q = [gemm(x[:n_src], *Ws[0 if l >= 0 else 1]) if n_src else x.new_zeros((1, LOSS_DIM))
             for x, l in zip(feats, term_layers)]
    f32 = dict(dtype=torch.float32, device=dev)
    st = dict(geo=geo, keys=keys, term_layers=term_layers, feats=feats, Ws=Ws, q=q, n_src=n_src, shape=(nl, N),
              vals=torch.empty(len(keys), **f32), dlogit=torch.empty((nl, N), **f32), dcorr=torch.empty((nl, N, 3), **f32),
              src_gt=torch.empty((N, 3), **f32), pos=torch.empty(N, dtype=torch.int32, device=dev),
              anchor=torch.empty(N, dtype=torch.int32, device=dev), lse=torch.empty((T, N), **f32),
              row_loss=torch.empty((T, N), **f32), pair_loss=torch.empty((T, B), dtype=torch.float64, device=dev),
              n_anchor=torch.empty(B, dtype=torch.int32, device=dev))
    ws = workspace(L.regtr_loss_ws_bytes(N, nl), dev, 'loss')
    a = np.zeros((), LOSS_ARGS)
    for f, t in (('xyz', xyz), ('offs', offs), ('pose', pose), ('w', w), ('logit', logit), ('corr', corr), ('ws', ws)):
        a[f] = t.data_ptr()
    for f in ('dlogit', 'dcorr', 'src_gt', 'pos', 'anchor', 'lse', 'row_loss', 'pair_loss', 'n_anchor', 'vals'):
        a[f] = st[f].data_ptr()
    a['ws_bytes'], a['rp2'], a['rn2'] = ws.numel(), geo.r_p * geo.r_p, geo.r_n * geo.r_n
    a['N'], a['B'], a['L'], a['n_terms'], a['n_vals'] = N, B, nl, T, len(keys)
    a['max_src'], a['max_tgt'] = max(geo.lens[:B]), max(geo.lens[B:])
    a['ov_val'][:], a['corr_val'][:] = -1, -1
    for i in geo.overlap_on:
        a['ov_val'][i] = keys.index(f'overlap_{i}')
    for i in geo.corr_on:
        a['corr_val'][i] = keys.index(f'corr_{i}')
    for t, l in enumerate(term_layers):
        a['feat'][t] = feats[t].data_ptr()
        if not circle:
            a['q'][t] = q[t].data_ptr()
        a['term_val'][t] = keys.index(f'feature_{l}' if l >= 0 else 'feature_un')
    st['args'], st['hold'] = a, (xyz, offs, pose, w, logit, corr)
    s = _stream()
    _lib.check(L.regtr_loss_pointwise(a.ctypes.data, _p(geo.norm), s), 'regtr_loss_pointwise')
    if circle:
        _circle_forward(L, st, a, s)
        return st
    _lib.check(L.regtr_infonce_match(a.ctypes.data, s), 'regtr_infonce_match')
    _lib.check(L.regtr_infonce_fwd(a.ctypes.data, s), 'regtr_infonce_fwd')
    _lib.check(L.regtr_loss_finalize(a.ctypes.data, _p(geo.norm), s), 'regtr_loss_finalize')
    _count(int(N > 0 and nl > 0) + 2 * int(a['max_src'] > 0) + 1)
    return st


def loss_backward(st, g):
    """Gradients of loss_forward's inputs for the upstream gradient g of its values vector (read on the device).
    -> (d both_un (N, 256), d cond (L, N, 256), d corr (L, N, 3), d logit (L, N, 1), dW, dW_un)."""
    L = _lib.load()
    g = _chk(g.contiguous(), torch.float32, 'g', 1)
    nl, N = st['shape']
    n_src, term_layers, q = st['n_src'], st['term_layers'], st['q']
    dev = g.device
    f32 = dict(dtype=torch.float32, device=dev)
    d_logit, d_corr = torch.empty((nl, N, 1), **f32), torch.empty((nl, N, 3), **f32)
    d_un, d_cond = torch.zeros((N, LOSS_DIM), **f32), torch.zeros((nl, N, LOSS_DIM), **f32)
    if st['geo'].feature_loss == 'circle':
        return _circle_backward(L, st, g, d_un, d_cond, d_corr, d_logit)
    dq = torch.zeros((len(term_layers), max(n_src, 1), LOSS_DIM), **f32)
    dfeat = [d_cond[l] if l >= 0 else d_un for l in term_layers]
    a = st['args'].copy()
    a['g'], a['dlogit_out'], a['dcorr_out'] = g.data_ptr(), d_logit.data_ptr(), d_corr.data_ptr()
    for t in range(len(term_layers)):
        a['dq'][t], a['dfeat'][t] = dq[t].data_ptr(), dfeat[t].data_ptr()
    s = _stream()
    _lib.check(L.regtr_loss_pointwise_bwd(a.ctypes.data, s), 'regtr_loss_pointwise_bwd')
    _lib.check(L.regtr_infonce_bwd(a.ctypes.data, _p(st['geo'].norm), s), 'regtr_infonce_bwd')
    _count(int(N > 0 and nl > 0) + int(a['max_src'] > 0) + int(a['max_tgt'] > 0))
    dW = [torch.zeros((LOSS_DIM, LOSS_DIM), **f32), torch.zeros((LOSS_DIM, LOSS_DIM), **f32)]
    if n_src:
        for t, l in enumerate(term_layers):
            k = 0 if l >= 0 else 1
            gemm(dq[t, :n_src], *st['Ws'][k], out=dfeat[t][:n_src])          # Ws is symmetric: dA = dQ Ws = dQ Ws^T
            dWs, _ = linear_wgrad(st['feats'][t][:n_src], dq[t, :n_src], False)
            sym_weight_bwd(dWs, dW[k])
    return d_un, d_cond, d_corr, d_logit, dW[0], dW[1]


def _circle_forward(L, st, a, s):
    """loss_forward's circle part (regtr_circle_*): geometry, row and column log-sum-exps, values."""
    geo, N, B, T = st['geo'], st['shape'][1], st['geo'].B, len(st['term_layers'])
    dev = st['vals'].device
    i32 = dict(dtype=torch.int32, device=dev)
    st.update(n_pos=torch.empty(N, **i32), n_neg=torch.empty(N, **i32), n_sel=torch.empty(2 * B, **i32),
              lse_pos=torch.empty((T, N), dtype=torch.float64, device=dev),
              lse_neg=torch.empty((T, N), dtype=torch.float64, device=dev))
    c = np.zeros((), CIRCLE_ARGS)
    for f in CIRCLE_ARGS.names:
        c[f] = st[f].data_ptr()
    st['circle_args'] = c
    _lib.check(L.regtr_circle_match(a.ctypes.data, c.ctypes.data, s), 'regtr_circle_match')
    _lib.check(L.regtr_circle_fwd(a.ctypes.data, c.ctypes.data, s), 'regtr_circle_fwd')
    _lib.check(L.regtr_circle_finalize(a.ctypes.data, c.ctypes.data, _p(geo.norm), s), 'regtr_circle_finalize')
    n_launch = int(N > 0 and st['shape'][0] > 0) + int(max(a['max_src'], a['max_tgt']) > 0) + \
        int(a['max_src'] > 0) + int(a['max_tgt'] > 0) + 1
    _count(n_launch)


def _circle_backward(L, st, g, d_un, d_cond, d_corr, d_logit):
    """loss_backward's circle part: both sides' feature gradients come from regtr_circle_bwd; there is no W."""
    nl, N = st['shape']
    a = st['args'].copy()
    a['g'], a['dlogit_out'], a['dcorr_out'] = g.data_ptr(), d_logit.data_ptr(), d_corr.data_ptr()
    for t, l in enumerate(st['term_layers']):
        a['dfeat'][t] = (d_cond[l] if l >= 0 else d_un).data_ptr()
    c, s = st['circle_args'], _stream()
    _lib.check(L.regtr_loss_pointwise_bwd(a.ctypes.data, s), 'regtr_loss_pointwise_bwd')
    _lib.check(L.regtr_circle_bwd(a.ctypes.data, c.ctypes.data, _p(st['geo'].norm), s), 'regtr_circle_bwd')
    _count(int(N > 0 and nl > 0) + int(a['max_src'] > 0) + int(a['max_tgt'] > 0))
    return d_un, d_cond, d_corr, d_logit, None, None


class _LossFn(torch.autograd.Function):
    """values vector of loss_forward; backward on loss_backward."""

    @staticmethod
    def forward(ctx, both_un, cond, corr, logit, W, W_un, geo):
        st = loss_forward(both_un, cond, corr, logit, W, W_un, geo)
        ctx.st = {k: v for k, v in st.items() if k != 'vals'}    # the output must not be reachable from its own node
        return st['vals']

    @staticmethod
    def backward(ctx, g):
        need = ctx.needs_input_grad
        grads = loss_backward(ctx.st, g)
        return tuple(d if n else None for d, n in zip(grads, need)) + (None,)


def loss_values(both_un, cond, corr, logit, W, W_un, geo: LossGeometry):
    """The fp32 vector of geo.keys() loss values, differentiable with respect to the packed predictions and both W
    (for the circle loss, `geo.feature_loss == 'circle'`, W and W_un are None)."""
    return _LossFn.apply(both_un, cond, corr, logit, W, W_un, geo)
