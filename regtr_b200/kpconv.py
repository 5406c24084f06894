"""KPConv backbone on the H100 kernels: pyramid pre-processor, KPConv op, blocks, encoder.

Host-side mirror of the reference modules (same class names, constructor arguments,
forward signatures and state_dict keys) for the parts of
/root/reference/src/models/backbone_kpconv/{kpconv.py,kpconv_blocks.py} that lie on the
RegTR hot path (SURVEY.md section 2 rows 2-3): `PreprocessorGPU`, `KPFEncoder`, `KPConv`,
`BatchNormBlock` (per-cloud InstanceNorm), `UnaryBlock`, `SimpleBlock`,
`ResnetBottleneckBlock`, `max_pool`.  Deformable / modulated KPConv, the `closest` /
`gaussian` / `constant` modes and the decoder blocks are outside the hot path and raise
NotImplementedError.

Every numeric step runs a kernel from libregtr_b200.so (regtr_b200.ops); dense Linear
layers go through torch (cuBLAS) as plain library GEMMs.
"""
from __future__ import annotations

import logging
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .config import pyramid_plan
from .lazy import LazyDict
from .weights import kernel_disposition

_CELL_SLACK = 1.0001   # cell = radius * slack: keeps |dx| < r inside the 27-cell stencil under fp32 rounding


# ------------------------------------------------------------------ pre-processing

def level_capacities(cfg, cap0: int, ratio: float = 0.40, quantum: int = 256):
    """Row capacities of every pyramid level for a static-shape (CUDA-graph) pipeline.
    Each voxel-grid level keeps 19-27 % of the previous one on 3DMatch-like data (SURVEY.md 8:
    38061 -> 10088 -> 2753 -> 751); `ratio` leaves ~50 % head-room and overflow is detected on the
    device (REGTR_STATUS_CAPACITY), never silently wrong."""
    levels, _, _ = pyramid_plan(cfg)
    caps = [int(cap0)]
    for _ in levels[1:]:
        c = int(caps[-1] * ratio) + 1
        caps.append(min(caps[-1], (c + quantum - 1) // quantum * quantum))
    return caps


class DenseGridOverflow(RuntimeError):
    """REGTR_STATUS_GRID: redo the pyramid with the sort-based voxel sub-sampling (`build(dense=False)`)."""


class Pyramid:
    """Device-resident KPConv pyramid with capacity-shaped buffers.  Level sizes live in
    `offs_all[level]` (int32, device); nothing here requires a host synchronisation."""

    def __init__(self, n_clouds, levels, caps, points, offs_all, conv32, conv64, pool32, pool64, up64, status,
                 grids=None):
        self.n_clouds, self.levels, self.caps = n_clouds, levels, caps
        self.points, self.offs_all = points, offs_all
        self.conv32, self.conv64, self.pool32, self.pool64, self.up64 = conv32, conv64, pool32, pool64, up64
        self.status = status
        self.grids = grids            # cell list per level (kept for the lazily computed `upsamples`)

    def upsample_indices(self, li):
        """`upsamples[li]` (kpconv.py:503-507): for every point of level li its first-K neighbours of level
        li+1 inside radius 2 r_li, int64, capacity-shaped.  Computed on demand from the retained cell lists:
        RegTR.forward never reads it."""
        if self.up64[li] is not None or not self.levels[li]['strided']:
            return self.up64[li]
        lvl = self.levels[li]           # NOT cached here: a graph-owned pyramid is refilled by every replay
        return ops.ball_query(self.points[li], self.offs_all[li], self.points[li + 1], self.offs_all[li + 1],
                              self.grids[li + 1], lvl['K'], 2 * lvl['radius'], q_order=self.grids[li].order,
                              want32=False)[1]

    def n_dev(self, level):
        """1-element int32 device view holding the number of points of `level`."""
        return self.offs_all[level, self.n_clouds:]

    def private(self, static=True):
        """Private keys the encoder blocks consume (capacity tensors + device counts)."""
        return dict(_points=self.points, _offs=[self.offs_all[l] for l in range(len(self.levels))],
                    _neighbors32=self.conv32, _pools32=self.pool32,
                    _ndev=[self.n_dev(l) for l in range(len(self.levels))] if static else None,
                    _n_clouds=self.n_clouds)


class PreprocessorGPU(nn.Module):
    """Computes the KPConv pyramid metadata on the GPU, deterministically.

    Same contract as the reference PreprocessorGPU.forward (kpconv.py:426-537): returns a
    dict of per-level lists `points`, `neighbors`, `pools`, `upsamples`, `stack_lengths`
    (int64 indices, shadow index = number of supports).  Differences by design:
      * bit-reproducible (sorted voxel order, index-ordered fp32 sums) where the reference
        is not (MinkowskiEngine hash order, Readme.md:99);
      * ONE host synchronisation for the whole pyramid (`finalize`), where the reference
        synchronises at every `.item()` / python loop (kpconv.py:239,276-285); `build` alone
        is sync-free and CUDA-graph capturable.
    Extra private keys (`_offs`, `_neighbors32`, `_pools32`, `_lens`, ...) carry the int32 /
    device-offset forms the encoder kernels consume.
    """

    def __init__(self, cfg, compute_upsamples: bool = True):
        super().__init__()
        self.cfg = cfg
        self.compute_upsamples = compute_upsamples

    @torch.no_grad()
    def build(self, points, offs0, n_clouds: int, caps=None, want64: bool = True, upsamples: bool = None,
              dense: bool = True) -> Pyramid:
        """points (cap0,3) f32 packed clouds, offs0 (n_clouds+1) int32 device offsets.
        caps: per-level row capacities (default: every level as large as level 0).
        upsamples: compute the `upsamples` lists (default: the module's `compute_upsamples`).
        dense: voxel sub-sampling by counting sort over a dense grid (default; sets status bit 4 when a cloud's
        bounding box exceeds the cell budget) or, dense=False, by the sort-based variant."""
        upsamples = self.compute_upsamples if upsamples is None else upsamples
        levels, _, _ = pyramid_plan(self.cfg)
        device = points.device
        cap0 = points.shape[0]
        caps = [cap0] * len(levels) if caps is None else list(caps)
        assert caps[0] == cap0
        status = ops.new_status(device)
        offs_all = torch.zeros((len(levels), n_clouds + 1), dtype=torch.int32, device=device)
        offs_all[0].copy_(offs0)
        pts_l, conv32, conv64, pool32, pool64, up64, grids = [], [], [], [], [], [], []
        cur = points
        grid = ops.CellGrid(cur, offs_all[0], n_clouds, levels[0]['radius'] * _CELL_SLACK, status)
        for li, lvl in enumerate(levels):
            r, K = lvl['radius'], lvl['K']
            offs = offs_all[li]
            pts_l.append(cur)
            grids.append(grid)
            if lvl['has_conv']:
                c32, c64 = ops.ball_query(cur, offs, cur, offs, grid, K, r, q_order=grid.order, want64=want64)
            else:
                c32 = c64 = None
            conv32.append(c32); conv64.append(c64)
            if lvl['strided']:
                nxt, _ = ops.grid_subsample(cur, offs, n_clouds, lvl['dl'], status, out_cap=caps[li + 1],
                                            out_offs=offs_all[li + 1], dense=dense)
                p32, p64 = ops.ball_query(nxt, offs_all[li + 1], cur, offs, grid, K, r, want64=want64)
                nxt_grid = ops.CellGrid(nxt, offs_all[li + 1], n_clouds, 2 * r * _CELL_SLACK, status)
                u64 = None
                if upsamples and want64:
                    _, u64 = ops.ball_query(cur, offs, nxt, offs_all[li + 1], nxt_grid, K, 2 * r,
                                            q_order=grid.order, want32=False)
                pool32.append(p32); pool64.append(p64); up64.append(u64)
                cur, grid = nxt, nxt_grid
            else:
                pool32.append(None); pool64.append(None); up64.append(None)
        return Pyramid(n_clouds, levels, caps, pts_l, offs_all, conv32, conv64, pool32, pool64, up64, status, grids)

    @staticmethod
    def check_status(code: int):
        if code & 4:
            raise DenseGridOverflow('a cloud spans more voxels than the dense-grid budget (16 cells per point)')
        if code & 1:
            raise RuntimeError('point coordinates exceed the +-32766-cell key range of the voxel / cell grid')
        if code & 2:
            raise RuntimeError('a pyramid level overflowed its static capacity')

    @staticmethod
    def finalize(pyr: Pyramid, host=None, lazy_upsamples: bool = True):
        """The single host synchronisation: read the level sizes, narrow the capacity buffers to
        exact shapes and assemble the reference's dict.  `host` may carry an already-downloaded
        (offs_all, status) pair.  `upsamples` lists that the pyramid did not compute are produced on
        first access of the key (LazyDict) unless lazy_upsamples=False."""
        n_clouds, levels = pyr.n_clouds, pyr.levels
        device = pyr.points[0].device
        if host is None:
            flat = torch.cat([pyr.offs_all.reshape(-1), pyr.status]).cpu()
            offs_host, code = flat[:-1].reshape(len(levels), n_clouds + 1), int(flat[-1])
        else:
            offs_host, code = host
        PreprocessorGPU.check_status(code)
        lens = [(offs_host[l, 1:] - offs_host[l, :-1]).tolist() for l in range(len(levels))]
        totals = [int(offs_host[l, -1]) for l in range(len(levels))]
        e_idx = torch.zeros((0, 1), dtype=torch.int64, device=device)
        data = LazyDict(None, None, points=[], neighbors=[], pools=[], stack_lengths=[],
                        _points=[], _offs=[], _neighbors32=[], _pools32=[], _lens=lens, _ndev=None,
                        _n_clouds=n_clouds)

        def upsamples():
            ups = []
            for li, lvl in enumerate(levels):
                u = pyr.upsample_indices(li) if lvl['strided'] else None
                ups.append(u[:totals[li]] if u is not None else e_idx)
            return ups

        lens_dev = (pyr.offs_all[:, 1:] - pyr.offs_all[:, :-1]).to(torch.int64)     # (levels, n_clouds), one tiny kernel
        for li, lvl in enumerate(levels):
            n = totals[li]
            data['points'].append(pyr.points[li][:n])
            data['_points'].append(pyr.points[li][:n])
            data['neighbors'].append(pyr.conv64[li][:n] if pyr.conv64[li] is not None else e_idx)
            data['_neighbors32'].append(pyr.conv32[li][:n] if pyr.conv32[li] is not None else None)
            if lvl['strided']:
                n2 = totals[li + 1]
                data['pools'].append(pyr.pool64[li][:n2] if pyr.pool64[li] is not None else e_idx)
                data['_pools32'].append(pyr.pool32[li][:n2])
            else:
                data['pools'].append(e_idx)
                data['_pools32'].append(None)
            data['stack_lengths'].append(lens_dev[li])
            data['_offs'].append(pyr.offs_all[li])
        if lazy_upsamples:
            data._lazy['upsamples'] = upsamples
        else:
            data['upsamples'] = upsamples()
        return data

    @torch.no_grad()
    def forward(self, pts: List[torch.Tensor], lazy_upsamples: bool = False):
        device = pts[0].device
        points = torch.cat([p.to(torch.float32) for p in pts], dim=0).contiguous()
        offs0 = ops.make_offsets([int(p.shape[0]) for p in pts], device)
        up = False if lazy_upsamples else None
        try:
            return self.finalize(self.build(points, offs0, len(pts), upsamples=up), lazy_upsamples=lazy_upsamples)
        except DenseGridOverflow:          # sparse / very large extent: sort-based sub-sampling, same results
            return self.finalize(self.build(points, offs0, len(pts), upsamples=up, dense=False),
                                 lazy_upsamples=lazy_upsamples)


def _meta_private(meta, device):
    """Private (int32 / offsets) form of a pyramid dict; derived on the fly for a foreign
    (reference-produced) dict."""
    if '_offs' not in meta:
        lens = [l.tolist() for l in meta['stack_lengths']]
        meta.update(
            _points=list(meta['points']), _offs=[ops.make_offsets(l, device) for l in lens],
            _neighbors32=[n.to(torch.int32).contiguous() if n.numel() and n.shape[1] > 1 else None
                          for n in meta['neighbors']],
            _pools32=[p.to(torch.int32).contiguous() if p.numel() and p.shape[1] > 1 else None
                      for p in meta['pools']],
            _lens=lens, _ndev=None, _n_clouds=len(lens[0]))
    return meta


# --------------------------------------------------------------------------- blocks

def max_pool(x, inds):
    """kpconv_blocks.py:127-143.  `inds` int64 (reference contract) or int32."""
    return ops.max_pool(x.contiguous(), inds if inds.dtype == torch.int32 else inds.to(torch.int32))


class KPConv(nn.Module):
    """Rigid kernel-point convolution (kpconv_blocks.py:176-414), same constructor signature."""

    def __init__(self, kernel_size, p_dim, in_channels, out_channels, KP_extent, radius,
                 fixed_kernel_points='center', KP_influence='linear', aggregation_mode='sum',
                 deformable=False, modulated=False):
        super().__init__()
        if deformable or modulated:
            raise NotImplementedError('deformable / modulated KPConv is outside the hot path')
        if KP_influence != 'linear' or aggregation_mode != 'sum':
            raise NotImplementedError("only KP_influence='linear', aggregation_mode='sum' are on the hot path")
        if kernel_size != 15 or p_dim != 3:
            raise NotImplementedError('the fused kernel is specialised for 15 kernel points in 3-D')
        self.K, self.p_dim = kernel_size, p_dim
        self.in_channels, self.out_channels = in_channels, out_channels
        self.radius, self.KP_extent = radius, KP_extent
        self.weights = nn.Parameter(torch.empty((kernel_size, in_channels, out_channels), dtype=torch.float32))
        bound = 1.0 / (in_channels * out_channels) ** 0.5      # kaiming_uniform_(a=sqrt(5)) fan-in rule
        nn.init.uniform_(self.weights, -bound, bound)
        # checkpoints overwrite this (the reference stores its randomised disposition in the state_dict)
        self.kernel_points = nn.Parameter(torch.from_numpy(kernel_disposition(radius, kernel_size)),
                                          requires_grad=False)

    def forward(self, q_pts, s_pts, neighb_inds, x, nq_dev=None, ns_dev=None, row_flags=None, instats=None):
        """instats=(offs, n_clouds): also return the per-cloud InstanceNorm statistics of the output, accumulated
        in the contraction GEMM's epilogue -> (out, stats)."""
        idx = neighb_inds if neighb_inds.dtype == torch.int32 else neighb_inds.to(torch.int32)
        return ops.kpconv(q_pts.contiguous(), s_pts.contiguous(), idx.contiguous(), x.contiguous(),
                          self.weights, self.kernel_points, self.KP_extent, nq_dev=nq_dev, ns_dev=ns_dev,
                          row_flags=row_flags, instats=instats)

    def __repr__(self):
        return 'KPConv(radius: {:.2f}, extent: {:.2f}, in_feat: {:d}, out_feat: {:d})'.format(
            self.radius, self.KP_extent, self.in_channels, self.out_channels)


class BatchNormBlock(nn.Module):
    """Per-cloud InstanceNorm (use_bn=True) or bias (kpconv_blocks.py:474-530).
    `fuse(x, offs, n_clouds, res, slope)` is the fused norm(+residual)(+LeakyReLU) entry."""

    def __init__(self, in_dim, use_bn, bn_momentum):
        super().__init__()
        self.in_dim, self.use_bn, self.bn_momentum = in_dim, use_bn, bn_momentum
        if not use_bn:
            self.bias = nn.Parameter(torch.zeros(in_dim, dtype=torch.float32))

    def fuse(self, x, offs, n_clouds, res=None, slope=-1.0, want_flags=False):
        if self.use_bn:
            return ops.instnorm_act(x, offs, n_clouds, res=res, slope=slope, want_flags=want_flags)
        if want_flags:
            raise NotImplementedError('row flags are only fused into the InstanceNorm pass')
        y = x + self.bias
        if res is not None:
            y = y + res
        return F.leaky_relu(y, slope) if slope >= 0 else y

    def apply(self, x, stats, offs, n_clouds, res=None, slope=-1.0, want_flags=False):
        """Normalise with statistics that the producing GEMM accumulated in its epilogue (differentiable in x and
        res: the backward recomputes the statistics from x)."""
        return ops.instnorm_apply(x, offs, n_clouds, stats, res=res, slope=slope, want_flags=want_flags)

    def forward(self, x, stack_lengths):
        offs = ops.make_offsets(stack_lengths, x.device)
        return self.fuse(x.contiguous(), offs, offs.numel() - 1)


class UnaryBlock(nn.Module):
    """Linear(no bias) -> InstanceNorm -> LeakyReLU(0.1) (kpconv_blocks.py:533-567)."""

    def __init__(self, in_dim, out_dim, use_bn, bn_momentum, no_relu=False):
        super().__init__()
        self.in_dim, self.out_dim, self.use_bn, self.no_relu = in_dim, out_dim, use_bn, no_relu
        self.mlp = nn.Linear(in_dim, out_dim, bias=False)
        self.batch_norm = BatchNormBlock(out_dim, use_bn, bn_momentum)

    def fuse(self, x, offs, n_clouds, res=None, final_slope=None, m_dev=None, want_flags=False, skip=False):
        """skip=True also returns x, as the last element, for the block's shortcut branch: in training its gradient
        is then added in this layer's dX GEMM (ops.linear_instats) instead of by autograd."""
        slope = final_slope if final_slope is not None else (-1.0 if self.no_relu else 0.1)
        if self.use_bn and self.out_dim % 32 == 0:
            # Linear with the InstanceNorm statistics accumulated in the GEMM epilogue, then the apply pass
            y, stats, *xs = ops.linear_instats(x, self.mlp.weight, offs, n_clouds, m_dev=m_dev, skip=skip)
            out = self.batch_norm.apply(y, stats, offs, n_clouds, res=res, slope=slope, want_flags=want_flags)
        else:
            xs = [x]
            out = self.batch_norm.fuse(ops.linear(x, self.mlp.weight, m_dev=m_dev), offs, n_clouds, res=res,
                                       slope=slope, want_flags=want_flags)
        if not skip:
            return out
        return (*out, xs[0]) if want_flags else (out, xs[0])

    def forward(self, x, stack_lengths=None):
        offs = ops.make_offsets(stack_lengths, x.device)
        return self.fuse(x, offs, offs.numel() - 1)


def _block_io(block, batch):
    """-> (q_pts, s_pts, idx32, offs_pre, offs_post, nq_dev, ns_dev, n_clouds) for a block."""
    m = _meta_private(batch, batch['points'][0].device if 'points' in batch else batch['_points'][0].device)
    li = block.layer_ind
    pts, offs, nd = m['_points'], m['_offs'], m['_ndev']
    if 'strided' in block.block_name:
        return (pts[li + 1], pts[li], m['_pools32'][li], offs[li], offs[li + 1],
                nd[li + 1] if nd else None, nd[li] if nd else None, m['_n_clouds'])
    return (pts[li], pts[li], m['_neighbors32'][li], offs[li], offs[li],
            nd[li] if nd else None, nd[li] if nd else None, m['_n_clouds'])


class SimpleBlock(nn.Module):
    """KPConv -> InstanceNorm -> LeakyReLU(0.1) (kpconv_blocks.py:590-646)."""

    def __init__(self, block_name, in_dim, out_dim, radius, layer_ind, config):
        super().__init__()
        self.block_name, self.layer_ind = block_name, layer_ind
        self.in_dim, self.out_dim = in_dim, out_dim
        extent = radius * config.KP_extent / config.conv_radius
        self.KPConv = KPConv(config.num_kernel_points, config.in_points_dim, in_dim, out_dim // 2, extent, radius,
                             fixed_kernel_points=config.fixed_kernel_points, KP_influence=config.KP_influence,
                             aggregation_mode=config.aggregation_mode, deformable='deform' in block_name,
                             modulated=config.modulated)
        self.batch_norm = BatchNormBlock(out_dim // 2, config.use_batch_norm, config.batch_norm_momentum)

    def forward(self, x, batch):
        q, s, idx, _, offs_post, nq_dev, ns_dev, nc = _block_io(self, batch)
        y = self.KPConv(q, s, idx, x, nq_dev, ns_dev)
        return self.batch_norm.fuse(y, offs_post, nc, slope=0.1)


class ResnetBottleneckBlock(nn.Module):
    """unary1 -> KPConv -> IN -> LReLU -> unary2(no relu) ; shortcut (max_pool if strided,
    optional unary) ; LReLU(x + shortcut)  (kpconv_blocks.py:649-741)."""

    def __init__(self, block_name, in_dim, out_dim, radius, layer_ind, config):
        super().__init__()
        self.block_name, self.layer_ind = block_name, layer_ind
        self.in_dim, self.out_dim = in_dim, out_dim
        bn, mom = config.use_batch_norm, config.batch_norm_momentum
        self.use_bn = bn
        extent = radius * config.KP_extent / config.conv_radius
        mid = out_dim // 4
        self.unary1 = UnaryBlock(in_dim, mid, bn, mom) if in_dim != mid else nn.Identity()
        self.KPConv = KPConv(config.num_kernel_points, config.in_points_dim, mid, mid, extent, radius,
                             fixed_kernel_points=config.fixed_kernel_points, KP_influence=config.KP_influence,
                             aggregation_mode=config.aggregation_mode, deformable='deform' in block_name,
                             modulated=config.modulated)
        self.batch_norm_conv = BatchNormBlock(mid, bn, mom)
        self.unary2 = UnaryBlock(mid, out_dim, bn, mom, no_relu=True)
        self.unary_shortcut = UnaryBlock(in_dim, out_dim, bn, mom, no_relu=True) if in_dim != out_dim \
            else nn.Identity()

    def forward(self, features, batch):
        q, s, idx, offs_pre, offs_post, nq_dev, ns_dev, nc = _block_io(self, batch)
        flags = None
        if isinstance(self.unary1, UnaryBlock) and self.use_bn:
            # the normalisation pass also emits the KPConv's "row sums to > 0" neighbour-count flags; `features`
            # continues as unary1's skip output, so that the shortcut's gradient joins unary1's dX in one GEMM
            x, flags, features = self.unary1.fuse(features, offs_pre, nc, m_dev=ns_dev, want_flags=True, skip=True)
        else:
            x = self.unary1.fuse(features, offs_pre, nc, m_dev=ns_dev) if isinstance(self.unary1, UnaryBlock) \
                else features
        if self.use_bn and self.KPConv.out_channels % 32 == 0:
            x, stats = self.KPConv(q, s, idx, x, nq_dev, ns_dev, row_flags=flags, instats=(offs_post, nc))
            x = self.batch_norm_conv.apply(x, stats, offs_post, nc, slope=0.1)
        else:
            x = self.KPConv(q, s, idx, x, nq_dev, ns_dev, row_flags=flags)
            x = self.batch_norm_conv.fuse(x, offs_post, nc, slope=0.1)
        shortcut = ops.max_pool(features, idx, ns_dev) if 'strided' in self.block_name else features
        if isinstance(self.unary_shortcut, UnaryBlock):
            shortcut = self.unary_shortcut.fuse(shortcut, offs_post, nc, m_dev=nq_dev)
        # LeakyReLU(unary2(x) + shortcut), fused into unary2's normalisation pass
        return self.unary2.fuse(x, offs_post, nc, res=shortcut, final_slope=0.1, m_dev=nq_dev)


def block_decider(block_name, radius, in_dim, out_dim, layer_ind, config):
    """kpconv_blocks.py:429-471, restricted to the block kinds either config selects."""
    if block_name in ('simple', 'simple_strided'):
        return SimpleBlock(block_name, in_dim, out_dim, radius, layer_ind, config)
    if block_name in ('resnetb', 'resnetb_strided'):
        return ResnetBottleneckBlock(block_name, in_dim, out_dim, radius, layer_ind, config)
    raise NotImplementedError(f'block {block_name!r} is outside the RegTR hot path (SURVEY.md 2 row 3)')


class KPFEncoder(nn.Module):
    """KPConv encoder (kpconv.py:22-88): same constructor, `encoder_blocks`, `encoder_skip_dims`."""

    def __init__(self, config, d_bottle, increase_channel_when_downsample=True):
        super().__init__()
        self.logger = logging.getLogger(__name__)
        octave = 0
        r = config.first_subsampling_dl * config.conv_radius
        in_dim, out_dim = config.in_feats_dim, config.first_feats_dim
        self.encoder_blocks = nn.ModuleList()
        self.encoder_skip_dims, self.encoder_skips = [], []
        block = None
        for block_i, block in enumerate(config.architecture):
            if any(t in block for t in ('pool', 'strided', 'upsample', 'global')):
                self.encoder_skips.append(block_i)
                self.encoder_skip_dims.append(in_dim)
            if 'upsample' in block:
                break
            self.encoder_blocks.append(block_decider(block, r, in_dim, out_dim, octave, config))
            in_dim = out_dim // 2 if 'simple' in block else out_dim
            if 'pool' in block or 'strided' in block:
                octave += 1
                r *= 2
                if increase_channel_when_downsample:
                    out_dim *= 2
        if 'upsample' not in block:
            self.encoder_skips.append(block_i)
            self.encoder_skip_dims.append(in_dim)

    def forward(self, x, batch):
        skip_x = []
        for block_i, block_op in enumerate(self.encoder_blocks):
            if block_i in self.encoder_skips:
                skip_x.append(x)
            x = block_op(x, batch)
        return x, skip_x
