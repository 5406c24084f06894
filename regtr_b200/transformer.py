"""Stacked self/cross attention over the down-sampled point features, on the H100 kernels.

Host-side mirror of /root/reference/src/models/transformer/{transformers.py,
position_embedding.py} for the branches both configs select: pre-norm
`TransformerCrossEncoderLayer.forward_pre` (transformers.py:183-244), `TransformerCrossEncoder`
with `return_intermediate` + final norm (18-59) and `PositionEmbeddingCoordsSine` (7-50) -- plus
the alternative branches of SURVEY.md 8f N4: `forward_post` (121-181) and
`PositionEmbeddingLearned` (position_embedding.py:53-72).
Same constructor signatures and state_dict keys (`self_attn.in_proj_weight`, ...).

Design: the reference pads every cloud to the longest one ((L,B,D) tensors + key-padding
masks).  Here tokens stay PACKED in one (N,D) matrix -- src clouds first, then tgt clouds,
the order the KPConv encoder already produces -- and attention runs over explicit
(query range, key range) problems, so no FLOP or byte is spent on padding.  The padded
reference-style `forward` is kept as a thin adaptor around `forward_packed`.
"""
from __future__ import annotations

import copy
import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor

from . import ops


class PositionEmbeddingCoordsSine(nn.Module):
    """position_embedding.py:7-50 (same constructor)."""

    def __init__(self, n_dim: int = 1, d_model: int = 256, temperature=10000, scale=None):
        super().__init__()
        self.n_dim, self.d_model, self.temperature = n_dim, d_model, temperature
        self.num_pos_feats = d_model // n_dim // 2 * 2
        self.padding = d_model - self.num_pos_feats * n_dim
        self.scale_arg = 1.0 if scale is None else scale

    def forward(self, xyz: Tensor) -> Tensor:
        lead = xyz.shape[:-1]
        out = ops.pos_embed_sine(xyz.reshape(-1, self.n_dim).contiguous(), self.d_model, self.temperature,
                                 self.scale_arg)
        return out.reshape(*lead, self.d_model)


class PositionEmbeddingLearned(nn.Module):
    """position_embedding.py:53-72: MLP n_dim -> 32 -> 64 -> 128 -> 256 -> d_model with ReLUs (same
    constructor and `mlp.{0,2,4,6,8}` state_dict keys); every layer runs on the library GEMM."""

    def __init__(self, n_dim: int = 1, d_model: int = 256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(n_dim, 32), nn.ReLU(), nn.Linear(32, 64), nn.ReLU(),
                                 nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 256), nn.ReLU(),
                                 nn.Linear(256, d_model))

    def forward(self, xyz: Tensor) -> Tensor:
        lead = xyz.shape[:-1]
        x = xyz.reshape(-1, xyz.shape[-1])
        first = self.mlp[0]
        pad = (-x.shape[1]) % 4                 # the tensor-core GEMM needs a 16-byte row pitch: zero-pad K
        if pad:
            w = first.weight
            cache = self.__dict__.setdefault('_padded_w', {})
            key = (w._version, w.data_ptr())
            if key not in cache:
                cache.clear()
                cache[key] = F.pad(w.detach(), (0, pad)).contiguous()
            x, w0 = F.pad(x, (0, pad)).contiguous(), cache[key]
        else:
            x, w0 = x.contiguous(), first.weight
        h = ops.linear(x, w0, first.bias, relu=True)
        for i in (2, 4, 6):
            h = ops.linear(h, self.mlp[i].weight, self.mlp[i].bias, relu=True)
        h = ops.linear(h, self.mlp[8].weight, self.mlp[8].bias)
        return h.reshape(*lead, -1)


class _MHAParams(nn.Module):
    """Parameter container with nn.MultiheadAttention's state_dict layout."""

    def __init__(self, d_model, nhead):
        super().__init__()
        self.embed_dim, self.num_heads = d_model, nhead
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d_model, d_model))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d_model))
        self.out_proj = nn.Linear(d_model, d_model)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.zeros_(self.out_proj.bias)


class AttentionPlan:
    """Device-side (start,len) tables of the self and cross attention problems of a batch:
    problem c = cloud c of the (src x B, tgt x B) stack; its cross partner is the other cloud of
    the pair.  `max_len` is a host-side upper bound of the sequence lengths (grid sizing only);
    `n_dev` (static-shape pipelines only) is the device-side total token count, so that the dense
    layers skip the capacity padding rows."""

    def __init__(self, lens=None, device=None, table=None, max_len=None, n_dev=None, max_tiles=None):
        if table is None:
            n2 = len(lens)
            B = n2 // 2
            lens = list(map(int, lens))
            starts = [0]
            for v in lens:
                starts.append(starts[-1] + v)
            other = [B + c if c < B else c - B for c in range(n2)]
            t64, t128 = [0], [0]
            for v in lens:
                t64.append(t64[-1] + (v + 63) // 64); t128.append(t128[-1] + (v + 127) // 128)
            rows = [starts[:n2] + [0], lens + [0],                                    # query ranges
                    [starts[o] for o in other] + [0], [lens[o] for o in other] + [0],  # cross key ranges
                    t64, t128]                                                        # tile prefixes (total last)
            table = torch.tensor(rows, dtype=torch.int32).to(device)
            max_len = max(lens) if n2 else 0
            max_tiles = (t64[-1], t128[-1])
            self.lens = lens                # host lengths: only plans built from them can record attention maps
        else:
            self.lens = None
        self.map_dims = None                # (Ns, Nt) of the recorded maps; None: the longest src / tgt cloud
        self._map_tables = None
        n2 = table.shape[1] - 1
        self.q_start, self.q_len = table[0, :n2], table[1, :n2]
        self.xk_start, self.xk_len = table[2, :n2], table[3, :n2]
        self.max_len = int(max_len)
        self.n_dev = n_dev
        # (device tile table, host bound of the total) for the 64-query (mma.sync) and 128-query (wgmma) cores
        self.tiles64 = (table[4], int(max_tiles[0]))
        self.tiles128 = (table[5], int(max_tiles[1]))

    @classmethod
    def from_device(cls, offs, B: int, max_len: int):
        """Sync-free construction from device offsets (static-shape / CUDA-graph pipelines)."""
        n2 = 2 * B                          # sum_p ceil(len_p / T) <= capacity / T + number of problems
        return cls(table=ops.attention_plan(offs, B), max_len=max_len, n_dev=offs[2 * B:2 * B + 1],
                   max_tiles=(max_len // 64 + n2, max_len // 128 + n2))

    def map_tables(self, device):
        """Device (offset, pitch) tables of the self and cross problems into one flat per-layer map buffer, built once
        per plan (see `attention_map_layout`)."""
        if self.lens is None:
            raise RuntimeError('recording attention maps needs host-side cloud lengths (an eager forward); '
                               'this plan was built on the device')
        if self._map_tables is None:
            lay = attention_map_layout(self.lens, *(self.map_dims or (None, None)))
            dev = lambda v, dt: torch.tensor(v, dtype=dt).to(device)
            self._map_tables = dict(lay, self_tab=(dev(lay['self_offset'], torch.int64), dev(lay['self_pitch'], torch.int32)),
                                    cross_tab=(dev(lay['cross_offset'], torch.int64), dev(lay['cross_pitch'], torch.int32)))
        return self._map_tables


def attention_map_layout(lens, Ns=None, Nt=None):
    """Where the head-averaged attention maps of a (src x B, tgt x B) batch go in one flat buffer, in the reference's
    padded layout: src_satt (B, Ns, Ns) | tgt_satt (B, Nt, Nt) | src_xatt (B, Ns, Nt) | tgt_xatt (B, Nt, Ns).
    Ns / Nt default to the longest src / tgt cloud.  Problem c of the plan (cloud c as query, itself or its partner
    as key) writes its (len_q, len_k) block at `*_offset[c]` with row pitch `*_pitch[c]`; the rest stays as filled.
    Host only (plain Python): -> dict(self_offset, self_pitch, cross_offset, cross_pitch, shapes, numel, Ns, Nt)."""
    lens = [int(v) for v in lens]
    B = len(lens) // 2
    s, t = lens[:B], lens[B:]
    Ns = max(s, default=0) if Ns is None else int(Ns)
    Nt = max(t, default=0) if Nt is None else int(Nt)
    if any(v > Ns for v in s) or any(v > Nt for v in t):
        raise ValueError(f'attention_map_layout: cloud lengths {lens} exceed the map sizes ({Ns}, {Nt})')
    shapes = [(B, Ns, Ns), (B, Nt, Nt), (B, Ns, Nt), (B, Nt, Ns)]
    base = [0]
    for sh in shapes:
        base.append(base[-1] + sh[0] * sh[1] * sh[2])
    self_off = [base[0] + c * Ns * Ns for c in range(B)] + [base[1] + c * Nt * Nt for c in range(B)]
    cross_off = [base[2] + c * Ns * Nt for c in range(B)] + [base[3] + c * Nt * Ns for c in range(B)]
    return dict(self_offset=self_off, self_pitch=[Ns] * B + [Nt] * B, cross_offset=cross_off,
                cross_pitch=[Nt] * B + [Ns] * B, shapes=shapes, bases=base[:4], numel=base[4], Ns=Ns, Nt=Nt)


class TransformerCrossEncoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu",
                 normalize_before=False, sa_val_has_pos_emb=False, ca_val_has_pos_emb=False,
                 attention_type='dot_prod', attention_impl='fp32'):
        super().__init__()
        if attention_impl not in ('fp32', 'tf32_tc', 'bf16_tc'):
            raise ValueError("attention_impl: 'tf32_tc' (wgmma 3xTF32, fp32-accurate), 'fp32' (mma.sync 3xTF32) or 'bf16_tc'")
        self.attention_impl = attention_impl
        if attention_type != 'dot_prod':
            raise NotImplementedError
        if activation != 'relu':
            raise NotImplementedError('only relu is on the hot path')
        if not (isinstance(dropout, (int, float)) and 0.0 <= dropout < 1.0):
            raise ValueError(f'dropout must be in [0, 1), got {dropout!r}')
        # the six dropouts of forward_pre apply in forward_train_packed (training mode only); they add no state
        self.dropout_p = float(dropout)
        self.self_attn = _MHAParams(d_model, nhead)
        self.multihead_attn = _MHAParams(d_model, nhead)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.norm3 = nn.LayerNorm(d_model)
        self.nhead = nhead
        self.normalize_before = normalize_before
        self.sa_val_has_pos_emb, self.ca_val_has_pos_emb = sa_val_has_pos_emb, ca_val_has_pos_emb
        # analysis only (reference: get_attentions): filled by every forward while record_attentions is on
        self.satt_weights, self.xatt_weights = None, None
        self.record_attentions = False

    def _attend(self, mha: _MHAParams, x2, x2p, val_has_pos, plan: AttentionPlan, cross: bool):
        E = mha.embed_dim
        W, b = mha.in_proj_weight, mha.in_proj_bias
        ks, kl = (plan.xk_start, plan.xk_len) if cross else (plan.q_start, plan.q_len)
        nd = plan.n_dev
        q = k = None
        if self.attention_impl == 'bf16_tc' and val_has_pos:
            # fast mode: in-projection with a bf16 epilogue + wgmma attention core (TMA-fed, register accumulators)
            o = ops.mha_bf16_tc(x2p, W, b, plan.q_start, plan.q_len, ks, kl, plan.max_len, self.nhead, m_dev=nd)
        elif self.attention_impl == 'tf32_tc' and val_has_pos:
            # parity mode on the tensor cores: split-epilogue in-projection + TMA-fed wgmma 3xTF32 attention core
            o = ops.mha_tf32_tc(x2p, W, b, plan.q_start, plan.q_len, ks, kl, plan.max_len, self.nhead,
                                m_dev=nd, tiles=plan.tiles128)
        else:
            if val_has_pos:
                qkv = ops.linear(x2p, W, b, m_dev=nd)         # one packed in-projection GEMM
                q, k, v = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
            else:
                qk = ops.linear(x2p, W[:2 * E], b[:2 * E], m_dev=nd)
                q, k = qk[:, :E], qk[:, E:]
                v = ops.linear(x2, W[2 * E:], b[2 * E:], m_dev=nd)
            o = ops.mha_varlen(q, k, v, plan.q_start, plan.q_len, ks, kl, plan.max_len, self.nhead, tiles=plan.tiles64)
        if self.record_attentions:
            if q is None:
                # the fused tensor-core in-projections never hold fp32 q and k: project them on the library GEMM (the
                # maps are then the fp32 attention of the same weights, also under bf16_tc)
                qk = ops.linear(x2p, W[:2 * E], b[:2 * E], m_dev=nd)
                q, k = qk[:, :E], qk[:, E:]
            self._record_map(q, k, plan, cross)
        return o

    def _record_map(self, q, k, plan: AttentionPlan, cross: bool):
        """Head-averaged probabilities of this attention into a fresh zero-filled buffer in the reference's padded
        layout (`attention_map_layout`): sets satt_weights after the self attention, xatt_weights after the cross."""
        tabs = plan.map_tables(q.device)
        if not cross:       # self attention runs first in both layer variants: one buffer per layer and forward
            self._map_buf = torch.zeros(tabs['numel'], dtype=torch.float32, device=q.device)
        buf = self._map_buf
        off, pitch = tabs['cross_tab' if cross else 'self_tab']
        ks, kl = (plan.xk_start, plan.xk_len) if cross else (plan.q_start, plan.q_len)
        ops.mha_probs_avg(q, k, buf, off, pitch, plan.q_start, plan.q_len, ks, kl, plan.max_len, self.nhead)
        i = 2 if cross else 0
        views = tuple(buf.narrow(0, tabs['bases'][j], math.prod(tabs['shapes'][j])).view(tabs['shapes'][j])
                      for j in (i, i + 1))
        if cross:
            self.xatt_weights = views
            del self._map_buf
        else:
            self.satt_weights = views

    def forward_packed(self, x, pos, plan: AttentionPlan):
        """x, pos: (N,E) packed tokens (src clouds then tgt clouds).  Returns updated x."""
        if not self.normalize_before:
            return self.forward_post_packed(x, pos, plan)
        has_pos = pos is not None
        nd = plan.n_dev
        # self attention (shared weights for src and tgt: one launch over all 2B clouds)
        x2, x2p = ops.layernorm_pos(x, self.norm1.weight, self.norm1.bias, pos, self.norm1.eps,
                                    want_plain=not self.sa_val_has_pos_emb, want_pos=True, n_dev=nd)
        o = self._attend(self.self_attn, x2, x2p, self.sa_val_has_pos_emb or not has_pos, plan, cross=False)
        x = ops.linear(o, self.self_attn.out_proj.weight, self.self_attn.out_proj.bias, residual=x, m_dev=nd)
        # cross attention, both directions from the same pre-update normalised features
        x2, x2p = ops.layernorm_pos(x, self.norm2.weight, self.norm2.bias, pos, self.norm2.eps,
                                    want_plain=not self.ca_val_has_pos_emb, want_pos=True, n_dev=nd)
        o = self._attend(self.multihead_attn, x2, x2p, self.ca_val_has_pos_emb or not has_pos, plan, cross=True)
        x = ops.linear(o, self.multihead_attn.out_proj.weight, self.multihead_attn.out_proj.bias, residual=x, m_dev=nd)
        # position-wise feed-forward
        x2, _ = ops.layernorm_pos(x, self.norm3.weight, self.norm3.bias, None, self.norm3.eps,
                                  want_plain=True, want_pos=False, n_dev=nd)
        h = ops.linear(x2, self.linear1.weight, self.linear1.bias, relu=True, m_dev=nd)
        x = ops.linear(h, self.linear2.weight, self.linear2.bias, residual=x, m_dev=nd)
        return x


    def forward_train_packed(self, x, pos, plan: AttentionPlan, drop=None, layer_idx: int = 0):
        """Differentiable pre-norm layer (exact shapes) for the branches both reference configs select: pre-norm,
        values carrying the position embedding, the default 3xTF32 attention core.  Same math as `forward_packed`;
        every LayerNorm also hands x on to the residual add that follows it (layernorm_pos(skip=True)), so the
        residual gradient is added inside the LayerNorm backward.
        drop (an ops.DropoutKey, or None): apply the six dropouts of layer `layer_idx` (transformers.py:183-244, train
        mode) and return (x, z).  Without dropout the out-projection and linear2 GEMMs add the residual in their
        epilogue and the layer returns x.  With it they run without residual=, and each dropped branch z is added as
        x + m * scale * z in the prologue of the LayerNorm that follows it (norm2, norm3, then the encoder's final
        norm), which also hands x' on: the last branch z = linear2(...) is returned not yet added."""
        has_pos = pos is not None
        site = lambda s: None if drop is None else drop.site(layer_idx, s)

        def branch(h, lin, x):
            if drop is None:
                return ops.linear(h, lin.weight, lin.bias, residual=x), None
            return x, ops.linear(h, lin.weight, lin.bias)

        z = z_site = None
        for mha, norm, cross, att_site, out_site in (
                (self.self_attn, self.norm1, False, ops.SITE_SELF_ATTN, ops.SITE_SELF_OUT),
                (self.multihead_attn, self.norm2, True, ops.SITE_CROSS_ATTN, ops.SITE_CROSS_OUT)):
            y, yp, x = ops.layernorm_pos(x, norm.weight, norm.bias, pos, norm.eps, want_plain=not has_pos,
                                         want_pos=has_pos, skip=True, z=z, drop=z_site)
            qkv = ops.linear(yp if has_pos else y, mha.in_proj_weight, mha.in_proj_bias)
            ks, kl = (plan.xk_start, plan.xk_len) if cross else (plan.q_start, plan.q_len)
            o = ops.mha_packed(qkv, plan.q_start, plan.q_len, ks, kl, plan.max_len, self.nhead, drop=site(att_site))
            x, z = branch(o, mha.out_proj, x)
            z_site = site(out_site)
        x2, _, x = ops.layernorm_pos(x, self.norm3.weight, self.norm3.bias, None, self.norm3.eps,
                                     want_plain=True, want_pos=False, skip=True, z=z, drop=z_site)
        h = ops.linear(x2, self.linear1.weight, self.linear1.bias, relu=True, drop=site(ops.SITE_FFN))
        x, z = branch(h, self.linear2, x)
        return x if drop is None else (x, z)

    def forward_post_packed(self, x, pos, plan: AttentionPlan):
        """Post-norm layer (transformers.py:121-181): attention on x (+pos), then LayerNorm(x + update)."""
        has_pos = pos is not None
        nd = plan.n_dev
        ln = lambda y, norm, want_pos: ops.layernorm_pos(y, norm.weight, norm.bias, pos if want_pos else None,
                                                         norm.eps, want_plain=True, want_pos=want_pos and has_pos,
                                                         n_dev=nd)
        xp = x + pos if has_pos else x
        o = self._attend(self.self_attn, x, xp, self.sa_val_has_pos_emb or not has_pos, plan, cross=False)
        y = ops.linear(o, self.self_attn.out_proj.weight, self.self_attn.out_proj.bias, residual=x, m_dev=nd)
        x, xp = ln(y, self.norm1, True)
        xp = xp if has_pos else x
        o = self._attend(self.multihead_attn, x, xp, self.ca_val_has_pos_emb or not has_pos, plan, cross=True)
        y = ops.linear(o, self.multihead_attn.out_proj.weight, self.multihead_attn.out_proj.bias, residual=x, m_dev=nd)
        x, _ = ln(y, self.norm2, False)
        h = ops.linear(x, self.linear1.weight, self.linear1.bias, relu=True, m_dev=nd)
        y = ops.linear(h, self.linear2.weight, self.linear2.bias, residual=x, m_dev=nd)
        x, _ = ln(y, self.norm3, False)
        return x


def warn_dropout_eval_only(module):
    """One warning per module when an inference executor runs a dropout > 0 model in training mode."""
    enc = module if isinstance(module, TransformerCrossEncoder) else getattr(module, 'transformer_encoder', None)
    if enc is None or not module.training or enc.dropout_p == 0.0 or module.__dict__.get('_dropout_warned'):
        return
    module.__dict__['_dropout_warned'] = True
    import logging
    logging.getLogger(type(module).__name__).warning(
        f'dropout={enc.dropout_p} is applied by forward_train only; this forward is an inference executor and runs '
        'without dropout (as in eval mode)')


def _get_clones(module, N):
    return nn.ModuleList([copy.deepcopy(module) for _ in range(N)])


class TransformerCrossEncoder(nn.Module):
    def __init__(self, cross_encoder_layer, num_layers, norm=None, return_intermediate=False):
        super().__init__()
        self.layers = _get_clones(cross_encoder_layer, num_layers)
        self.num_layers = num_layers
        self.norm = norm
        self.return_intermediate = return_intermediate
        self._record_attentions = False

    @property
    def record_attentions(self) -> bool:
        """Opt-in analysis switch (off by default).  While on, every eager forward (`forward_packed`, hence
        `RegTR.forward`, and the padded `forward`) also computes each layer's head-averaged attention maps for
        `get_attentions()`; the forward's own outputs are unchanged, bit for bit.  Turning it off drops the maps."""
        return self._record_attentions

    @record_attentions.setter
    def record_attentions(self, on: bool):
        self._record_attentions = bool(on)
        for layer in self.layers:
            layer.record_attentions = bool(on)
            if not on:
                layer.satt_weights, layer.xatt_weights = None, None

    def get_attentions(self):
        """For analysis: the attention maps of the last recorded forward (transformers.py:61-81), stacked over the
        layers: ((src_satt, tgt_satt), (src_xatt, tgt_xatt)) of shapes (L, B, Ns, Ns), (L, B, Nt, Nt), (L, B, Ns, Nt),
        (L, B, Nt, Ns), Ns / Nt the longest src / tgt cloud (the padded length in the padded `forward`).  Each map is
        the head average of the softmax probabilities; padded key columns and padded query rows are 0.  Under
        attention_impl='bf16_tc' the maps are the fp32 attention of the same weights, not the bf16 core's own."""
        if any(layer.satt_weights is None or layer.xatt_weights is None for layer in self.layers):
            raise RuntimeError('get_attentions: no attention maps recorded; set record_attentions = True on the '
                               'TransformerCrossEncoder and run a forward first')
        st = lambda side, which: torch.stack([getattr(layer, which)[side] for layer in self.layers])
        return (st(0, 'satt_weights'), st(1, 'satt_weights')), (st(0, 'xatt_weights'), st(1, 'xatt_weights'))

    def forward_packed(self, x, pos, plan: AttentionPlan):
        """-> (n_out, N, E): final-normed output of every layer (return_intermediate) or the last."""
        outs = []
        for layer in self.layers:
            x = layer.forward_packed(x, pos, plan)
            if self.return_intermediate:
                outs.append(self._final(x, plan.n_dev))
        if not self.return_intermediate:
            outs.append(self._final(x, plan.n_dev))
        return torch.stack(outs)

    @property
    def dropout_p(self) -> float:
        return self.layers[0].dropout_p if len(self.layers) else 0.0

    def forward_train_packed(self, x, pos, plan: AttentionPlan, drop=None):
        """Differentiable `forward_packed` (pre-norm layers with a final norm, return_intermediate): -> (L, N, E).
        The final norm of each intermediate output passes x on to the next layer (skip=True).
        drop (an ops.DropoutKey, or None): the masks of the six dropouts of every layer; layer l's dropout3 and
        residual add run in the prologue of its final norm."""
        if self.record_attentions:
            raise RuntimeError('attention maps are recorded by the inference forward only; turn record_attentions off '
                               'to train')
        if drop is not None and len(self.layers) > 16:
            raise ValueError('dropout: more than 16 layers are outside the mask counter layout')
        outs = []
        for li, layer in enumerate(self.layers):
            if drop is None:
                x, z = layer.forward_train_packed(x, pos, plan), None
            else:
                x, z = layer.forward_train_packed(x, pos, plan, drop, li)
            y, _, x = ops.layernorm_pos(x, self.norm.weight, self.norm.bias, None, self.norm.eps, True, False, skip=True,
                                        z=z, drop=None if drop is None else drop.site(li, ops.SITE_FFN_OUT))
            outs.append(y)
        return torch.stack(outs)

    def _final(self, x, n_dev=None):
        if self.norm is None:
            return x
        y, _ = ops.layernorm_pos(x, self.norm.weight, self.norm.bias, None, self.norm.eps, True, False, n_dev=n_dev)
        return y

    def forward(self, src, tgt, src_mask: Optional[Tensor] = None, tgt_mask: Optional[Tensor] = None,
                src_key_padding_mask: Optional[Tensor] = None, tgt_key_padding_mask: Optional[Tensor] = None,
                src_pos: Optional[Tensor] = None, tgt_pos: Optional[Tensor] = None):
        """Reference-compatible padded interface (transformers.py:27-59): (L,B,D) in, (n_out,L,B,D) out.
        Padded rows of the outputs are zero (the reference leaves unspecified values there).  An inference executor:
        dropout never applies here (see `forward_train_packed`)."""
        warn_dropout_eval_only(self)
        assert src_mask is None and tgt_mask is None, 'Masking not implemented'
        B = src.shape[1]
        s_lens = (~src_key_padding_mask).sum(1).tolist() if src_key_padding_mask is not None else [src.shape[0]] * B
        t_lens = (~tgt_key_padding_mask).sum(1).tolist() if tgt_key_padding_mask is not None else [tgt.shape[0]] * B

        def pack(padded, lens):
            return [padded[:l, b] for b, l in enumerate(lens)]
        x = torch.cat(pack(src, s_lens) + pack(tgt, t_lens), 0).contiguous()
        pos = None
        if src_pos is not None:
            pos = torch.cat(pack(src_pos, s_lens) + pack(tgt_pos, t_lens), 0).contiguous()
        plan = AttentionPlan(s_lens + t_lens, x.device)
        plan.map_dims = (src.shape[0], tgt.shape[0])        # recorded maps in the caller's padded sizes
        out = self.forward_packed(x, pos, plan)
        parts = torch.split(out, s_lens + t_lens, dim=1)
        pad = torch.nn.utils.rnn.pad_sequence
        src_out = pad([p.transpose(0, 1) for p in parts[:B]]).permute(2, 0, 1, 3)
        tgt_out = pad([p.transpose(0, 1) for p in parts[B:]]).permute(2, 0, 1, 3)
        return src_out, tgt_out
