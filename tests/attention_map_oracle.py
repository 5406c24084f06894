"""CPU oracle of the cross-encoder's attention maps (the reference's `TransformerCrossEncoder.get_attentions()`).

A restatement next to oracle/regtr_oracle.py, which it imports and leaves unchanged: `cross_encoder_layer_maps` is
`regtr_oracle.cross_encoder_layer` (forward_pre / forward_post, one un-padded pair) that also returns the four
head-averaged attention maps of the layer, and `attention_maps` runs the oracle forward up to the cross-encoder and
pads the maps into the reference's (L, B, Ns, Ns) / (L, B, Nt, Nt) / (L, B, Ns, Nt) / (L, B, Nt, Ns) layout, padded
rows and columns 0.  Any dtype: float64 gives the yardstick the GPU maps are measured against.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import pre, regtr_oracle as O


def mha_probs(q_in, k_in, in_w, in_b, nhead, stats=None):
    """Head-averaged softmax(q k^T / sqrt(dh)) of nn.MultiheadAttention (average_attn_weights=True): (Lq, Lk).
    stats (a dict, optional): 's_max' becomes the largest |score| seen."""
    E = q_in.shape[-1]
    dh = E // nhead
    q = (q_in @ in_w[:E].t() + in_b[:E]).view(-1, nhead, dh).transpose(0, 1)
    k = (k_in @ in_w[E:2 * E].t() + in_b[E:2 * E]).view(-1, nhead, dh).transpose(0, 1)
    s = (q / math.sqrt(dh)) @ k.transpose(1, 2)
    if stats is not None and s.numel():
        stats['s_max'] = max(stats.get('s_max', 0.0), float(s.abs().max()))
    return torch.softmax(s, dim=-1).mean(0)


def head_probs(q, k, nhead):
    """Head-averaged probabilities from projected q (Lq, E) and k (Lk, E)."""
    E = q.shape[-1]
    dh = E // nhead
    qh = q.reshape(-1, nhead, dh).transpose(0, 1)
    kh = k.reshape(-1, nhead, dh).transpose(0, 1)
    return torch.softmax((qh / math.sqrt(dh)) @ kh.transpose(1, 2), dim=-1).mean(0)


def cross_encoder_layer_maps(sd, cfg, i, src, tgt, sp, tp, prefix='transformer_encoder.', stats=None):
    """regtr_oracle.cross_encoder_layer plus its maps: -> (src, tgt, (satt_s, satt_t), (xatt_s, xatt_t))."""
    E, H = cfg.d_embed, cfg.nhead
    dt = src.dtype
    p = f'{prefix}layers.{i}.'
    g = lambda k: sd[p + k].to(dt)
    maps = lambda m, q, k: mha_probs(q, k, g(m + '.in_proj_weight'), g(m + '.in_proj_bias'), H, stats)
    ln = lambda x, k: F.layer_norm(x, (E,), g(k + '.weight'), g(k + '.bias'), 1e-5)
    if not cfg.pre_norm:
        swp, twp = src + sp, tgt + tp
        satt = (maps('self_attn', swp, swp), maps('self_attn', twp, twp))
        s1 = ln(src + _att(g, H, 'self_attn', swp, swp, swp if cfg.sa_val_has_pos_emb else src), 'norm1')
        t1 = ln(tgt + _att(g, H, 'self_attn', twp, twp, twp if cfg.sa_val_has_pos_emb else tgt), 'norm1')
        swp, twp = s1 + sp, t1 + tp
        xatt = (maps('multihead_attn', swp, twp), maps('multihead_attn', twp, swp))
    else:
        s2p, t2p = ln(src, 'norm1') + sp, ln(tgt, 'norm1') + tp
        satt = (maps('self_attn', s2p, s2p), maps('self_attn', t2p, t2p))
        s_mid, t_mid = _pre_self(sd, cfg, i, src, tgt, sp, tp, prefix)
        s2p, t2p = ln(s_mid, 'norm2') + sp, ln(t_mid, 'norm2') + tp
        xatt = (maps('multihead_attn', s2p, t2p), maps('multihead_attn', t2p, s2p))
    src, tgt = O.cross_encoder_layer(sd, cfg, i, src, tgt, sp, tp, prefix=prefix)
    return src, tgt, satt, xatt


def _att(g, H, m, q, k, v):
    return O.mha(q, k, v, g(m + '.in_proj_weight'), g(m + '.in_proj_bias'), g(m + '.out_proj.weight'),
                 g(m + '.out_proj.bias'), H)


def _pre_self(sd, cfg, i, src, tgt, sp, tp, prefix):
    """Pre-norm layer state after its self-attention residual (the cross attention's input), as in forward_pre."""
    E, H = cfg.d_embed, cfg.nhead
    p = f'{prefix}layers.{i}.'
    g = lambda k: sd[p + k].to(src.dtype)
    ln = lambda x: F.layer_norm(x, (E,), g('norm1.weight'), g('norm1.bias'), 1e-5)
    s2 = ln(src); s2p = s2 + sp
    t2 = ln(tgt); t2p = t2 + tp
    src = src + _att(g, H, 'self_attn', s2p, s2p, s2p if cfg.sa_val_has_pos_emb else s2)
    tgt = tgt + _att(g, H, 'self_attn', t2p, t2p, t2p if cfg.sa_val_has_pos_emb else t2)
    return src, tgt


def pad_maps(per_pair, Ns, Nt, dtype):
    """per_pair: per layer, per pair ((satt_s, satt_t), (xatt_s, xatt_t)) -> the four padded (L, B, ., .) stacks."""
    L, B = len(per_pair), len(per_pair[0])
    dims = [(Ns, Ns), (Nt, Nt), (Ns, Nt), (Nt, Ns)]
    out = [torch.zeros((L, B) + d, dtype=dtype) for d in dims]
    for li, layer in enumerate(per_pair):
        for b, (satt, xatt) in enumerate(layer):
            for j, m in enumerate(satt + xatt):
                out[j][li, b, :m.shape[0], :m.shape[1]] = m
    return (out[0], out[1]), (out[2], out[3])


def attention_maps(sd, cfg, src_list, tgt_list, dtype=torch.float32, meta=None, stats=None):
    """`get_attentions()` after RegTR.forward (regtr_oracle.forward's pipeline up to the cross-encoder), CPU:
    -> ((src_satt, tgt_satt), (src_xatt, tgt_xatt)), padded, plus the per-cloud coarse lengths."""
    B = len(src_list)
    if meta is None:
        meta = pre.preprocess(cfg, list(src_list) + list(tgt_list), True)
    slens = [int(v) for v in meta['stack_lengths'][-1]]
    feats = O.encoder(sd, cfg, meta, dtype)
    both = feats @ sd['feat_proj.weight'].to(dtype).t() + sd['feat_proj.bias'].to(dtype)
    xyz_c = O._t(meta['points'][-1], dtype)
    if cfg.get('pos_emb_type', 'sine') == 'sine':
        pe = O.pos_embed_sine(xyz_c, cfg.d_embed, scale=cfg.get('pos_emb_scaling', 1.0))
    else:
        pe = O.pos_embed_learned({k: v.to(dtype) for k, v in sd.items() if k.startswith('pos_embed.')}, xyz_c)
    f_split, p_split = torch.split(both, slens), torch.split(pe, slens)
    use_pe = cfg.transformer_encoder_has_pos_emb
    per_layer = [[] for _ in range(cfg.num_encoder_layers)]
    for b in range(B):
        s, t = f_split[b], f_split[B + b]
        sp = p_split[b] if use_pe else torch.zeros_like(s)
        tp = p_split[B + b] if use_pe else torch.zeros_like(t)
        for i in range(cfg.num_encoder_layers):
            s, t, satt, xatt = cross_encoder_layer_maps(sd, cfg, i, s, t, sp, tp, stats=stats)
            per_layer[i].append((satt, xatt))
    Ns, Nt = max(slens[:B]), max(slens[B:])
    return pad_maps(per_layer, Ns, Nt, dtype), slens
