"""ORACLE (test infrastructure only) -- CPU restatement of RegTR.forward.

A functional PyTorch-CPU restatement of the reference hot path, stage by stage,
consuming a reference-layout `state_dict` (SURVEY.md 8b).  It is what the CUDA
product is checked against on the GPU box, where /root/reference does not
exist; `tests/golden/make_golden.py` pins it against the unmodified reference
modules in the build container.  Every function cites the reference lines it
follows.  `dtype=torch.float64` evaluates the same algorithm in double (used to
measure the fp32 spread the tolerances are derived from).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from regtr_b200.config import pyramid_plan
from . import pre


def _t(x, dtype):
    return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(dtype)


# ----------------------------------------------------------------------- KPConv

def kpconv(q_pts, s_pts, inds, x, weights, kernel_points, extent, chunk=8192, count=None):
    """Rigid KPConv, linear influence, sum aggregation.

    Follows KPConv.forward, /root/reference/src/models/backbone_kpconv/kpconv_blocks.py:
    shadow point at 1e6 (309), neighbourhood centring (312-315), squared distance
    to the kernel points (325-329), linear influence clamp (368), zero shadow
    feature row (388), gather (391), influence-weighted sum (394), per-kernel-point
    weight contraction and sum (401-406), division by the number of neighbours
    whose feature row sums to > 0 (409-412).  `count` (Nq,) fixes that divisor
    (see `kpconv_count`).
    """
    dt = x.dtype
    s_aug = torch.cat([s_pts, torch.full_like(s_pts[:1], 1e6)], 0)
    x_aug = torch.cat([x, torch.zeros_like(x[:1])], 0)
    outs = []
    for a in range(0, q_pts.shape[0], chunk):
        idx = inds[a:a + chunk]
        nb = s_aug[idx] - q_pts[a:a + chunk, None, :]                  # (n,K,3)
        diff = nb[:, :, None, :] - kernel_points[None, None]           # (n,K,P,3)
        d2 = (diff ** 2).sum(-1)
        infl = torch.clamp(1 - torch.sqrt(d2) / extent, min=0.0).transpose(1, 2)  # (n,P,K)
        nx = x_aug[idx]                                                # (n,K,Cin)
        wf = infl @ nx                                                 # (n,P,Cin)
        out = torch.einsum('npc,pco->no', wf, weights.to(dt))
        cnt = (nx.sum(-1) > 0).sum(-1).clamp(min=1) if count is None else count[a:a + chunk]
        outs.append(out / cnt[:, None].to(dt))
    return torch.cat(outs, 0) if outs else x.new_zeros((0, weights.shape[-1]))


def kpconv_count(inds, x):
    """kpconv's divisor per query: the number of neighbours whose feature row sums to > 0, at least 1."""
    pos = torch.cat([x.detach().sum(-1) > 0, torch.zeros(1, dtype=torch.bool)])
    return pos[inds].sum(-1).clamp(min=1)


def instance_norm(x, lens, eps=1e-5):
    """Per-cloud InstanceNorm1d(affine=False, no running stats): biased variance over
    the points of each cloud (kpconv_blocks.py:489, 505-519)."""
    out = torch.empty_like(x)
    a = 0
    for n in map(int, lens):
        seg = x[a:a + n]
        mu = seg.mean(0, keepdim=True)
        var = seg.var(0, unbiased=False, keepdim=True)
        out[a:a + n] = (seg - mu) / torch.sqrt(var + eps)
        a += n
    return out


def _act(x, slope, decisions=None, site=None):
    """LeakyReLU(slope), ReLU for slope 0.  With `decisions`, the elements that take the identity branch are the
    boolean mask decisions[site] (recorded there as x > 0 when absent); the math stays smooth in x."""
    if decisions is None:
        return F.relu(x) if slope == 0 else F.leaky_relu(x, slope)
    mask = decisions.setdefault(site, x.detach() > 0)
    return torch.where(mask, x, x * slope)


def unary(x, w, lens, relu=True, decisions=None, site=None):
    """UnaryBlock: Linear(no bias) -> InstanceNorm -> LeakyReLU(0.1) (kpconv_blocks.py:533-561)."""
    y = instance_norm(x @ w.t(), lens)
    return _act(y, 0.1, decisions, site) if relu else y


def max_pool(x, inds, winner=None):
    """kpconv_blocks.py:127-143: max over the K gathered rows, zero shadow row.  `winner` (Nq,C) fixes the slot
    that each output takes (see `max_pool_winner`)."""
    x_aug = torch.cat([x, torch.zeros_like(x[:1])], 0)
    if winner is None:
        return x_aug[inds].max(1).values
    return x_aug[inds].gather(1, winner[:, None, :]).squeeze(1)


def max_pool_winner(x, inds):
    """The first slot of each (query, channel) that holds the maximum, (Nq,C) int64."""
    g = torch.cat([x.detach(), torch.zeros_like(x[:1])], 0)[inds]
    return (g == g.max(1, keepdim=True).values).to(torch.uint8).argmax(1)


def encoder_block(sd, cfg, i, x, meta, dtype=torch.float32, decisions=None, prefix='kpf_encoder.encoder_blocks.'):
    """Encoder block i: SimpleBlock (kpconv_blocks.py:632-646) or ResnetBottleneckBlock (706-741).

    `decisions` (a dict, optional) fixes the block's branches; every site absent from it is filled in with the
    choice this evaluation takes, so `{}` records them.  Sites: 'kpconv' the KPConv divisor per query (Nq,);
    'pool' the max-pool winner slot per (query, channel); 'unary1', 'conv', 'out' the LeakyReLU masks after
    unary1, after the KPConv's InstanceNorm and at the block output ('out' alone for a SimpleBlock)."""
    b = pyramid_plan(cfg)[1][i]
    g = lambda k: sd[f'{prefix}{i}.{k}'].to(dtype)
    d = decisions
    lv = b['level']
    lens = [np.asarray(l) for l in meta['stack_lengths']]
    if b['strided']:
        q, s, idx, l_post = (_t(meta['points'][lv + 1], dtype), _t(meta['points'][lv], dtype),
                             _t(meta['pools'][lv], torch.long), lens[lv + 1])
    else:
        s = _t(meta['points'][lv], dtype)
        q, idx, l_post = s, _t(meta['neighbors'][lv], torch.long), lens[lv]
    conv = lambda h: kpconv(q, s, idx, h, g('KPConv.weights'), g('KPConv.kernel_points'), b['extent'],
                            count=None if d is None else d.setdefault('kpconv', kpconv_count(idx, h)))
    if b['kind'] == 'simple':
        return _act(instance_norm(conv(x), l_post), 0.1, d, 'out')
    mid = b['out_dim'] // 4
    h = unary(x, g('unary1.mlp.weight'), lens[lv], decisions=d, site='unary1') if b['in_dim'] != mid else x
    h = _act(instance_norm(conv(h), l_post), 0.1, d, 'conv')
    h = unary(h, g('unary2.mlp.weight'), l_post, relu=False)
    sc = x
    if b['strided']:
        sc = max_pool(x, idx, None if d is None else d.setdefault('pool', max_pool_winner(x, idx)))
    if b['in_dim'] != b['out_dim']:
        sc = unary(sc, g('unary_shortcut.mlp.weight'), l_post, relu=False)
    return _act(h + sc, 0.1, d, 'out')


def encoder(sd, cfg, meta, dtype=torch.float32, prefix='kpf_encoder.encoder_blocks.'):
    """KPFEncoder.forward (kpconv.py:81-88): the blocks in sequence on a constant input feature."""
    _, blocks, _ = pyramid_plan(cfg)
    x = torch.ones((len(meta['points'][0]), 1), dtype=dtype)           # regtr.py:122
    for i in range(len(blocks)):
        x = encoder_block(sd, cfg, i, x, meta, dtype, prefix=prefix)
    return x


# ------------------------------------------------------------------ transformer

def pos_embed_sine(xyz, d_model=256, temperature=10000.0, scale=1.0):
    """PositionEmbeddingCoordsSine.forward (transformer/position_embedding.py:29-50)."""
    n_dim = xyz.shape[-1]
    npf = d_model // n_dim // 2 * 2
    dim_t = torch.arange(npf, dtype=torch.float32)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode='trunc') / npf)
    v = (xyz * (scale * 2 * math.pi)).unsqueeze(-1) / dim_t.to(xyz.dtype)
    emb = torch.stack([v[..., 0::2].sin(), v[..., 1::2].cos()], dim=-1).reshape(*xyz.shape[:-1], -1)
    return F.pad(emb, (0, d_model - npf * n_dim))


def pos_embed_learned(sd, xyz, prefix='pos_embed.'):
    """PositionEmbeddingLearned.forward (transformer/position_embedding.py:53-72): 5-layer MLP, ReLU between."""
    h = xyz
    for i in (0, 2, 4, 6, 8):
        h = h @ sd[f'{prefix}mlp.{i}.weight'].to(xyz.dtype).t() + sd[f'{prefix}mlp.{i}.bias'].to(xyz.dtype)
        if i != 8:
            h = F.relu(h)
    return h


def mha(q_in, k_in, v_in, in_w, in_b, out_w, out_b, nhead):
    """nn.MultiheadAttention forward on ONE un-padded sequence pair (no mask needed):
    packed in-projection, per-head softmax(q k^T / sqrt(dh)) v, out-projection.
    q_in (Lq,E), k_in/v_in (Lk,E).  Equivalent to the padded/masked call the reference
    makes (transformers.py:197-226) because masked keys get exactly zero weight."""
    E = q_in.shape[-1]
    dh = E // nhead
    q = (q_in @ in_w[:E].t() + in_b[:E]).view(-1, nhead, dh).transpose(0, 1)
    k = (k_in @ in_w[E:2 * E].t() + in_b[E:2 * E]).view(-1, nhead, dh).transpose(0, 1)
    v = (v_in @ in_w[2 * E:].t() + in_b[2 * E:]).view(-1, nhead, dh).transpose(0, 1)
    att = torch.softmax((q / math.sqrt(dh)) @ k.transpose(1, 2), dim=-1)
    o = (att @ v).transpose(0, 1).reshape(-1, E)
    return o @ out_w.t() + out_b


def cross_encoder_layer(sd, cfg, i, src, tgt, sp, tp, decisions=None, prefix='transformer_encoder.'):
    """TransformerCrossEncoderLayer i: forward_pre (transformers.py:183-244) or, without pre_norm, forward_post
    (121-181), on one pair of un-padded sequences; sp / tp are the position embeddings the layer adds (zeros when
    it adds none).  `decisions` (a dict, optional) fixes the feed-forward ReLU masks, sites 'ffn_src' and
    'ffn_tgt', as in `encoder_block`.  Returns (src, tgt)."""
    E, H = cfg.d_embed, cfg.nhead
    dt = src.dtype
    p = f'{prefix}layers.{i}.'
    g = lambda k: sd[p + k].to(dt)
    ln = lambda x, k: F.layer_norm(x, (E,), g(k + '.weight'), g(k + '.bias'), 1e-5)
    att = lambda m, q, k, v: mha(q, k, v, g(m + '.in_proj_weight'), g(m + '.in_proj_bias'),
                                 g(m + '.out_proj.weight'), g(m + '.out_proj.bias'), H)
    ffn = lambda x, site: _act(x @ g('linear1.weight').t() + g('linear1.bias'), 0, decisions, site) \
        @ g('linear2.weight').t() + g('linear2.bias')
    if not cfg.pre_norm:
        swp, twp = src + sp, tgt + tp
        src = ln(src + att('self_attn', swp, swp, swp if cfg.sa_val_has_pos_emb else src), 'norm1')
        tgt = ln(tgt + att('self_attn', twp, twp, twp if cfg.sa_val_has_pos_emb else tgt), 'norm1')
        swp, twp = src + sp, tgt + tp
        s3 = att('multihead_attn', swp, twp, twp if cfg.ca_val_has_pos_emb else tgt)
        t3 = att('multihead_attn', twp, swp, swp if cfg.ca_val_has_pos_emb else src)
        src, tgt = ln(src + s3, 'norm2'), ln(tgt + t3, 'norm2')
        return ln(src + ffn(src, 'ffn_src'), 'norm3'), ln(tgt + ffn(tgt, 'ffn_tgt'), 'norm3')
    s2 = ln(src, 'norm1'); s2p = s2 + sp
    src = src + att('self_attn', s2p, s2p, s2p if cfg.sa_val_has_pos_emb else s2)
    t2 = ln(tgt, 'norm1'); t2p = t2 + tp
    tgt = tgt + att('self_attn', t2p, t2p, t2p if cfg.sa_val_has_pos_emb else t2)
    s2, t2 = ln(src, 'norm2'), ln(tgt, 'norm2')
    s2p, t2p = s2 + sp, t2 + tp
    s3 = att('multihead_attn', s2p, t2p, t2p if cfg.ca_val_has_pos_emb else t2)
    t3 = att('multihead_attn', t2p, s2p, s2p if cfg.ca_val_has_pos_emb else s2)
    src, tgt = src + s3, tgt + t3
    return src + ffn(ln(src, 'norm3'), 'ffn_src'), tgt + ffn(ln(tgt, 'norm3'), 'ffn_tgt')


def cross_encoder(sd, cfg, src, tgt, src_pe, tgt_pe, prefix='transformer_encoder.'):
    """TransformerCrossEncoder.forward with return_intermediate and final norm
    (transformers.py:27-59) over `cross_encoder_layer`.
    Operates per pair on un-padded sequences; returns (L,S,E), (L,T,E)."""
    E = cfg.d_embed
    dt = src.dtype
    use_pe = cfg.transformer_encoder_has_pos_emb
    sp = src_pe if use_pe else torch.zeros_like(src)
    tp = tgt_pe if use_pe else torch.zeros_like(tgt)
    # no final norm without pre_norm (regtr.py:64)
    ln = (lambda x: F.layer_norm(x, (E,), sd[prefix + 'norm.weight'].to(dt), sd[prefix + 'norm.bias'].to(dt), 1e-5)) \
        if cfg.pre_norm else (lambda x: x)
    outs_s, outs_t = [], []
    for i in range(cfg.num_encoder_layers):
        src, tgt = cross_encoder_layer(sd, cfg, i, src, tgt, sp, tp, prefix=prefix)
        outs_s.append(ln(src))
        outs_t.append(ln(tgt))
    return torch.stack(outs_s), torch.stack(outs_t)


def regressor(sd, feats, prefix='correspondence_decoder.'):
    """CorrespondenceRegressor.forward (regtr.py:413-443) on an un-padded (L,S,E) tensor."""
    g = lambda k: sd[prefix + k].to(feats.dtype)
    h = F.relu(feats @ g('coor_mlp.0.weight').t() + g('coor_mlp.0.bias'))
    h = F.relu(h @ g('coor_mlp.2.weight').t() + g('coor_mlp.2.bias'))
    corr = h @ g('coor_mlp.4.weight').t() + g('coor_mlp.4.bias')
    logit = feats @ g('conf_logits_decoder.weight').t() + g('conf_logits_decoder.bias')
    return corr, logit


def corr_decoder(sd, cfg, feats_q, feats_k, pe_q, pe_k, xyz_k, prefix='correspondence_decoder.'):
    """CorrespondenceDecoder (regtr.py:297-396) for one direction of one pair, un-padded:
    feats_q (L,Q,E), feats_k (L,S,E) conditioned features, pe_* position embeddings, xyz_k (S,3).
    simple_attention (316-351): q = q_proj(f_q + pe)/sqrt(E), k = k_proj(f_k + pe), softmax over keys,
    weighted sum of the key coordinates; logits from the plain features (383).  q_norm is unused (306)."""
    g = lambda k: sd[prefix + k].to(feats_q.dtype)
    use_pe = cfg.corr_decoder_has_pos_emb
    fq = feats_q + pe_q if use_pe else feats_q
    fk = feats_k + pe_k if use_pe else feats_k
    q = (fq @ g('q_proj.weight').t() + g('q_proj.bias')) / math.sqrt(fq.shape[-1])
    k = fk @ g('k_proj.weight').t() + g('k_proj.bias')
    attn = torch.softmax(q @ k.transpose(-2, -1), dim=-1)               # (L,Q,S)
    corr = attn @ xyz_k
    logit = feats_q @ g('conf_logits_decoder.weight').t() + g('conf_logits_decoder.bias')
    return corr, logit


def kabsch(a, b, w):
    """compute_rigid_transform (utils/se3_torch.py:108-154), weighted branch."""
    wn = w[..., None] / torch.clamp_min(w.sum(-1, keepdim=True)[..., None], 1e-6)
    ca, cb = (a * wn).sum(-2), (b * wn).sum(-2)
    ac, bc = a - ca[..., None, :], b - cb[..., None, :]
    cov = ac.transpose(-2, -1) @ (bc * wn)
    u, _, vh = torch.linalg.svd(cov)
    v = vh.transpose(-2, -1)
    rp = v @ u.transpose(-2, -1)
    vn = v.clone(); vn[..., 2] *= -1
    rn = vn @ u.transpose(-2, -1)
    R = torch.where(torch.det(rp)[..., None, None] > 0, rp, rn)
    t = -R @ ca[..., :, None] + cb[..., :, None]
    return torch.cat([R, t], -1)


# ---------------------------------------------------------------------- forward

def forward(sd, cfg, src_list, tgt_list, dtype=torch.float32, meta=None, with_upsamples=True):
    """RegTR.forward (/root/reference/src/models/regtr.py:104-235) on the CPU.

    `meta` may carry a precomputed pyramid (e.g. from the CUDA path, to isolate the
    float stages); by default the oracle pre-processing in oracle/pre.py is used.
    Returns the reference's output dict (torch CPU tensors) plus 'kpconv_meta'.
    """
    B = len(src_list)
    if meta is None:
        meta = pre.preprocess(cfg, list(src_list) + list(tgt_list), with_upsamples)
    slens = [int(v) for v in meta['stack_lengths'][-1]]
    feats = encoder(sd, cfg, meta, dtype)
    both = feats @ sd['feat_proj.weight'].to(dtype).t() + sd['feat_proj.bias'].to(dtype)
    xyz_c = _t(meta['points'][-1], dtype)
    if cfg.get('pos_emb_type', 'sine') == 'sine':
        pe = pos_embed_sine(xyz_c, cfg.d_embed, scale=cfg.get('pos_emb_scaling', 1.0))
    else:
        pe = pos_embed_learned({k: v.to(dtype) for k, v in sd.items() if k.startswith('pos_embed.')}, xyz_c)
    f_split, x_split, p_split = (torch.split(v, slens) for v in (both, xyz_c, pe))
    out = {k: [] for k in ('src_feat_un', 'tgt_feat_un', 'src_feat', 'tgt_feat', 'src_kp', 'tgt_kp',
                           'src_kp_warped', 'tgt_kp_warped', 'src_overlap', 'tgt_overlap')}
    poses = []
    for b in range(B):
        fs, ft = f_split[b], f_split[B + b]
        xs, xt = x_split[b], x_split[B + b]
        cs, ct = cross_encoder(sd, cfg, fs, ft, p_split[b], p_split[B + b])
        if cfg.get('direct_regress_coor', False):
            s_corr, s_log = regressor(sd, cs)
            t_corr, t_log = regressor(sd, ct)
        else:
            s_corr, s_log = corr_decoder(sd, cfg, cs, ct, p_split[b], p_split[B + b], xt)
            t_corr, t_log = corr_decoder(sd, cfg, ct, cs, p_split[B + b], p_split[b], xs)
        L = cs.shape[0]
        a = torch.cat([xs.expand(L, -1, -1), t_corr], 1)               # regtr.py:185-190
        bb = torch.cat([s_corr, xt.expand(L, -1, -1)], 1)
        w = torch.cat([torch.sigmoid(s_log[..., 0]), torch.sigmoid(t_log[..., 0])], 1)
        poses.append(kabsch(a, bb, w))
        for k, v in (('src_feat_un', fs), ('tgt_feat_un', ft), ('src_feat', cs), ('tgt_feat', ct),
                     ('src_kp', xs), ('tgt_kp', xt), ('src_kp_warped', s_corr),
                     ('tgt_kp_warped', t_corr), ('src_overlap', s_log), ('tgt_overlap', t_log)):
            out[k].append(v)
    out['pose'] = torch.stack(poses, 1)                                 # (L,B,3,4)
    out['kpconv_meta'] = meta
    return out
