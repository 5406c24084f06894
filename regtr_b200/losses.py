"""Loss values of a forward pass (SURVEY.md 8f N1/N3: `test_step` reports them, `training_step` needs them).

Mirror of
  * `RegTR.compute_loss` (/root/reference/src/models/regtr.py:237-294) and its `weight_dict` (regtr.py:89-93),
  * `compute_overlaps` (/root/reference/src/models/backbone_kpconv/kpconv.py:540-566),
  * `CorrCriterion` (/root/reference/src/models/losses/corr_loss.py:9-40),
  * `InfoNCELossFull` (/root/reference/src/models/losses/feature_loss.py:246-314),
  * `CircleLossFull(dist_type='euclidean')` (/root/reference/src/models/losses/feature_loss.py:160-243).
`compute_loss` is plain torch ops on whatever device the predictions live on: the restatement pinned against the
reference, and the yardstick of `compute_loss_device`, the same losses on the library's kernels (csrc/loss.cu), which
`RegTR.compute_loss` takes for the model's own CUDA outputs.  Differentiable: on outputs of `RegTR.forward_train` the gradient flows on into the library's backward
kernels (everything after the KPConv encoder)."""
from __future__ import annotations

from typing import Dict, List

import torch
import torch.nn.functional as F

_EPS = 1e-6


def se3_transform_list(pose, xyz: List[torch.Tensor]):
    """utils/se3_torch.py:70-90: pose (B,3,4) or list, xyz list(B) of ([L,] N, 3)."""
    return [x @ pose[b][:3, :3].transpose(-1, -2) + pose[b][:3, 3] for b, x in enumerate(xyz)]


def se3_inv(pose):
    r = pose[..., :3, :3].transpose(-1, -2)
    return torch.cat([r, -(r @ pose[..., :3, 3:4])], dim=-1)


def compute_overlaps(batch) -> Dict[str, torch.Tensor]:
    """Ground-truth overlap per level: level 0 = the dataset's masks, coarser levels = unweighted mean over
    the valid pooling indices, clamped to [0,1]  (kpconv.py:540-566)."""
    meta = batch['kpconv_meta']
    out = {'pyr_0': torch.cat(list(batch['src_overlap']) + list(batch['tgt_overlap']), dim=0).type(torch.float)}
    invalid = [s.sum() for s in meta['stack_lengths']]
    for p in range(1, len(meta['points'])):
        pool = meta['pools'][p - 1].clone()
        valid = pool < invalid[p - 1]
        pool[~valid] = 0
        g = out[f'pyr_{p - 1}'][pool] * valid
        out[f'pyr_{p}'] = torch.clamp(torch.sum(g, dim=1) / torch.sum(valid, dim=1), min=0, max=1)
    return out


def corr_loss(kp_before, kp_warped_pred, pose_gt, overlap_weights=None):
    """CorrCriterion(metric='mae')  (corr_loss.py:19-40)."""
    gt = se3_transform_list(pose_gt, kp_before)
    err = torch.sum(torch.abs(torch.cat(kp_warped_pred, dim=0) - torch.cat(gt, dim=0)), dim=-1)
    if overlap_weights is None:
        return torch.mean(err, dim=1)
    w = torch.cat(list(overlap_weights))
    return torch.sum(w * err) / torch.clamp_min(torch.sum(w), _EPS)


def infonce_loss(W, src_feat, tgt_feat, src_xyz, tgt_xyz, r_p: float, r_n: float):
    """InfoNCELossFull.forward (feature_loss.py:268-314): bilinear logits with the symmetrised upper triangle
    of W; positive = nearest target point if closer than r_p; other points within r_n are ignored."""
    Wt = torch.triu(W)
    Ws = Wt + Wt.T
    per_pair = []
    for a, p, ax, px in zip(src_feat, tgt_feat, src_xyz, tgt_xyz):
        logits = torch.einsum('ic,cd,jd->ij', a, Ws, p)
        with torch.no_grad():
            d = torch.cdist(ax, px)
            d1, i1 = d.topk(k=1, dim=-1, largest=False)
            mask = d1[..., 0] < r_p
            ignore = d < r_n
            ignore.scatter_(-1, i1, 0)
        logits = logits.masked_fill(ignore, -float('inf'))
        loss = -torch.gather(logits, -1, i1).squeeze(-1) + torch.logsumexp(logits, dim=-1)
        per_pair.append(torch.sum(loss[mask]) / torch.sum(mask))
    return torch.mean(torch.stack(per_pair))


def circle_loss(src_feat, tgt_feat, src_xyz, tgt_xyz, r_p: float, r_n: float, log_scale: float = 10.0,
                pos_margin: float = 0.1, neg_margin: float = 1.4):
    """CircleLossFull.forward / get_circle_loss (feature_loss.py:191-243) with dist_type='euclidean', as written:
    feature distances from explicit differences plus 1e-12 under the square root, masked entries offset by 1e5 so
    that their detached weight is 0 and exp(0) = 1 enters every log-sum-exp, F.softplus (linear above 20), and the
    mean over an empty selection, which is NaN.  The pair losses are meaned over the pairs."""
    total = 0
    for a, p, ax, px in zip(src_feat, tgt_feat, src_xyz, tgt_xyz):
        coords = torch.cdist(ax, px)
        feats = torch.sqrt(torch.sum((a.T[..., :, None] - p.T[..., None, :]) ** 2, dim=-3) + 1e-12)
        pos_mask, neg_mask = coords < r_p, coords > r_n
        row_sel = ((pos_mask.sum(-1) > 0) * (neg_mask.sum(-1) > 0)).detach()
        col_sel = ((pos_mask.sum(-2) > 0) * (neg_mask.sum(-2) > 0)).detach()
        pos = feats - 1e5 * (~pos_mask).to(feats.dtype)
        pos_weight = torch.clamp_min(pos - pos_margin, min=0).detach()
        zp = log_scale * (pos - pos_margin) * pos_weight
        neg = feats + 1e5 * (~neg_mask).to(feats.dtype)
        neg_weight = torch.clamp_min(neg_margin - neg, min=0).detach()
        zn = log_scale * (neg_margin - neg) * neg_weight
        loss_row = F.softplus(torch.logsumexp(zp, dim=-1) + torch.logsumexp(zn, dim=-1)) / log_scale
        loss_col = F.softplus(torch.logsumexp(zp, dim=-2) + torch.logsumexp(zn, dim=-2)) / log_scale
        total = total + (loss_row[row_sel].mean() + loss_col[col_sel].mean()) / 2
    return total / len(src_feat)


def loss_weights(cfg) -> Dict[str, float]:
    """regtr.py:89-93."""
    wd = {}
    for k in ('overlap', 'feature', 'corr'):
        for i in cfg.get(f'{k}_loss_on', [cfg.num_encoder_layers - 1]):
            wd[f'{k}_{i}'] = cfg.get(f'wt_{k}')
    wd['feature_un'] = cfg.wt_feature_un
    return wd


def compute_loss(model, pred: Dict, batch: Dict) -> Dict[str, torch.Tensor]:
    """RegTR.compute_loss (regtr.py:237-294).  `model` supplies cfg and, for the InfoNCE feature loss, the two InfoNCE
    matrices (`feature_criterion.W`, `feature_criterion_un.W`; the circle loss has no parameter); batch needs
    `kpconv_meta`, `pose`, `src_overlap`, `tgt_overlap` (the dataset's level-0 overlap masks)."""
    cfg = model.cfg
    if cfg.feature_loss_type not in ('infonce', 'circle'):
        raise NotImplementedError(f'feature_loss_type {cfg.feature_loss_type!r}')
    meta, pose_gt = batch['kpconv_meta'], batch['pose']
    p = len(meta['stack_lengths']) - 1
    batch['overlap_pyr'] = compute_overlaps(batch)
    lens = [int(v) for v in meta['stack_lengths'][p]]
    B = len(lens) // 2
    parts = torch.split(batch['overlap_pyr'][f'pyr_{p}'], lens)
    src_ov, tgt_ov = parts[:B], parts[B:]
    losses = {}
    all_pred = torch.cat(list(pred['src_overlap']) + list(pred['tgt_overlap']), dim=-2)
    all_gt = batch['overlap_pyr'][f'pyr_{p}']
    for i in cfg.overlap_loss_on:
        losses[f'overlap_{i}'] = F.binary_cross_entropy_with_logits(all_pred[i, :, 0], all_gt)
    src_kp_gt = se3_transform_list(pose_gt, list(pred['src_kp']))
    if cfg.feature_loss_type == 'circle':
        feature = lambda _crit, s, t: circle_loss(s, t, src_kp_gt, list(pred['tgt_kp']), cfg.r_p, cfg.r_n)
    else:
        feature = lambda crit, s, t: infonce_loss(crit.W, s, t, src_kp_gt, list(pred['tgt_kp']), cfg.r_p, cfg.r_n)
    for i in cfg.feature_loss_on:
        losses[f'feature_{i}'] = feature(getattr(model, 'feature_criterion', None), [s[i] for s in pred['src_feat']],
                                         [t[i] for t in pred['tgt_feat']])
    losses['feature_un'] = feature(getattr(model, 'feature_criterion_un', None), list(pred['src_feat_un']),
                                   list(pred['tgt_feat_un']))
    for i in cfg.corr_loss_on:
        s = corr_loss(list(pred['src_kp']), [w[i] for w in pred['src_kp_warped']], pose_gt, src_ov)
        t = corr_loss(list(pred['tgt_kp']), [w[i] for w in pred['tgt_kp_warped']],
                      torch.stack([se3_inv(q) for q in pose_gt]), tgt_ov)
        losses[f'corr_{i}'] = s + t
    wd = loss_weights(cfg)
    losses['total'] = torch.sum(torch.stack([losses[k] * wd[k] for k in losses]))
    return losses


def loss_keys(cfg) -> List[str]:
    """The keys of `compute_loss_device`'s result in order (`ops.LossGeometry.keys` and 'total')."""
    return [f'overlap_{i}' for i in cfg.overlap_loss_on] + [f'feature_{i}' for i in cfg.feature_loss_on] + \
        ['feature_un'] + [f'corr_{i}' for i in cfg.corr_loss_on] + ['total']


_weight_vectors = {}


def _weight_vector(wd: Dict[str, float], keys, device) -> torch.Tensor:
    """fp32 device vector of the weights of `keys`, uploaded once per (device, weights)."""
    key = (str(device), tuple((k, float(wd[k])) for k in keys))
    if key not in _weight_vectors:
        _weight_vectors[key] = torch.tensor([wd[k] for k in keys], dtype=torch.float32, device=device)
    return _weight_vectors[key]


def device_route(model, pred, batch) -> bool:
    """True when `compute_loss_device` applies: `pred` carries the packed CUDA tensors its views were cut from, at
    exact shapes and 256 channels, the InfoNCE or the circle loss is configured, and the pyramid has an int32 pooling
    table for every level."""
    core = getattr(pred, 'core', None)
    if core is None or model.cfg.feature_loss_type not in ('infonce', 'circle') or not core['both_un'].is_cuda:
        return False
    from . import ops
    from .kpconv import _meta_private
    meta = _meta_private(batch['kpconv_meta'], core['both_un'].device)
    n = sum(meta['_lens'][-1])
    return (core['both_un'].shape == (n, ops.LOSS_DIM) and core['cond'].shape[1] == n and
            core['cond'].shape[0] <= ops.LOSS_MAX_LAYERS and len(meta['_points']) <= ops.LOSS_MAX_LEVELS and
            len(meta['_lens'][-1]) >= 2 and all(p is not None for p in meta['_pools32'][:len(meta['_points']) - 1]))


def compute_loss_device(model, pred, batch, reduce_norms=None) -> Dict[str, torch.Tensor]:
    """`compute_loss` on the library's loss kernels (csrc/loss.cu), for a `pred` that `device_route` accepts: same
    keys in the same order, same total.  Reads the packed tensors `pred.core`, not the per-cloud views; the number of
    launches does not depend on the number of pairs and nothing synchronises with the host.  Fills
    batch['overlap_pyr'] like `compute_loss`.

    reduce_norms: for a batch that is a slice of a larger one (data parallelism), a callable that sums the (4,) fp64
    normaliser vector of `ops.loss_norms` in place over every slice (an all-reduce); the values and their gradients
    are then this slice's share of the whole batch's losses, and the shares add up to them."""
    from . import ops
    from .kpconv import _meta_private
    cfg, core = model.cfg, pred.core
    dev = core['both_un'].device
    meta = _meta_private(batch['kpconv_meta'], dev)
    n_lvl = len(meta['_points'])
    pyr0 = torch.cat(list(batch['src_overlap']) + list(batch['tgt_overlap']), dim=0).type(torch.float)
    pyr = ops.overlap_pyramid(pyr0, meta['_pools32'][:n_lvl - 1], meta['_offs'], meta['_n_clouds'])
    batch['overlap_pyr'] = {f'pyr_{p}': t for p, t in enumerate(pyr)}
    pose = batch['pose']
    pose = pose if torch.is_tensor(pose) else torch.stack(list(pose))
    pose = pose[..., :3, :].to(device=dev, dtype=torch.float32).contiguous()
    geo = ops.LossGeometry(core['xyz_c'], meta['_offs'][-1], meta['_lens'][-1], pose, pyr[-1], cfg.overlap_loss_on,
                           cfg.feature_loss_on, cfg.corr_loss_on, cfg.r_p, cfg.r_n, feature_loss=cfg.feature_loss_type)
    if reduce_norms is not None:
        geo.norm = ops.loss_norms(geo)
        reduce_norms(geo.norm)
    circle = cfg.feature_loss_type == 'circle'                  # CircleLossFull has no parameter
    vals = ops.loss_values(core['both_un'], core['cond'], core['corr'], core['logit'],
                           None if circle else model.feature_criterion.W,
                           None if circle else model.feature_criterion_un.W, geo)
    keys = geo.keys()
    losses = {k: vals[j] for j, k in enumerate(keys)}
    losses['total'] = torch.sum(vals * _weight_vector(loss_weights(cfg), keys, dev))
    return losses
