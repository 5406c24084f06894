"""RegTR forward on the H100 kernels -- the drop-in boundary.

`RegTR(cfg)` keeps the reference's constructor, sub-module names, state_dict layout
(168 keys for the 3DMatch config, loadable with strict=True) and
`forward(batch: dict) -> dict` contract (/root/reference/src/models/regtr.py:23-235):

    batch['src_xyz'], batch['tgt_xyz']: lists (B) of (Ni,3) CUDA tensors
    -> outputs: src_feat_un/tgt_feat_un (tuples of (S,256)), src_feat/tgt_feat (lists of
       (6,S,256)), src_kp/tgt_kp, src_kp_warped/tgt_kp_warped (lists of (6,S,3)),
       src_overlap/tgt_overlap (lists of (6,S,1) logits), pose (6,B,3,4);
       side effect batch['kpconv_meta'] (regtr.py:118).

What differs from the reference is *how*: packed tokens instead of padded ones, one host
sync for the pyramid sizes, hand-written sm_90a kernels for the neighbour search, the
KPConv gather/aggregation, normalisations, attention core and Kabsch, and a fused
correspondence-assembly + sigmoid + Kabsch kernel (regtr.py:185-203 in one launch).
`forward_train(batch)` is the differentiable variant for fine-tuning everything after the KPConv encoder (the
encoder runs without grad and must be frozen); `forward_train(batch, train_encoder=True)` trains the encoder as well.
`compute_loss` of its outputs is differentiable, and the backward runs on the library's backward kernels (attention,
LayerNorm, dense layers, and for the encoder KPConv, max-pool and per-cloud InstanceNorm).
"""
from __future__ import annotations

import contextlib
import logging
import time
import weakref

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .kpconv import KPFEncoder, PreprocessorGPU
from .lazy import LazyDict
from .transformer import (AttentionPlan, PositionEmbeddingCoordsSine, PositionEmbeddingLearned, warn_dropout_eval_only,
                          TransformerCrossEncoder, TransformerCrossEncoderLayer)


class _LossParam(nn.Module):
    """Keeps `feature_criterion*.W` loadable (InfoNCELossFull's only parameter; training-only)."""

    def __init__(self, d_embed):
        super().__init__()
        self.W = nn.Parameter(torch.zeros(d_embed, d_embed), requires_grad=True)


class PackedOutput(dict):
    """The reference's output dict, plus `core`: the packed tensors (`both_un`, `xyz_c`, `cond`, `corr`, `logit`,
    `pose`) its per-cloud views were cut from.  Keys and values are those of a plain dict; `compute_loss` reads `core`
    to run the loss kernels on the packed tokens."""

    core = None


class CorrespondenceRegressor(nn.Module):
    """MLP 256->256->256->3 + Linear 256->1 on every layer's features (regtr.py:399-443)."""

    def __init__(self, d_embed):
        super().__init__()
        self.coor_mlp = nn.Sequential(nn.Linear(d_embed, d_embed), nn.ReLU(), nn.Linear(d_embed, d_embed),
                                      nn.ReLU(), nn.Linear(d_embed, 3))
        self.conf_logits_decoder = nn.Linear(d_embed, 1)

    def forward_packed(self, feats, xyz=None, pe=None, plan=None):
        """feats (L,N,E) packed -> corr (L,N,3), logits (L,N,1)."""
        L_, n, E = feats.shape
        x = feats.reshape(L_ * n, E)
        h = ops.linear(x, self.coor_mlp[0].weight, self.coor_mlp[0].bias, relu=True)
        h = ops.linear(h, self.coor_mlp[2].weight, self.coor_mlp[2].bias, relu=True)
        corr = ops.linear(h, self.coor_mlp[4].weight, self.coor_mlp[4].bias)
        logit = ops.linear(x, self.conf_logits_decoder.weight, self.conf_logits_decoder.bias)
        return corr.view(L_, n, 3), logit.view(L_, n, 1)


class CorrespondenceDecoder(nn.Module):
    """Attention-based correspondence decoding (regtr.py:297-396, `direct_regress_coor: False`):
    q_proj / k_proj of the conditioned features (+ position embedding), single-head softmax attention
    over the OTHER cloud's tokens, values = that cloud's coordinates; overlap logits from the plain
    features.  Same constructor and state_dict keys (`q_norm` is defined but never applied, as in the
    reference; `pos_embed` is the shared embedding module).  `num_neighbors > 0` is not supported."""

    def __init__(self, d_embed, use_pos_emb, pos_embed=None, num_neighbors=0):
        super().__init__()
        assert use_pos_emb is False or pos_embed is not None, \
            'Position encoder must be supplied if use_pos_emb is True'
        if num_neighbors > 0:
            raise NotImplementedError('top-k neighbour masking is unused by every reference config')
        self.use_pos_emb = use_pos_emb
        self.pos_embed = pos_embed
        self.q_norm = nn.LayerNorm(d_embed)
        self.q_proj = nn.Linear(d_embed, d_embed)
        self.k_proj = nn.Linear(d_embed, d_embed)
        self.conf_logits_decoder = nn.Linear(d_embed, 1)
        self.num_neighbors = num_neighbors

    def forward_packed(self, feats, xyz, pe, plan: AttentionPlan):
        """feats (L,N,E) packed, xyz (N,3), pe (N,E) -> corr (L,N,3), logits (L,N,1)."""
        L_, n, E = feats.shape
        f2 = (feats + pe[None]) if self.use_pos_emb else feats                      # regtr.py:379-380
        f2 = f2.reshape(L_ * n, E)
        qp = ops.linear(f2, self.q_proj.weight, self.q_proj.bias)
        kp = ops.linear(f2, self.k_proj.weight, self.k_proj.bias)
        corr = ops.corr_decode(qp, kp, xyz, plan.q_start, plan.q_len, plan.xk_start, plan.xk_len, plan.max_len, L_)
        logit = ops.linear(feats.reshape(L_ * n, E), self.conf_logits_decoder.weight, self.conf_logits_decoder.bias)
        return corr.view(L_, n, 3), logit.view(L_, n, 1)


class RegTR(nn.Module):
    def __init__(self, cfg, *args, **kwargs):
        super().__init__()
        self.cfg = cfg
        self.logger = logging.getLogger(self.__class__.__name__)
        self.preprocessor = PreprocessorGPU(cfg)
        self.kpf_encoder = KPFEncoder(cfg, cfg.d_embed)
        self.feat_proj = nn.Linear(self.kpf_encoder.encoder_skip_dims[-1], cfg.d_embed, bias=True)
        if cfg.get('pos_emb_type', 'sine') == 'sine':
            self.pos_embed = PositionEmbeddingCoordsSine(3, cfg.d_embed, scale=cfg.get('pos_emb_scaling', 1.0))
        elif cfg['pos_emb_type'] == 'learned':
            self.pos_embed = PositionEmbeddingLearned(3, cfg.d_embed)
        else:
            raise NotImplementedError
        layer = TransformerCrossEncoderLayer(
            cfg.d_embed, cfg.nhead, cfg.d_feedforward, cfg.dropout, activation=cfg.transformer_act,
            normalize_before=cfg.pre_norm, sa_val_has_pos_emb=cfg.sa_val_has_pos_emb,
            ca_val_has_pos_emb=cfg.ca_val_has_pos_emb, attention_type=cfg.attention_type,
            attention_impl=cfg.get('attention_impl', 'fp32'))
        norm = nn.LayerNorm(cfg.d_embed) if cfg.pre_norm else None
        self.transformer_encoder = TransformerCrossEncoder(layer, cfg.num_encoder_layers, norm,
                                                           return_intermediate=True)
        if cfg.get('direct_regress_coor', False):
            self.correspondence_decoder = CorrespondenceRegressor(cfg.d_embed)
        else:
            self.correspondence_decoder = CorrespondenceDecoder(cfg.d_embed, cfg.corr_decoder_has_pos_emb,
                                                                self.pos_embed)
        if cfg.feature_loss_type == 'infonce':
            self.feature_criterion = _LossParam(cfg.d_embed)
            self.feature_criterion_un = _LossParam(cfg.d_embed)

    @property
    def device(self):
        return next(self.parameters()).device

    # ------------------------------------------------------------------ core (sync-free)
    # The three stages after the pyramid, at the reference's own `_TIMEIT` boundaries (regtr.py:108-216:
    # preprocess | encoder | attention + decoder | pose).  None synchronises with the host, so any prefix /
    # suffix of them is CUDA-graph capturable (GraphedRegTR captures them as one graph, or one per stage
    # when stage times are wanted).
    def _stage_encoder(self, meta):
        """KPConv encoder + feature projection + position embedding (regtr.py:122-154)."""
        pts = meta['_points']
        feats0 = torch.ones_like(pts[0][:, 0:1])                                   # regtr.py:122
        feats_un, _ = self.kpf_encoder(feats0, meta)                               # regtr.py:136
        nd = meta.get('_ndev')
        both_un = ops.linear(feats_un, self.feat_proj.weight, self.feat_proj.bias,
                             m_dev=nd[-1] if nd else None)                         # regtr.py:145
        xyz_c = pts[-1]
        pe = self.pos_embed(xyz_c)                                                 # regtr.py:149-154
        return dict(both_un=both_un.contiguous(), xyz_c=xyz_c, pe=pe)

    def _stage_attention(self, enc, plan: AttentionPlan):
        """Cross-encoder + correspondence decoder on all layers (regtr.py:156-183)."""
        cfg = self.cfg
        cond = self.transformer_encoder.forward_packed(
            enc['both_un'], enc['pe'] if cfg.transformer_encoder_has_pos_emb else None, plan)   # (L,N,E)
        corr, logit = self.correspondence_decoder.forward_packed(cond, enc['xyz_c'], enc['pe'], plan)
        return dict(cond=cond, corr=corr, logit=logit)

    def _stage_pose(self, enc, att, offs_c, B: int):
        """Correspondence assembly + sigmoid + weighted Kabsch, one launch (regtr.py:185-203)."""
        return ops.pose_from_corr(enc['xyz_c'], att['corr'].contiguous(), att['logit'][..., 0].contiguous(), offs_c, B)

    def _core(self, meta, B: int, plan: AttentionPlan):
        enc = self._stage_encoder(meta)
        att = self._stage_attention(enc, plan)
        pose = self._stage_pose(enc, att, meta['_offs'][-1], B)
        return dict(both_un=enc['both_un'], xyz_c=enc['xyz_c'], cond=att['cond'], corr=att['corr'],
                    logit=att['logit'], pose=pose)

    @staticmethod
    def _assemble(core, lens_c, B):
        """Per-cloud views in the reference's output layout (regtr.py:218-234)."""
        n = sum(lens_c)
        split = lambda t, dim=0: torch.split(t.narrow(dim, 0, n), lens_c, dim=dim)
        un, kp = split(core['both_un']), split(core['xyz_c'])
        feat, warped, ovl = split(core['cond'], 1), split(core['corr'], 1), split(core['logit'], 1)
        out = PackedOutput({
            'src_feat_un': un[:B], 'tgt_feat_un': un[B:],
            'src_feat': list(feat[:B]), 'tgt_feat': list(feat[B:]),
            'src_kp': kp[:B], 'src_kp_warped': list(warped[:B]),
            'tgt_kp': kp[B:], 'tgt_kp_warped': list(warped[B:]),
            'src_overlap': list(ovl[:B]), 'tgt_overlap': list(ovl[B:]),
            'pose': core['pose'],
        })
        out.core = core
        return out

    def compute_loss(self, pred, batch):
        """Losses of a forward (regtr.py:237-294: overlap BCE, InfoNCE or circle feature losses (cfg.feature_loss_type),
        L1 correspondence loss, weighted total).  For outputs of `forward_train` (which carry autograd history) `total` is differentiable;
        for outputs of `forward` the values are computed without grad, as `test_step` reports them.
        Needs batch['pose'], ['src_overlap'], ['tgt_overlap'], ['kpconv_meta'].
        An output of this model's own `forward` / `forward_train` on CUDA goes through the loss kernels
        (`losses.compute_loss_device`: no host synchronisation, a launch count independent of B); any other `pred`
        (a hand-built or oracle dict, CPU tensors) goes through the torch restatement `losses.compute_loss`."""
        from . import losses
        fn = losses.compute_loss_device if losses.device_route(self, pred, batch) else losses.compute_loss
        if torch.is_grad_enabled() and pred['src_feat'][0].requires_grad:
            return fn(self, pred, batch)
        with torch.no_grad():
            return fn(self, pred, batch)

    def configure_optimizers(self):
        """The reference's solver (generic_reg_model.py:28-62) over self.parameters(), on the library's optimizer:
        cfg.optimizer 'AdamW' / 'Adam' (lr cfg.base_lr, weight_decay cfg.weight_decay) and cfg.scheduler 'step'
        (StepLR(*cfg.scheduler_param)) or 'none' (StepLR(50, 1.0)).  Sets and returns (self.optimizer, self.scheduler).
        Clip the gradients to cfg.grad_clip with regtr_b200.optim.clip_grad_norm_ before every optimizer.step()."""
        from . import optim
        cfg = self.cfg
        scheduler_type = cfg.get('scheduler', None)
        if scheduler_type == 'warmup':
            raise NotImplementedError("configure_optimizers: scheduler 'warmup' (no shipped config selects it)")
        if scheduler_type not in (None, 'none', 'step'):
            raise NotImplementedError(f'configure_optimizers: scheduler {scheduler_type!r}')
        if cfg.optimizer == 'AdamW':
            self.optimizer = optim.AdamW(self.parameters(), lr=cfg.base_lr, weight_decay=cfg.weight_decay)
        elif cfg.optimizer == 'Adam':
            self.optimizer = optim.Adam(self.parameters(), lr=cfg.base_lr, weight_decay=cfg.weight_decay)
        else:
            raise NotImplementedError(f'configure_optimizers: optimizer {cfg.optimizer!r}')
        if scheduler_type == 'step':
            self.scheduler = torch.optim.lr_scheduler.StepLR(self.optimizer, cfg.scheduler_param[0],
                                                             cfg.scheduler_param[1])
        else:
            self.scheduler = torch.optim.lr_scheduler.StepLR(self.optimizer, 50, 1.0)
        self.logger.info(f'Using optimizer {self.optimizer} with scheduler {self.scheduler}')
        return self.optimizer, self.scheduler

    def _check_trainable(self, train_encoder: bool = False):
        """forward_train covers the branches both reference configs select; anything else raises."""
        cfg = self.cfg
        if not train_encoder and any(p.requires_grad for p in self.kpf_encoder.parameters()):
            raise ValueError('forward_train: the KPConv encoder has parameters that require grad; pass '
                             'train_encoder=True to train it, or freeze it with model.kpf_encoder.requires_grad_(False)')
        if train_encoder:
            if not cfg.use_batch_norm:
                raise NotImplementedError('forward_train(train_encoder=True): no backward for use_batch_norm=False')
            for name, p in self.kpf_encoder.named_parameters():
                if name.endswith('kernel_points') and p.requires_grad:
                    raise NotImplementedError(f'forward_train(train_encoder=True): kpf_encoder.{name} requires grad, but '
                                              'the kernel disposition is fixed (no gradient through the influences)')
        unsupported = []
        if not cfg.pre_norm:
            unsupported.append('pre_norm=False')
        if not cfg.get('direct_regress_coor', False):
            unsupported.append('direct_regress_coor=False (CorrespondenceDecoder)')
        if cfg.get('pos_emb_type', 'sine') != 'sine':
            unsupported.append(f"pos_emb_type={cfg['pos_emb_type']!r}")
        if not (cfg.sa_val_has_pos_emb and cfg.ca_val_has_pos_emb):
            unsupported.append('sa/ca_val_has_pos_emb=False')
        if cfg.get('attention_impl', 'fp32') != 'fp32':
            unsupported.append(f"attention_impl={cfg['attention_impl']!r}")
        if unsupported:
            raise NotImplementedError('forward_train: no backward for ' + ', '.join(unsupported))

    def _stage_attention_train(self, feats_un, xyz_c, offs_c, B: int, plan: AttentionPlan, drop=None):
        """Differentiable stages after the encoder: feature projection, cross-encoder, correspondence heads.
        The position embedding and the pose carry no gradient (the reference loss does not use the pose).
        drop: the cross-encoder's dropout masks (ops.DropoutKey) or None."""
        cfg = self.cfg
        both_un = ops.linear(feats_un, self.feat_proj.weight, self.feat_proj.bias)             # regtr.py:145
        with torch.no_grad():
            pe = self.pos_embed(xyz_c)
        cond = self.transformer_encoder.forward_train_packed(
            both_un, pe if cfg.transformer_encoder_has_pos_emb else None, plan, drop=drop)
        corr, logit = self.correspondence_decoder.forward_packed(cond, xyz_c, pe, plan)
        with torch.no_grad():
            pose = ops.pose_from_corr(xyz_c, corr.detach().contiguous(), logit.detach()[..., 0].contiguous(), offs_c, B)
        return dict(both_un=both_un, xyz_c=xyz_c, cond=cond, corr=corr, logit=logit, pose=pose)

    def forward_train(self, batch, train_encoder: bool = False, *, dropout_key=None):
        """`forward` with autograd: same output dict, whose src/tgt_feat(_un), *_kp_warped and *_overlap carry
        history back to every parameter after the KPConv encoder.  The pyramid always runs without grad.
        train_encoder=False: the encoder runs without grad and must be frozen
        (model.kpf_encoder.requires_grad_(False)).  train_encoder=True: the encoder runs under autograd too, on the
        encoder backward kernels, and every encoder parameter that requires grad receives one (kernel_points must
        stay frozen, as in the reference); its output is bit-identical to the inference encoder's.
        Dropout (cfg.dropout > 0, training mode only): the cross-encoder applies the reference's six dropouts, with
        masks drawn from dropout_key = (seed, step, pair_base) -- pair_base the global index of the batch's first
        pair, so a pair gets the same masks in any batch, on any rank, and a resumed run repeats them.  dropout_key
        None draws a fresh seed from torch's default CPU generator on every call.  In eval mode or at dropout 0 the
        key is ignored and the step runs exactly as without it.
        Exact shapes, eager only."""
        if self.transformer_encoder.record_attentions:
            raise RuntimeError('forward_train: attention maps are recorded by the eager inference forward only; set '
                               'transformer_encoder.record_attentions = False to train')
        self._check_trainable(train_encoder)
        B = len(batch['src_xyz'])
        with torch.no_grad():
            meta = self.preprocessor(list(batch['src_xyz']) + list(batch['tgt_xyz']), lazy_upsamples=True)
            batch['kpconv_meta'] = meta
        pts = meta['_points']
        with contextlib.nullcontext() if train_encoder else torch.no_grad():
            feats_un, _ = self.kpf_encoder(torch.ones_like(pts[0][:, 0:1]), meta)             # regtr.py:122-136
        lens_c = meta['_lens'][-1]
        plan = AttentionPlan(lens_c, pts[-1].device)
        drop = None
        p = self.transformer_encoder.dropout_p
        if self.training and p > 0.0:
            if dropout_key is None:
                dropout_key = (int(torch.randint(0, 2 ** 62, (1,)).item()), 0, 0)
            seed, step, pair_base = dropout_key
            drop = ops.DropoutKey(p, seed, step, pair_base, B, offs=meta['_offs'][-1], max_len=plan.max_len)
        core = self._stage_attention_train(feats_un, pts[-1], meta['_offs'][-1], B, plan, drop)
        return self._assemble(core, lens_c, B)

    @torch.no_grad()
    def forward(self, batch):
        """Eager path: exact shapes, one host sync (pyramid sizes) before the encoder.  An inference executor: dropout
        never applies (a training-mode model with dropout > 0 logs one warning; see forward_train)."""
        warn_dropout_eval_only(self)
        B = len(batch['src_xyz'])
        meta = self.preprocessor(list(batch['src_xyz']) + list(batch['tgt_xyz']), lazy_upsamples=True)   # regtr.py:117-118
        batch['kpconv_meta'] = meta
        lens_c = meta['_lens'][-1]
        plan = AttentionPlan(lens_c, meta['_points'][-1].device)
        return self._assemble(self._core(meta, B, plan), lens_c, B)


class GraphedRegTR:
    """CUDA-graph executor of `RegTR.forward` for latency-bound serving (batch 1..B pairs).

    The eager forward is launch-bound: a few hundred kernels of a few microseconds each (SURVEY.md H6).
    Here the whole forward -- pyramid, encoder, cross-encoder, regressor, Kabsch -- is captured
    ONCE per (pairs, level-0 capacity bucket) into a CUDA graph over capacity-shaped buffers;
    data-dependent level sizes stay on the device (int32 offsets read by every kernel), so a
    replay needs no host round trip.  Per call: one H2D/D2D copy per cloud into the packed buffer, one
    graph launch, ONE small D2H (level sizes + status + pose) and a single synchronisation.

    Outputs are views into the graph's static buffers: valid until the next call with the same
    bucket; the per-cloud views (and `batch['kpconv_meta']`) are built lazily on first access, `pose`
    and `host_pose` (pinned host copy, not part of the reference contract) are always there.  If a
    level overflows its static capacity (REGTR_STATUS_CAPACITY) the call falls back to the eager
    forward, so results are never silently truncated.

    `stages=True` captures the four `_TIMEIT` stages of the reference (regtr.py:108-216) as four graphs
    replayed back to back with CUDA events in between: `stage_ms()` then reports where a pair's
    latency goes (bench.py).  Every captured graph owns a private scratch namespace (ops.new_namespace):
    no graph ever shares or outlives a buffer another graph writes.

    Training with validation in between: after the library optimizer's step() (regtr_b200.optim.AdamW / Adam) the
    captured graphs stay valid -- the step rewrites the split weights they read in place.  After a torch optimizer's
    step the cached splits are dropped and rebuilt elsewhere, so call `invalidate()` before the next call.
    """

    STAGES = ('preprocess', 'encoder', 'attention_decoder', 'pose')

    def __init__(self, model: RegTR, bucket: int = 8192, full_meta: bool = True, ratio: float = 0.30,
                 retry_ratio: float = 0.45, stages: bool = False):
        self.model = model
        self.bucket = int(bucket)
        self.full_meta = full_meta
        self.ratio, self.retry_ratio = ratio, retry_ratio   # level-to-level capacity ratio (real data: 0.19-0.27)
        self.stages = stages
        self.ratios = {}
        self.sparse = set()             # buckets whose clouds overflowed the dense voxel grid: captured sort-based
        self.graphs = {}
        self.fallbacks = 0
        self.wait_s = 0.0               # host time spent blocked in result() waiting for the GPU (diagnostics)
        # the graphs bake in pointers to the split (hi, lo) weights: load_state_dict bumps the model's epoch and
        # every graph is re-captured on its next use; regtr_b200.optim's step() rewrites the splits in place (the
        # graphs stay valid); any other in-place edit of a parameter (a torch optimizer's step) needs invalidate()
        self._epoch = getattr(model, '_weights_epoch', 0)
        if not hasattr(model, '_weights_epoch'):
            model._weights_epoch = 0
            model.register_load_state_dict_post_hook(GraphedRegTR._bump_epoch)
        weakref.finalize(self, GraphedRegTR._release_all, self.graphs)

    @staticmethod
    def _bump_epoch(module, incompatible_keys):
        module._weights_epoch = getattr(module, '_weights_epoch', 0) + 1

    def invalidate(self):
        """Drop every captured graph (weights were modified in place)."""
        for key in list(self.graphs):
            self._drop(key)

    @staticmethod
    def _release_all(graphs):
        for st in graphs.values():
            ops.release_namespace(st['ns'])
        graphs.clear()

    def _drop(self, key):
        st = self.graphs.pop(key, None)
        if st is not None:
            torch.cuda.synchronize(self.model.device)        # no replay of this graph is in flight any more
            ops.release_namespace(st['ns'])

    def _capture(self, B: int, cap0: int):
        ns = ops.new_namespace()                 # private scratch for THIS graph (never freed while it lives)
        with ops.scratch_namespace(ns):
            st = self._capture_impl(B, cap0)
        st['ns'] = ns
        return st

    def _capture_impl(self, B: int, cap0: int):
        from .kpconv import level_capacities
        model = self.model
        dev = model.device
        caps = level_capacities(model.cfg, cap0, ratio=self.ratios.get((B, cap0), self.ratio))
        st = dict(points=torch.zeros((cap0, 3), dtype=torch.float32, device=dev),
                  offs0=torch.zeros(2 * B + 1, dtype=torch.int32, device=dev), caps=caps)
        box = {}

        def s_pre():
            box['pyr'] = model.preprocessor.build(st['points'], st['offs0'], 2 * B, caps=caps,
                                                  want64=self.full_meta, upsamples=False,
                                                  dense=(B, cap0) not in self.sparse)
            box['plan'] = AttentionPlan.from_device(box['pyr'].offs_all[-1], B, caps[-1])
            box['meta'] = box['pyr'].private(static=True)

        def s_enc():
            box['enc'] = model._stage_encoder(box['meta'])

        def s_att():
            box['att'] = model._stage_attention(box['enc'], box['plan'])

        def s_pose():
            pyr = box['pyr']
            box['pose'] = model._stage_pose(box['enc'], box['att'], box['meta']['_offs'][-1], B)
            # everything the host needs, in ONE buffer / one D2H: level offsets | status | pose bits
            box['tail'] = torch.cat([pyr.offs_all.reshape(-1), pyr.status.view(torch.int32),
                                     box['pose'].reshape(-1).view(torch.int32)])

        fns = [s_pre, s_enc, s_att, s_pose]

        def run():
            for f in fns:
                f()

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):           # warm-up (sizes the scratch buffers, caches) before capture
            n = cap0 // (2 * B)                 # a plausible offset table so that the warm-up exercises every kernel
            st['offs0'].copy_(torch.arange(0, 2 * B + 1, dtype=torch.int32, device=dev) * n)
            st['points'].uniform_(-1.0, 1.0)
            for _ in range(2):
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        n0 = ops.LAUNCHES
        graphs = []
        if self.stages:
            pool = None
            for f in fns:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, pool=pool):
                    f()
                pool = pool or g.pool()
                graphs.append(g)
        else:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                run()
            graphs.append(g)
        pyr, tail = box['pyr'], box['tail']
        core = dict(both_un=box['enc']['both_un'], xyz_c=box['enc']['xyz_c'], cond=box['att']['cond'],
                    corr=box['att']['corr'], logit=box['att']['logit'], pose=box['pose'])
        n_tail = tail.numel()
        tail_host = torch.empty(n_tail, dtype=torch.int32).pin_memory()
        n_meta = pyr.offs_all.numel() + 1
        st.update(graphs=graphs, pyr=pyr, core=core, tail=tail, tail_host=tail_host,
                  n_launches=ops.LAUNCHES - n0,           # hand-written kernels per replay (launch accounting)
                  tail_np=tail_host.numpy(), n_meta=n_meta,
                  host_pose=tail_host[n_meta:].view(torch.float32).view(tuple(core['pose'].shape)),
                  offs_host=torch.empty(2 * B + 1, dtype=torch.int32).pin_memory(),
                  done=torch.cuda.Event(),
                  stage_ev=[torch.cuda.Event(enable_timing=True) for _ in range(len(fns) + 1)]
                  if self.stages else None)
        st['offs_np'] = st['offs_host'].numpy()
        return st

    @torch.no_grad()
    def submit(self, batch):
        """Enqueue one forward on the current stream (no host synchronisation): copy the clouds into the
        static buffers, replay the graph, start the D2H of (level sizes, status, pose).  Returns a ticket
        for `result`."""
        if self.model.transformer_encoder.record_attentions:
            raise RuntimeError('GraphedRegTR: attention maps are recorded by the eager RegTR.forward only (the captured '
                               'graphs never record them); set transformer_encoder.record_attentions = False')
        src, tgt = batch['src_xyz'], batch['tgt_xyz']
        B = len(src)
        clouds = list(src) + list(tgt)
        lens0 = [c.shape[0] for c in clouds]
        n0 = sum(lens0)
        cap0 = max(self.bucket, (n0 + self.bucket - 1) // self.bucket * self.bucket)
        key = (B, cap0)
        if self._epoch != self.model._weights_epoch:          # weights were reloaded since the graphs were captured
            self.invalidate()
            self._epoch = self.model._weights_epoch
        st = self.graphs.get(key)
        if st is None:
            st = self.graphs[key] = self._capture(B, cap0)
        offs = st['offs_np']
        a = 0
        pts = st['points']
        for i, c in enumerate(clouds):          # H2D (pinned sources: asynchronous, no staging pass) or D2D
            offs[i] = a
            pts[a:a + lens0[i]].copy_(c, non_blocking=True)
            a += lens0[i]
        offs[2 * B] = a
        st['offs0'].copy_(st['offs_host'], non_blocking=True)
        if st['stage_ev'] is None:
            st['graphs'][0].replay()
        else:
            ev = st['stage_ev']
            ev[0].record()
            for g, e in zip(st['graphs'], ev[1:]):
                g.replay()
                e.record()
        ops.LAUNCHES += st['n_launches']
        st['tail_host'].copy_(st['tail'], non_blocking=True)
        st['done'].record()
        return (key, st, batch, B)

    def stage_ms(self, key=None):
        """{stage: milliseconds} of the LAST finished replay (stages=True executors only)."""
        st = self.graphs[key] if key is not None else next(iter(self.graphs.values()))
        ev = st['stage_ev']
        return {nm: ev[i].elapsed_time(ev[i + 1]) for i, nm in enumerate(self.STAGES)}

    @torch.no_grad()
    def result(self, ticket):
        """Wait for a submitted forward and return the reference's output dict (views into the graph's
        static buffers: valid until the next submit on the same capacity bucket)."""
        key, st, batch, B = ticket
        model = self.model
        t0 = time.perf_counter()
        st['done'].synchronize()
        self.wait_s += time.perf_counter() - t0
        pyr = st['pyr']
        n_lvl = len(pyr.levels)
        n_meta = st['n_meta']
        code = int(st['tail_np'][n_meta - 1])
        if code & 6:                            # a level overflowed its capacity (2) or the dense voxel grid (4):
            self.fallbacks += 1                 # redo eagerly and re-capture this bucket differently next time
            if code & 4 and key not in self.sparse:
                self.sparse.add(key)
                self._drop(key)
            elif code & 2 and self.ratios.get(key, self.ratio) < self.retry_ratio:
                self.ratios[key] = self.retry_ratio
                self._drop(key)
            dev = model.device                  # the eager forward has no host path: move host clouds first
            eager = {k: [c.to(dev, non_blocking=True) for c in batch[k]] for k in ('src_xyz', 'tgt_xyz')}
            out = model.forward(eager)
            batch['kpconv_meta'] = eager['kpconv_meta']
            out['host_pose'] = out['pose'].cpu()
            return out
        offs_np = st['tail_np'][:n_meta - 1].copy()          # this call's level sizes (the pinned buffer is reused)

        def make_meta():
            return model.preprocessor.finalize(pyr, host=(torch.from_numpy(offs_np).reshape(n_lvl, 2 * B + 1), code))

        meta = LazyDict(make_meta)
        batch['kpconv_meta'] = meta

        def make_out():
            return model._assemble(st['core'], meta['_lens'][-1], B)

        return LazyDict(make_out, pose=st['core']['pose'], host_pose=st['host_pose'])

    def __call__(self, batch):
        return self.result(self.submit(batch))


class PipelinedRegTR:
    """`depth` CUDA-graph executors on private streams, used round-robin: while the GPU finishes pair i,
    pairs i+1 .. i+depth-1 are already enqueued, so the many small latency-bound kernels of one forward
    overlap with another pair's (independent pairs; SURVEY.md 8e).  `submit` returns immediately;
    `result` of the oldest ticket is taken when its slot is needed again or on `drain`."""

    def __init__(self, model: RegTR, depth: int = 2, **kw):
        self.slots = [GraphedRegTR(model, **kw) for _ in range(depth)]
        self.streams = [torch.cuda.Stream(device=model.device) for _ in range(depth)]
        self.pending = [None] * depth
        self.i = 0

    def submit(self, batch, pre_hook=None):
        """Returns the finished output of the forward that previously used this slot (or None).
        `pre_hook()` (e.g. a benchmark's L2 flush) runs on the slot's stream right before the forward."""
        k = self.i % len(self.slots)
        self.i += 1
        done = None
        if self.pending[k] is not None:
            done = self.slots[k].result(self.pending[k])
        self.streams[k].wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.streams[k]):
            if pre_hook is not None:
                pre_hook()
            self.pending[k] = self.slots[k].submit(batch)
        return done

    def warm(self, batches):
        """Capture every (slot, capacity bucket) graph needed by `batches` ahead of time."""
        for k, slot in enumerate(self.slots):
            with torch.cuda.stream(self.streams[k]):
                for b in batches:
                    slot(dict(b))
        torch.cuda.synchronize()

    def join(self):
        """Make the current stream wait for every slot stream (for event timing on the current stream)."""
        for st in self.streams:
            torch.cuda.current_stream().wait_stream(st)

    def drain(self):
        outs = []
        n = len(self.slots)
        for j in range(n):
            k = (self.i + j) % n
            if self.pending[k] is not None:
                outs.append(self.slots[k].result(self.pending[k]))
                self.pending[k] = None
        return outs
