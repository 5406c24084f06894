"""Recording of the model's stages on its own activations, and the oracle's restatement of one stage, shared by the
stage-by-stage tests of the training backward (tests/test_gpu_grad_stages.py) and of the inference forward
(tests/test_gpu_forward_stages.py).

`record` wraps every KPConv-encoder block and every cross-encoder layer of a model (and, for an inference forward,
the final norm, the position embedding and the correspondence head) and the ops they call: per stage it keeps the
input, the other arguments, the output and every recorded op call with its arguments and result.  The op results
carry the GPU's branch decisions (LeakyReLU / ReLU masks, max-pool winners, KPConv neighbour counts), which
`gpu_decisions` turns into the oracle's terms so that `oracle_block` / `oracle_layer` can evaluate the same stage in
float64 and fp32 with the GPU's decisions.
"""
import inspect
import os
import sys

import numpy as np
import pytest
import torch

from conftest import FORWARD_CASES, REAL_CASES, make_case, make_real_case

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402

DEV = 'cuda:0'
ENC = 'kpf_encoder.encoder_blocks.'
XENC = 'transformer_encoder.layers.'
RECORDED_OPS = ('instnorm_act', 'instnorm_apply', 'max_pool', 'kpconv', 'linear_instats', 'linear', 'mha_varlen_lse')
INFERENCE_OPS = RECORDED_OPS + ('layernorm_pos', 'mha_varlen', 'mha_tf32_tc', 'corr_decode', 'pos_embed_sine',
                                'pose_from_corr')


class Tap(torch.autograd.Function):
    """Identity that keeps a copy of the gradient flowing back through it in box[key]."""

    @staticmethod
    def forward(ctx, x, box, key):
        ctx.box, ctx.key = box, key
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        ctx.box[ctx.key] = g.clone()
        return g, None, None


def record(model, mp, inference=False):
    """Wrap every encoder block's forward, every cross-encoder layer's forward_train_packed (inference: its
    forward_packed, which runs forward_post_packed for a post-norm layer) and the ops they call.
    Per block / layer: 'x' (input), 'rest' (the other arguments), 'calls' [(op, arguments, result)], 'y' (output),
    and after a backward 'dout' (gradient at the output) and 'dx' (gradient the block sends to its input, if it needs
    one).  Every attention-core backward is kept in rec['mha_bwd'], keyed by the address of the O it was given: its
    dO and copies of the dq, dk, dv it wrote.
    inference=True: the ops of INFERENCE_OPS are recorded, and so are rec['final'] (the cross-encoder's final norm,
    one box per call), rec['pe'] (the position embedding), rec['head'] (the correspondence head's forward_packed) and
    rec['top'] (the op calls outside every box: the feature projection and the pose)."""
    from regtr_b200 import ops
    rec = dict(enc=[], xenc=[], final=[], pe={}, head={}, top=[], mha_bwd={})
    rec['cur'] = rec['top'] if inference else None

    def recording(name, fn):
        sig = inspect.signature(fn)

        def wrapped(*a, **k):
            r = fn(*a, **k)
            if rec['cur'] is not None:
                bound = sig.bind(*a, **k)
                bound.apply_defaults()
                rec['cur'].append((name, dict(bound.arguments), r))
            return r
        return wrapped

    for name in (INFERENCE_OPS if inference else RECORDED_OPS):
        mp.setattr(ops, name, recording(name, getattr(ops, name)))
    mha_bwd = ops.mha_varlen_bwd
    bwd_sig = inspect.signature(mha_bwd)

    def recording_bwd(*a, **k):
        mha_bwd(*a, **k)
        b = bwd_sig.bind(*a, **k).arguments
        rec['mha_bwd'][b['o'].data_ptr()] = dict(d_o=b['d_o'], **{t: b[t].clone() for t in ('dq', 'dk', 'dv')})
    mp.setattr(ops, 'mha_varlen_bwd', recording_bwd)

    def tap(mod, method, box):
        fn = getattr(mod, method)

        def wrapped(x, *rest):
            box.update(x=x.detach(), rest=rest, calls=[])
            outer, rec['cur'] = rec['cur'], box['calls']
            y = fn(Tap.apply(x, box, 'dx') if x.requires_grad else x, *rest)
            rec['cur'] = outer
            box['y'] = y.detach() if torch.is_tensor(y) else tuple(t.detach() for t in y)
            return Tap.apply(y, box, 'dout') if torch.is_tensor(y) and y.requires_grad else y
        mp.setattr(mod, method, wrapped)

    for blk in model.kpf_encoder.encoder_blocks:
        rec['enc'].append({})
        tap(blk, 'forward', rec['enc'][-1])
    for layer in model.transformer_encoder.layers:
        rec['xenc'].append({})
        tap(layer, 'forward_packed' if inference else 'forward_train_packed', rec['xenc'][-1])
    if inference:
        final = model.transformer_encoder._final

        def recording_final(x, n_dev=None):
            rec['final'].append({})
            box = rec['final'][-1]
            box.update(x=x.detach(), calls=[])
            outer, rec['cur'] = rec['cur'], box['calls']
            y = final(x, n_dev)
            rec['cur'] = outer
            box['y'] = y.detach()
            return y
        mp.setattr(model.transformer_encoder, '_final', recording_final)
        tap(model.pos_embed, 'forward', rec['pe'])
        tap(model.correspondence_decoder, 'forward_packed', rec['head'])
    return rec


def pairs(case):
    from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair
    return [(make_modelnet_pair if kind == 'modelnet' else make_3dmatch_pair)(*args)
            for kind, args in FORWARD_CASES[case][2]]


def meta_cpu(meta):
    return {k: [torch.as_tensor(v).cpu() for v in meta[k]] for k in ('points', 'neighbors', 'pools', 'stack_lengths')}


_TRAIN_RUNS = {}


def train_run(case):
    """The recorded training step of a case (computed once per session)."""
    if case in _TRAIN_RUNS:
        return _TRAIN_RUNS[case]
    from regtr_b200.regtr import RegTR
    cfg, sd0, src, tgt = make_case(case)
    sd = ei.loss_state_dict(sd0)
    model = RegTR(cfg).to(DEV)
    model.load_state_dict(sd, strict=True)
    li = ei.loss_inputs(pairs(case), [len(s) for s in src], [len(t) for t in tgt])
    batch = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt],
             'pose': li['pose'].to(DEV), 'src_overlap': [m.to(DEV) for m in li['src_overlap']],
             'tgt_overlap': [m.to(DEV) for m in li['tgt_overlap']]}
    with pytest.MonkeyPatch.context() as mp:
        rec = record(model, mp)
        model.compute_loss(model.forward_train(batch, train_encoder=True), batch)['total'].backward()
    meta = batch['kpconv_meta']
    run = dict(cfg=cfg, sd=sd, model=model, rec=rec, meta=meta, src=src, tgt=tgt, li=li,
               grads={n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None},
               meta_cpu=meta_cpu(meta))
    _TRAIN_RUNS[case] = run
    return run


_INFERENCE_RUNS = {}


def inference_run(case):
    """The recorded eager inference forward of a case -- a synthetic or variant fixture, or a real-data one --
    (computed once per session)."""
    if case in _INFERENCE_RUNS:
        return _INFERENCE_RUNS[case]
    from regtr_b200.regtr import RegTR
    cfg, sd, src, tgt = make_real_case(case) if case in REAL_CASES else make_case(case)
    src, tgt = ([src], [tgt]) if case in REAL_CASES else (src, tgt)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    batch = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    with pytest.MonkeyPatch.context() as mp:
        rec = record(model, mp, inference=True)
        out = model(batch)
    torch.cuda.synchronize()
    meta = batch['kpconv_meta']
    run = dict(cfg=cfg, sd=sd, model=model, rec=rec, meta=meta, src=src, tgt=tgt, out=out, meta_cpu=meta_cpu(meta))
    _INFERENCE_RUNS[case] = run
    return run


def trainable(model, prefix):
    return [(n, p) for n, p in model.named_parameters() if n.startswith(prefix) and p.requires_grad]


def leaves(sd, names, dtype):
    return {n: sd[n].detach().clone().to(dtype).requires_grad_(True) for n in names}


# ----------------------------------------------------------------------------------------------- decisions

def block_sites(cfg, i):
    from regtr_b200.config import pyramid_plan
    b = pyramid_plan(cfg)[1][i]
    if b['kind'] == 'simple':
        return b, ['out']
    return b, (['unary1'] if b['in_dim'] != b['out_dim'] // 4 else []) + ['conv', 'out']


def gpu_decisions(cfg, i, calls):
    """The branch decisions the GPU took in encoder block i, in oracle.regtr_oracle.encoder_block's terms."""
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    b, sites = block_sites(cfg, i)
    acts = [r for name, a, r in calls if name in ('instnorm_act', 'instnorm_apply') and a['slope'] >= 0]
    assert len(acts) == len(sites), (i, len(acts), sites)
    d = {site: ((r[0] if isinstance(r, tuple) else r).detach() > 0).cpu() for site, r in zip(sites, acts)}
    (_, a, _), = [c for c in calls if c[0] == 'kpconv']
    x, flags = a['x'].detach(), a['row_flags']
    if flags is None:           # counted by the aggregation itself: from x's row sums (Cin > 1) or from x (Cin = 1)
        flags = ops._kpconv_wf(a['q_pts'], a['s_pts'], a['idx32'], x, a['kernel_points'], a['extent'], None)[1] \
            if x.shape[1] > 1 else x[:, 0] > 0
    flags = torch.cat([flags[:x.shape[0]].bool().cpu(), torch.zeros(1, dtype=torch.bool)])
    d['kpconv'] = flags[a['idx32'].long().cpu()].sum(-1).clamp(min=1)
    pools = [c for c in calls if c[0] == 'max_pool']
    assert len(pools) == (b['strided'] and b['kind'] != 'simple')
    for _, a, r in pools:
        xs, idx = a['x'].detach().cpu(), a['idx32'].long().cpu()
        d['pool'] = O.max_pool_winner(xs, idx)
        assert torch.equal(O.max_pool(xs, idx, d['pool']), r.detach().cpu())      # the slots the GPU's output took
    return d


def flips(gpu, free, pool_idx=None):
    """Number of decisions the unforced float64 forward takes differently, per site (a max-pool decision is the
    winning support row; all shadow slots are one row)."""
    out = []
    for k, v in gpu.items():
        w = free[k]
        if k == 'pool':
            v, w = pool_idx.gather(1, v), pool_idx.gather(1, w)
        out.append(f'{k} {int((v != w).sum())}/{v.numel()}')
    return ', '.join(out)


# ------------------------------------------------------------------------------------- oracle stages

def oracle_block(run, i, x, need_dx, dout, dtype, decisions, names):
    """float64 / fp32 autograd of oracle.regtr_oracle.encoder_block i on x with the GPU's decisions; dout None: the
    block's output instead of its gradients."""
    from oracle import regtr_oracle as O
    sd = run['sd']
    lv = leaves(sd, names, dtype)
    sdd = {k: lv.get(k, v) for k, v in sd.items() if k.startswith(f'{ENC}{i}.')}
    xin = x.detach().cpu().to(dtype).requires_grad_(need_dx)
    d = dict(decisions)
    y = O.encoder_block(sdd, run['cfg'], i, xin, run['meta_cpu'], dtype, d)
    assert d.keys() == decisions.keys()                  # every branch of the block was forced
    if dout is None:
        return y.detach()
    ins = ([xin] if xin.requires_grad else []) + [lv[n] for n in names]
    return torch.autograd.grad(y, ins, dout.cpu().to(dtype))


def oracle_layer(run, i, x, pos, dout, dtype, masks, names):
    """float64 / fp32 autograd of oracle.cross_encoder_layer over the pairs of the packed tokens x; masks: the
    feed-forward ReLU masks per packed row, or None for the unforced forward (-> its masks, no gradients); dout
    None: the layer's packed output instead of its gradients."""
    from oracle import regtr_oracle as O
    lens = [int(v) for v in run['meta']['_lens'][-1]]
    st = np.concatenate([[0], np.cumsum(lens)])
    B = len(lens) // 2
    lv = leaves(run['sd'], names, dtype)
    xin = x.cpu().to(dtype).requires_grad_(True)
    pe = pos.cpu().to(dtype) if pos is not None else torch.zeros_like(xin)
    outs, gouts, free = [], [], []
    for b in range(B):
        rs, rt = slice(st[b], st[b + 1]), slice(st[B + b], st[B + b + 1])
        d = {} if masks is None else {'ffn_src': masks[rs], 'ffn_tgt': masks[rt]}
        so, to = O.cross_encoder_layer(lv if names else run['sd'], run['cfg'], i, xin[rs], xin[rt], pe[rs], pe[rt], d)
        assert len(d) == 2
        outs += [so, to]
        if dout is not None:
            gouts += [dout[rs].cpu().to(dtype), dout[rt].cpu().to(dtype)]
        free.append(d)
    if masks is None:                                     # packed order: the B sources, then the B targets
        return torch.cat([d['ffn_src'] for d in free] + [d['ffn_tgt'] for d in free])
    if dout is None:
        return torch.cat(outs[0::2] + outs[1::2]).detach()
    return torch.autograd.grad(outs, [xin] + [lv[n] for n in names], gouts)
