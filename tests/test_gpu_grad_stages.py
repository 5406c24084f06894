"""GPU tests of the training backward stage by stage, on the model's own activations.

One forward_train(train_encoder=True) -> compute_loss -> backward() per case records, for every KPConv-encoder block
and every cross-encoder layer, its input, the gradient that reaches its output and its input, and the outputs of the
ops it calls (which carry the GPU's branch decisions: LeakyReLU / ReLU masks, max-pool winners, KPConv neighbour
counts).  Then:
  * each block / layer is re-run alone on its recorded input and upstream gradient: dx and every parameter gradient
    must be bit-identical to the full backward's (no state leaks between blocks: CSR caches, workspaces, gradient
    accumulation);
  * the same gradients are compared with float64 autograd of the oracle's block / layer, run with the GPU's
    decisions, under the fp32 yardstick (tests/grad_yardstick.py), and the decisions that the unforced float64
    forward takes differently are counted;
  * the float64 oracle's d(feats_un) is fed to the GPU encoder alone, and every encoder parameter gradient is compared
    with the float64 oracle encoder's under the same yardstick;
  * each attention core's recorded q, k, v, O, lse and output gradient are run through the core's backward alone and
    checked as tests/test_gpu_attention_backward.py checks synthetic inputs (tests/attention_oracle.py).
"""
import inspect
import os
import sys
import types

import numpy as np
import pytest
import torch

import attention_oracle as ao
from conftest import FORWARD_CASES, make_case
from grad_yardstick import Yardstick, errors

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
CASES = ['fwd_3dmatch_small_b2', 'fwd_modelnet_b1']
ENC = 'kpf_encoder.encoder_blocks.'
XENC = 'transformer_encoder.layers.'
_RECORDED_OPS = ('instnorm_act', 'instnorm_apply', 'max_pool', 'kpconv', 'linear_instats', 'linear', 'mha_varlen_lse')


class _Tap(torch.autograd.Function):
    """Identity that keeps a copy of the gradient flowing back through it in box[key]."""

    @staticmethod
    def forward(ctx, x, box, key):
        ctx.box, ctx.key = box, key
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        ctx.box[ctx.key] = g.clone()
        return g, None, None


def _record(model, mp):
    """Wrap every encoder block's forward, every cross-encoder layer's forward_train_packed and the ops they call.
    Per block / layer: 'x' (input), 'rest' (the other arguments), 'calls' [(op, arguments, result)], and after the
    backward 'dout' (gradient at the output) and 'dx' (gradient the block sends to its input, if it needs one).
    Every attention-core backward is kept in rec['mha_bwd'], keyed by the address of the O it was given: its dO and
    copies of the dq, dk, dv it wrote."""
    from regtr_b200 import ops
    rec = dict(enc=[], xenc=[], cur=None, mha_bwd={})

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

    for name in _RECORDED_OPS:
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
            rec['cur'] = box['calls']
            y = fn(_Tap.apply(x, box, 'dx') if x.requires_grad else x, *rest)
            rec['cur'] = None
            box['y'] = y.detach()
            return _Tap.apply(y, box, 'dout')
        mp.setattr(mod, method, wrapped)

    for blk in model.kpf_encoder.encoder_blocks:
        rec['enc'].append({})
        tap(blk, 'forward', rec['enc'][-1])
    for layer in model.transformer_encoder.layers:
        rec['xenc'].append({})
        tap(layer, 'forward_train_packed', rec['xenc'][-1])
    return rec


def _pairs(case):
    from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair
    return [(make_modelnet_pair if kind == 'modelnet' else make_3dmatch_pair)(*args)
            for kind, args in FORWARD_CASES[case][2]]


_RUNS = {}


def _full_run(case):
    """The recorded training step of a case (computed once per session)."""
    if case in _RUNS:
        return _RUNS[case]
    from regtr_b200.regtr import RegTR
    cfg, sd0, src, tgt = make_case(case)
    sd = ei.loss_state_dict(sd0)
    model = RegTR(cfg).to(DEV)
    model.load_state_dict(sd, strict=True)
    li = ei.loss_inputs(_pairs(case), [len(s) for s in src], [len(t) for t in tgt])
    batch = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt],
             'pose': li['pose'].to(DEV), 'src_overlap': [m.to(DEV) for m in li['src_overlap']],
             'tgt_overlap': [m.to(DEV) for m in li['tgt_overlap']]}
    with pytest.MonkeyPatch.context() as mp:
        rec = _record(model, mp)
        model.compute_loss(model.forward_train(batch, train_encoder=True), batch)['total'].backward()
    meta = batch['kpconv_meta']
    run = dict(cfg=cfg, sd=sd, model=model, rec=rec, meta=meta, src=src, tgt=tgt, li=li,
               grads={n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None},
               meta_cpu={k: [torch.as_tensor(v).cpu() for v in meta[k]]
                         for k in ('points', 'neighbors', 'pools', 'stack_lengths')})
    _RUNS[case] = run
    return run


def _trainable(model, prefix):
    return [(n, p) for n, p in model.named_parameters() if n.startswith(prefix) and p.requires_grad]


def _leaves(sd, names, dtype):
    return {n: sd[n].detach().clone().to(dtype).requires_grad_(True) for n in names}


# ----------------------------------------------------------------------------------------------- decisions

def _block_sites(cfg, i):
    from regtr_b200.config import pyramid_plan
    b = pyramid_plan(cfg)[1][i]
    if b['kind'] == 'simple':
        return b, ['out']
    return b, (['unary1'] if b['in_dim'] != b['out_dim'] // 4 else []) + ['conv', 'out']


def _gpu_decisions(cfg, i, calls):
    """The branch decisions the GPU took in encoder block i, in oracle.regtr_oracle.encoder_block's terms."""
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    b, sites = _block_sites(cfg, i)
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


def _flips(gpu, free, pool_idx=None):
    """Number of decisions the unforced float64 forward takes differently, per site (a max-pool decision is the
    winning support row; all shadow slots are one row)."""
    out = []
    for k, v in gpu.items():
        w = free[k]
        if k == 'pool':
            v, w = pool_idx.gather(1, v), pool_idx.gather(1, w)
        out.append(f'{k} {int((v != w).sum())}/{v.numel()}')
    return ', '.join(out)


# ------------------------------------------------------------------------------------- block-local encoder

def _oracle_block(run, i, x, need_dx, dout, dtype, decisions, names):
    from oracle import regtr_oracle as O
    sd = run['sd']
    leaves = _leaves(sd, names, dtype)
    sdd = {k: leaves.get(k, v) for k, v in sd.items() if k.startswith(f'{ENC}{i}.')}
    xin = x.detach().cpu().to(dtype).requires_grad_(need_dx)
    d = dict(decisions)
    y = O.encoder_block(sdd, run['cfg'], i, xin, run['meta_cpu'], dtype, d)
    assert d.keys() == decisions.keys()                  # every branch of the block was forced
    ins = ([xin] if xin.requires_grad else []) + [leaves[n] for n in names]
    return torch.autograd.grad(y, ins, dout.cpu().to(dtype))


@pytest.mark.parametrize('case', CASES)
def test_encoder_blocks_backward_block_local(case):
    from oracle import regtr_oracle as O
    run = _full_run(case)
    cfg, model, meta = run['cfg'], run['model'], run['meta']
    ys = Yardstick(f'{case}: encoder blocks, block-local backward (GPU decisions)')
    not_identical, flips = [], []
    for i, (blk, r) in enumerate(zip(model.kpf_encoder.encoder_blocks, run['rec']['enc'])):
        named = _trainable(model, f'{ENC}{i}.')
        names = [n for n, _ in named]
        x = r['x'].clone().requires_grad_('dx' in r)
        out = blk(x, meta)
        ins = ([x] if x.requires_grad else []) + [p for _, p in named]
        rerun = torch.autograd.grad(out, ins, r['dout'])
        full = ([r['dx']] if x.requires_grad else []) + [run['grads'][n] for n in names]
        labels = (['dx'] if x.requires_grad else []) + [n[len(f'{ENC}{i}.'):] for n in names]
        not_identical += [f'{i}.{lab}' for lab, a, b in zip(labels, rerun, full) if not torch.equal(a, b)]
        dec = _gpu_decisions(cfg, i, r['calls'])
        g64 = _oracle_block(run, i, r['x'], 'dx' in r, r['dout'], torch.float64, dec, names)
        g32 = _oracle_block(run, i, r['x'], 'dx' in r, r['dout'], torch.float32, dec, names)
        for lab, g, a, b in zip(labels, full, g32, g64):
            ys.add(f'{i}.{lab}', g, a, b)
        free = {}
        with torch.no_grad():
            O.encoder_block(run['sd'], cfg, i, r['x'].cpu().double(), run['meta_cpu'], torch.float64, free)
        b, _ = _block_sites(cfg, i)
        pool_idx = run['meta_cpu']['pools'][b['level']].long() if 'pool' in dec else None
        flips.append(f'  block {i}: {_flips(dec, free, pool_idx)}')
    ys.report()
    print('  decisions of the unforced float64 forward that differ from the GPU\'s:\n' + '\n'.join(flips))
    assert not not_identical, f'block-local rerun not bit-identical to the full backward: {not_identical}'
    assert not ys.failures(), ys.failures()


# -------------------------------------------------------------------------------- layer-local cross-encoder

def _oracle_layer(run, i, x, pos, dout, dtype, masks, names):
    """float64 / fp32 autograd of oracle.cross_encoder_layer over the pairs of the packed tokens x; masks: the
    feed-forward ReLU masks per packed row, or None for the unforced forward (-> its masks, no gradients)."""
    from oracle import regtr_oracle as O
    lens = [int(v) for v in run['meta']['_lens'][-1]]
    st = np.concatenate([[0], np.cumsum(lens)])
    B = len(lens) // 2
    leaves = _leaves(run['sd'], names, dtype)
    xin = x.cpu().to(dtype).requires_grad_(True)
    pe = pos.cpu().to(dtype) if pos is not None else torch.zeros_like(xin)
    outs, gouts, free = [], [], []
    for b in range(B):
        rs, rt = slice(st[b], st[b + 1]), slice(st[B + b], st[B + b + 1])
        d = {} if masks is None else {'ffn_src': masks[rs], 'ffn_tgt': masks[rt]}
        so, to = O.cross_encoder_layer(leaves, run['cfg'], i, xin[rs], xin[rt], pe[rs], pe[rt], d)
        assert len(d) == 2
        outs += [so, to]
        gouts += [dout[rs].cpu().to(dtype), dout[rt].cpu().to(dtype)]
        free.append(d)
    if masks is None:                                     # packed order: the B sources, then the B targets
        return torch.cat([d['ffn_src'] for d in free] + [d['ffn_tgt'] for d in free])
    return torch.autograd.grad(outs, [xin] + [leaves[n] for n in names], gouts)


def _add_in_proj_rows(ys, label, g, a, b):
    """The q, k and v row blocks of an in-projection gradient, one yardstick row each: the k / v blocks are much
    larger than the q block, so a whole-tensor row would hide an error in dQ.  The k block of the bias gradient is
    sum_j dK_j, zero in exact arithmetic (softmax ignores a vector added to every key): it is measured against the
    larger of the q and v blocks instead of itself."""
    E = g.shape[0] // 3
    for part, blk in zip('qkv', (slice(0, E), slice(E, 2 * E), slice(2 * E, 3 * E))):
        if part == 'k' and label.endswith('bias'):
            scale = max(float(b[:E].abs().max()), float(b[2 * E:].abs().max()))
            ys.add_abs(f'{label}[k]', g[blk], a[blk], b[blk], scale)
        else:
            ys.add(f'{label}[{part}]', g[blk], a[blk], b[blk])


@pytest.mark.parametrize('case', CASES)
def test_cross_encoder_layers_backward_layer_local(case):
    run = _full_run(case)
    model = run['model']
    ys = Yardstick(f'{case}: cross-encoder layers, layer-local backward (GPU ReLU masks)')
    not_identical, flips = [], []
    for i, (layer, r) in enumerate(zip(model.transformer_encoder.layers, run['rec']['xenc'])):
        named = _trainable(model, f'{XENC}{i}.')
        names = [n for n, _ in named]
        pos, plan = r['rest']
        x = r['x'].clone().requires_grad_(True)
        out = layer.forward_train_packed(x, pos, plan)
        rerun = torch.autograd.grad(out, [x] + [p for _, p in named], r['dout'])
        full = [r['dx']] + [run['grads'][n] for n in names]
        labels = ['dx'] + [n[len(f'{XENC}{i}.'):] for n in names]
        not_identical += [f'{i}.{lab}' for lab, a, b in zip(labels, rerun, full) if not torch.equal(a, b)]
        (h,) = [res for name, a, res in r['calls'] if name == 'linear' and a['relu']]
        mask = (h.detach() > 0).cpu()
        g64 = _oracle_layer(run, i, r['x'], pos, r['dout'], torch.float64, mask, names)
        g32 = _oracle_layer(run, i, r['x'], pos, r['dout'], torch.float32, mask, names)
        for lab, g, a, b in zip(labels, full, g32, g64):
            if lab.endswith('.in_proj_weight') or lab.endswith('.in_proj_bias'):
                _add_in_proj_rows(ys, f'{i}.{lab}', g, a, b)
            else:
                ys.add(f'{i}.{lab}', g, a, b)
        with torch.no_grad():
            free = _oracle_layer(run, i, r['x'], pos, r['dout'], torch.float64, None, names)
        flips.append(f'  layer {i}: ReLU {int((free != mask).sum())}/{mask.numel()}')
    ys.report()
    print('  decisions of the unforced float64 forward that differ from the GPU\'s:\n' + '\n'.join(flips))
    assert not not_identical, f'layer-local rerun not bit-identical to the full backward: {not_identical}'
    assert not ys.failures(), ys.failures()


@pytest.mark.parametrize('case', CASES)
def test_cross_encoder_attention_cores_on_recorded_tensors(case):
    """Every cross-encoder layer's self- and cross-attention core, on the q, k, v, O, lse and output gradient the
    training step gave it: the step's dq / dk / dv equal a rerun of the backward bit for bit and meet the yardstick as
    separate rows against float64 autograd of the core, and the invariants of tests/attention_oracle.py hold per
    problem and head (the dQ(k + c) check reruns the forward and backward with shifted keys)."""
    run = _full_run(case)
    H = run['model'].transformer_encoder.layers[0].nhead
    ys = Yardstick(f'{case}: cross-encoder attention cores on the recorded tensors')
    inv, not_identical = [], []
    for i, r in enumerate(run['rec']['xenc']):
        cores = [(a, res) for name, a, res in r['calls'] if name == 'mha_varlen_lse']
        assert len(cores) == 2, (i, len(cores))
        for which, (a, (o, lse)) in zip(('self', 'cross'), cores):
            b = run['rec']['mha_bwd'][o.data_ptr()]
            q, k, v, d_o = a['q'], a['k'], a['v'], b['d_o']
            problems = ao.problems_of(a['q_start'], a['q_len'], a['k_start'], a['k_len'])
            rerun = ao.run_kernel(q, k, v, d_o, problems, H, o, lse)
            not_identical += [f'{i}.{which}.{t}' for t in rerun if not torch.equal(rerun[t], b[t].cpu())]
            got = {t: b[t].cpu() for t in ('dq', 'dk', 'dv')}
            ks = k.cpu() + ao.key_shift(k, problems, H)
            r64, r32 = (ao.reference(q, k, v, d_o, problems, H, dt) for dt in (torch.float64, torch.float32))
            s64, s32 = (ao.reference(q, ks, v, d_o, problems, H, dt) for dt in (torch.float64, torch.float32))
            ao.add_rows(ys, f'{i}.{which} ', problems, got, r32, r64)
            got_shift = ao.run_kernel(q, ks, v, d_o, problems, H)
            inv += [(f'{i}.{which} {c}',) + tuple(rest) for c, *rest in
                    ao.invariants(problems, H, d_o, got, r32, r64, got_shift, s32, s64)]
    ys.report()
    ao.report_invariants(f'{case}: cross-encoder attention cores on the recorded tensors', inv)
    assert not not_identical, f'attention backward rerun not bit-identical to the training step: {not_identical}'
    assert not ys.failures(), ys.failures()
    assert not ao.failed(inv), ao.failed(inv)[:8]


# ------------------------------------------------------------------------------------------------ stage chain

def _oracle_feats_un_grad(run, dtype, feats_un=None):
    """d(total)/d(feats_un) of the oracle's forward and loss in `dtype` on the GPU's pyramid; feats_un: evaluate the
    stages after the encoder at this encoder output instead of the oracle's own."""
    from oracle import regtr_oracle as O
    from regtr_b200 import losses as LS
    cfg, meta = run['cfg'], run['meta_cpu']
    sdo = {k: (v.detach().to(dtype) if v.is_floating_point() else v) for k, v in run['sd'].items()}
    leaf = {}
    enc = O.encoder

    def encoder_leaf(*a, **k):
        f = enc(*a, **k) if feats_un is None else feats_un.cpu().to(dtype)
        leaf['f'] = f.detach().requires_grad_(True)
        return leaf['f']
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(O, 'encoder', encoder_leaf)
        pred = O.forward(sdo, cfg, run['src'], run['tgt'], dtype=dtype, meta=meta)
    bo = {'kpconv_meta': {k: meta[k] for k in ('points', 'pools', 'stack_lengths')}}
    bo.update({k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in run['li'].items()})
    mo = types.SimpleNamespace(cfg=cfg, feature_criterion=types.SimpleNamespace(W=sdo['feature_criterion.W']),
                               feature_criterion_un=types.SimpleNamespace(W=sdo['feature_criterion_un.W']))
    LS.compute_loss(mo, pred, bo)['total'].backward()
    return leaf['f'].grad


def _diag_errs(g, w, name):
    """tests/diag_grad_accuracy.py's measures: norm (relative), largest sampled entry / rms, largest entry / rms."""
    g, w = g.detach().double().reshape(-1).cpu(), w.detach().double().reshape(-1)
    idx = torch.from_numpy(ei.grad_sample_index(name, w.numel()))
    rms = max(float(w.norm()) / np.sqrt(w.numel()), 1e-30)
    return (abs(float(g.norm()) - float(w.norm())) / float(w.norm()), float((g[idx] - w[idx]).abs().max()) / rms,
            float((g - w).abs().max()) / rms)


@pytest.mark.parametrize('case', CASES)
def test_encoder_backward_from_float64_feats_un_gradient(case):
    """The float64 oracle's d(feats_un), cast to fp32, through the GPU encoder alone; the yardstick is the fp32 oracle
    encoder fed the same gradient, both oracle encoders run with the GPU's decisions.  Also reports how far the
    d(feats_un) of the full step is from float64, on the GPU and in the fp32 oracle (not asserted)."""
    from oracle import regtr_oracle as O
    run = _full_run(case)
    cfg, model, meta, sd = run['cfg'], run['model'], run['meta'], run['sd']
    d64 = _oracle_feats_un_grad(run, torch.float64)
    d32 = _oracle_feats_un_grad(run, torch.float32)
    last = run['rec']['enc'][-1]
    d64g = _oracle_feats_un_grad(run, torch.float64, last['y'])
    print(f'\n{case}: d(feats_un) of the full step against the float64 oracle\'s: max-abs / max|ref|, relative '
          'Frobenius | norm rel, sampled entry / rms, max entry / rms')
    for who, g, ref in (('GPU', last['dout'], d64), ('fp32 oracle', d32, d64),
                        ('GPU, float64 evaluated at the GPU\'s feats_un', last['dout'], d64g),
                        ('float64 at the GPU\'s feats_un', d64g, d64)):
        a, b = errors(g, ref), _diag_errs(g, ref, 'feats_un')
        print(f'  {who:46s} {a[0]:9.2e} {a[1]:9.2e} | {b[0]:8.1e} {b[1]:8.1e} {b[2]:8.1e}')
    print(f'  encoder output, GPU against float64: max-abs / max|ref| {errors(last["y"], O.encoder(sd, cfg, run["meta_cpu"], torch.float64))[0]:.2e}')
    named = _trainable(model, 'kpf_encoder.')
    for _, p in named:
        p.grad = None
    feats_un, _ = model.kpf_encoder(torch.ones_like(meta['_points'][0][:, 0:1]), meta)
    assert feats_un.shape == d64.shape
    torch.autograd.backward(feats_un, d64.float().to(DEV))
    gpu = {n: p.grad for n, p in named}
    decs = [_gpu_decisions(cfg, i, r['calls']) for i, r in enumerate(run['rec']['enc'])]

    def chain(dtype):
        leaves = _leaves(sd, list(gpu), dtype)
        sdd = {k: leaves.get(k, v) for k, v in sd.items() if k.startswith(ENC)}
        x = torch.ones((len(run['meta_cpu']['points'][0]), 1), dtype=dtype)
        for i, dec in enumerate(decs):
            d = dict(dec)
            x = O.encoder_block(sdd, cfg, i, x, run['meta_cpu'], dtype, d)
            assert d.keys() == dec.keys()
        return dict(zip(leaves, torch.autograd.grad(x, list(leaves.values()), d64.to(dtype))))
    o64, o32 = chain(torch.float64), chain(torch.float32)
    ys = Yardstick(f'{case}: encoder parameters from the float64 d(feats_un) (GPU decisions)')
    print(f'\n{case}: encoder parameters from the float64 d(feats_un), errors against the float64 oracle '
          '(norm rel | sampled entry / rms | max entry / rms)')
    print(f'{"parameter":40s} {"GPU":>28s}   {"fp32 oracle":>28s}')
    for n in gpu:
        ys.add(n[len(ENC):], gpu[n], o32[n], o64[n])
        a, b = _diag_errs(gpu[n], o64[n], n), _diag_errs(o32[n], o64[n], n)
        print(f'{n[len(ENC):]:40s} {a[0]:8.1e} {a[1]:8.1e} {a[2]:8.1e}   {b[0]:8.1e} {b[1]:8.1e} {b[2]:8.1e}')
    ys.report()
    assert not ys.failures(), ys.failures()
