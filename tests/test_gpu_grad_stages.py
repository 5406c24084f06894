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
import types

import numpy as np
import pytest
import torch

import attention_oracle as ao
from grad_yardstick import Yardstick, errors
from stage_oracle import (DEV, ENC, XENC, ei, flips as _flips, gpu_decisions as _gpu_decisions, leaves as _leaves,
                          oracle_block as _oracle_block, oracle_layer as _oracle_layer, block_sites as _block_sites,
                          train_run as _full_run, trainable as _trainable)

pytestmark = pytest.mark.gpu

CASES = ['fwd_3dmatch_small_b2', 'fwd_modelnet_b1']


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
