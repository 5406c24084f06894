"""GPU tests of the inference forward stage by stage, on the model's own activations.

One eager RegTR.forward per case records (tests/stage_oracle.py), for every KPConv-encoder block, every cross-encoder
layer, the final norm, the position embedding and the correspondence head, its input, its output and the ops it
calls.  Then:
  * each block / layer is re-run alone on its recorded input: its output must be bit-identical to the full forward's;
  * each block's output is compared with oracle.regtr_oracle.encoder_block in float64 under the fp32 yardstick
    (tests/grad_yardstick.py), both oracles run with the GPU's decisions (LeakyReLU masks, max-pool winners, KPConv
    divisors), and so is each op inside it on that op's own recorded inputs (the KPConv output, the Linear of
    `linear_instats` with its mean and rstd, the InstanceNorm passes); max_pool must equal the oracle's bit for bit;
  * each cross-encoder layer against oracle.cross_encoder_layer under the GPU's feed-forward ReLU masks, and each
    attention core's O with the O(k + c) = O and O(v + c) = O + c invariants (tests/attention_oracle.py);
  * the stages after the encoder on their recorded inputs: feature projection, position embedding, final LayerNorm,
    correspondence head, and the pose within 1e-6 of a float64 Kabsch with the reference's flip rule;
  * a chain table (printed, not asserted): every stage of the full GPU forward and of the full fp32 oracle forward
    against the full float64 oracle forward on the GPU's pyramid, and the first stage where the GPU's error grows
    past 10x the fp32 oracle's.
Every family of rows is shown to be sharp: an output multiplied by (1 + 1e-5) fails it.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attention_oracle as ao
from grad_yardstick import Yardstick, errors
import stage_oracle as so

pytestmark = pytest.mark.gpu

CASES = ['fwd_3dmatch_small_b2', 'fwd_modelnet_b1', 'var_modelnet_attndec_b1', 'var_modelnet_postnorm_b1',
         'real_3dmatch_redkitchen_0_5']


def _lens(offs):
    o = offs.cpu().tolist()
    return [b - a for a, b in zip(o[:-1], o[1:])]


def _stats(y, lens, dtype):
    means, rstds, a = [], [], 0
    for n in lens:
        seg = y[a:a + n].to(dtype)
        means.append(seg.mean(0))
        rstds.append(1.0 / torch.sqrt(seg.var(0, unbiased=False) + 1e-5))
        a += n
    return torch.stack(means), torch.stack(rstds)


def _first(r):
    return r[0] if isinstance(r, tuple) else r


# ------------------------------------------------------------------------------------------- encoder blocks

def _block_op_rows(ys, i, calls, dec, scale):
    """One row per recorded op of block i on its own recorded inputs."""
    from oracle import regtr_oracle as O
    for name, a, r in calls:
        if name == 'kpconv':
            args = {dt: [a[k].detach().cpu().to(dt) for k in ('q_pts', 's_pts', 'x', 'weights', 'kernel_points')]
                    for dt in (torch.float64, torch.float32)}
            idx = a['idx32'].long().cpu()
            ref = {dt: O.kpconv(q, s, idx, x, W, kp, a['extent'], count=dec['kpconv'])
                   for dt, (q, s, x, W, kp) in args.items()}
            ys.add(f'{i}.kpconv', _first(r).cpu() * scale, ref[torch.float32], ref[torch.float64])
            if a['instats'] is not None:
                lens = _lens(a['instats'][0])
                (m64, s64), (m32, s32) = (_stats(ref[dt], lens, dt) for dt in (torch.float64, torch.float32))
                ys.add(f'{i}.kpconv mean', r[1][..., 0].cpu() * scale, m32, m64)
                ys.add(f'{i}.kpconv rstd', r[1][..., 1].cpu() * scale, s32, s64)
        elif name == 'linear_instats':
            ref = {dt: a['x'].detach().cpu().to(dt) @ a['weight'].detach().cpu().to(dt).t()
                   for dt in (torch.float64, torch.float32)}
            lens = _lens(a['offs'])
            ys.add(f'{i}.linear_instats', r[0].cpu() * scale, ref[torch.float32], ref[torch.float64])
            (m64, s64), (m32, s32) = (_stats(ref[dt], lens, dt) for dt in (torch.float64, torch.float32))
            ys.add(f'{i}.linear_instats mean', r[1][..., 0].cpu() * scale, m32, m64)
            ys.add(f'{i}.linear_instats rstd', r[1][..., 1].cpu() * scale, s32, s64)
        elif name in ('instnorm_act', 'instnorm_apply'):
            out = _first(r).cpu()
            lens = _lens(a['offs'])
            mask = out > 0 if a['slope'] >= 0 else None
            ref = {}
            for dt in (torch.float64, torch.float32):
                y = O.instance_norm(a['x'].detach().cpu().to(dt), lens)
                if a['res'] is not None:
                    y = y + a['res'].detach().cpu().to(dt)
                ref[dt] = torch.where(mask, y, y * a['slope']) if mask is not None else y
            ys.add(f'{i}.{name}', out * scale, ref[torch.float32], ref[torch.float64])


def _encoder_rows(run, scale=1.0):
    from oracle import regtr_oracle as O
    cfg = run['cfg']
    ys = Yardstick(f'{run["case"]}: encoder blocks, block-local forward (GPU decisions)')
    flips, pools = [], []
    for i, r in enumerate(run['rec']['enc']):
        dec = so.gpu_decisions(cfg, i, r['calls'])
        y64, y32 = (so.oracle_block(run, i, r['x'], False, None, dt, dec, []) for dt in (torch.float64, torch.float32))
        ys.add(f'{i}.block', r['y'].cpu() * scale, y32, y64)
        _block_op_rows(ys, i, r['calls'], dec, scale)
        for _, a, res in [c for c in r['calls'] if c[0] == 'max_pool']:
            pools.append(torch.equal(O.max_pool(a['x'].detach().cpu(), a['idx32'].long().cpu()), res.cpu()))
        if scale == 1.0:
            free = {}
            with torch.no_grad():
                O.encoder_block(run['sd'], cfg, i, r['x'].cpu().double(), run['meta_cpu'], torch.float64, free)
            b, _ = so.block_sites(cfg, i)
            pool_idx = run['meta_cpu']['pools'][b['level']].long() if 'pool' in dec else None
            flips.append(f'  block {i}: {so.flips(dec, free, pool_idx)}')
    return ys, flips, pools


@pytest.mark.parametrize('case', CASES)
def test_encoder_blocks_forward_block_local(case):
    run = _run(case)
    model = run['model']
    not_identical = []
    with torch.no_grad():
        for i, (blk, r) in enumerate(zip(model.kpf_encoder.encoder_blocks, run['rec']['enc'])):
            if not torch.equal(blk(r['x'], *r['rest']), r['y']):
                not_identical.append(i)
    ys, flips, pools = _encoder_rows(run)
    ys.report()
    print('  decisions of the unforced float64 forward that differ from the GPU\'s:\n' + '\n'.join(flips))
    assert not not_identical, f'blocks whose rerun is not bit-identical to the full forward: {not_identical}'
    assert pools and all(pools), 'max_pool differs from the oracle\'s'
    assert not ys.failures(), ys.failures()


# ---------------------------------------------------------------------------------- cross-encoder layers

def _attention_rows(ys, inv, i, calls, H, scale):
    """O of every recorded attention core against float64 on its own inputs, and the O(k + c), O(v + c) invariants
    (the core re-run with shifted keys / values)."""
    from regtr_b200 import ops
    cores = [(n, a, r) for n, a, r in calls if n in ('mha_varlen', 'mha_tf32_tc')]
    assert len(cores) == 2, (i, [c[0] for c in calls])
    for which, (name, a, o) in zip(('self', 'cross'), cores):
        problems = ao.problems_of(a['q_start'], a['q_len'], a['k_start'], a['k_len'])
        if name == 'mha_varlen':
            q, k, v = (a[t].detach() for t in 'qkv')
            args = lambda kk, vv: ops.mha_varlen(q.contiguous(), kk.contiguous(), vv.contiguous(), a['q_start'],
                                                 a['q_len'], a['k_start'], a['k_len'], a['max_q_len'], H)
            qkv = {dt: (q.cpu().to(dt), k.cpu().to(dt), v.cpu().to(dt)) for dt in (torch.float64, torch.float32)}
        else:
            x, W, b = a['x'].detach(), a['in_w'].detach(), a['in_b'].detach()
            E = x.shape[1]
            qkv = {}
            for dt in (torch.float64, torch.float32):
                y = x.cpu().to(dt) @ W.cpu().to(dt).t() + b.cpu().to(dt)
                qkv[dt] = (y[:, :E], y[:, E:2 * E], y[:, 2 * E:])
            q, k, v = (t.float().to(so.DEV) for t in qkv[torch.float32])
            args = lambda kk, vv: ops.mha_varlen(q, kk.contiguous(), vv.contiguous(), a['q_start'], a['q_len'],
                                                 a['k_start'], a['k_len'], a['max_q_len'], H)
        (r64, _), (r32, _) = (ao.forward_reference(*qkv[dt], problems, H, dt) for dt in (torch.float64, torch.float32))
        rows = ao.rows_of([p for p in problems if p[3] > 0], 'q')
        ys.add(f'{i}.{which} attention O', o.cpu()[rows] * scale, r32[rows], r64[rows])
        if scale != 1.0 or name != 'mha_varlen':
            continue
        ck = ao.key_shift(k, problems, H, 0).to(so.DEV)
        cv = ao.key_shift(v, problems, H, 1).to(so.DEV)
        o_k, o_v = args(k + ck, v).cpu(), args(k, v + cv).cpu()
        k32 = ao.forward_reference(q, k + ck, v, problems, H, torch.float32)[0]
        v32 = ao.forward_reference(q, k, v + cv, problems, H, torch.float32)[0]
        cvd = cv.cpu().double()
        inv += [(f'{i}.{which} {n}',) + t[1:] for n, t in
                [('O(k + c) = O', t) for t in ao.per_problem('', problems, H, ao.HD, o_k, k32, r64)] +
                [('O(v + c) = O + c', t) for t in ao.per_problem('', problems, H, ao.HD, o_v.double() - cvd,
                                                                  v32.double() - cvd, r64)]]


def _layer_rows(run, scale=1.0):
    model = run['model']
    H = model.transformer_encoder.layers[0].nhead
    ys = Yardstick(f'{run["case"]}: cross-encoder layers, layer-local forward (GPU ReLU masks)')
    inv, flips = [], []
    for i, r in enumerate(run['rec']['xenc']):
        pos, _ = r['rest']
        (h,) = [res for name, a, res in r['calls'] if name == 'linear' and a['relu']]
        mask = (h > 0).cpu()
        y64, y32 = (so.oracle_layer(run, i, r['x'], pos, None, dt, mask, []) for dt in (torch.float64, torch.float32))
        ys.add(f'{i}.layer', r['y'].cpu() * scale, y32, y64)
        _attention_rows(ys, inv, i, r['calls'], H, scale)
        if scale == 1.0:
            with torch.no_grad():
                free = so.oracle_layer(run, i, r['x'], pos, None, torch.float64, None, [])
            flips.append(f'  layer {i}: ReLU {int((free != mask).sum())}/{mask.numel()}')
    return ys, inv, flips


@pytest.mark.parametrize('case', CASES)
def test_cross_encoder_layers_forward_layer_local(case):
    run = _run(case)
    not_identical = []
    with torch.no_grad():
        for i, (layer, r) in enumerate(zip(run['model'].transformer_encoder.layers, run['rec']['xenc'])):
            if not torch.equal(layer.forward_packed(r['x'], *r['rest']), r['y']):
                not_identical.append(i)
    ys, inv, flips = _layer_rows(run)
    ys.report()
    ao.report_invariants(f'{case}: cross-encoder attention cores on the recorded tensors', inv)
    print('  decisions of the unforced float64 forward that differ from the GPU\'s:\n' + '\n'.join(flips))
    assert not not_identical, f'layers whose rerun is not bit-identical to the full forward: {not_identical}'
    assert not ys.failures(), ys.failures()
    assert not ao.failed(inv), ao.failed(inv)[:8]


# ------------------------------------------------------------------------------------- after the encoder

def _pair_slices(run):
    lens = [int(v) for v in run['meta']['_lens'][-1]]
    st = np.concatenate([[0], np.cumsum(lens)])
    B = len(lens) // 2
    return B, [(slice(st[b], st[b + 1]), slice(st[B + b], st[B + b + 1])) for b in range(B)]


def _post_rows(run, scale=1.0):
    from oracle import regtr_oracle as O
    cfg, sd, model, rec = run['cfg'], run['sd'], run['model'], run['rec']
    ys = Yardstick(f'{run["case"]}: stages after the encoder, on their recorded inputs')
    g = lambda k, dt: sd[k].to(dt)
    dts = (torch.float64, torch.float32)
    (fp,) = [(a, r) for n, a, r in rec['top'] if n == 'linear' and a['weight'] is model.feat_proj.weight]
    ref = {dt: fp[0]['x'].cpu().to(dt) @ g('feat_proj.weight', dt).t() + g('feat_proj.bias', dt) for dt in dts}
    ys.add('feat_proj', fp[1].cpu() * scale, ref[torch.float32], ref[torch.float64])
    xyz = rec['pe']['x'].cpu()
    if cfg.get('pos_emb_type', 'sine') == 'sine':         # float64 on the same fp32 xyz and fp32 frequency table
        ref = {dt: O.pos_embed_sine(xyz.to(dt), cfg.d_embed, scale=cfg.get('pos_emb_scaling', 1.0)) for dt in dts}
    else:
        ref = {dt: O.pos_embed_learned({k: v.to(dt) for k, v in sd.items() if k.startswith('pos_embed.')}, xyz.to(dt))
               for dt in dts}
    ys.add('pos_embed', rec['pe']['y'].cpu() * scale, ref[torch.float32], ref[torch.float64])
    if cfg.pre_norm:
        for j, f in enumerate(rec['final']):
            ref = {dt: F.layer_norm(f['x'].cpu().to(dt), (cfg.d_embed,), g('transformer_encoder.norm.weight', dt),
                                    g('transformer_encoder.norm.bias', dt), 1e-5) for dt in dts}
            ys.add(f'final norm {j}', f['y'].cpu() * scale, ref[torch.float32], ref[torch.float64])
    head = rec['head']
    cond, (xyz_c, pe, _) = head['x'].cpu(), head['rest']
    corr, logit = head['y']
    B, sl = _pair_slices(run)
    ref = {}
    for dt in dts:
        c, lg = torch.zeros(corr.shape, dtype=dt), torch.zeros(logit.shape, dtype=dt)
        sdd = {k: v.to(dt) for k, v in sd.items() if k.startswith('correspondence_decoder.')}
        for rs, rt in sl:
            if cfg.get('direct_regress_coor', False):
                for rows in (rs, rt):
                    c[:, rows], lg[:, rows] = O.regressor(sdd, cond[:, rows].to(dt))
            else:
                x, p = xyz_c.cpu().to(dt), pe.cpu().to(dt)
                c[:, rs], lg[:, rs] = O.corr_decoder(sdd, cfg, cond[:, rs].to(dt), cond[:, rt].to(dt), p[rs], p[rt], x[rt])
                c[:, rt], lg[:, rt] = O.corr_decoder(sdd, cfg, cond[:, rt].to(dt), cond[:, rs].to(dt), p[rt], p[rs], x[rs])
        ref[dt] = (c, lg)
    ys.add('head corr', corr.cpu() * scale, ref[torch.float32][0], ref[torch.float64][0])
    ys.add('head logit', logit.cpu() * scale, ref[torch.float32][1], ref[torch.float64][1])
    (pc,) = [(a, r) for n, a, r in rec['top'] if n == 'pose_from_corr']
    kp, cr, lgt = (pc[0][k].cpu() for k in ('kp', 'corr', 'logit'))
    ref = {}
    for dt in dts:
        poses = []
        for rs, rt in sl:
            L_ = cr.shape[0]
            a = torch.cat([kp[rs].to(dt).expand(L_, -1, -1), cr[:, rt].to(dt)], 1)
            b = torch.cat([cr[:, rs].to(dt), kp[rt].to(dt).expand(L_, -1, -1)], 1)
            w = torch.sigmoid(torch.cat([lgt[:, rs], lgt[:, rt]], 1).to(dt))
            poses.append(O.kabsch(a, b, w))
        ref[dt] = torch.stack(poses, 1)
    got = pc[1].cpu()
    # fp32 SVD is 1e-6 to 1e-5 off float64 here, too loose to serve as the yardstick: the pose is held to 1e-6 of
    # float64 (the float64 reference stands in for the fp32 one, so the bound is the yardstick's floor)
    ys.add('pose R', got[..., :3] * scale, ref[torch.float64][..., :3], ref[torch.float64][..., :3])
    ys.add('pose t', got[..., 3] * scale, ref[torch.float64][..., 3], ref[torch.float64][..., 3])
    return ys


@pytest.mark.parametrize('case', CASES)
def test_stages_after_encoder_on_recorded_inputs(case):
    ys = _post_rows(_run(case))
    ys.report()
    assert not ys.failures(), ys.failures()


# ------------------------------------------------------------------------------------------- chain table

def _oracle_chain(run, dtype):
    """Every stage output of the unforced oracle forward in `dtype` on the GPU's pyramid, packed as the GPU packs
    them: encoder blocks, feature projection, cross-encoder layers (and their final norm)."""
    from oracle import regtr_oracle as O
    cfg, sd = run['cfg'], run['sd']
    out = {}
    x = torch.ones((len(run['meta_cpu']['points'][0]), 1), dtype=dtype)
    with torch.no_grad():
        for i in range(len(run['rec']['enc'])):
            x = O.encoder_block(sd, cfg, i, x, run['meta_cpu'], dtype)
            out[f'encoder block {i}'] = x
        both = x @ sd['feat_proj.weight'].to(dtype).t() + sd['feat_proj.bias'].to(dtype)
        out['feat_proj'] = both
        xyz = run['meta_cpu']['points'][-1].to(dtype)
        pe = O.pos_embed_sine(xyz, cfg.d_embed, scale=cfg.get('pos_emb_scaling', 1.0)) \
            if cfg.get('pos_emb_type', 'sine') == 'sine' else \
            O.pos_embed_learned({k: v.to(dtype) for k, v in sd.items() if k.startswith('pos_embed.')}, xyz)
        use_pe = cfg.transformer_encoder_has_pos_emb
        B, sl = _pair_slices(run)
        cur = both.clone()
        for i in range(cfg.num_encoder_layers):
            nxt = cur.clone()
            for rs, rt in sl:
                z = torch.zeros_like(cur[rs]), torch.zeros_like(cur[rt])
                nxt[rs], nxt[rt] = O.cross_encoder_layer(sd, cfg, i, cur[rs], cur[rt], pe[rs] if use_pe else z[0],
                                                         pe[rt] if use_pe else z[1])
            cur = nxt
            out[f'cross-encoder layer {i}'] = cur
            if cfg.pre_norm:
                out[f'final norm {i}'] = F.layer_norm(cur, (cfg.d_embed,), sd['transformer_encoder.norm.weight'].to(dtype),
                                                      sd['transformer_encoder.norm.bias'].to(dtype), 1e-5)
    return out


@pytest.mark.parametrize('case', CASES)
def test_forward_chain_table(case):
    """Printed, not asserted: each stage of the full GPU forward and of the full fp32 oracle forward against the full
    float64 oracle forward (unforced, on the GPU's pyramid)."""
    run = _run(case)
    rec = run['rec']
    gpu = {f'encoder block {i}': r['y'] for i, r in enumerate(rec['enc'])}
    gpu['feat_proj'] = [r for n, a, r in rec['top'] if n == 'linear' and a['weight'] is run['model'].feat_proj.weight][0]
    for i, r in enumerate(rec['xenc']):
        gpu[f'cross-encoder layer {i}'] = r['y']
        if run['cfg'].pre_norm:
            gpu[f'final norm {i}'] = rec['final'][i]['y']
    o64, o32 = _oracle_chain(run, torch.float64), _oracle_chain(run, torch.float32)
    print(f'\n{case}: full forward, each stage against the full float64 oracle forward (max-abs / max|ref|, '
          'relative Frobenius)')
    print(f'  {"stage":24s} {"GPU max":>9s} {"GPU fro":>9s}   {"fp32 max":>9s} {"fp32 fro":>9s}   GPU / fp32')
    first = None
    for name, g in gpu.items():
        eg, ef = errors(g, o64[name]), errors(o32[name], o64[name])
        ratio = eg[0] / max(ef[0], 1e-30)
        if first is None and ratio > 10 and eg[0] > 1e-6:
            first = name
        print(f'  {name:24s} {eg[0]:9.2e} {eg[1]:9.2e}   {ef[0]:9.2e} {ef[1]:9.2e}   {ratio:8.2f}')
    print(f'  first stage where the GPU\'s error exceeds 10x the fp32 oracle\'s (and 1e-6): {first or "none"}')
    assert set(gpu) == set(o64)


# ------------------------------------------------------------------------------------------- sharpness

def test_forward_stage_checks_are_sharp():
    """Every row family -- encoder block, KPConv, linear_instats (out, mean, rstd), InstanceNorm pass, cross-encoder
    layer, attention O, feature projection, position embedding, final norm, head, pose -- fails with its GPU output
    multiplied by (1 + 1e-5)."""
    run = _run('fwd_3dmatch_small_b2')
    s = 1 + 1e-5
    fails = _encoder_rows(run, s)[0].failures() + _layer_rows(run, s)[0].failures() + _post_rows(run, s).failures()
    families = ['.block', '.kpconv', '.linear_instats', '.linear_instats mean', '.linear_instats rstd', '.instnorm_',
                '.layer', 'attention O', 'feat_proj', 'pos_embed', 'final norm', 'head corr', 'head logit', 'pose R',
                'pose t']
    missing = [f for f in families if not any(f in name for name in fails)]
    print(f'\nrows failing with outputs x (1 + 1e-5): {len(fails)}')
    assert not missing, missing


def _run(case):
    run = so.inference_run(case)
    run['case'] = case
    return run
