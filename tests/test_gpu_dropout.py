"""GPU tests of the cross-encoder dropout (model.dropout > 0, forward_train in training mode): the keep masks against
the Python rule (tests/dropout_rule.py), the attention core and the whole cross-encoder against float64 with the same
masks under the fp32 yardstick, bit-identity with the dropout-free model wherever dropout does not apply, launch
counts, determinism and the rank invariance of the masks."""
import math

import numpy as np
import pytest
import torch

import dropout_rule as R
from grad_yardstick import Yardstick
from test_gpu_backward import _batch, _model

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
P = 0.1
SEED, STEP = 20261017, 9


def _offs(lens):
    return torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------- keep masks

def test_keep_mask_equals_the_python_rule_on_every_site():
    """ops.dropout_keep_mask (the kernels' device function) against the restatement, bit for bit: every layer, site
    and head of a modelnet-sized step, at pair_base 0 and inside a batch starting at pair 3."""
    from regtr_b200 import ops
    for lens, pair_base in (([212, 190], 0), ([64, 131, 17, 200], 3)):
        B = len(lens) // 2
        for layer in range(6):
            for site in R.SITES:
                for c in range(2 * B):
                    partner = (c + B) % (2 * B)
                    cols = {1: lens[c], 3: lens[partner], 5: 1024}.get(site, 256)
                    for head in (range(8) if site in (1, 3) else (0,)):
                        got = ops.dropout_keep_mask(P, SEED, STEP, pair_base, B, c, layer, site, head, lens[c], cols)
                        want = R.local_keep_mask(P, SEED, STEP, pair_base, B, c, layer, site, head, lens[c], cols)
                        assert np.array_equal(got.cpu().numpy().astype(bool), want), (lens, layer, site, c, head)


# --------------------------------------------------------------------------------------------- attention core

def _mask_tensor(p, key, B, c, layer, site, head, rows, cols, dtype):
    m = R.local_keep_mask(p, *key, B, c, layer, site, head, rows, cols)
    return torch.from_numpy(m).to(dtype) * float(R.scale(p))


def _attention_ref(qkv, d_o, lens, cross, key, layer, site, dtype):
    """float64 / float32 autograd of the dropped attention over the plan's problems -> (O, dqkv)."""
    B = len(lens) // 2
    off = np.concatenate([[0], np.cumsum(lens)])
    E, H = qkv.shape[1] // 3, 8
    x = qkv.detach().cpu().to(dtype).requires_grad_(True)
    o = torch.zeros(x.shape[0], E, dtype=dtype)
    for c in range(2 * B):
        kc = (c + B) % (2 * B) if cross else c
        qs, ql, ks, kl = off[c], lens[c], off[kc], lens[kc]
        if ql == 0 or kl == 0:
            continue
        q = x[qs:qs + ql, :E].view(ql, H, 32).transpose(0, 1)
        k = x[ks:ks + kl, E:2 * E].view(kl, H, 32).transpose(0, 1)
        v = x[ks:ks + kl, 2 * E:].view(kl, H, 32).transpose(0, 1)
        pr = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(32), -1)
        m = torch.stack([_mask_tensor(P, key, B, c, layer, site, h, ql, kl, dtype) for h in range(H)])
        o[qs:qs + ql] = ((pr * m) @ v).transpose(0, 1).reshape(ql, E)
    (o * d_o.cpu().to(dtype)).sum().backward()
    return o.detach(), x.grad


@pytest.mark.parametrize('cross', [False, True])
def test_attention_core_drop_argument_matches_float64(cross):
    """Dropout forward, dQ, dK and dV against float64 autograd with the same masks (fp32 yardstick), uneven clouds
    of 2 pairs; sum_k dK = 0 over every key range (sum_j dS_ij = 0 in the backward's own arithmetic)."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    lens = [37, 130, 64, 9]
    B, E, H = 2, 256, 8
    n = sum(lens)
    g = torch.Generator().manual_seed(3)
    qkv = (torch.randn(n, 3 * E, generator=g) * 1.5).to(DEV)
    qkv[:, E:2 * E] += 0.7                  # a shared key offset: softmax ignores it, so sum_k dK must vanish
    d_o = torch.randn(n, E, generator=g).to(DEV)
    plan = AttentionPlan(lens, DEV)
    ks, kl = (plan.xk_start, plan.xk_len) if cross else (plan.q_start, plan.q_len)
    site, layer = (3 if cross else 1), 4
    key = ops.DropoutKey(P, SEED, STEP, 0, B)
    drop = key.site(layer, site)
    q, k, v = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    o, lse = ops.mha_varlen_lse(q, k, v, plan.q_start, plan.q_len, ks, kl, plan.max_len, H, drop=drop)
    _, lse0 = ops.mha_varlen_lse(q, k, v, plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
    assert torch.equal(lse, lse0)                                   # lse of the undropped probabilities
    d = torch.zeros_like(qkv)
    ops.mha_varlen_bwd(q, k, v, o, lse, d_o, d[:, :E], d[:, E:2 * E], d[:, 2 * E:], plan.q_start, plan.q_len,
                       ks, kl, plan.max_len, plan.max_len, H, drop=drop)
    torch.cuda.synchronize()
    kk = (SEED, STEP, 0)
    o64, d64 = _attention_ref(qkv, d_o, lens, cross, kk, layer, site, torch.float64)
    o32, d32 = _attention_ref(qkv, d_o, lens, cross, kk, layer, site, torch.float32)
    ys = Yardstick(f'attention with dropout, {"cross" if cross else "self"} problems')
    ys.add('O', o, o32, o64)
    dc = d.cpu()
    for name, sl in (('dq', slice(0, E)), ('dk', slice(E, 2 * E)), ('dv', slice(2 * E, 3 * E))):
        ys.add(name, dc[:, sl], d32[:, sl], d64[:, sl])
    off = np.concatenate([[0], np.cumsum(lens)])
    scale = float(d64[:, E:2 * E].abs().max())
    for c in range(2 * B):
        r = slice(off[c], off[c + 1])
        ys.add_abs(f'sum dK cloud {c}', dc[r, E:2 * E].sum(0), d32[r, E:2 * E].sum(0),
                   torch.zeros(E, dtype=torch.float64), scale)
    ys.report()
    assert not ys.failures(), ys.failures()
    # the mask matters: without it the result is far off
    o_nodrop = ops.mha_varlen(q, k, v, plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
    assert float((o_nodrop - o).abs().max()) > 1e-2
    d2 = torch.zeros_like(qkv)
    ops.mha_varlen_bwd(q, k, v, o, lse, d_o, d2[:, :E], d2[:, E:2 * E], d2[:, 2 * E:], plan.q_start,
                       plan.q_len, ks, kl, plan.max_len, plan.max_len, H, drop=drop)
    assert torch.equal(d, d2)


def test_dropout_arguments_come_together():
    """The attention forward and the LayerNorm forward and backward take their dropout arguments as optional pointers
    that are all given or all NULL: every mixed combination returns its error code and launches nothing (the
    NaN-filled outputs stay untouched)."""
    from regtr_b200 import lib, ops
    from regtr_b200.transformer import AttentionPlan
    L = lib.load()
    ERR_ARG, ERR_UNSUPPORTED = -1, -3
    st = torch.cuda.current_stream().cuda_stream
    lens, E, H = [37, 64], 256, 8
    n = sum(lens)
    g = torch.Generator().manual_seed(5)
    qkv, x, z, dy = (torch.randn(n, c, generator=g).to(DEV) for c in (3 * E, E, E, E))
    gamma, beta = torch.ones(E, device=DEV), torch.zeros(E, device=DEV)
    offs, n_dev = _offs(lens), torch.tensor([n], dtype=torch.int32, device=DEV)
    key = ops.DropoutKey(P, SEED, STEP, 0, 1, offs=offs, max_len=max(lens))
    plan = AttentionPlan(lens, DEV)
    p = lambda t: None if t is None else t.data_ptr()
    nan = lambda *shape: torch.full(shape, float('nan'), device=DEV)
    untouched = lambda *ts: all(bool(t.isnan().all()) for t in ts if t is not None)

    # attention forward: a dropout key needs lse; a tile table takes neither lse nor a key
    att = key.site(0, ops.SITE_SELF_ATTN).ptr
    q, k, v = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    tb, mt = plan.tiles64
    for want_lse, tiles, drop, rc in ((False, None, att, ERR_ARG), (True, tb, None, ERR_UNSUPPORTED),
                                      (False, tb, att, ERR_UNSUPPORTED), (True, tb, att, ERR_UNSUPPORTED)):
        o, lse = nan(n, E), (nan(n, H) if want_lse else None)
        got = L.regtr_mha_varlen_fwd(p(q), 3 * E, p(k), 3 * E, p(v), 3 * E, p(o), E, p(lse), p(plan.q_start),
                                     p(plan.q_len), p(plan.q_start), p(plan.q_len), 2, plan.max_len, p(tiles),
                                     mt if tiles is not None else 0, H, 32, 1 / math.sqrt(32), drop, st)
        assert got == rc, (want_lse, tiles is not None, drop is not None)
        assert untouched(o, lse)

    # LayerNorm forward: z, offs, x_out and the key together, and no n_dev with the key
    res = key.site(0, ops.SITE_SELF_OUT).ptr
    xo = nan(n, E)
    full = dict(z=z, offs=offs, x_out=xo, drop=res)
    for kw in (dict(z=z), dict(offs=offs), dict(x_out=xo), dict(full, drop=None), dict(drop=res),
               dict(z=z, offs=offs, drop=res), dict(full, n_dev=n_dev)):
        a = dict(dict.fromkeys(('z', 'offs', 'x_out', 'drop', 'n_dev')), **kw)
        y = nan(n, E)
        got = L.regtr_layernorm_pos(p(x), p(a['z']), p(gamma), p(beta), None, n, p(a['n_dev']), p(a['offs']), E, 1e-5,
                                    p(y), None, p(a['x_out']), a['drop'], st)
        assert got == ERR_ARG, sorted(k for k, t in kw.items() if t is not None)
        assert untouched(y, xo)

    # LayerNorm backward: offs, dz and the key together
    ws = torch.empty(L.regtr_layernorm_bwd_ws_bytes(n, E), dtype=torch.uint8, device=DEV)
    dz = nan(n, E)
    for kw in (dict(offs=offs), dict(dz=dz), dict(offs=offs, dz=dz), dict(drop=res), dict(offs=offs, drop=res),
               dict(dz=dz, drop=res)):
        a = dict(dict.fromkeys(('offs', 'dz', 'drop')), **kw)
        dx, dg, db = nan(n, E), nan(E), nan(E)
        got = L.regtr_layernorm_bwd(p(x), p(gamma), p(dy), None, None, n, p(a['offs']), E, 1e-5, p(dx), p(a['dz']),
                                    p(dg), p(db), a['drop'], p(ws), ws.numel(), st)
        assert got == ERR_ARG, sorted(kw)
        assert untouched(dx, dg, db, dz)


# --------------------------------------------------------------------------------------------- cross-encoder

def _ln(x, w, b):
    return torch.nn.functional.layer_norm(x, (x.shape[1],), w, b, 1e-5)


def _encoder_ref(x, pos, lens, prm, n_layers, key, dtype, relu_pass=None):
    """transformers.py forward_pre (train mode) + the final norm of every layer, packed, with the Python masks.
    relu_pass (one bool tensor per layer): the GPU's ReLU decisions, taken instead of the reference's own (a
    pre-activation within rounding of 0 may fall on either side, which moves one gradient entry by a whole term)."""
    B = len(lens) // 2
    off = np.concatenate([[0], np.cumsum(lens)])
    E, H = x.shape[1], 8
    s = float(R.scale(P))

    def rows_mask(layer, site, cols):
        return torch.cat([torch.from_numpy(R.local_keep_mask(P, *key, B, c, layer, site, 0, lens[c], cols))
                          for c in range(2 * B)]).to(dtype) * s

    def attend(y, pfx, layer, cross):
        site = 3 if cross else 1
        qkv = y @ prm[pfx + 'in_proj_weight'].T + prm[pfx + 'in_proj_bias']
        outs = []
        for c in range(2 * B):
            kc = (c + B) % (2 * B) if cross else c
            ql, kl = lens[c], lens[kc]
            q = qkv[off[c]:off[c + 1], :E].view(ql, H, 32).transpose(0, 1)
            k = qkv[off[kc]:off[kc + 1], E:2 * E].view(kl, H, 32).transpose(0, 1)
            v = qkv[off[kc]:off[kc + 1], 2 * E:].view(kl, H, 32).transpose(0, 1)
            pr = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(32), -1)
            m = torch.stack([torch.from_numpy(R.local_keep_mask(P, *key, B, c, layer, site, h, ql, kl)).to(dtype)
                             for h in range(H)]) * s
            outs.append(((pr * m) @ v).transpose(0, 1).reshape(ql, E))
        o = torch.cat(outs)
        return o @ prm[pfx + 'out_proj.weight'].T + prm[pfx + 'out_proj.bias']

    res = []
    for li in range(n_layers):
        L = f'layers.{li}.'
        y = _ln(x, prm[L + 'norm1.weight'], prm[L + 'norm1.bias']) + pos
        x = x + attend(y, L + 'self_attn.', li, False) * rows_mask(li, 2, E)
        y = _ln(x, prm[L + 'norm2.weight'], prm[L + 'norm2.bias']) + pos
        x = x + attend(y, L + 'multihead_attn.', li, True) * rows_mask(li, 4, E)
        y = _ln(x, prm[L + 'norm3.weight'], prm[L + 'norm3.bias'])
        pre = y @ prm[L + 'linear1.weight'].T + prm[L + 'linear1.bias']
        h = torch.relu(pre) if relu_pass is None else pre * relu_pass[li].to(dtype)
        h = h * rows_mask(li, 5, h.shape[1])
        x = x + (h @ prm[L + 'linear2.weight'].T + prm[L + 'linear2.bias']) * rows_mask(li, 6, E)
        res.append(_ln(x, prm['norm.weight'], prm['norm.bias']))
    return torch.stack(res)


def _encoder(n_layers, p):
    import torch.nn as nn
    from regtr_b200.transformer import TransformerCrossEncoder, TransformerCrossEncoderLayer
    torch.manual_seed(0)
    layer = TransformerCrossEncoderLayer(256, 8, 1024, p, normalize_before=True, sa_val_has_pos_emb=True,
                                         ca_val_has_pos_emb=True)
    enc = TransformerCrossEncoder(layer, n_layers, nn.LayerNorm(256), return_intermediate=True)
    with torch.no_grad():
        for name, t in enc.named_parameters():
            if 'norm' in name:
                t.copy_((1.0 if name.endswith('weight') else 0.0) + 0.1 * torch.randn_like(t))
            elif name.endswith('bias'):
                t.copy_(0.05 * torch.randn_like(t))
    return enc.to(DEV)


def _model_activations(case):
    """The cross-encoder of a case's model with its own input: feat_proj output, position embedding, coarse lengths."""
    _, m1, src, tgt = _models(case)
    with torch.no_grad():
        b = _batch(case, src, tgt)
        meta = m1.preprocessor(list(b['src_xyz']) + list(b['tgt_xyz']), lazy_upsamples=True)
        enc = m1._stage_encoder(meta)
    return m1.transformer_encoder, enc['both_un'].cpu(), enc['pe'].cpu(), [int(v) for v in meta['_lens'][-1]]


@pytest.mark.parametrize('inputs', ['random', 'fwd_modelnet_b1', 'fwd_3dmatch_small_b2'])
def test_cross_encoder_drop_argument_matches_float64(inputs):
    """Pre-norm layers with all six dropouts (forward_train_packed with a DropoutKey) against float64 autograd of
    the reference's forward_pre with the same masks: every output and every gradient under the fp32 yardstick.
    'random': two layers with perturbed norms on randn tokens of two uneven pairs; the model cases: the model's own
    six-layer cross-encoder on its own feat_proj output and position embedding."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    E = 256
    g = torch.Generator().manual_seed(1)
    if inputs == 'random':
        lens = [150, 41, 97, 230]                       # two pairs, uneven
        n_layers, pair_base = 2, 5
        enc = _encoder(n_layers, P)
        x0 = torch.randn(sum(lens), E, generator=g)
        pos = torch.randn(sum(lens), E, generator=g)
    else:
        enc, x0, pos, lens = _model_activations(inputs)
        n_layers, pair_base = len(enc.layers), 2
        enc.requires_grad_(True)
    B = len(lens) // 2
    gout = torch.randn(n_layers, sum(lens), E, generator=g)
    x = x0.to(DEV).requires_grad_(True)
    plan = AttentionPlan(lens, DEV)
    drop = ops.DropoutKey(P, SEED, STEP, pair_base, B, offs=_offs(lens), max_len=max(lens))
    hs, real = [], ops.linear

    def spy(*a, **k):
        h = real(*a, **k)
        if k.get('drop') is not None:                   # the feed-forward block's dropout(relu(linear1))
            hs.append(h.detach().cpu())
        return h
    ops.linear = spy
    try:
        out = enc.forward_train_packed(x, pos.to(DEV), plan, drop=drop)
    finally:
        ops.linear = real
    (out * gout.to(DEV)).sum().backward()
    key = (SEED, STEP, pair_base)
    # the GPU's ReLU decisions: where a unit is kept, the dropped output is positive exactly where the ReLU passed
    # (where it is dropped the mask zeroes the unit whatever the decision)
    relu_pass = [h > 0 for h in hs]
    assert len(relu_pass) == n_layers
    ref = {}
    for dt in (torch.float64, torch.float32):
        prm = {n: t.detach().cpu().to(dt).requires_grad_(True) for n, t in enc.named_parameters()}
        xr = x0.to(dt).requires_grad_(True)
        o = _encoder_ref(xr, pos.to(dt), lens, prm, n_layers, key, dt, relu_pass)
        (o * gout.to(dt)).sum().backward()
        ref[dt] = (o.detach(), xr.grad, {n: t.grad for n, t in prm.items()})
    ys = Yardstick(f'cross-encoder with dropout ({inputs}: {n_layers} layers, {B} pairs)')
    ys.add('out', out, ref[torch.float32][0], ref[torch.float64][0])
    ys.add('dx', x.grad, ref[torch.float32][1], ref[torch.float64][1])
    for n, t in enc.named_parameters():
        ys.add('d ' + n, t.grad, ref[torch.float32][2][n], ref[torch.float64][2][n])
    ys.report()
    assert not ys.failures(), ys.failures()
    # the masks are those of the global pairs: another pair_base gives another result
    out2 = enc.forward_train_packed(x, pos.to(DEV), plan,
                                    drop=ops.DropoutKey(P, SEED, STEP, 0, B, offs=_offs(lens), max_len=max(lens)))
    assert float((out2 - out).abs().max()) > 1e-3


# ------------------------------------------------------------------------------------------------ whole model

def _models(case='fwd_modelnet_b1'):
    """(p = 0 model in training mode, p = 0.1 model with the same weights, src, tgt)."""
    from regtr_b200.regtr import RegTR
    cfg, sd, m0, src, tgt = _model(case)
    cfg1 = cfg.copy()
    cfg1.dropout = P
    m1 = RegTR(cfg1).to(DEV)
    m1.load_state_dict(sd, strict=True)
    m1.kpf_encoder.requires_grad_(False)
    return m0, m1, src, tgt


def _train_step(model, case, src, tgt, **kw):
    from regtr_b200 import ops
    model.zero_grad(set_to_none=True)
    batch = _batch(case, src, tgt)
    n0 = ops.LAUNCHES
    pred = model.forward_train(batch, **kw)
    total = model.compute_loss(pred, batch)['total']
    total.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    return pred, total.detach(), grads, ops.LAUNCHES - n0


def _same(a, b):
    pa, ta, ga, _ = a
    pb, tb, gb, _ = b
    assert torch.equal(ta, tb)
    for k in ('src_feat', 'tgt_feat', 'src_kp_warped', 'tgt_overlap'):
        for u, v in zip(pa[k], pb[k]):
            assert torch.equal(u, v), k
    assert ga.keys() == gb.keys()
    for n in ga:
        assert torch.equal(ga[n], gb[n]), n


def test_unchanged_at_p0_and_in_eval_mode():
    """A p = 0.1 model in eval mode: forward, GraphedRegTR and forward_train (outputs and gradients) bit-identical to
    the p = 0 model with the same weights, with the same number of launches; the training-mode forward warns once."""
    from regtr_b200.regtr import GraphedRegTR
    case = 'fwd_modelnet_b1'
    m0, m1, src, tgt = _models(case)
    m1.eval()
    a, b = m0(_batch(case, src, tgt)), m1(_batch(case, src, tgt))
    for k in ('src_feat', 'tgt_kp_warped', 'src_overlap'):
        assert torch.equal(a[k][0], b[k][0]), k
    assert torch.equal(a['pose'], b['pose'])
    ga, gb = GraphedRegTR(m0)(_batch(case, src, tgt)), GraphedRegTR(m1)(_batch(case, src, tgt))
    assert torch.equal(ga['pose'], gb['pose'])
    r0 = _train_step(m0, case, src, tgt)
    r1 = _train_step(m1, case, src, tgt, dropout_key=(1, 2, 3))
    _same(r0, r1)
    assert r0[3] == r1[3]
    r0b = _train_step(m0, case, src, tgt, dropout_key=(1, 2, 3))       # p = 0: the key is ignored
    r1b = _train_step(m1, case, src, tgt, dropout_key=(4, 5, 6))
    _same(r0, r0b)
    _same(r0b, r1b)
    assert r0b[3] == r1b[3]                  # second steps: weight splits and index caches are built by the first


def test_dropout_step_is_keyed_deterministic_and_within_the_launch_budget(caplog):
    case = 'fwd_modelnet_b1'
    m0, m1, src, tgt = _models(case)
    base = _train_step(m0, case, src, tgt)
    a = _train_step(m1, case, src, tgt, dropout_key=(SEED, STEP, 0))
    b = _train_step(m1, case, src, tgt, dropout_key=(SEED, STEP, 0))
    _same(a, b)
    c = _train_step(m1, case, src, tgt, dropout_key=(SEED, STEP + 1, 0))
    assert not torch.equal(a[0]['src_feat'][0], c[0]['src_feat'][0])
    assert not torch.equal(a[0]['src_feat'][0], base[0]['src_feat'][0])
    n_layers = len(m1.transformer_encoder.layers)
    print('launches: p=0', base[3], 'p=0.1', a[3])
    assert a[3] <= base[3] + n_layers
    torch.manual_seed(7)
    d = _train_step(m1, case, src, tgt)
    torch.manual_seed(7)
    e = _train_step(m1, case, src, tgt)
    _same(d, e)                                         # dropout_key None: reproducible under torch.manual_seed
    import logging
    with caplog.at_level(logging.WARNING):
        m1(_batch(case, src, tgt)); m1(_batch(case, src, tgt))
    assert sum('forward_train' in r.getMessage() for r in caplog.records) == 1


def test_masks_follow_the_global_pair_not_the_batch():
    """Pair 1 of fwd_3dmatch_small_b2 trained alone with pair_base 1 sees the masks it sees inside the batch of two
    (pair_base 0): its features agree to GEMM rounding, and differ with pair_base 0."""
    case = 'fwd_3dmatch_small_b2'
    _, m1, src, tgt = _models(case)
    with torch.no_grad():
        both = m1.forward_train(_batch(case, src, tgt), dropout_key=(SEED, STEP, 0))
        b1 = _batch(case, src, tgt)
        one = {k: b1[k][1:2] for k in ('src_xyz', 'tgt_xyz')}
        alone = m1.forward_train(one, dropout_key=(SEED, STEP, 1))
        wrong = m1.forward_train(dict(one), dropout_key=(SEED, STEP, 0))
    for k in ('src_feat', 'tgt_feat'):
        ref = both[k][1]
        err = float((alone[k][0] - ref).abs().max() / ref.abs().max())
        off = float((wrong[k][0] - ref).abs().max() / ref.abs().max())
        print(k, err, off)
        assert err <= 1e-4 and off > 1e-2


def test_training_with_dropout_lowers_the_loss():
    """SGD steps at p = 0.1 (trainer-style keys: one step index per update) lower the eval-mode loss."""
    case = 'fwd_modelnet_b1'
    _, m1, src, tgt = _models(case)
    opt = torch.optim.SGD([p for p in m1.parameters() if p.requires_grad], lr=2e-3)

    def eval_loss():
        m1.eval()
        b = _batch(case, src, tgt)
        v = float(m1.compute_loss(m1(b), b)['total'])
        m1.train()
        return v
    before = eval_loss()
    for step in range(1, 7):
        opt.zero_grad(set_to_none=True)
        b = _batch(case, src, tgt)
        m1.compute_loss(m1.forward_train(b, dropout_key=(SEED, step, 0)), b)['total'].backward()
        opt.step()
    after = eval_loss()
    print('eval loss', before, '->', after)
    assert after < before


# ----------------------------------------------------------------------------------------- against the reference

@pytest.mark.parametrize('case', ['fwd_modelnet_b1', 'fwd_3dmatch_small_b2'])
def test_forward_train_with_dropout_matches_the_reference(case):
    """forward_train -> compute_loss -> backward at dropout 0.1, encoder frozen, against the unmodified reference run
    in train mode with the same masks served through F.dropout (tests/golden/dropout.npz): the loss to rtol 2e-5 and
    every post-encoder gradient to the norm / sampled-entry criteria of test_forward_train_gradients_match_reference_
    backward."""
    from conftest import load_golden
    from test_gpu_backward import _check_grads
    fx = load_golden('dropout')
    seed, step, pair_base = (int(v) for v in fx[f'{case}|key'])
    assert float(fx[f'{case}|p']) == P
    _, m1, src, tgt = _models(case)
    batch = _batch(case, src, tgt)
    losses = m1.compute_loss(m1.forward_train(batch, dropout_key=(seed, step, pair_base)), batch)
    for k, v in losses.items():
        np.testing.assert_allclose(float(v.detach()), float(fx[f'{case}|loss_{k}']), rtol=2e-5, atol=1e-7, err_msg=k)
    losses['total'].backward()
    params = dict(m1.named_parameters())
    names = [k.split('|', 2)[2] for k in fx if k.startswith(f'{case}|g|') and '|g|kpf_encoder.' not in k]
    assert len(names) == sum(1 for n, p in params.items() if not n.startswith('kpf_encoder.'))
    worst = dict(norm=0.0, entry=0.0)
    _check_grads({n: params[n].grad for n in names}, {n: fx[f'{case}|g|{n}'] for n in names}, worst)
    print(case, 'worst vs reference with dropout:', worst)


# -------------------------------------------------------------------------------------------------- trainer

def test_trainer_resume_is_exact_with_dropout(tmp_path):
    """dropout 0.1: 6 steps equal 3 steps + save + resume + 3 steps bit for bit (masks keyed by the trainer's seed
    and step), as test_exact_resume_and_checkpoints at dropout 0; the trainer passes (seed, step, 0)."""
    import os
    from regtr_b200 import trainer as T
    from regtr_b200.config import get_config
    from test_gpu_trainer import datasets, make_model, make_opt, state_equal, write_synthetic
    data = write_synthetic(tmp_path / 'data', n_train=7, n_val=2)
    keys = []

    def run(name, niter, resume=None, spy=False):
        cfg = get_config('3dmatch', train_batch_size=2, val_batch_size=2, dropout=P)
        train_set, val_set = datasets(data)
        trainer = T.Trainer(make_opt(tmp_path / name, validate_every=3, resume=resume), niter=niter,
                            grad_clip=cfg.grad_clip, seed=5)
        model = make_model(cfg, seed=12)
        if spy:
            real = model.forward_train

            def forward_train(batch, train_encoder=False, **kw):
                keys.append(kw.get('dropout_key'))
                return real(batch, train_encoder=train_encoder, **kw)
            model.forward_train = forward_train
        trainer.fit(model, train_set, val_set)
        return str(tmp_path / name / 'ckpt')
    ck_a = run('a', 6, spy=True)
    ck_b = run('b', 3)
    ck_c = run('c', 3, resume=os.path.join(ck_b, 'model-3.pth'))
    assert keys == [(5, s, 0) for s in range(1, 7)]
    a = torch.load(os.path.join(ck_a, 'model-6.pth'))
    c = torch.load(os.path.join(ck_c, 'model-6.pth'))
    assert a['step'] == c['step'] == 6
    for k in ('state_dict', 'optimizer', 'scheduler', 'trainer'):
        assert state_equal(a[k], c[k]), k
    # the dropout run differs from a dropout-free one
    from test_gpu_trainer import _run
    _, ck_z = _run(tmp_path, 'z', data, niter=6)
    z = torch.load(os.path.join(ck_z, 'model-6.pth'))
    assert not state_equal(a['state_dict'], z['state_dict'])
