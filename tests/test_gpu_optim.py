"""GPU tests of the library optimizer step (regtr_b200.optim): gradient-norm clipping and Adam / AdamW against torch's
and a float64 restatement, state_dict interop with torch's optimizers, the in-place refresh of the split-weight cache
(CUDA graphs captured before the steps stay valid), launch counts, no host sync, no foreign kernel, and a short
training run at model level."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import FORWARD_CASES, make_case

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
OPT_KERNELS = ('k_sumsq_chunks', 'k_norm_finalize', 'k_scale_chunks', 'k_adam_chunks', 'k_split_refresh')


def _model_grad_shapes():
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    return [tuple(p.shape) for p in RegTR(get_config('3dmatch')).parameters()]


# ------------------------------------------------------------------------------------------------------------ clip

@pytest.mark.parametrize('scale', [1e-4, 1.0, 1e3])
def test_clip_matches_torch_and_float64(scale):
    from regtr_b200 import optim
    gen = torch.Generator(device=DEV).manual_seed(7)
    shapes = [(0,), (1,), (3,), (4097,), (983040,)] + _model_grad_shapes()
    grads = [torch.randn(s, generator=gen, device=DEV) * scale for s in shapes]
    grads[5] = grads[5][1:].clone()                       # an unaligned element count among the model's shapes
    max_norm = 0.1 * len(shapes) ** 0.5
    ps = [torch.nn.Parameter(torch.zeros_like(g)) for g in grads]
    qs = [torch.nn.Parameter(torch.zeros_like(g)) for g in grads]
    for p, q, g in zip(ps, qs, grads):
        p.grad, q.grad = g.clone(), g.clone()
    want64 = float(torch.cat([g.double().reshape(-1) for g in grads]).norm())
    tot = optim.clip_grad_norm_(ps, max_norm)
    ref = torch.nn.utils.clip_grad_norm_(qs, max_norm)
    assert tot.dim() == 0 and tot.dtype == torch.float32 and tot.is_cuda
    assert abs(float(tot) - want64) <= 1e-6 * want64, (float(tot), want64)
    below = want64 < max_norm
    for p, q in zip(ps, qs):
        if below:
            assert torch.equal(p.grad, q.grad)            # coefficient 1: untouched bits
        else:
            d = (p.grad - q.grad).abs()
            assert bool((d <= 1e-6 * q.grad.abs()).all()), float(d.max())
    # two runs are bit-identical
    rs = [torch.nn.Parameter(torch.zeros_like(g)) for g in grads]
    for r, g in zip(rs, grads):
        r.grad = g.clone()
    tot2 = optim.clip_grad_norm_(rs, max_norm)
    assert torch.equal(tot, tot2) and all(torch.equal(p.grad, r.grad) for p, r in zip(ps, rs))
    print(f'scale {scale}: total {float(tot):.9g}  float64 {want64:.9g}  torch {float(ref):.9g}')


def test_clip_edge_cases():
    from regtr_b200 import optim
    assert float(optim.clip_grad_norm_([torch.nn.Parameter(torch.zeros(3, device=DEV))], 1.0)) == 0.0
    z = torch.nn.Parameter(torch.zeros(0, device=DEV))
    z.grad = torch.zeros(0, device=DEV)
    assert float(optim.clip_grad_norm_([z], 1.0)) == 0.0
    for bad in (float('inf'), float('nan'), 'both'):
        ps, qs = [], []
        for n in (5, 4097):
            g = torch.randn(n, device=DEV)
            if n == 4097:
                if bad == 'both':
                    g[3], g[9] = float('inf'), float('nan')
                else:
                    g[17] = bad
            for lst in (ps, qs):
                t = torch.nn.Parameter(torch.zeros(n, device=DEV))
                t.grad = g.clone()
                lst.append(t)
        a = optim.clip_grad_norm_(ps, 1.0)
        b = torch.nn.utils.clip_grad_norm_(qs, 1.0)
        assert torch.equal(a.isnan(), b.isnan()) and torch.equal(a.isinf(), b.isinf()), (bad, a, b)
        for p, q in zip(ps, qs):
            assert torch.equal(p.grad.isnan(), q.grad.isnan()) and torch.equal(p.grad.isinf(), q.grad.isinf()), bad
            fin = q.grad.isfinite()
            assert torch.equal(p.grad[fin], q.grad[fin]), bad


# ---------------------------------------------------------------------------------------------------------- update

def _adam64(p, grads, groups_of, hp, decoupled):
    """Float64 restatement of the update (torch's algorithm, no intermediate rounding)."""
    p = [x.double().cpu() for x in p]
    m = [torch.zeros_like(x) for x in p]
    v = [torch.zeros_like(x) for x in p]
    for t, gs in enumerate(grads, 1):
        for i, g in enumerate(gs):
            if g is None:
                continue
            lr, wd = hp[groups_of[i]]
            b1, b2, eps = 0.9, 0.999, 1e-8
            g = g.double().cpu()
            if decoupled:
                p[i] = p[i] * (1 - lr * wd)
            else:
                g = g + wd * p[i]
            m[i] = m[i] + (1 - b1) * (g - m[i])
            v[i] = b2 * v[i] + (1 - b2) * g * g
            denom = v[i].sqrt() / (1 - b2 ** t) ** 0.5 + eps
            p[i] = p[i] - lr / (1 - b1 ** t) * m[i] / denom
    return p, m, v


@pytest.mark.parametrize('decoupled', [True, False], ids=['AdamW', 'Adam'])
def test_update_matches_torch_and_float64(decoupled):
    from regtr_b200 import optim
    gen = torch.Generator(device=DEV).manual_seed(11)
    shapes = [(256, 256), (1000,), (33, 7), (4097,), (15, 32, 64), (5,)]
    groups_of = [0, 0, 1, 1, 0, 1]
    hp = [(1e-3, 1e-2), (3e-4, 0.1)]
    init = [torch.randn(s, generator=gen, device=DEV) for s in shapes]
    lib_p = [torch.nn.Parameter(x.clone()) for x in init]
    ref_p = [torch.nn.Parameter(x.clone()) for x in init]
    nograd = len(shapes) - 1                               # never gets a gradient

    def groups(ps):
        return [dict(params=[p for p, k in zip(ps, groups_of) if k == j], lr=hp[j][0], weight_decay=hp[j][1])
                for j in range(2)]
    LibC, RefC = (optim.AdamW, torch.optim.AdamW) if decoupled else (optim.Adam, torch.optim.Adam)
    lib = LibC(groups(lib_p))
    ref = RefC(groups(ref_p), foreach=False)
    v0 = lib_p[nograd]._version
    all_grads = []
    for _ in range(10):
        gs = [None if i == nograd else torch.randn(s, generator=gen, device=DEV) * 0.1 for i, s in enumerate(shapes)]
        all_grads.append(gs)
        for p, q, g in zip(lib_p, ref_p, gs):
            p.grad = None if g is None else g.clone()
            q.grad = None if g is None else g.clone()
        lib.step()
        ref.step()
    torch.cuda.synchronize()
    p64, m64, v64 = _adam64(init, all_grads, groups_of, hp, decoupled)
    same = total = 0
    for i, (p, q) in enumerate(zip(lib_p, ref_p)):
        if i == nograd:
            assert p not in lib.state and p._version == v0 and torch.equal(p.detach(), init[i])
            continue
        sl, sr = lib.state[p], ref.state[q]
        assert sl['step'].device.type == 'cpu' and sl['step'].dtype == torch.float32 and float(sl['step']) == 10.0
        for a, b, w in ((p.detach(), q.detach(), p64[i]), (sl['exp_avg'], sr['exp_avg'], m64[i]),
                        (sl['exp_avg_sq'], sr['exp_avg_sq'], v64[i])):
            scale = float(b.abs().max())
            assert float((a - b).abs().max()) <= 1e-6 * scale
            e_lib = float((a.double().cpu() - w).abs().max())
            e_ref = float((b.double().cpu() - w).abs().max())
            assert e_lib <= 2 * e_ref, (i, e_lib, e_ref)
            same += int((a == b).sum())
            total += a.numel()
    print(f'{"AdamW" if decoupled else "Adam"}: {same / total:.6f} of p / m / v entries bit-identical to torch')


def test_state_dict_interop_with_torch():
    from regtr_b200 import optim
    gen = torch.Generator(device=DEV).manual_seed(5)
    shapes = [(64, 32), (31,), (4097,)]
    init = [torch.randn(s, generator=gen, device=DEV) for s in shapes]
    grads = [[torch.randn(s, generator=gen, device=DEV) for s in shapes] for _ in range(6)]

    def make(cls, ps, **kw):
        return cls([dict(params=ps[:2], lr=1e-3, weight_decay=1e-2), dict(params=ps[2:], lr=5e-4, weight_decay=0.0)],
                   **kw)

    def steps(opt, ps, gs):
        for g in gs:
            for p, x in zip(ps, g):
                p.grad = x.clone()
            opt.step()

    for first, second, kw1, kw2 in ((optim.AdamW, torch.optim.AdamW, {}, dict(foreach=False)),
                                    (torch.optim.AdamW, optim.AdamW, dict(foreach=False), {})):
        a = [torch.nn.Parameter(x.clone()) for x in init]
        o1 = make(first, a, **kw1)
        steps(o1, a, grads[:3])
        o2 = make(second, a, **kw2)
        o2.load_state_dict(o1.state_dict())
        steps(o2, a, grads[3:])
        b = [torch.nn.Parameter(x.clone()) for x in init]
        o3 = make(first, b, **kw1)
        steps(o3, b, grads)
        for p, q in zip(a, b):
            for x, y in ((p.detach(), q.detach()), (o2.state[p]['exp_avg'], o3.state[q]['exp_avg']),
                         (o2.state[p]['exp_avg_sq'], o3.state[q]['exp_avg_sq'])):
                assert float((x - y).abs().max()) <= 1e-6 * float(y.abs().max())
            assert float(o2.state[p]['step']) == 6.0 and o2.state[p]['step'].device.type == 'cpu'
    # StepLR drives the library optimizer's lr exactly as torch's
    lrs = []
    for cls, kw in ((optim.AdamW, {}), (torch.optim.AdamW, dict(foreach=False))):
        ps = [torch.nn.Parameter(x.clone()) for x in init]
        opt = make(cls, ps, **kw)
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.5)
        seq = []
        for g in grads:
            for p, x in zip(ps, g):
                p.grad = x.clone()
            opt.step()
            sched.step()
            seq.append([grp['lr'] for grp in opt.param_groups])
        lrs.append(seq)
    assert lrs[0] == lrs[1] and lrs[0][-1] == [1e-3 * 0.125, 5e-4 * 0.125]


# --------------------------------------------------------------------------------------------- model-level helpers

def _model(case, base_lr=None):
    from regtr_b200.regtr import RegTR
    cfg, sd0, src, tgt = make_case(case)
    if base_lr is not None:
        cfg.base_lr = base_lr
    sd = ei.loss_state_dict(sd0)
    model = RegTR(cfg).to(DEV)
    model.load_state_dict(sd, strict=True)
    return cfg, sd, model, src, tgt


def _batch(case, src, tgt):
    from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair
    pairs = [(make_modelnet_pair if kind == 'modelnet' else make_3dmatch_pair)(*args)
             for kind, args in FORWARD_CASES[case][2]]
    b = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    li = ei.loss_inputs(pairs, [len(s) for s in src], [len(t) for t in tgt])
    b['pose'] = li['pose'].to(DEV)
    b['src_overlap'] = [m.to(DEV) for m in li['src_overlap']]
    b['tgt_overlap'] = [m.to(DEV) for m in li['tgt_overlap']]
    return b


def _fresh_split(p, key):
    from regtr_b200 import lib, ops
    off, shape, stride, transpose = key[:4]
    view = torch.as_strided(p.detach(), shape, stride, off)
    src = (view.t() if transpose else view).contiguous()
    hi, lo = torch.empty_like(src), torch.empty_like(src)
    L = lib.load()
    lib.check(L.regtr_split_tf32(src.data_ptr(), src.numel(), hi.data_ptr(), lo.data_ptr(), ops._stream()), 'split')
    return hi, lo


def _check_split_caches(model):
    n = 0
    for name, p in model.named_parameters():
        for key, (hi, lo) in p.__dict__.get('_regtr_split', {}).items():
            assert key[-1] == p._version, name
            fh, fl = _fresh_split(p, key)
            assert torch.equal(hi, fh) and torch.equal(lo, fl), (name, key)
            n += 1
    return n


class _SplitCounter:
    def __init__(self, L):
        self.fn, self.calls = L.regtr_split_tf32, 0

    def __call__(self, *a):
        self.calls += 1
        return self.fn(*a)


@pytest.mark.parametrize('case', ['fwd_3dmatch_small_b2', 'fwd_modelnet_b1'])
def test_steps_refresh_split_caches_and_keep_graphs_valid(case, monkeypatch):
    from regtr_b200 import lib, optim
    from regtr_b200.regtr import GraphedRegTR, RegTR
    cfg, sd, model, src, tgt = _model(case)
    opt, sched = model.configure_optimizers()
    runner = GraphedRegTR(model, bucket=8192)
    plain = lambda: {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    runner(plain())                                        # captured before any step
    counter = _SplitCounter(lib.load())
    monkeypatch.setattr(lib.load(), 'regtr_split_tf32', counter)
    for step in range(3):
        batch = _batch(case, src, tgt)
        opt.zero_grad(set_to_none=True)
        calls = counter.calls
        model.compute_loss(model.forward_train(batch, train_encoder=True), batch)['total'].backward()
        if step > 0:                                       # every split the step needs was refreshed in place
            assert counter.calls == calls, (step, counter.calls - calls)
        optim.clip_grad_norm_(model.parameters(), cfg.grad_clip)
        opt.step()
        sched.step()
        n = _check_split_caches(model)
        assert n > 0
    got = runner(plain())                                  # no invalidate()
    fresh = RegTR(cfg).to(DEV)
    fresh.load_state_dict(model.state_dict(), strict=True)
    want = GraphedRegTR(fresh, bucket=8192)(plain())
    eager = model(plain())
    for k in ('src_feat_un', 'src_feat', 'tgt_overlap', 'src_kp_warped', 'tgt_kp_warped'):
        for b in range(len(src)):
            assert torch.equal(got[k][b], want[k][b]), k
            s = float(eager[k][b].abs().max())
            assert float((got[k][b] - eager[k][b]).abs().max()) <= 2e-5 * max(s, 1.0), k
    assert torch.equal(got['pose'], want['pose'])
    assert float((got['pose'] - eager['pose']).abs().max()) <= 5e-5
    assert torch.equal(eager['pose'], fresh(plain())['pose'])
    print(f'{case}: {n} split-cache entries refreshed per step, bit-equal to fresh splits')


def test_step_is_sync_free_and_launches_library_kernels_only():
    from torch.profiler import ProfilerActivity, profile
    from regtr_b200 import ops, optim
    case = 'fwd_modelnet_b1'
    cfg, sd, model, src, tgt = _model(case)
    opt, sched = model.configure_optimizers()
    for step in range(2):
        batch = _batch(case, src, tgt)
        opt.zero_grad(set_to_none=True)
        model.compute_loss(model.forward_train(batch, train_encoder=True), batch)['total'].backward()
        torch.cuda.synchronize()
        if step == 0:
            n0 = ops.LAUNCHES
            torch.cuda.set_sync_debug_mode('error')
            try:
                optim.clip_grad_norm_(model.parameters(), cfg.grad_clip)
                n1 = ops.LAUNCHES
                opt.step()
                sched.step()
            finally:
                torch.cuda.set_sync_debug_mode('default')
            assert n1 - n0 <= 3 and ops.LAUNCHES - n1 <= 2, (n1 - n0, ops.LAUNCHES - n1)
        else:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                optim.clip_grad_norm_(model.parameters(), cfg.grad_clip)
                opt.step()
                sched.step()
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            kernels = [nm for nm in names if 'memcpy' not in nm.lower()]
            assert kernels and all(any(k in nm for k in OPT_KERNELS) for nm in kernels), sorted(set(kernels))
            print('CUDA activity of clip + step + scheduler:', sorted(set(names)))


def _train(case, n=5, base_lr=1e-3):
    """n iterations of the library solver and, from the same start, of torch's.  Every iteration's backward runs on the
    library model, and its raw gradients are also handed to the torch model, so the two optimizers step on the same
    gradients and the arms differ by their arithmetic alone.  (Each arm running its own backward made the comparison
    a test of how this unstable 5-step run amplifies rounding: the arms' losses drifted apart about 10x per step.)
    -> per arm: losses (each from that arm's own forward), clip norms, final state dict."""
    from regtr_b200 import optim
    cfg, sd, model, src, tgt = _model(case, base_lr=base_lr)
    _, _, model_t, _, _ = _model(case, base_lr=base_lr)
    opt, sched = model.configure_optimizers()
    opt_t = torch.optim.AdamW(model_t.parameters(), lr=cfg.base_lr, weight_decay=cfg.weight_decay, foreach=False)
    sched_t = torch.optim.lr_scheduler.StepLR(opt_t, cfg.scheduler_param[0], cfg.scheduler_param[1])
    losses, norms, losses_t, norms_t = [], [], [], []
    for _ in range(n):
        batch, batch_t = _batch(case, src, tgt), _batch(case, src, tgt)
        opt.zero_grad(set_to_none=True)
        opt_t.zero_grad(set_to_none=True)
        total = model.compute_loss(model.forward_train(batch, train_encoder=True), batch)['total']
        losses.append(total.detach().clone())
        total.backward()
        total_t = model_t.compute_loss(model_t.forward_train(batch_t, train_encoder=True), batch_t)['total']
        losses_t.append(total_t.detach().clone())
        del total_t                                         # the torch arm's own graph is not differentiated
        for p, pt in zip(model.parameters(), model_t.parameters()):
            pt.grad = None if p.grad is None else p.grad.clone()
        norms.append(optim.clip_grad_norm_(model.parameters(), cfg.grad_clip).detach().clone())
        norms_t.append(torch.nn.utils.clip_grad_norm_(model_t.parameters(), cfg.grad_clip).detach().clone())
        opt.step()
        sched.step()
        opt_t.step()
        sched_t.step()
    state = lambda m: {k: v.clone() for k, v in m.state_dict().items()}
    return ((torch.stack(losses).cpu(), torch.stack(norms).cpu(), state(model)),
            (torch.stack(losses_t).cpu(), torch.stack(norms_t).cpu(), state(model_t)))


def test_training_iterations_on_shared_gradients_match_torch_and_lower_the_loss():
    """5 iterations of the reference's solver (clip to grad_clip, AdamW, StepLR) on one batch, library vs torch from
    the same start and on the same gradients.  base_lr is raised from 1e-4 to 1e-3 so that 5 steps lower the loss
    clearly."""
    case = 'fwd_modelnet_b1'
    (l1, n1, s1), (l3, n3, _) = _train(case)
    (l2, n2, s2), _ = _train(case)
    assert torch.equal(l1, l2) and torch.equal(n1, n2) and all(torch.equal(s1[k], s2[k]) for k in s1)
    assert float(((l1 - l3).abs() / l3.abs()).max()) <= 1e-4, (l1, l3)
    assert float(((n1 - n3).abs() / n3.abs()).max()) <= 1e-4, (n1, n3)
    print('losses library', l1.tolist(), 'torch', l3.tolist(), 'grad norms', n1.tolist())
    assert l1[-1] < l1[0]
