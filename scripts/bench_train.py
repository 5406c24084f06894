"""Time training steps of the fine-tuning path: RegTR.forward_train + compute_loss + backward() with the KPConv
encoder frozen (gradients of every parameter after the encoder), or with --train-encoder the full training step
(forward_train(batch, train_encoder=True): gradients of every parameter except the kernel points).

    python scripts/bench_train.py [--config 2|3] [--pairs B] [--steps K] [--warmup W] [--train-encoder]
                                  [--optimizer none|library|torch]

--optimizer none (default) times forward + loss + backward only.  library / torch add the rest of the reference's
training iteration to every step: clip_grad_norm_(cfg.grad_clip), AdamW.step() and StepLR.step() of
RegTR.configure_optimizers() (regtr_b200.optim: library kernels) or of torch (torch.optim.AdamW with its default
foreach path and torch.nn.utils.clip_grad_norm_).  The optimizer's time is reported from CUDA events of its own,
with the library kernel launches per step (ops.LAUNCHES).

Same workload as bench.py: seeded random weights, the synthetic 3DMatch-shaped pairs of the chosen BASELINE config
(config 2: 1 pair per step, config 3: 8), the attention_impl='fp32' core.  CUDA events around the forward + loss
and around the backward of every step; the 256 MB L2 flush between steps is not timed.  The loss targets are
synthetic (identity ground-truth pose, seeded level-0 overlap masks); the timing does not depend on their values.
Prints one JSON line with the card's name and power limit beside the numbers.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from regtr_b200 import ops  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.regtr import RegTR  # noqa: E402
from regtr_b200.synthetic import make_batch  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

WEIGHT_SEED = 2024
POOL = 8


def card():
    """(name, power limit) of cuda:0 -- a read-only nvidia-smi query."""
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', type=int, default=2, choices=[2, 3])
    ap.add_argument('--pairs', type=int, default=None, help='pairs per step (default: 1 for config 2, 8 for 3)')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--train-encoder', action='store_true', help='train the KPConv encoder too (full training step)')
    ap.add_argument('--optimizer', default='none', choices=['none', 'library', 'torch'],
                    help='add clip + AdamW + StepLR on the library kernels or torch\'s to every step')
    ap.add_argument('--dropout', type=float, default=0.0,
                    help='model.dropout: the six transformer dropouts in training mode (masks keyed by the step)')
    ap.add_argument('--kernel-times', action='store_true',
                    help='also report the GPU time per step of the attention forward and backward kernels '
                         '(torch.profiler over the timed steps)')
    args = ap.parse_args()
    if args.steps < 1:
        ap.error('--steps must be >= 1')
    assert torch.cuda.is_available(), 'bench_train.py needs a CUDA device (no CPU fallback)'
    dev = torch.device('cuda:0')
    B = args.pairs or {2: 1, 3: 8}[args.config]

    cfg = get_config('3dmatch', dropout=args.dropout) if args.dropout else get_config('3dmatch')
    model = RegTR(cfg).to(dev)
    model.load_state_dict(random_state_dict(cfg, WEIGHT_SEED), strict=True)
    if not args.train_encoder:
        model.kpf_encoder.requires_grad_(False)
    opt = sched = clip = None
    if args.optimizer == 'library':
        from regtr_b200 import optim
        opt, sched = model.configure_optimizers()
        clip = optim.clip_grad_norm_
    elif args.optimizer == 'torch':
        opt = torch.optim.AdamW(model.parameters(), lr=cfg.base_lr, weight_decay=cfg.weight_decay)
        sched = torch.optim.lr_scheduler.StepLR(opt, cfg.scheduler_param[0], cfg.scheduler_param[1])
        clip = torch.nn.utils.clip_grad_norm_
    opt_launches = []
    n_pool = max(POOL, B)
    b = make_batch(2, n_pool)
    pool = [(torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev)) for s, t in zip(b['src_xyz'], b['tgt_xyz'])]
    gen = torch.Generator().manual_seed(WEIGHT_SEED)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step(i, evs=None):
        ids = [(i * B + j) % n_pool for j in range(B)]
        batch = {'src_xyz': [pool[k][0] for k in ids], 'tgt_xyz': [pool[k][1] for k in ids],
                 'pose': torch.eye(3, 4, device=dev).expand(B, 3, 4).contiguous()}
        batch['src_overlap'] = [(torch.rand(len(s), generator=gen) < 0.5).to(dev) for s in batch['src_xyz']]
        batch['tgt_overlap'] = [(torch.rand(len(t), generator=gen) < 0.5).to(dev) for t in batch['tgt_xyz']]
        model.zero_grad(set_to_none=True)
        if evs:
            evs[0].record()
        pred = model.forward_train(batch, train_encoder=args.train_encoder, dropout_key=(WEIGHT_SEED, i, 0))
        total = model.compute_loss(pred, batch)['total']
        if evs:
            evs[1].record()
        total.backward()
        if evs:
            evs[2].record()
        if opt is not None:
            n0 = ops.LAUNCHES
            clip(model.parameters(), cfg.grad_clip)
            opt.step()
            sched.step()
            if evs:
                evs[3].record()
                opt_launches.append(ops.LAUNCHES - n0)

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    timed = []
    for i in range(args.steps):
        flush.zero_()
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(3 if opt is None else 4)]
        step(args.warmup + i, evs)
        timed.append(evs)
    torch.cuda.synchronize()
    prof = None
    if args.kernel_times:            # a separate pass after the timed steps: the step times above are untraced
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
        with prof:
            for i in range(args.steps):
                flush.zero_()
                step(args.warmup + args.steps + i)
            torch.cuda.synchronize()
        kt = {}
        for ev in prof.key_averages():
            for tag, pat in (('attention_fwd', 'k_mha_tf32x3'), ('attention_bwd_dq', 'k_mha_bwd_dq'),
                             ('attention_bwd_dkv', 'k_mha_bwd_dkv'), ('dropout_rows', 'k_dropout_rows')):
                if pat in ev.key:
                    kt[tag + '_ms_per_step'] = kt.get(tag + '_ms_per_step', 0.0) + \
                        getattr(ev, 'device_time_total', getattr(ev, 'cuda_time_total', 0.0)) / 1e3 / args.steps
    fwd = sum(e[0].elapsed_time(e[1]) for e in timed)
    bwd = sum(e[1].elapsed_time(e[2]) for e in timed)
    name, power = card()
    extra = {}
    if args.dropout:
        extra['dropout'] = args.dropout
    if prof is not None:
        extra.update(kt)
    if opt is not None:
        ost = sum(e[2].elapsed_time(e[3]) for e in timed)
        extra.update(optimizer=args.optimizer, optimizer_ms_per_step=ost / args.steps,
                     train_ms_per_step_with_optimizer=(fwd + bwd + ost) / args.steps,
                     optimizer_library_launches_per_step=sum(opt_launches[:args.steps]) / args.steps)
    print(json.dumps(dict(
        metric='training steps/s of forward_train + compute_loss + backward ' +
               ('(KPConv encoder trained)' if args.train_encoder else '(KPConv encoder frozen)'),
        train_encoder=args.train_encoder,
        workload=f'BASELINE config {args.config}: synthetic 3DMatch-like pairs, ~20k pts/cloud, {B} pair(s)/step',
        steps=args.steps, warmup=args.warmup, train_pairs_per_s=B * args.steps / ((fwd + bwd) * 1e-3),
        train_ms_per_step=(fwd + bwd) / args.steps, train_forward_ms_per_step=fwd / args.steps,
        train_backward_ms_per_step=bwd / args.steps, train_backward_share=bwd / (fwd + bwd),
        **extra, gpu=name, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
