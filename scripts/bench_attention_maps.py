"""Cost of recording the cross-encoder's attention maps (`transformer_encoder.record_attentions`, get_attentions()).

    python scripts/bench_attention_maps.py [--steps 20] [--blocks 3] [--warmup 3]

At 1 and 8 pairs (the 3DMatch config, random weights, synthetic 3DMatch-shaped pairs of ~20k points per cloud):
  * forward_ms_off / forward_ms_on: eager `RegTR.forward` with recording off and on.  Each block times --steps
    forwards between two CUDA events after --warmup untimed ones; median and range over --blocks blocks, off and on
    alternating block by block;
  * map kernel: every `regtr_mha_probs_avg` launch of one recorded forward (2 per layer), re-launched alone --steps
    times per block between CUDA events (median over blocks), its total per forward;
  * bytes written by the map kernel (4 bytes per (query, key) entry of every problem) and the rate that makes;
  * the kernel's share of its bound, computed from shapes below: tensor-core work 2 sweeps x 3 TF32 MMAs (3xTF32)
    x 2 E FLOP per (query, key) entry against the data sheet's 495 TFLOP/s dense TF32, and the bytes written against
    3.35 TB/s of HBM3; the larger of the two times is the bound.  Data-sheet figures are for a 700 W H100 SXM.
The card's name and power limit are read in the same run.  One JSON line per batch size; writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench_train import WEIGHT_SEED, card  # noqa: E402
from regtr_b200 import ops  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.regtr import RegTR  # noqa: E402
from regtr_b200.synthetic import make_batch  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

TF32_PEAK, HBM_PEAK = 495e12, 3.35e12      # H100 SXM data sheet (dense TF32 tensor FLOP/s, HBM3 bytes/s), 700 W


def kernel_work(pairs_qk: int, E: int):
    """(tensor-core FLOP, bytes written) of one regtr_mha_probs_avg launch over pairs_qk (query, key) entries."""
    return 2 * 3 * 2 * E * pairs_qk, 4 * pairs_qk


def timed(fn, steps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        fn()
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--blocks', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_attention_maps.py needs a CUDA device (no CPU fallback)'
    dev = torch.device('cuda:0')
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(dev).eval()
    model.load_state_dict(random_state_dict(cfg, WEIGHT_SEED), strict=True)
    xenc = model.transformer_encoder
    name, power = card()
    stat = lambda v: dict(median=statistics.median(v), min=min(v), max=max(v))
    for B in (1, 8):
        b = make_batch(3, B)
        batch = {'src_xyz': [torch.from_numpy(s).to(dev) for s in b['src_xyz']],
                 'tgt_xyz': [torch.from_numpy(t).to(dev) for t in b['tgt_xyz']]}
        fwd = lambda: model(dict(batch))
        for on in (False, True):
            xenc.record_attentions = on
            for _ in range(args.warmup):
                fwd()
        times = {False: [], True: []}
        for _ in range(args.blocks):
            for on in (False, True):
                xenc.record_attentions = on
                times[on].append(timed(fwd, args.steps))
        # the map kernel alone: its launches of one recorded forward, re-timed
        xenc.record_attentions = True
        ops.TRACE = []
        fwd()
        trace = [t for t in ops.TRACE if t[0] == 'mha_probs']
        ops.TRACE = None
        torch.cuda.synchronize()
        relaunch = lambda: [t[2]() for t in trace]
        relaunch()
        k_ms = [timed(relaunch, args.steps) for _ in range(args.blocks)]
        xenc.record_attentions = False
        flop = sum(kernel_work(t[1]['pairs_qk'], t[1]['E'])[0] for t in trace)
        nbytes = sum(kernel_work(t[1]['pairs_qk'], t[1]['E'])[1] for t in trace)
        k_s = statistics.median(k_ms) * 1e-3
        t_flop, t_byte = flop / TF32_PEAK, nbytes / HBM_PEAK
        bound = 'tensor (TF32)' if t_flop >= t_byte else 'HBM write'
        tokens = sum(t[1]['tokens'] for t in trace) // max(len(trace), 1)
        print(json.dumps(dict(
            pairs=B, coarse_tokens=tokens, launches_per_forward=len(trace),
            forward_ms_off=stat(times[False]), forward_ms_on=stat(times[True]),
            map_kernel_ms_per_forward=stat(k_ms), map_bytes_per_forward=nbytes,
            map_write_GBps=nbytes / k_s / 1e9, map_tensor_TFLOPs=flop / k_s / 1e12,
            bound=bound, share_of_bound=max(t_flop, t_byte) / k_s,
            gpu=name, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
