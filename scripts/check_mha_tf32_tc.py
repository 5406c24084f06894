"""wgmma 3xTF32 attention block vs float64 and vs the mma.sync core (error + time)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from regtr_b200 import ops
from regtr_b200.transformer import AttentionPlan
DEV = 'cuda:0'
torch.manual_seed(0)
E, H = 256, 8
for lens in ([410, 339], [130, 7, 300, 129], [64, 64], [410, 380, 395, 402, 350, 339, 360, 345] * 2):
    n = sum(lens)
    x = torch.randn(n, E, device=DEV) * 0.8
    W = torch.randn(3 * E, E, device=DEV) / E ** 0.5 * 1.5
    b = torch.randn(3 * E, device=DEV) * 0.1
    plan = AttentionPlan(lens, DEV)
    qkv = ops.linear(x, W, b)
    qkv64 = x.double() @ W.double().t() + b.double()
    for name, ks, kl in (('self', plan.q_start, plan.q_len), ('cross', plan.xk_start, plan.xk_len)):
        want = ops.mha_varlen(qkv[:, :E].contiguous(), qkv[:, E:2 * E].contiguous(), qkv[:, 2 * E:].contiguous(), plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
        got = ops.mha_tf32_tc(x, W, b, plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
        torch.cuda.synchronize()
        # float64 reference
        st = np.concatenate([[0], np.cumsum(lens)]); B = len(lens) // 2
        ref = torch.zeros(n, E, dtype=torch.float64, device=DEV)
        ksl, kll = ks.tolist(), kl.tolist()
        for c in range(len(lens)):
            q = qkv64[st[c]:st[c + 1], :E].reshape(-1, H, 32).transpose(0, 1)
            k = qkv64[ksl[c]:ksl[c] + kll[c], E:2 * E].reshape(-1, H, 32).transpose(0, 1)
            v = qkv64[ksl[c]:ksl[c] + kll[c], 2 * E:].reshape(-1, H, 32).transpose(0, 1)
            w = torch.softmax(q @ k.transpose(1, 2) / 32 ** 0.5, -1)
            ref[st[c]:st[c + 1]] = (w @ v).transpose(0, 1).reshape(-1, E)
        e_tc = float((got.double() - ref).abs().max()); e_mma = float((want.double() - ref).abs().max())
        print(f'lens {lens[:4]}.. n={n} {name}: wgmma err {e_tc:.2e}  mma.sync err {e_mma:.2e}  finite {bool(torch.isfinite(got).all())}')
    # timing (graph-free, back to back; includes the in-projection for the wgmma path)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for _ in range(3):
        ops.mha_tf32_tc(x, W, b, plan.q_start, plan.q_len, plan.xk_start, plan.xk_len, plan.max_len, H)
    e[0].record()
    for _ in range(20):
        ops.mha_tf32_tc(x, W, b, plan.q_start, plan.q_len, plan.xk_start, plan.xk_len, plan.max_len, H)
    e[1].record()
    for _ in range(20):
        qkv = ops.linear(x, W, b)
        ops.mha_varlen(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], plan.q_start, plan.q_len, plan.xk_start, plan.xk_len, plan.max_len, H)
    e[2].record(); torch.cuda.synchronize()
    print(f'   block time (in-proj + core): wgmma {e[0].elapsed_time(e[1]) / 20 * 1e3:.1f} us, mma.sync {e[1].elapsed_time(e[2]) / 20 * 1e3:.1f} us')
