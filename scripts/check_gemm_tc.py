# Accuracy of the 3xTF32 wgmma GEMM against float64 at the model's shapes, then per-shape timings.
#   --save DIR      write every accuracy-case output to DIR/<M>x<N>x<K>.npy
#   --compare DIR   check that every output is bit-identical to the one saved in DIR (e.g. by an older build)
import argparse, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from regtr_b200 import ops
ap = argparse.ArgumentParser()
ap.add_argument('--save', metavar='DIR')
ap.add_argument('--compare', metavar='DIR')
args = ap.parse_args()
if args.save:
    os.makedirs(args.save, exist_ok=True)
# H100 SXM data sheet: dense TF32 tensor rate and HBM3 bandwidth (a power-limited card reaches less)
PEAK_TF32, PEAK_HBM = 495e12, 3.35e12
torch.manual_seed(0)
dev = 'cuda:0'
ok = True
for (M, N, K, bias, res, relu) in [(300, 64, 64, False, False, False), (128, 128, 32, True, False, False),
                                   (1000, 32, 480, False, False, False), (38061, 128, 64, False, False, False),
                                   (749, 256, 3840, False, False, False), (700, 768, 256, True, False, False),
                                   (700, 256, 1024, True, True, False), (700, 1024, 256, True, False, True),
                                   (650, 3, 256, True, False, False), (9977, 64, 960, False, False, False)]:
    a = torch.randn(M, K, device=dev) * 1.7
    w = torch.randn(N, K, device=dev) / K ** 0.5
    b = torch.randn(N, device=dev) if bias else None
    r = torch.randn(M, N, device=dev) if res else None
    want = a.double() @ w.double().t()
    if bias: want = want + b.double()
    if res: want = want + r.double()
    if relu: want = want.relu()
    got = ops.linear(a, w, b, residual=r, relu=relu)
    torch.cuda.synchronize()
    err = float((got.double() - want).abs().max()); scale = float(want.abs().max())
    ref32 = a @ w.t()
    if bias: ref32 = ref32 + b
    if res: ref32 = ref32 + r
    if relu: ref32 = ref32.relu()
    err32 = float((ref32.double() - want).abs().max())
    good = err <= 2e-6 * scale * max(1.0, (K / 64) ** 0.5)
    name = f'{M}x{N}x{K}.npy'
    if args.save:
        np.save(os.path.join(args.save, name), got.cpu().numpy())
    if args.compare:
        same = np.array_equal(np.load(os.path.join(args.compare, name)).view(np.uint32), got.cpu().numpy().view(np.uint32))
        print(f'  {name}: {"bit-identical" if same else "DIFFERS"} to {args.compare}')
        good &= same
    ok &= good
    print(f'M={M:6d} N={N:5d} K={K:5d} err {err:.3e} (cublas fp32 err {err32:.3e}) scale {scale:.2f} {"OK" if good else "FAIL"}')
# device-side row count
a = torch.randn(512, 64, device=dev); w = torch.randn(96, 64, device=dev)
md = torch.tensor([300], dtype=torch.int32, device=dev)
out = torch.full((512, 96), 7.0, device=dev)
hi, lo = ops.split_weight(w)
ops.gemm(a, hi, lo, m_dev=md, out=out)
torch.cuda.synchronize()
e = float((out[:300].double() - (a[:300].double() @ w.double().t())).abs().max())
print('m_dev: err', e, 'untouched rows', bool((out[300:] == 7.0).all()))
ok &= e < 1e-4 and bool((out[300:] == 7.0).all())
# timing
import time
for (M, N, K) in [(38061, 128, 64), (38061, 32, 64), (38061, 32, 480), (38061, 128, 32), (9977, 64, 960), (9977, 256, 64),
                  (2741, 128, 1920), (749, 256, 3840), (750, 768, 256), (750, 256, 1024), (6000, 768, 256), (6000, 1024, 256),
                  (6000, 256, 1024), (304000, 32, 480), (80000, 64, 960)]:
    a = torch.randn(M, K, device=dev); w = torch.randn(N, K, device=dev)
    hi, lo = ops.split_weight(w)
    for _ in range(3): ops.gemm(a, hi, lo); (a @ w.t())
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    for _ in range(20): ops.gemm(a, hi, lo)
    e1.record()
    for _ in range(20): a @ w.t()
    e2.record(); torch.cuda.synchronize()
    fl = 2 * M * N * K
    t = e0.elapsed_time(e1) / 20 * 1e-3
    nbytes = 4 * (M * K + 2 * N * K + M * N)           # algorithmic: A, B_hi, B_lo read once, C written once
    bound = 'tensor' if 3 * fl / PEAK_TF32 >= nbytes / PEAK_HBM else 'hbm'
    print(f'M={M} N={N} K={K}: tc3x {t*1e6:.1f} us ({fl/t/1e12:.1f} TF/s fp32-equiv, {3*fl/t/1e12:.1f} TF/s 3xTF32 MMA, '
          f'{nbytes/t/1e9:.0f} GB/s algorithmic, {bound}-bound)  cublas fp32 {e1.elapsed_time(e2)/20*1e3:.1f} us')
print('ALL OK' if ok else 'SOME FAILED')
