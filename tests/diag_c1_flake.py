"""Flake hunt for the Cin = 1, Cout = 64 KPConv comparison (random points near the origin, K = 40): which side varies
on the first call of a process?  tests/test_gpu_forward_ops.py::test_kpconv_vs_float64 prints both sides' errors
against float64 on every path."""
import os, sys
import numpy as np, torch
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, HERE)
from oracle import regtr_oracle as O
from regtr_b200 import ops
DEV = 'cuda:0'
G = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if dt is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV).to(dt)
cin, cout = 1, 64
rng = np.random.default_rng(cin)
Nq, Ns, K = 301, 457, 40
q = rng.normal(size=(Nq, 3)).astype(np.float32) * 0.05
s = rng.normal(size=(Ns, 3)).astype(np.float32) * 0.05
idx = rng.integers(0, Ns + 1, size=(Nq, K))
idx[:, 30:] = np.where(rng.random((Nq, 10)) < 0.7, Ns, idx[:, 30:])
idx[7] = Ns
x = rng.normal(size=(Ns, cin)).astype(np.float32) + 1.0
W = (rng.normal(size=(15, cin, cout)) / np.sqrt(15 * cin)).astype(np.float32)
kp = (rng.normal(size=(15, 3)) * 0.03).astype(np.float32)
def oracle(dt=torch.float32):
    return O.kpconv(torch.from_numpy(q).to(dt), torch.from_numpy(s).to(dt), torch.from_numpy(idx), torch.from_numpy(x).to(dt),
                    torch.from_numpy(W).to(dt), torch.from_numpy(kp).to(dt), 0.05).numpy()
def gpu():
    return ops.kpconv(G(q), G(s), G(idx, torch.int32), G(x), G(W), G(kp), 0.05).cpu().numpy()
order = sys.argv[1] if len(sys.argv) > 1 else 'og'
res = {}
for ch in order:
    res.setdefault(ch, []).append(oracle() if ch == 'o' else gpu())
w64 = oracle(torch.float64)
sc = np.abs(w64).max()
for k, v in res.items():
    for i, a in enumerate(v):
        print(order, k, i, 'vs f64 %.2e' % (np.abs(a - w64).max() / sc), 'vs first %.2e' % (np.abs(a - v[0]).max() / sc))
