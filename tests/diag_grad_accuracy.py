"""How far are the encoder gradients from float64?  (diagnostic, not collected by pytest)

    python tests/diag_grad_accuracy.py [case]

Runs forward_train(train_encoder=True) -> compute_loss -> backward() of one golden case on the GPU, and the CPU
oracle's autograd in fp32 and in float64 on the same inputs.  Prints, per encoder parameter, the error of the GPU
gradient and of the fp32 oracle's gradient against float64, with the criteria of tests/test_oracle_grad.py: norm
(relative) and the largest of the 32 sampled entries (relative to the rms entry), plus the largest entry over the
whole tensor.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, HERE); sys.path.insert(0, os.path.join(HERE, 'golden'))
import eval_inputs as ei                                         # noqa: E402
from conftest import FORWARD_CASES, make_case                    # noqa: E402
from oracle import regtr_oracle as O                             # noqa: E402
from regtr_b200 import losses as LS                              # noqa: E402
from regtr_b200.regtr import RegTR                               # noqa: E402
from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair  # noqa: E402

case = sys.argv[1] if len(sys.argv) > 1 else 'fwd_3dmatch_small_b2'
cfg, sd0, src, tgt = make_case(case)
sd = ei.loss_state_dict(sd0)
pairs = [(make_modelnet_pair if k == 'modelnet' else make_3dmatch_pair)(*a) for k, a in FORWARD_CASES[case][2]]
li = ei.loss_inputs(pairs, [len(s) for s in src], [len(t) for t in tgt])


def oracle_grads(dtype):
    leaves = {k: (v.clone().to(dtype).requires_grad_(not k.endswith('kernel_points')) if v.is_floating_point() else v)
              for k, v in sd.items()}
    pred = O.forward(leaves, cfg, src, tgt, dtype=dtype)
    meta = pred['kpconv_meta']
    b = {'kpconv_meta': {k: [torch.as_tensor(np.asarray(v)) for v in meta[k]] for k in ('points', 'pools', 'stack_lengths')}}
    b.update({k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in li.items()})
    m = types.SimpleNamespace(cfg=cfg, feature_criterion=types.SimpleNamespace(W=leaves['feature_criterion.W']),
                              feature_criterion_un=types.SimpleNamespace(W=leaves['feature_criterion_un.W']))
    LS.compute_loss(m, pred, b)['total'].backward()
    return {k: v.grad.double().reshape(-1) for k, v in leaves.items() if torch.is_tensor(v) and v.grad is not None}


dev = 'cuda:0'
model = RegTR(cfg).to(dev)
model.load_state_dict(sd, strict=True)
batch = {'src_xyz': [torch.from_numpy(s).to(dev) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(dev) for t in tgt],
         'pose': li['pose'].to(dev), 'src_overlap': [m.to(dev) for m in li['src_overlap']],
         'tgt_overlap': [m.to(dev) for m in li['tgt_overlap']]}
model.compute_loss(model.forward_train(batch, train_encoder=True), batch)['total'].backward()
gpu = {n: p.grad.detach().double().reshape(-1).cpu() for n, p in model.named_parameters() if p.grad is not None}
o32, o64 = oracle_grads(torch.float32), oracle_grads(torch.float64)


def errs(g, w, name):
    idx = torch.from_numpy(ei.grad_sample_index(name, w.numel()))
    rms = max(float(w.norm()) / np.sqrt(w.numel()), 1e-30)
    return (abs(float(g.norm()) - float(w.norm())) / float(w.norm()), float((g[idx] - w[idx]).abs().max()) / rms,
            float((g - w).abs().max()) / rms)


print(f'{case}: encoder parameters, errors against the float64 oracle (norm rel | sampled entry / rms | max entry / rms)')
print(f'{"parameter":55s} {"GPU":>28s}   {"fp32 oracle":>28s}   GPU vs fp32 oracle (sampled)')
for n in gpu:
    if not n.startswith('kpf_encoder.'):
        continue
    a, b = errs(gpu[n], o64[n], n), errs(o32[n], o64[n], n)
    c = errs(gpu[n], o32[n], n)[1]
    print(f'{n[len("kpf_encoder.encoder_blocks."):]:55s} {a[0]:8.1e} {a[1]:8.1e} {a[2]:8.1e}   {b[0]:8.1e} {b[1]:8.1e} {b[2]:8.1e}   {c:8.1e}')
