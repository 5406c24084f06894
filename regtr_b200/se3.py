"""Rigid-transform solve on the H100 kernel.

`compute_rigid_transform(a, b, weights)` keeps the reference signature and semantics
(/root/reference/src/utils/se3_torch.py:108-154): `a`, `b` ([*,] N, 3), `weights` ([*,] N)
-> ([*,] 3, 4) with T*a = b.  One warp per problem, fp64 accumulation, Jacobi 3x3 SVD
(regtr_b200/csrc/kabsch.cu).  The reference's `assert weights.min() >= 0 and
weights.max() <= 1` forces a device->host sync; it is only evaluated when
`check_weights=True`.
"""
from __future__ import annotations

import torch

from . import ops


def compute_rigid_transform(a: torch.Tensor, b: torch.Tensor, weights: torch.Tensor = None,
                            check_weights: bool = False):
    assert a.shape == b.shape
    assert a.shape[-1] == 3
    lead = a.shape[:-2]
    n = a.shape[-2]
    if weights is None:
        weights = torch.ones(a.shape[:-1], dtype=torch.float32, device=a.device)
    else:
        assert a.shape[:-1] == weights.shape
        if check_weights:
            assert weights.min() >= 0 and weights.max() <= 1
    n_prob = 1
    for d in lead:
        n_prob *= int(d)
    offs = torch.arange(0, (n_prob + 1) * n, n, dtype=torch.int32, device=a.device)
    T = ops.kabsch(a.reshape(-1, 3).to(torch.float32).contiguous(), b.reshape(-1, 3).to(torch.float32).contiguous(),
                   weights.reshape(-1).to(torch.float32).contiguous(), offs)
    return T.reshape(*lead, 3, 4)


def se3_transform(pose, xyz):
    """Rx + t (se3_torch.py:52-69); plain torch, not on the hot path."""
    rot, trans = pose[..., :3, :3], pose[..., :3, 3:4]
    return torch.einsum('...ij,...bj->...bi', rot, xyz) + trans.transpose(-1, -2)
