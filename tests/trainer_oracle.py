"""Float64 restatement of the training loop's bookkeeping, the yardstick of ops.meter_update / ops.pose_errors:
AverageMeter.update (utils/misc.py), the loss_smooth EMA of trainer.py:127-134, and se3_compare (fp64)."""
import math

import numpy as np


class Meter:
    """AverageMeter.update with Python floats: NaN skipped, +-inf accumulated."""

    def __init__(self):
        self.val, self.sum, self.sq_sum, self.count = 0, 0.0, 0.0, 0

    def update(self, v: float):
        if math.isnan(v):
            return
        self.val = v
        self.sum += v * 1
        self.count += 1
        self.sq_sum += v ** 2 * 1

    def row(self):
        return [float(self.val) if self.count else 0.0, self.sum, self.sq_sum, float(self.count)]


class Smooth:
    """loss_smooth: the first value as it is, then skip non-finite values (their steps are logged), else the EMA."""

    def __init__(self):
        self.value, self.skipped = None, []

    def update(self, v: float, step: int):
        if self.value is None:
            self.value = v
        elif not math.isfinite(v):
            self.skipped.append(step)
        else:
            self.value = 0.99 * self.value + 0.01 * v


def pose_errors(pred: np.ndarray, gt: np.ndarray):
    """pred (L,B,3,4), gt (B,3,4) -> rot_deg (L,B), trans (L,B) in float64.  Every sum is written out left to right
    with elementwise numpy operations (no BLAS, no FMA), so that the cosine is the same double as the kernel's: near
    0 and 180 degrees acos turns a last-bit difference of the cosine into ~1e-6 degrees."""
    P, G = np.asarray(pred, np.float64), np.asarray(gt, np.float64)[None]
    R = [[(P[..., i, 0] * G[..., j, 0] + P[..., i, 1] * G[..., j, 1]) + P[..., i, 2] * G[..., j, 2]
          for j in range(3)] for i in range(3)]
    tr = (R[0][0] + R[1][1]) + R[2][2]
    rot = np.arccos(np.clip(0.5 * (tr - 1.0), -1.0, 1.0)) * (180.0 / np.pi)
    n2 = 0.0
    for i in range(3):
        d = P[..., i, 3] - ((R[i][0] * G[..., 0, 3] + R[i][1] * G[..., 1, 3]) + R[i][2] * G[..., 2, 3])
        n2 = n2 + d * d
    return rot, np.sqrt(n2)
