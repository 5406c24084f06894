"""The fp32 yardstick for gradient tests.

A CUDA gradient is compared with float64 autograd of the CPU oracle's math, and so is the same oracle evaluated in
fp32 on the same inputs and with the same branch decisions.  The fp32 oracle's error says how well fp32 can do on
that tensor; the CUDA kernel passes when its error is within FACTOR times that, plus FLOOR.  Both errors are measured
as max-abs over max|ref| and as relative Frobenius norm, and the rule holds for each measure.
"""
import torch

FACTOR, FLOOR = 10.0, 1e-6


def errors(got, ref):
    """(max|got - ref| / max|ref|, ||got - ref|| / ||ref||) against a float64 reference."""
    ref = ref.detach().double().cpu()
    if ref.numel() == 0:
        return 0.0, 0.0
    d = got.detach().double().cpu() - ref
    return (float(d.abs().max() / ref.abs().max().clamp_min(1e-300)),
            float(d.norm() / ref.norm().clamp_min(1e-300)))


class Yardstick:
    """Collects one row per compared tensor; `report()` prints the table, `failures()` names the rows over the bound."""

    def __init__(self, title):
        self.title, self.rows = title, []

    def add(self, name, gpu, fp32, ref):
        eg, ef = errors(gpu, ref), errors(fp32, ref)
        ok = all(a <= FACTOR * b + FLOOR for a, b in zip(eg, ef))
        self.rows.append((name, eg, ef, ok))
        return ok

    def add_abs(self, name, gpu, fp32, ref, scale):
        """A row for a tensor that is zero in exact arithmetic: both measures are taken against `scale` (max-abs /
        scale and rms / scale) instead of the reference's own size."""
        def err(t):
            d = t.detach().double().cpu() - ref.detach().double().cpu()
            return (float(d.abs().max()) / scale, float(d.norm()) / (scale * max(d.numel(), 1) ** 0.5)) \
                if d.numel() else (0.0, 0.0)
        eg, ef = err(gpu), err(fp32)
        ok = all(a <= FACTOR * b + FLOOR for a, b in zip(eg, ef))
        self.rows.append((name, eg, ef, ok))
        return ok

    def report(self):
        w = max([len(r[0]) for r in self.rows] + [6])
        print(f'\n{self.title}\n  errors against float64: max-abs / max|ref| and relative Frobenius norm; '
              f'pass: GPU <= {FACTOR:g} x fp32 oracle + {FLOOR:g}')
        print(f'  {"tensor":{w}s}  {"GPU max":>9s} {"GPU fro":>9s}   {"fp32 max":>9s} {"fp32 fro":>9s}')
        for name, eg, ef, ok in self.rows:
            print(f'  {name:{w}s}  {eg[0]:9.2e} {eg[1]:9.2e}   {ef[0]:9.2e} {ef[1]:9.2e}   {"ok" if ok else "FAIL"}')

    def failures(self):
        return [r[0] for r in self.rows if not r[3]]
