"""The KPConv-encoder backward's checks are sharp: on the model of the kernels' arithmetic (tests/kpconv_bwd_oracle.py)
the shipped design meets the fp32 yardstick on every output-gradient family, and every emulated wrong kernel fails the
yardstick row, the max-pool criterion or the bit-exactness assertion that targets it.  The model's own KPConv and
max-pool shapes lie inside the domain tests/test_gpu_kpconv_backward_domain.py runs.  CPU only."""
import numpy as np
import pytest
import torch

import kpconv_bwd_oracle as kb
from grad_yardstick import Yardstick
from test_gpu_forward_ops import _kp_inputs

NQ, COUT = 65, 32                  # query 64, the last, has shadow slots next to support Ns - 1


def _case(cin, K, family, c=None):
    c = _kp_inputs(cin, K, NQ) if c is None else c
    nq = len(c['q'])
    rng = np.random.default_rng(cin * 7 + K)
    W = (rng.standard_normal((15, cin, COUT)) / np.sqrt(15 * cin)).astype(np.float32)
    g = kb.gout_family(family, nq, COUT, cin + K)
    dwf = (g.astype(np.float64) @ W.reshape(15 * cin, COUT).astype(np.float64).T).astype(np.float32)
    flags = (c['x'].astype(np.float64).sum(1) > 0).astype(np.uint8)
    (dx64, _), = kb.kpconv_grads(c, W, [g], torch.float64, need_w=False)
    (dx32, _), = kb.kpconv_grads(c, W, [g], torch.float32, need_w=False)
    return c, dwf, flags, dx32, dx64


def _applies(variant, cin):
    nv = 1 if cin <= 32 else 2 if cin <= 64 else 4
    return variant != 'tail_dropped' or cin % (32 * nv) != 0


@pytest.mark.parametrize('cin,K', [(4, 40), (12, 72), (64, 40)])
@pytest.mark.parametrize('family', kb.FAMILIES)
def test_yardstick_separates_kpconv_dx_models(cin, K, family):
    c, dwf, flags, dx32, dx64 = _case(cin, K, family)
    assert (c['idx'][-1] == c['Ns']).any(), 'the last query needs shadow slots for shadow_to_last'
    ys = Yardstick(f'KPConv dx model, Cin={cin} K={K} Nq={NQ}, gout {family}')
    for v in kb.VARIANTS:
        ys.add(v, torch.from_numpy(kb.model_dx(c, dwf, flags, variant=v)), dx32, dx64)
    ys.add('shipped, count from x', torch.from_numpy(kb.model_dx(c, dwf, None)), dx32, dx64)
    ys.report()
    failed = set(ys.failures())
    want = {v for v in kb.VARIANTS if v not in ('shipped', 'fill_order') and _applies(v, cin)}
    assert not failed & {'shipped', 'shipped, count from x'}, ys.failures()
    assert want <= failed, sorted(want - failed)
    print('caught:', ', '.join(sorted(want)))


def test_fill_order_is_caught_by_bit_exactness():
    """Summing each support's rows in a scheduling-dependent order stays within the yardstick, so only the GPU file's
    bit-identity assertions (two passes; a cloud alone and stacked) catch it: two such orders give different bits."""
    c, dwf, flags, dx32, dx64 = _case(64, 16, 'zero_mean', kb.dense_case(200, 16, 50, 64, 3))
    assert np.bincount(c['idx'][c['idx'] < 50]).max() > 40
    base = kb.model_dx(c, dwf, flags)
    a = kb.model_dx(c, dwf, flags, 'fill_order', seed=1)
    b = kb.model_dx(c, dwf, flags, 'fill_order', seed=2)
    assert not np.array_equal(a, b) and not np.array_equal(a, base)
    assert np.array_equal(base, kb.model_dx(c, dwf, flags))
    ys = Yardstick('KPConv dx model, shared supports, Cin=64 K=16 Nq=200 Ns=50')
    for name, t in (('shipped', base), ('fill_order 1', a), ('fill_order 2', b)):
        ys.add(name, torch.from_numpy(t), dx32, dx64)
    ys.report()
    assert not ys.failures(), ys.failures()
    print('caught: fill_order (bits differ between two scheduling orders)')


@pytest.mark.parametrize('C,K', [(6, 40), (33, 255), (1, 1)])
def test_max_pool_criterion_separates_models(C, K):
    x, idx, g = kb.max_pool_case(C, K)
    want = kb.max_pool_dx(x, idx, g, torch.float64)
    rows = []
    for v in kb.MP_VARIANTS:
        rows.append((v, kb.max_pool_failures(torch.from_numpy(kb.model_max_pool_dx(x, idx, g, v)), want)))
    print(f'\nmax-pool dx model, C={C} K={K}: ' + '; '.join(f'{v}: {f or "ok"}' for v, f in rows))
    fails = dict(rows)
    assert not fails['shipped'], fails['shipped']
    expect = {'shadow_leak'} | ({'ties_last'} if K > 1 else set())
    assert all(fails[v] for v in expect), fails
    print('caught:', ', '.join(sorted(expect)))


def test_model_shapes_lie_inside_the_tested_domain():
    """Every (Cin, K) of a KPConv and (C, K) of a max-pool in RegTR(cfg).kpf_encoder, for the 3DMatch and ModelNet
    configs and the variant configs of the golden cases, is a case of the GPU file's grid."""
    from conftest import VARIANT_CASES
    from regtr_b200 import kpconv as kc
    from regtr_b200.config import get_config, pyramid_plan
    from regtr_b200.regtr import RegTR
    kp_cases = {(c, k) for c, k, _ in kb.kpconv_cases()}
    pool_cases = {(c, k) for c in kb.POOL_C for k in kb.POOL_K}
    seen_kp, seen_pool = set(), set()
    for name, over in [('3dmatch', {}), ('modelnet', {})] + [(v[0], v[3]) for v in VARIANT_CASES.values()]:
        cfg = get_config(name, **over)
        levels = pyramid_plan(cfg)[0]
        for b in RegTR(cfg).kpf_encoder.encoder_blocks:
            K = levels[b.layer_ind]['K']
            seen_kp.add((b.KPConv.in_channels, K))
            if isinstance(b, kc.ResnetBottleneckBlock) and 'strided' in b.block_name:
                seen_pool.add((b.in_dim, K))
    print('KPConv (Cin, K):', sorted(seen_kp), '\nmax-pool (C, K):', sorted(seen_pool))
    assert seen_kp and seen_pool
    assert seen_kp <= kp_cases, sorted(seen_kp - kp_cases)
    assert seen_pool <= pool_cases, sorted(seen_pool - pool_cases)
    assert max(kb.POOL_K) == 255 and max(kb.KPCONV_K) == 128 and max(kb.KPCONV_CIN) == 256


def test_kpconv_cases_cover_the_grid():
    cases = kb.kpconv_cases()
    pairs = {(c, k) for c, k, _ in cases}
    assert {(c, 40) for c in kb.KPCONV_CIN} <= pairs
    assert {(c, k) for c in kb.SWEEP_CIN for k in kb.KPCONV_K} <= pairs
    for c, k in kb.CORNERS:
        assert {m for cc, kk, m in cases if (cc, kk) == (c, k)} == set(kb.MODES)
    assert {m for _, _, m in cases} == set(kb.MODES)
