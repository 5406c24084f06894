"""pytest configuration: registers the `gpu` marker and shared helpers/fixtures."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: test needs a CUDA device (an H100)')


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + '.npz')))


@pytest.fixture(scope='session')
def ops_golden():
    return load_golden('ops')


# (fixture name) -> (config name, weight seed, [(maker, args)...]) ; mirrors tests/golden/make_golden.py
FORWARD_CASES = {
    'fwd_modelnet_b1': ('modelnet', 11, [('modelnet', (1000,))]),
    'fwd_3dmatch_small_b1': ('3dmatch', 12, [('3dmatch', (2000, 3000))]),
    'fwd_3dmatch_small_b2': ('3dmatch', 13, [('3dmatch', (2001, 2500)), ('3dmatch', (2002, 4000))]),
}
# alternative config branches (SURVEY.md 8f N4): (config, weight seed, makers, config overrides)
VARIANT_CASES = {
    'var_modelnet_attndec_b1': ('modelnet', 14, [('modelnet', (1001,))], dict(direct_regress_coor=False)),
    'var_modelnet_postnorm_b1': ('modelnet', 15, [('modelnet', (1002,))], dict(pre_norm=False)),
    'var_modelnet_learnedpe_attndec_b2': ('modelnet', 16, [('modelnet', (1003,)), ('modelnet', (1004,))],
                                          dict(pos_emb_type='learned', direct_regress_coor=False)),
}


def make_case(name):
    """Regenerate (cfg, state_dict, src_list, tgt_list) of a golden forward case from its seeds."""
    from regtr_b200.config import get_config
    from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair
    from regtr_b200.weights import random_state_dict
    cfg_name, wseed, makers, *rest = (FORWARD_CASES.get(name) or VARIANT_CASES[name])
    cfg = get_config(cfg_name, **(rest[0] if rest else {}))
    sd = random_state_dict(cfg, wseed)
    pairs = [(make_modelnet_pair if kind == 'modelnet' else make_3dmatch_pair)(*args)
             for kind, args in makers]
    return cfg, sd, [p['src_xyz'] for p in pairs], [p['tgt_xyz'] for p in pairs]


def check_forward_against_golden(out, meta, fx, n_pairs, feat_rtol, corr_atol, logit_atol, pose_atol,
                                 exact_points=True):
    """Shared comparison of a forward output dict (numpy-convertible) with a golden fixture."""
    def npy(t):
        return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)
    n_lvl = len(meta['points'])
    step = int(fx['row_step']) if 'row_step' in fx else 7
    for lvl in range(n_lvl):
        assert np.array_equal(npy(meta['stack_lengths'][lvl]), fx[f'stack_lengths_{lvl}']), f'stack_lengths[{lvl}]'
        if f'neighbors_{lvl}' not in fx:        # variant fixtures carry the float outputs only
            continue
        for key in ('neighbors', 'pools', 'upsamples'):
            got = npy(meta[key][lvl])
            want = fx[f'{key}_{lvl}']
            assert got.shape == want.shape, (key, lvl, got.shape, want.shape)
            assert np.array_equal(got, want), f'{key}[{lvl}] indices differ'
        if lvl > 0:
            got, want = npy(meta['points'][lvl]), fx[f'points_{lvl}']
            if exact_points:
                assert np.array_equal(got, want), f'points[{lvl}] not bit-exact'
            else:
                np.testing.assert_allclose(got, want, rtol=0, atol=1e-6)
    for b in range(n_pairs):
        for side in ('src', 'tgt'):
            fu, fc = npy(out[f'{side}_feat_un'][b]), npy(out[f'{side}_feat'][b])
            s_un, s_c = float(fx[f'{side}_feat_un_{b}_absmax']), float(fx[f'{side}_feat_{b}_absmax'])
            assert np.abs(fu[::step] - fx[f'{side}_feat_un_{b}_rows']).max() <= feat_rtol * s_un
            assert np.abs(fc[:, ::step] - fx[f'{side}_feat_{b}_rows']).max() <= feat_rtol * s_c
            assert abs(fu.astype(np.float64).sum() - float(fx[f'{side}_feat_un_{b}_sum'])) \
                <= feat_rtol * s_un * fu.size ** 0.5 * 4
            assert np.abs(npy(out[f'{side}_kp_warped'][b]) - fx[f'{side}_kp_warped_{b}']).max() <= corr_atol
            assert np.abs(npy(out[f'{side}_overlap'][b]) - fx[f'{side}_overlap_{b}']).max() <= logit_atol
    assert np.abs(npy(out['pose']) - fx['pose']).max() <= pose_atol


# ---- the reference's own sample clouds (tests/golden/real/, outputs from the unmodified reference) -------------
REAL_CASES = {   # fixture name -> (config, weight seed); mirrors tests/golden/make_golden.py
    'real_3dmatch_redkitchen_0_5': ('3dmatch', 31),
    'real_3dmatch_sun3d_home_38_41': ('3dmatch', 32),
    'real_3dmatch_sun3d_hotel3_8_15': ('3dmatch', 33),
    'real_modelnet_2': ('modelnet', 34),
    'real_modelnet_630': ('modelnet', 35),
}


def make_real_case(name):
    """(cfg, state_dict, src, tgt) of a real-data golden case: the committed input clouds + seeded weights."""
    from regtr_b200.config import get_config
    from regtr_b200.weights import random_state_dict
    cfg_name, wseed = REAL_CASES[name]
    cfg = get_config(cfg_name)
    inp = np.load(os.path.join(GOLDEN, 'real', name + '_input.npz'))
    return cfg, random_state_dict(cfg, wseed), inp['src_xyz'], inp['tgt_xyz']


def sha256_of(a):
    import hashlib
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def check_real_pyramid_against_golden(meta, fx):
    """Level sizes, level >= 1 points (bit-exact) and every index array (SHA-256 of the int64 array + a strided
    row sample that localises a mismatch) against a real-data fixture."""
    def npy(t):
        return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)
    n_lvl = len(meta['points'])
    for lvl in range(n_lvl):
        assert np.array_equal(npy(meta['stack_lengths'][lvl]), fx[f'stack_lengths_{lvl}']), f'stack_lengths[{lvl}]'
        if lvl > 0:
            assert np.array_equal(npy(meta['points'][lvl]), fx[f'points_{lvl}']), f'points[{lvl}] not bit-exact'
        for key in ('neighbors', 'pools', 'upsamples'):
            got = npy(meta[key][lvl]).astype(np.int64)
            assert tuple(got.shape) == tuple(fx[f'{key}_{lvl}_shape']), (key, lvl, got.shape)
            assert np.array_equal(got[::97].astype(np.int32), fx[f'{key}_{lvl}_rows']), f'{key}[{lvl}] sample rows differ'
            assert np.array_equal(sha256_of(got), fx[f'{key}_{lvl}_sha256']), f'{key}[{lvl}] SHA-256 differs'


def check_real_forward_against_golden(out, meta, fx, feat_rtol, corr_atol, logit_atol, pose_atol):
    def npy(t):
        return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)
    check_real_pyramid_against_golden(meta, fx)
    step = int(fx['row_step'])
    for side in ('src', 'tgt'):
        fu, fc = npy(out[f'{side}_feat_un'][0]), npy(out[f'{side}_feat'][0])
        s_un, s_c = float(fx[f'{side}_feat_un_0_absmax']), float(fx[f'{side}_feat_0_absmax'])
        assert np.abs(fu[::step] - fx[f'{side}_feat_un_0_rows']).max() <= feat_rtol * s_un
        assert np.abs(fc[:, ::step] - fx[f'{side}_feat_0_rows']).max() <= feat_rtol * s_c
        assert abs(fu.astype(np.float64).sum() - float(fx[f'{side}_feat_un_0_sum'])) <= feat_rtol * s_un * fu.size ** 0.5 * 4
        assert np.abs(npy(out[f'{side}_kp_warped'][0]) - fx[f'{side}_kp_warped_0']).max() <= corr_atol
        assert np.abs(npy(out[f'{side}_overlap'][0]) - fx[f'{side}_overlap_0']).max() <= logit_atol
    assert np.abs(npy(out['pose']) - fx['pose']).max() <= pose_atol
