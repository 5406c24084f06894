"""The 3xTF32 GEMM's yardstick is sharp: on the model of the kernel's arithmetic (tests/gemm_oracle.py), the shipped
design meets the fp32 yardstick and every emulated wrong kernel fails it, on the input families of
tests/test_gpu_gemm.py at K = 1024 and 3840.  CPU only."""
import numpy as np
import pytest

import gemm_oracle as go


@pytest.mark.parametrize('K', [1024, 3840])
@pytest.mark.parametrize('family', go.FAMILIES)
def test_yardstick_separates_gemm_models(family, K):
    ys = go.emulation_table(family, 32, 32, K, seed=K)
    ys.report()
    failed = {name.replace(' per-row', '') for name in ys.failures()}
    assert 'shipped' not in failed, ys.failures()
    assert set(go.VARIANTS) - {'shipped'} <= failed, sorted(set(go.VARIANTS) - failed)


def test_tf32_roundings_restated():
    """The numpy roundings on constructed bit patterns: ties go to even (rne) or away from zero (rna)."""
    def f(u):
        return np.array(u, dtype=np.uint32).view(np.float32)
    one = 0x3F800000
    x = f([one | 0x1000, one | 0x3000, one | 0x0FFF, one | 0x1001, 0x80000000 | one | 0x1000, 0])
    assert go.tf32_rne(x).view(np.uint32).tolist() == [one, one | 0x4000, one, one | 0x2000, 0x80000000 | one, 0]
    assert go.tf32_rna(x).view(np.uint32).tolist() == [one | 0x2000, one | 0x4000, one, one | 0x2000,
                                                       0x80000000 | one | 0x2000, 0]
    assert go.tf32_trunc(x).view(np.uint32).tolist() == [one, one | 0x2000, one, one, 0x80000000 | one, 0]
    assert go.bf16_rne(f([one | 0x8000, one | 0x18000, one | 0x7FFF])).tolist() == [0x3F80, 0x3F82, 0x3F80]


def test_split_count_rule_covers_the_gpu_cases():
    """The shapes tests/test_gpu_gemm.py names after a split count take it under the restated rule."""
    for (M, N, K), s in {(128, 64, 512): 2, (256, 128, 1024): 4, (128, 256, 2048): 8, (64, 128, 9000): 16,
                         (1000, 260, 3840): 8}.items():
        assert go.choose_splits(M, N, K) == s, (M, N, K)
    # the last one only because of the rule of at most 16 k-blocks per plane: without it the count would be 6
    assert min(go.cdiv(go.NUM_SMS, 8 * 3), 3840 // 32 // 8, 8) == 6
    # the cap: 282 k-blocks in 16 planes of 18
    assert go.cdiv(go.cdiv(9000, 32), 16) == 18
