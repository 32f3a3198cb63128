"""Fused encoder at shapes whose candidate-GEMM tiles are partly empty: the tiles are 128 tokens x 256 features (two 128-feature
segments), so an odd number of segments leaves the last tile's second segment beyond d_sae."""
import pytest

from tests.test_sae_gpu import _check_against_float64, _fused_case


@pytest.mark.gpu
@pytest.mark.parametrize("rows,d,F,k,c_keep", [(300, 64, 384, 8, 8), (129, 96, 640, 16, 6), (64, 128, 1152, 8, 4)])
def test_fused_encode_topk_odd_segment_count(rows, d, F, k, c_keep):
    eng, hp = _fused_case(rows, d, F, k, seed=rows + F, c_keep=c_keep)
    _check_against_float64(eng, hp, k)
