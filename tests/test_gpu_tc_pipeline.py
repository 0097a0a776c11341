"""The wgmma engine's operand pipeline (3-stage raw ring, 4-stage B-operand ring, half-k-block commit groups) at shapes where every CTA
runs several tiles, so that the ring positions carry over from one tile to the next.  Same accuracy check as test_gpu_tc_engine."""
import pytest

import test_gpu_tc_engine as engine

pytestmark = pytest.mark.gpu

CASES = [
    # layout, epilogue, M, N, K
    # 320 tiles (2-3 per CTA) with 1-7 and 11 k-blocks per tile: every position of the raw and operand rings, also with fewer
    # k-blocks than stages
    (0, 0, 4096, 1280, 32), (0, 0, 4096, 1280, 64), (0, 0, 4096, 1280, 92), (0, 0, 4096, 1280, 128), (0, 0, 4096, 1280, 160),
    (0, 0, 4096, 1280, 188), (0, 0, 4096, 1280, 224), (0, 0, 4096, 1280, 348),
    # MN-major A and B (A fragments transposed by the consumers' reads), and K-major A with MN-major B, both with more tiles than CTAs
    (2, 0, 2048, 1536, 1000), (1, 2, 4096, 768, 260),
]


@pytest.mark.parametrize("layout,epi,M,N,K", CASES)
def test_tc_gemm_pipeline_across_tiles(layout, epi, M, N, K):
    engine.test_tc_gemm_is_fp32_accurate(layout, epi, M, N, K)
