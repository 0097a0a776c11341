"""Pre-split weights of the wgmma 3xTF32 engine: the tf32 hi / lo split kernel (rlx_debug_tf32_split_f32) bit-exact against the same mask
and subtraction in torch, and the pre-split engine instances (rlx_debug_gemm_f32 layouts 3 / 4) bit-identical to the converter instances
they replace in the PPO update: the forward layout with bias+tanh and the dX layout with tanh'.  C sits in the NaN guard buffer of
test_gpu_tc_epilogue: every output must be written and nothing outside it."""
import pytest
import torch

import test_gpu_tc_engine as engine
import test_gpu_tc_epilogue as epilogue

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _split_ref(x):
    hi = (x.view(torch.int32) & -8192).view(torch.float32)  # 0xFFFFE000: the low 13 mantissa bits cleared
    return hi, x - hi


@pytest.mark.parametrize("batch,rows,cols,trans", [(1, 512, 376, 0), (2, 256, 256, 1), (1, 512, 256, 0), (3, 45, 70, 0), (3, 45, 70, 1)])
def test_tf32_split_is_bit_exact(batch, rows, cols, trans):
    k = engine._k()
    g = torch.Generator().manual_seed(batch * 1000 + rows + cols + trans)
    x = torch.randn(batch, rows, cols, generator=g) * 0.05
    flat = x.view(-1)
    flat[:6] = torch.tensor([0.0, -0.0, 1e-40, -3e-39, 3.0e38, -1.0 + 2.0 ** -20])  # zeros, subnormals, a large value, a nonzero lo
    x = x.to(DEV)
    out_shape = (batch, cols, rows) if trans else (batch, rows, cols)
    hi = torch.full(out_shape, float("nan"), device=DEV)
    lo = torch.full(out_shape, float("nan"), device=DEV)
    k.debug_tf32_split(x, trans, hi, lo)
    torch.cuda.synchronize()
    hi_ref, lo_ref = _split_ref(x.transpose(1, 2).contiguous() if trans else x)
    assert torch.equal(hi.view(torch.int32), hi_ref.view(torch.int32))
    assert torch.equal(lo.view(torch.int32), lo_ref.view(torch.int32))
    assert torch.equal(hi + lo, x.transpose(1, 2) if trans else x)  # the split is exact


def _presplit_equals_converter(layout, M, N, K):
    """layout 3 (forward: layout 0, bias+tanh) or 4 (dX: layout 1, tanh') against its converter instance, bit for bit"""
    base, epi = layout - 3, (1 if layout == 3 else 2)
    k = engine._k()
    g = torch.Generator().manual_seed(M * 17 + N * 3 + K + layout)
    A, B, bias, aux, ref = epilogue._operands(base, epi, M, N, K, g)
    conv = epilogue._run(k, 1, base, epi, A, B, M, N, K, bias, aux, M, N)
    pre = epilogue._run(k, 1, layout, epi, A, B, M, N, K, bias, aux, M, N)
    assert torch.equal(pre, conv), "pre-split instance differs from the converter instance"
    bound = 6e-7 + 3.2e-9 * K
    assert engine._err(pre, ref)[0] < bound


CASES = [
    # layout, M, N, K: interior tiles only, then ragged M, N (N = 4 mod 8) and K (K = 376: the PPO layer-1 reduction)
    (3, 256, 256, 96), (3, 256, 512, 256), (4, 256, 256, 256), (4, 384, 384, 96),
    (3, 200, 132, 376), (3, 333, 260, 100), (3, 130, 201, 376), (4, 130, 132, 376), (4, 333, 260, 100), (4, 129, 201, 64),
]


@pytest.mark.parametrize("layout,M,N,K", CASES)
def test_presplit_matches_converter(layout, M, N, K):
    _presplit_equals_converter(layout, M, N, K)


# several tiles per CTA; 1, 3, 5 and 7 k-blocks per tile walk the start of consecutive tiles through every position of the 4-stage ring
@pytest.mark.parametrize("layout,M,N,K", [(3, 8192, 512, 32), (3, 4096, 1280, 96), (3, 4100, 516, 376), (4, 4096, 768, 160), (4, 4100, 260, 224)])
def test_presplit_matches_converter_across_tiles(layout, M, N, K):
    _presplit_equals_converter(layout, M, N, K)


def test_presplit_layouts_need_their_epilogue():
    k = engine._k()
    A, B, C = torch.randn(128, 32, device=DEV), torch.randn(128, 32, device=DEV), torch.full((128, 128), float("nan"), device=DEV)
    with pytest.raises(RuntimeError, match="unsupported epilogue/layout"):
        k.debug_gemm(1, 3, 0, A, B, C, 128, 128, 32)
    with pytest.raises(RuntimeError, match="unsupported epilogue/layout"):
        k.debug_gemm(0, 3, 1, A, B, C, 128, 128, 32, bias=torch.zeros(128, device=DEV))
