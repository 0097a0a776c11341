"""Every epilogue of the wgmma engine (rlx_debug_gemm_f32) at interior-only shapes and at ragged M and N (N = 4 mod 8, odd N), against
fp64 and the exact-fp32 SIMT engine.  C sits in a NaN-filled buffer with rows past M and a pitch past N: every output must be written and
the guard band left untouched (interior tiles store without bounds tests, edge tiles with them)."""
import pytest
import torch

import test_gpu_tc_engine as engine

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD_ROWS, GUARD_COLS = 5, 8


def _operands(layout, epi, M, N, K, g):
    if layout == 0:
        A, B = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * 0.3
        ref = A.double() @ B.double().T
    elif layout == 1:
        A, B = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) * 0.3
        ref = A.double() @ B.double()
    else:
        A, B = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g) * 0.3
        ref = A.double().T @ B.double()
    bias = torch.randn(N, generator=g) if epi in (1, 3, 5) else None
    aux = None
    if epi == 1:
        ref = torch.tanh(ref + bias.double())
    elif epi == 3:
        ref = torch.relu(ref + bias.double())
    elif epi == 5:
        ref = ref + bias.double()
    elif epi == 2:
        aux = torch.tanh(torch.randn(M, N, generator=g))
        ref = ref * (1 - aux.double() ** 2)
    elif epi == 4:
        aux = torch.randn(M, N, generator=g)
        ref = ref * (aux.double() > 0)
    return A, B, bias, aux, ref


def _padded(x, cols):
    """x in the leading columns of a contiguous buffer of row pitch `cols` (a multiple of 4 floats); the GEMM reads x's extent only"""
    buf = torch.zeros(x.shape[0], cols, device=DEV)
    buf[:, :x.shape[1]] = x.to(DEV)
    return buf


def _pitch(n):
    return (n + GUARD_COLS + 3) // 4 * 4


def _run(k, eng, layout, epi, A, B, M, N, K, bias, aux, out_rows, out_cols):
    C = torch.full((out_rows + GUARD_ROWS, _pitch(out_cols)), float("nan"), device=DEV)
    # operands at 16-byte pitches even when N is not a multiple of 4
    Ad = _padded(A, (A.shape[1] + 3) // 4 * 4)
    Bd = _padded(B, (B.shape[1] + 3) // 4 * 4)
    auxd = _padded(aux, (N + 3) // 4 * 4) if aux is not None else None
    k.debug_gemm(eng, layout, epi, Ad, Bd, C, M, N, K, bias=bias.to(DEV) if bias is not None else None, aux=auxd)
    torch.cuda.synchronize()
    out = C[:out_rows, :out_cols]
    assert torch.isfinite(out).all(), f"engine {eng} left unwritten / non-finite outputs"
    assert torch.isnan(C[out_rows:]).all() and torch.isnan(C[:, out_cols:]).all(), f"engine {eng} wrote outside the output"
    return out


CASES = [
    # layout, epilogue, M, N, K: interior tiles only, then ragged M and N
    (0, 0, 256, 256, 64), (0, 1, 256, 256, 96), (0, 3, 256, 256, 96), (0, 5, 256, 256, 96),
    (1, 0, 256, 384, 64), (1, 2, 256, 384, 96), (1, 4, 256, 384, 96),
    (2, 0, 256, 256, 300),
    (0, 0, 200, 132, 64), (0, 1, 200, 132, 96), (0, 3, 333, 133, 96), (0, 5, 129, 260, 96),
    (1, 0, 200, 132, 64), (1, 2, 200, 132, 96), (1, 4, 333, 133, 96), (1, 2, 130, 201, 64),
    (2, 0, 190, 140, 300), (2, 0, 131, 133, 40),
]


@pytest.mark.parametrize("layout,epi,M,N,K", CASES)
def test_tc_epilogue_matches_fp64_and_simt(layout, epi, M, N, K):
    k = engine._k()
    g = torch.Generator().manual_seed(M * 11 + N * 5 + K + epi)
    A, B, bias, aux, ref = _operands(layout, epi, M, N, K, g)
    out = {e: engine._err(_run(k, e, layout, epi, A, B, M, N, K, bias, aux, M, N), ref) for e in (0, 1)}
    (simt_fro, simt_max), (tc_fro, tc_max) = out[0], out[1]
    assert simt_fro < 2e-6
    bound = 6e-7 + 3.2e-9 * K
    assert tc_fro < bound, (out, bound, "3xTF32 engine is not fp32-accurate")
    assert tc_max < max(10 * bound, 4 * simt_max), (out, bound)


@pytest.mark.parametrize("layout,epi,M,N,K", [(0, 0, 4096, 1280, 96), (0, 1, 4096, 1280, 96), (1, 2, 4096, 768, 260), (1, 4, 4100, 260, 96)])
def test_tc_epilogue_across_tiles(layout, epi, M, N, K):
    """the epilogue tests repeated when every CTA runs several tiles (engine accuracy check of test_gpu_tc_engine)"""
    if epi <= 2:
        engine.test_tc_gemm_is_fp32_accurate(layout, epi, M, N, K)
    else:
        test_tc_epilogue_matches_fp64_and_simt(layout, epi, M, N, K)


@pytest.mark.parametrize("M,N,K", [(257, 256, 300), (377, 512, 1000), (129, 130, 64), (130, 133, 40), (384, 256, 96)])
def test_tc_transposed_store_with_extra_row(M, N, K):
    """epilogue 6: rows 0..M-2 of A^T B stored transposed, row M-1 (the bias-gradient row of the dW1 | db1 GEMM) into its own row.
    The same kernel main loop as the plain layout-2 GEMM, so the values must be bit-identical to it."""
    k = engine._k()
    g = torch.Generator().manual_seed(M * 13 + N + K)
    A, B = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g) * 0.3
    ref = A.double().T @ B.double()
    C = torch.full((N + 1 + GUARD_ROWS, _pitch(max(M - 1, N))), float("nan"), device=DEV)
    k.debug_gemm(1, 2, 6, _padded(A, (M + 3) // 4 * 4), _padded(B, (N + 3) // 4 * 4), C, M, N, K)
    torch.cuda.synchronize()
    ct, extra = C[:N, :M - 1], C[N, :N]
    assert torch.isfinite(ct).all() and torch.isfinite(extra).all(), "unwritten outputs"
    assert torch.isnan(C[:N, M - 1:]).all() and torch.isnan(C[N, N:]).all() and torch.isnan(C[N + 1:]).all(), "wrote outside the output"
    fro, mx = engine._err(ct, ref[:M - 1].T)
    bound = 6e-7 + 3.2e-9 * K
    assert fro < bound and mx < 10 * bound, (fro, mx, bound)
    assert engine._err(extra, ref[M - 1])[0] < bound
    plain = _run(k, 1, 2, 0, A, B, M, N, K, None, None, M, N)
    assert torch.equal(ct, plain[:M - 1].T) and torch.equal(extra, plain[M - 1])
