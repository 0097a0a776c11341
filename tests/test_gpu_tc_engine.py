"""The wgmma 3xTF32 GEMM engine in isolation (rlx_debug_gemm_f32): every operand layout / epilogue the MLP uses, with
M / N / K tails, against an fp64 reference and against the exact-fp32 SIMT engine."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _k():
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(376, 17, 256)


def _err(c, ref):
    c, ref = c.double().cpu(), ref.cpu()
    return float((c - ref).norm() / ref.norm()), float((c - ref).abs().max() / ref.abs().max())


CASES = [
    # layout, epilogue, M, N, K
    (0, 0, 128, 128, 32), (0, 0, 128, 256, 64), (0, 1, 4096, 512, 376), (0, 1, 40000, 512, 376), (0, 1, 130, 256, 256), (0, 0, 1000, 128, 64), (0, 1, 32, 512, 376),
    (1, 0, 256, 256, 256), (1, 2, 4100, 256, 256), (1, 2, 33, 256, 256),
    (2, 0, 128, 128, 64), (2, 0, 256, 256, 3000), (2, 0, 512, 380, 2752), (2, 0, 512, 380, 40), (2, 0, 256, 256, 5),
]


@pytest.mark.parametrize("layout,epi,M,N,K", CASES)
def test_tc_gemm_is_fp32_accurate(layout, epi, M, N, K):
    k = _k()
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    if layout == 0:
        A, B = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * 0.3
        ref = A.double() @ B.double().T
    elif layout == 1:
        A, B = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) * 0.3
        ref = A.double() @ B.double()
    else:
        A, B = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g) * 0.3
        ref = A.double().T @ B.double()
    bias = torch.randn(N, generator=g) if epi == 1 else None
    aux = torch.tanh(torch.randn(M, N, generator=g)) if epi == 2 else None
    if epi == 1:
        ref = torch.tanh(ref + bias.double())
    if epi == 2:
        ref = ref * (1 - aux.double() ** 2)
    out = {}
    for engine in (0, 1):
        C = torch.full((M, N), float("nan"), device=DEV)
        k.debug_gemm(engine, layout, epi, A.to(DEV), B.to(DEV), C, M, N, K, bias=bias.to(DEV) if bias is not None else None,
                     aux=aux.to(DEV) if aux is not None else None)
        torch.cuda.synchronize()
        assert torch.isfinite(C).all(), f"engine {engine} left unwritten / non-finite outputs"
        out[engine] = _err(C, ref)
    (simt_fro, simt_max), (tc_fro, tc_max) = out[0], out[1]
    assert simt_fro < 2e-6
    # Error model of the 3xTF32 engine: ~4e-7 from the split itself plus a few 1e-9 per reduction element from the tensor core's
    # accumulation rounding (production dW GEMMs keep chains <= 1024 via split-K).  Single-pass TF32 would sit at ~5e-4 here.
    bound = 6e-7 + 3.2e-9 * K
    assert tc_fro < bound, (out, bound, "3xTF32 engine is not fp32-accurate")
    assert tc_max < max(10 * bound, 4 * simt_max), (out, bound)


def test_tc_gemm_rejects_unaligned_shapes():
    k = _k()
    A, B, C = torch.randn(64, 30, device=DEV), torch.randn(64, 30, device=DEV), torch.empty(64, 64, device=DEV)
    with pytest.raises(RuntimeError, match="not supported by the wgmma engine"):
        k.debug_gemm(1, 0, 0, A, B, C, 64, 64, 30)


@pytest.mark.parametrize("engine", [-1, 2, 3, 4])
def test_debug_gemm_rejects_unknown_engines(engine):
    """Engines 2-4 once selected CTA-pair kernels: an old caller must get an error, not a silent SIMT result."""
    k = _k()
    A, B, C = torch.randn(128, 32, device=DEV), torch.randn(128, 32, device=DEV), torch.full((128, 128), float("nan"), device=DEV)
    with pytest.raises(RuntimeError, match="unknown engine"):
        k.debug_gemm(engine, 0, 0, A, B, C, 128, 128, 32)
    torch.cuda.synchronize()
    assert torch.isnan(C).all()
