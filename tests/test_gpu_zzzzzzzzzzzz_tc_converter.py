"""The B hi / lo conversion inside the wgmma 3xTF32 engine (gemm_tc.cu, convert_b): the consumer warps write the K-major swizzled hi and
lo tiles of every k-block's B that does not arrive pre-split.  The conversion is pure bit manipulation (hi = x with the low 13 mantissa
bits cleared, lo = x - hi, exact), and the MMA sequence does not depend on how the operands sat in global memory, so three products that
reach the tensor core through different paths must agree to the BIT, not merely within a tolerance:

  layout 2 (A and B MN-major: B through the conversion's transposing path, A through the consumers' transposing fragment reads)
      == layout 0 on explicitly transposed copies (K-major A and B: the element-wise path)
  layout 1 with tanh' (MN-major B through the conversion) == layout 4 (the same product with B split by tf32_split, no conversion)
  epilogue 6 (layout 2 stored transposed, the last row into the extra row) == layout 2 and a host transpose

Each call's GEMM path counters must show exactly the instance named, so a fallback or a different instance fails the test, and each
result is held to the float64 bar of test_gpu_zzzzzzzz_tc_gemm_float64.py.  Shapes: M and N 1 and 127 past a tile edge and off the
128 grid, K below one k-block, with a tail that is not a multiple of 32, and long enough for several turns of every ring, and more tiles
than SMs.  The bf16 instances (BF16: hi only, one MMA per k-slice) are reachable through the PPO update in bf16 mode only: the weight
gradient GEMMs there convert MN-major activations, checked by path, against the float64 autograd of the autocast oracle at the bf16 bar
of test_gpu_bf16.py, and for bit-identical repeats."""
import numpy as np
import pytest
import torch

import test_gpu_zzzzzz_tc_ppo_shapes as S
import test_gpu_zzzzzzzz_tc_gemm_float64 as F

_SM90 = pytest.mark.skipif(not (torch.cuda.is_available() and torch.cuda.get_device_capability() == (9, 0)),
                           reason="the wgmma engine needs an sm_90 device")


def gpu(test):
    return pytest.mark.gpu(_SM90(test))


DEV = "cuda"
BM, BN, BK = F.BM, F.BN, F.BK
# (M, N, K): one row / column, 1 and 127 past a tile edge, K of one k-slice, a 36 and a 1000 (tails of 4 and 8 past a k-block), 97 (not a
# multiple of 4: layout 4 cannot take it), and 2177 x 1027 = 162 tiles, more than the SMs of an H100
SHAPES = [(1, 129, 36), (BM + 1, 2 * BN - 1, 8), (2 * BM - 1, 1, 1000), (BM + 1, BN - 1, 97), (2 * BM - 1, 2 * BN - 1, 1000),
          (17 * BM + 1, 8 * BN + 3, 36), (17 * BM + 1, 8 * BN + 3, 1000), (17 * BM + 1, 8 * BN + 3, 97)]

# tc_gemm_kernel instance slot: A_KMAJ | B_KMAJ << 1 | EPI << 2 | BF16 << 5 | TRANS << 6 | SPLIT_B << 7 (S._tc_instances)
WANT = {(0, 0): {(True, True, 0, False, False, False): 1},
        (2, 0): {(False, False, 0, False, False, False): 1},
        (2, 6): {(False, False, 0, False, True, False): 1},
        (1, 2): {(True, False, 2, False, False, False): 1},
        (4, 2): {(True, True, 2, False, False, True): 1}}


@pytest.fixture(scope="module")
def k():
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(376, 17, 256)


@pytest.fixture(scope="module")
def lib():
    from rl_x_b200 import _native as nt
    return nt.load()


def _engine_gemm(k, lib, layout, epi, A, B, aux=None):
    """F._gemm with the path counters read around it: exactly the instance of (layout, epi) ran once, tf32_split only for layout 4, and
    nothing on the SIMT engine.  Returns the logical output (CPU float32)."""
    (out, buf, mask), counts = S._paths(lib, lambda: F._gemm(k, layout, epi, A, B, aux=aux))
    assert S._tc_instances(counts) == WANT[(layout, epi)], (layout, epi, counts)
    assert counts.get(S.GP_TF32_SPLIT, 0) == (1 if layout == 4 else 0), counts
    assert counts.get(S.GP_SGEMM, 0) == 0, counts
    ref, bound = F._reference(2 if epi == 2 else 0, A, B, None, aux)
    F._check(out, buf, mask, ref, bound, f"layout {layout} epilogue {epi} ({A.shape[0]}, {B.shape[0]}, {A.shape[1]})")
    return out


def _bits_equal(x, y, what):
    same = x.view(torch.int32) == y.view(torch.int32)
    if not bool(same.all()):
        m, n = divmod(int(torch.argmin(same.int())), x.shape[1])
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.numel()} outputs differ in their bits; first at ({m}, {n}): "
                             f"{float(x[m, n])!r} vs {float(y[m, n])!r}")


def _operands(M, N, K):
    g = torch.Generator().manual_seed(M * 7919 + N * 104729 + K)
    return torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * 0.3


@pytest.mark.parametrize("M,N,K", SHAPES)
@gpu
def test_mn_major_conversion_equals_k_major(k, lib, M, N, K):
    """C = A B^T through MN-major operands (layout 2) and through K-major copies of them (layout 0): bit for bit."""
    A, B = _operands(M, N, K)
    _bits_equal(_engine_gemm(k, lib, 2, 0, A, B), _engine_gemm(k, lib, 0, 0, A, B), f"layout 2 vs 0 ({M}, {N}, {K})")


@pytest.mark.parametrize("M,N,K", [s for s in SHAPES if s[2] % 4 == 0])
@gpu
def test_converted_b_equals_presplit_b(k, lib, M, N, K):
    """(A B^T) * tanh' with MN-major B converted in the kernel (layout 1) and with B split beforehand by tf32_split (layout 4)."""
    A, B = _operands(M, N, K)
    aux = torch.tanh(torch.randn(M, N, generator=torch.Generator().manual_seed(K)) * 2)
    _bits_equal(_engine_gemm(k, lib, 1, 2, A, B, aux), _engine_gemm(k, lib, 4, 2, A, B, aux), f"layout 1 vs 4 ({M}, {N}, {K})")


@pytest.mark.parametrize("M,N,K", [(max(M, 2), N, K) for M, N, K in SHAPES])
@gpu
def test_transposed_store_equals_host_transpose(k, lib, M, N, K):
    """Epilogue 6 stores the layout-2 product transposed (rows 0 .. M-2 into C[:N], row M-1 into the extra row); F._gemm reassembles it as
    [M, N], which must be the layout-2 output bit for bit."""
    A, B = _operands(M, N, K)
    _bits_equal(_engine_gemm(k, lib, 2, 6, A, B), _engine_gemm(k, lib, 2, 0, A, B), f"epilogue 6 vs layout 2 ({M}, {N}, {K})")


# ------------------------------------------------------------------------------------------------------------------- bf16 instances
BF16_DW = (False, False, 0, True, False, False)    # dW2 and the head's dW3: MN-major activations on both sides
BF16_DW1_T = (False, False, 0, True, True, False)  # dW1 | db1 stored transposed


@gpu
def test_bf16_instances_convert_mn_major_activations(lib):
    import test_gpu_bf16 as BF
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    from test_gpu_parity import _random_minibatch, _run_fwdbwd
    from oracle import ppo_oracle as O
    obs, act, hidden, m, ent = 128, 4, 384, 2048, 0.01
    assert lib.rlx_set_gemm_engine(1) == 1
    lib.rlx_set_autocast_bf16(1)
    try:
        kern = BF._kern(obs, act, hidden)
        pol, cri = O.init_params(obs, act, hidden, std_dev=0.9, seed=m)
        g = torch.Generator().manual_seed(m + 1)
        for w in list(pol.values()) + list(cri.values()):
            w.add_(0.02 * torch.randn(w.shape, generator=g))
        mb = _random_minibatch(obs, act, m, seed=m + 2)
        with torch.no_grad():
            lp, _ = O.get_logprob_entropy(pol, mb["states"], mb["actions"])
        mb["log_probs"] = lp + 0.15 * torch.randn(m, generator=g)
        runs = []
        for _ in range(2):
            fp = BF._flat(kern, pol, cri)
            (args, grads, metrics, st, keep), counts = S._paths(lib, lambda: _run_fwdbwd(kern, fp, mb, make_hparams(0.2, ent, 0.5, 0.5)))
            inst = S._tc_instances(counts)
            assert inst.get(BF16_DW, 0) >= 1 and inst.get(BF16_DW1_T, 0) == 1, counts
            assert all(key[3] for key in inst), counts  # every GEMM of the bf16 update on a BF16 instance
            assert counts.get(S.GP_SGEMM, 0) == 0, counts
            runs.append((grads.cpu(), fp))
    finally:
        lib.rlx_set_autocast_bf16(0)
        lib.rlx_set_gemm_engine(0)
    _bits_equal(runs[0][0][None], runs[1][0][None], "bf16 gradients of two runs")
    L = O.Learner(pol, cri, clip_range=0.2, entropy_coef=ent, critic_coef=0.5, bf16=True)
    gp, gc, _ = BF._grads_under_autocast(L, mb)
    gflat = runs[0][1].__class__(kern, DEV)
    gflat.flat.copy_(runs[0][0].to(DEV))
    gpol, gcri = gflat.state_dicts()
    for name, ref in {**gp, **gc}.items():
        ours = (gpol if name in gpol else gcri)[name]
        dist = BF._rel(ours.numpy(), ref.numpy())
        assert dist <= (5e-2 if name in ("critic.4.bias", "policy_mean.4.bias") else 1e-2), (name, dist)
        assert np.isfinite(ours.numpy()).all(), name
