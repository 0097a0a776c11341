"""The wgmma 3xTF32 GEMM engine (gemm_tc.cu) on its own, against float64 torch on the same float32 inputs, where a kernel goes wrong:
tile, k-slice, half-k-block and k-block edges, ring wrap-around, ragged epilogue columns, activation kinks, the precision class of the
hi / lo split of each operand, and pre-split weight copies after an in-place weight update.

Entry points, all through the test hook rlx_debug_gemm_f32 (PpoKernels.debug_gemm) except the last:
  layout 0  C = A B^T   (K-major A and B)      epilogues none, bias+tanh, bias+relu, bias
  layout 1  C = A B     (K-major A, MN-major B) epilogues none, tanh', relu'
  layout 2  C = A^T B   (MN-major A and B)      epilogue none, and the transposed store with an extra row (epilogue 6)
  layout 3 / 4          layout 0 with bias+tanh / layout 1 with tanh' through the pre-split instances (B split by tf32_split first)
  the PPO minibatch update, whose forward and input-gradient GEMMs read tf32_split's copies of the weights.
The engine has no beta / accumulate mode: every epilogue writes C without reading it.  So C starts as NaN everywhere: every element
inside the logical output must come out finite and right, and every element of the guard rows before and after it and of the columns
past it must still be NaN.  The operands sit in NaN-filled buffers too, with rows and columns past their extent, so a read outside an
operand poisons the result.  Batched operands and split-K chains are not reachable through the hook; the update tests
(test_gpu_zzzzzz_tc_ppo_shapes.py) cover them.

Bounds.  u = 2^-24.  For output (m, n) the float64 reference is x = sum_k A(m,k) B(n,k), and the error is measured against
s = sum_k |A(m,k)| |B(n,k)|, the scale of the accumulated terms.  An fp32 FMA loop is within K u s; the 3xTF32 engine adds up to about 32 u s
from the split (the dropped lo*lo term below 2^-20 |a||b|, the two cross terms' lo operands cut to tf32 on the way into the tensor core) and
adds each MMA's 8 products into an fp32 accumulator, at most about 2 u s per MMA.  So the bar is  |C - x| <= (32 + K / 4) u s,  plus one
rounding of the epilogue's own arithmetic; the activations are 1-Lipschitz.  On the inputs of test_precision_class_is_3xtf32 the engine
measured 1.8 to 10.8 u s and a single-pass TF32 product of the same inputs 520 to 3900 u s (H100 80GB HBM3, 700 W).

Sorted after the other GPU files: a kernel fault at a new shape takes the CUDA context with it, and then costs only this file."""
import os
import re

import pytest
import torch

_SM90 = pytest.mark.skipif(not (torch.cuda.is_available() and torch.cuda.get_device_capability() == (9, 0)),
                           reason="the wgmma engine needs an sm_90 device")


def gpu(test):
    return pytest.mark.gpu(_SM90(test))


DEV = "cuda"
U = 2.0 ** -24
NAN = float("nan")
LEAD_ROWS, GUARD_ROWS, GUARD_COLS = 2, 3, 8
TANH_REL = 1e-6  # tanh_fast (common.cuh): relative error below 5.5e-7 in its error model; the bar is its 1e-6 class

# ---------------------------------------------------------------------------------------------------- tile constants, from the source
_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rl_x_b200", "csrc")


def _source_constants():
    with open(os.path.join(_CSRC, "gemm_tc_common.cuh")) as fh:
        common = fh.read()
    with open(os.path.join(_CSRC, "gemm_tc.cu")) as fh:
        kernel = fh.read()
    c = {n: int(re.search(rf"constexpr int {n} = (\d+);", common).group(1)) for n in ("BM", "BN", "BK", "WG_K")}
    c.update({n: int(re.search(rf"\b{n} = (\d+)", kernel).group(1)) for n in ("RAW_STAGES", "OP_STAGES", "SPLIT_STAGES")})
    return c


TILE = _source_constants()
BM, BN, BK, WG_K = TILE["BM"], TILE["BN"], TILE["BK"], TILE["WG_K"]
HALF_KB = 2 * WG_K  # one commit group of the consumers: two k-slices
VEC = 2             # the epilogue stores adjacent columns as one float2


def _around(*edges):
    return sorted({v for e in edges for v in (e - 1, e, e + 1) if v >= 1})


# M: one row, either side of the consumer warpgroups' 64-row split and of the tile, one partial tile after a full one, three tiles with a
# ragged last one.  N: one pair and an odd tail, either side of an 8-column group and of the tile, N = 2 and 4 mod 8, a ragged second tile.
# K: below one k-slice, either side of a k-slice, a half k-block and a k-block; exactly the raw ring (RAW_STAGES k-blocks) and the
# operand / pre-split rings (OP_STAGES, SPLIT_STAGES k-blocks) and one more, each also with a ragged last k-block; several ring turns.
M_EDGES = sorted({1, 2 * BM + BM // 2 + 8, 3 * BM - 1} | set(_around(BM // 2, BM)))
N_EDGES = sorted({1, VEC, VEC + 1, BN + 2, BN + 4, BN + BN // 2 + 8, 2 * BN + 3} | set(_around(4 * VEC, BN)))
_RINGS = sorted({TILE["RAW_STAGES"], TILE["OP_STAGES"], TILE["SPLIT_STAGES"]})
K_EDGES = sorted({1, BK // 2 - 5, 11 * BK + 5} | set(_around(WG_K, HALF_KB, BK))
                 | {s * BK + r for d in _RINGS for s in (d, d + 1) for r in (0, 1)})
# layout 4 splits B^T into a copy of pitch K: K a multiple of 4
K_EDGES_4 = sorted({k for k in K_EDGES if k % 4 == 0} | {4, WG_K + 4, BK - 4, BK + 4} | {s * BK + 4 for d in _RINGS for s in (d, d + 1)})

# (layout, epilogue): every instance the hook reaches.  Epilogue 0 none, 1 bias+tanh, 2 tanh', 3 bias+relu, 4 relu', 5 bias, 6 transposed
INSTANCES = [(0, 0), (0, 1), (0, 3), (0, 5), (1, 0), (1, 2), (1, 4), (2, 0), (2, 6), (3, 1), (4, 2)]


def _sweep():
    """Per instance, every M, N and K edge at least once, with the three lists walked at different strides so that each instance
    meets other (M, N, K) combinations."""
    cases = []
    for j, (layout, epi) in enumerate(INSTANCES):
        ks = K_EDGES_4 if layout == 4 else K_EDGES
        n = max(len(M_EDGES), len(N_EDGES), len(ks))
        for i in range(n):
            M = M_EDGES[i % len(M_EDGES)]
            N = N_EDGES[(i + 3 * j) % len(N_EDGES)]
            K = ks[(5 * i + j) % len(ks)]
            cases.append((layout, epi, max(M, 2) if epi == 6 else M, N, K))
    return cases


SWEEP = _sweep()
# more tiles than SMs (2177 x 1027: 162 tiles), so the second tile of a CTA starts where the first left the rings: K of 4-6 k-blocks
RING_CARRY = [(0, 1, 2177, 1027, 97), (0, 3, 2177, 1027, 129), (1, 2, 2177, 1027, 129), (1, 4, 2177, 1027, 161), (2, 0, 2177, 1027, 161),
              (2, 6, 2177, 1027, 97), (3, 1, 2177, 1027, 161), (4, 2, 2177, 1027, 132)]


def test_sweep_brackets_every_tile_boundary():
    """the shape lists come from the constants in gemm_tc_common.cuh / gemm_tc.cu and straddle each boundary they define"""
    for edges, b in ((M_EDGES, BM), (M_EDGES, BM // 2), (N_EDGES, BN), (K_EDGES, WG_K), (K_EDGES, HALF_KB), (K_EDGES, BK)):
        assert {b - 1, b, b + 1} <= set(edges), (b, edges)
    assert 1 in M_EDGES and 1 in N_EDGES and 1 in K_EDGES
    assert any(k < BK for k in K_EDGES_4)
    assert any(n % VEC for n in N_EDGES) and any(n % 8 == 4 for n in N_EDGES)
    for depth in _RINGS:
        assert {depth * BK, (depth + 1) * BK} <= set(K_EDGES) and {depth * BK, (depth + 1) * BK} & set(K_EDGES_4)
    for layout, epi in INSTANCES:
        mine = [c for c in SWEEP if c[:2] == (layout, epi)]
        assert set(M_EDGES) - {1} <= {c[2] for c in mine} and set(N_EDGES) <= {c[3] for c in mine}
        assert set(K_EDGES_4 if layout == 4 else K_EDGES) <= {c[4] for c in mine}


# ------------------------------------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def k():
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(376, 17, 256)


def _pitch(cols):
    return (cols + GUARD_COLS + 3) // 4 * 4


def _in_guard(x):
    """x (CPU float32 [r, c]) at the top left of a NaN-filled device buffer with rows and columns past it; returns the [r, pitch] view the
    engine gets (its row pitch is the buffer's)"""
    r, c = x.shape
    buf = torch.full((r + GUARD_ROWS, _pitch(c)), NAN, device=DEV)
    buf[:r, :c] = x.to(DEV)
    return buf[:r]


def _nan_tail(v):
    return torch.cat([v, torch.full((4,), NAN)]).to(DEV)


def _gemm(k, layout, epi, A, B, bias=None, aux=None):
    """One GEMM on the wgmma engine.  A [M, K] and B [N, K] are the logical operands (CPU float32), laid out as the layout wants them.
    Returns (the logical output, the whole C buffer, a mask of the logical output in it); C starts as NaN."""
    M, K = A.shape
    N = B.shape[0]
    a_dev = _in_guard(A.T.contiguous() if layout == 2 else A)
    b_dev = _in_guard(B if layout in (0, 3) else B.T.contiguous())
    rows, cols = (N + 1, max(M - 1, N)) if epi == 6 else (M, N)
    buf = torch.full((LEAD_ROWS + rows + GUARD_ROWS, _pitch(cols)), NAN, device=DEV)
    C = buf[LEAD_ROWS:LEAD_ROWS + rows]
    k.debug_gemm(1, layout, epi, a_dev, b_dev, C, M, N, K, bias=None if bias is None else _nan_tail(bias),
                 aux=None if aux is None else _in_guard(aux))
    torch.cuda.synchronize()
    buf = buf.cpu()
    mask = torch.zeros(buf.shape, dtype=torch.bool)
    if epi == 6:  # rows 0 .. M-2 of the product transposed into C[:N], row M-1 into C[N]
        mask[LEAD_ROWS:LEAD_ROWS + N, :M - 1] = True
        mask[LEAD_ROWS + N, :N] = True
        out = torch.cat([buf[LEAD_ROWS:LEAD_ROWS + N, :M - 1].T, buf[LEAD_ROWS + N, :N][None]])
    else:
        mask[LEAD_ROWS:LEAD_ROWS + M, :N] = True
        out = buf[LEAD_ROWS:LEAD_ROWS + M, :N]
    return out, buf, mask


def _operands(layout, epi, M, N, K, g):
    A = torch.randn(M, K, generator=g)
    B = torch.randn(N, K, generator=g) * 0.3
    bias = torch.randn(N, generator=g) if epi in (1, 3, 5) else None
    aux = None
    if epi == 2:
        aux = torch.tanh(torch.randn(M, N, generator=g) * 2)
    elif epi == 4:
        aux = torch.randn(M, N, generator=g)
    return A, B, bias, aux


def _tol(K):
    return (32 + K / 4) * U


def _reference(epi, A, B, bias, aux):
    """(float64 reference output, per-element bound) for the engine's output"""
    a, b = A.double(), B.double()
    x = a @ b.T
    gemm = _tol(A.shape[1]) * (a.abs() @ b.abs().T)
    if epi in (0, 6):
        return x, gemm
    if epi in (1, 3, 5):
        z = x + bias.double()
        bound = gemm + U * z.abs()  # fp32 rounding of x + bias; tanh and relu are 1-Lipschitz
        if epi == 1:
            t = torch.tanh(z)
            return t, bound + TANH_REL * t.abs()
        return (torch.relu(z) if epi == 3 else z), bound
    e = aux.double()
    if epi == 2:
        d = 1 - e * e
        return x * d, d.abs() * gemm + 3 * U * x.abs()  # roundings of e * e, 1 - e e and the product
    return x * (e > 0), gemm * (e > 0)


def _check(out, buf, mask, ref, bound, what):
    assert torch.isnan(buf[~mask]).all(), f"{what}: wrote outside the output ({int((~torch.isnan(buf[~mask])).sum())} elements)"
    assert torch.isfinite(out).all(), f"{what}: {int((~torch.isfinite(out)).sum())} outputs unwritten or non-finite"
    err = (out.double() - ref).abs()
    bad = err > bound
    if bad.any():
        i = int(torch.argmax((err - bound) / bound.clamp_min(1e-300)))
        m, n = divmod(i, ref.shape[1])
        raise AssertionError(f"{what}: {int(bad.sum())} outputs out of bound; worst at ({m}, {n}): engine {float(out[m, n])!r}, "
                             f"float64 {float(ref[m, n])!r}, bound {float(bound[m, n]):.3e}")


# ------------------------------------------------------------------------------------------------------------------------- 1. shapes
@pytest.mark.parametrize("layout,epi,M,N,K", SWEEP + RING_CARRY)
@gpu
def test_gemm_vs_float64_at_tile_edges(k, layout, epi, M, N, K):
    g = torch.Generator().manual_seed(M * 7919 + N * 104729 + K * 13 + layout * 3 + epi)
    A, B, bias, aux = _operands(layout, epi, M, N, K, g)
    out, buf, mask = _gemm(k, layout, epi, A, B, bias, aux)
    ref, bound = _reference(epi, A, B, bias, aux)
    _check(out, buf, mask, ref, bound, f"layout {layout} epilogue {epi} ({M}, {N}, {K})")


# ------------------------------------------------------------------------------------------------------------- 2. precision class
def _tf32_hi(x):
    return (x.view(torch.int32) & -8192).view(torch.float32)  # the engine's split: the low 13 mantissa bits cleared


def _tf32_round(x):
    """float32 -> tf32, rounded to nearest (ties away from zero, as cvt.rna.tf32.f32)"""
    i = x.view(torch.int32).to(torch.int64)
    mag = ((i & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000
    return ((i & ~0x7FFFFFFF) | mag).to(torch.int32).view(torch.float32)


# (layout, epilogue): A split in the consumers' registers with B from the converter (K-major, then MN-major B), MN-major A, and B from
# tf32_split's copies (layouts 3 and 4; their epilogues are made transparent: bias 0 for tanh, aux 0 for tanh')
PRECISION = [(0, 0), (1, 0), (2, 0), (3, 1), (4, 2)]


@gpu
@pytest.mark.parametrize("K", [40, 376, 1000])
@pytest.mark.parametrize("low_bits", ["A", "B"])
@pytest.mark.parametrize("layout,epi", PRECISION)
def test_precision_class_is_3xtf32(k, layout, epi, low_bits, K):
    """Only one operand has mantissa bits below tf32's 10, the other is tf32-exact, so the engine's result rests on that operand's lo
    term alone: without it the engine is single-pass TF32.  The error, normalised per element by sum_k |A||B|, must be at the fp32 level
    (the module's bound) and at least 10x below a single-pass TF32 product of the same inputs (both operands rounded to tf32, product in
    float64)."""
    M, N = 256, 264
    g = torch.Generator().manual_seed(K * 31 + layout * 7 + (low_bits == "A"))
    A, B = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g)
    if low_bits == "A":
        B = _tf32_hi(B)
    else:
        A = _tf32_hi(A)
    low = A if low_bits == "A" else B
    assert (low != _tf32_hi(low)).float().mean() > 0.99
    bias = torch.zeros(N) if epi == 1 else None
    aux = torch.zeros(M, N) if epi == 2 else None
    out, buf, mask = _gemm(k, layout, epi, A, B, bias, aux)
    assert torch.isnan(buf[~mask]).all() and torch.isfinite(out).all()
    a, b = A.double(), B.double()
    x = a @ b.T
    scale = a.abs() @ b.abs().T
    ref = torch.tanh(x) if epi == 1 else x
    one_pass = _tf32_round(A).double() @ _tf32_round(B).double().T
    if epi == 1:
        one_pass = torch.tanh(one_pass)
    err = float(((out.double() - ref).abs() / scale).max())
    err_1x = float(((one_pass - ref).abs() / scale).max())
    allowance = _tol(K) + (TANH_REL if epi == 1 else 0.0)  # tanh_fast's own error, relative to |tanh x| <= |x| <= scale
    print(f"\nlayout {layout}, lo bits in {low_bits}, K {K}: max |C - C64| / (|A||B|) = {err / U:.2f} u; single-pass TF32 {err_1x / U:.0f} u")
    assert err <= allowance, (err / U, allowance / U, "not at fp32 level")
    assert err * 10 <= err_1x, (err / U, err_1x / U, "not 10x better than single-pass TF32")


# --------------------------------------------------------------------------------------------------------------- 3. epilogue edges
def _exact_product(M, N, rows):
    """A [M, 4], B [N, 4] whose product is exactly rows[m] in every column: A = [rows, 0, 0, 0], B = [1, 0, 0, 0].  rows must be tf32
    values, so that the split has no lo part and the tensor core multiplies them exactly."""
    A = torch.zeros(M, 4)
    A[:, 0] = rows
    assert torch.equal(_tf32_hi(A), A)
    B = torch.zeros(N, 4)
    B[:, 0] = 1.0
    return A, B


# pre-activations: zero of both signs, the relu kink, tanh_fast's polynomial / exponential branch point at 0.25, saturation
X_ROWS = torch.tensor([0.0, -0.0, 0.25, -0.25, 0.25 * (1 - 2 ** -10), 0.25 * (1 + 2 ** -10), 1.0, -1.0, 8.5, -8.5, 9.0, 10.0, -10.0,
                       15.0, 16.0, -16.0, 20.0, -20.0, 100.0, -100.0, 2 ** -20, -2 ** -20, 3.0, -3.0, 0.5])
# biases: signed zeros, tiny values of both signs (a subnormal among them), values that cancel rows exactly
BIASES = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1e-40, -1e-40, 2 ** -24, -2 ** -24, -0.25, 0.25, -1.0, 1.0, -10.0, 10.0, -3.0, 3.0, -0.5])


@pytest.mark.parametrize("layout,epi", [(0, 1), (0, 3), (0, 5), (3, 1)])
@gpu
def test_bias_epilogues_at_kinks_and_saturation(k, layout, epi):
    """The product is exact, so the engine's x + bias is the fp32 sum of the two, and relu and the plain bias must give exactly what that
    sum gives in torch: 0 for every z <= 0, z itself otherwise.  tanh: within TANH_REL of float64 tanh, never beyond +-1, odd (the rows
    hold +x and -x, the biases +b and -b, and -x + -b is exactly -(x + b) in fp32), and exactly 0 at z = 0."""
    M, N = len(X_ROWS), len(BIASES)
    A, B = _exact_product(M, N, X_ROWS)
    out, buf, mask = _gemm(k, layout, epi, A, B, bias=BIASES)
    assert torch.isnan(buf[~mask]).all() and torch.isfinite(out).all()
    z32 = X_ROWS[:, None] + BIASES[None, :]  # fp32 round to nearest, as on the device
    if epi == 5:
        assert torch.equal(out, z32)
    elif epi == 3:
        assert torch.equal(out, torch.relu(z32)) and bool((out[z32 <= 0] == 0).all())
    else:
        t = torch.tanh(z32.double())
        err = (out.double() - t).abs()
        assert bool((err <= TANH_REL * t.abs()).all()), float((err / t.abs().clamp_min(1e-300)).max())
        assert bool((out.abs() <= 1).all())
        assert bool((out[z32 == 0] == 0).all())
        xs, bs = X_ROWS.tolist(), BIASES.tolist()
        for i, xv in enumerate(xs):
            for j, bv in enumerate(bs):
                if -xv in xs and -bv in bs:
                    assert out[xs.index(-xv), bs.index(-bv)] == -out[i, j], (xv, bv)


# aux values: signed zeros, a subnormal and tiny values of both signs (relu'), and +-1, 1 - 2^-24, 1 - 2^-12 (tanh' at saturation)
AUX_COLS = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 1e-30, -1e-30, 1.0, -1.0, 1 - 2 ** -24, -(1 - 2 ** -24), 1 - 2 ** -12, -(1 - 2 ** -12), 0.5,
                         -0.5, 2.0 ** -12])


@pytest.mark.parametrize("layout,epi", [(1, 2), (1, 4), (4, 2)])
@gpu
def test_aux_epilogues_at_kinks_and_saturation(k, layout, epi):
    """relu': x where aux > 0, else exactly 0 (aux = -0 and negative subnormals give 0, positive subnormals pass x).  tanh': exactly 0 at
    aux = +-1, and x (1 - aux^2) within the roundings of the fp32 arithmetic elsewhere."""
    M, N = len(X_ROWS), len(AUX_COLS)
    A, B = _exact_product(M, N, X_ROWS)
    aux = AUX_COLS[None, :].expand(M, N).contiguous()
    out, buf, mask = _gemm(k, layout, epi, A, B, aux=aux)
    assert torch.isnan(buf[~mask]).all() and torch.isfinite(out).all()
    x = X_ROWS[:, None].expand(M, N)
    if epi == 4:
        assert torch.equal(out, torch.where(aux > 0, x, torch.zeros(()))), (out, aux)
    else:
        e = aux.double()
        ref = x.double() * (1 - e * e)
        assert bool(((out.double() - ref).abs() <= 3 * U * x.double().abs()).all())
        assert bool((out[aux.abs() == 1] == 0).all())


@pytest.mark.parametrize("pitch_extra,offset", [(2, 0), (1, 0), (0, 2), (0, 1)])
@gpu
def test_unaligned_output_is_rejected_untouched(k, pitch_extra, offset):
    """The engine stores rows of C with 8-byte stores from 16-byte-aligned rows: a row pitch that is not a multiple of 4 floats or a C that
    does not start on 16 bytes is refused with an error (the update's run_gemm then takes the SIMT engine), and C is left as it was."""
    M, N, K = 130, 130, 64
    g = torch.Generator().manual_seed(1)
    A, B = _in_guard(torch.randn(M, K, generator=g)), _in_guard(torch.randn(N, K, generator=g))
    ldc = _pitch(N) + pitch_extra
    flat = torch.full((offset + (M + 1) * ldc,), NAN, device=DEV)
    C = flat[offset:offset + M * ldc].view(M, ldc)
    with pytest.raises(RuntimeError, match="not supported by the wgmma engine"):
        k.debug_gemm(1, 0, 0, A, B, C, M, N, K)
    torch.cuda.synchronize()
    assert torch.isnan(flat).all()


# -------------------------------------------------------------------------------------------------------------- 5. determinism
@pytest.mark.parametrize("layout,epi,M,N,K", [(0, 1, 2177, 1027, 161), (1, 2, 2177, 1027, 129), (2, 0, 1027, 515, 1000), (2, 6, 1027, 515, 1000),
                                              (3, 1, 2177, 1027, 376), (4, 2, 2177, 1027, 132)])
@gpu
def test_same_inputs_give_the_same_bits(k, layout, epi, M, N, K):
    """DESIGN.md: every reduction has a fixed order (static tile schedule, no float atomics).  Two calls on the same inputs, with more
    tiles than SMs, must agree to the bit."""
    g = torch.Generator().manual_seed(M + N + K + layout)
    A, B, bias, aux = _operands(layout, epi, M, N, K, g)
    first, _, _ = _gemm(k, layout, epi, A, B, bias, aux)
    second, _, _ = _gemm(k, layout, epi, A, B, bias, aux)
    assert torch.equal(first.view(torch.int32), second.view(torch.int32))


# ------------------------------------------------------------------------------------------------ 4. pre-split weights after updates
@pytest.fixture
def tc_engine():
    from rl_x_b200 import _native as nt
    lib = nt.load()
    assert lib.rlx_set_gemm_engine(1) == 1
    yield lib
    lib.rlx_set_gemm_engine(0)


@pytest.mark.parametrize("update", ["clip_adam", "add_"])
@gpu
def test_presplit_weights_follow_in_place_updates(tc_engine, update):
    """The minibatch update's forward GEMMs and its input-gradient GEMM read tf32 hi / lo copies of W1cat, W2 and W2^T that the update
    makes from the parameters at the start of every call (ppo.cu, split_weights); there is no refresh call to make.  So after the
    parameters change in place - through clip + Adam, the optimiser step the PPO plugin runs after each fwdbwd, or through a plain
    add_ on a parameter view, as a checkpoint load or a user edit would - the next fwdbwd on the same workspace must give the float64
    gradient at the NEW parameters.  The gradient and the metrics are NaN before the second call, which must write them anew."""
    import test_gpu_zzzzzz_tc_ppo_shapes as S
    from test_gpu_parity import _flat_from_named, _run_fwdbwd
    obs, act, hidden, m = 64, 4, 128, 300
    k = S._kern(obs, act, hidden)
    pol, cri, mb = S._minibatch_case(obs, act, hidden, m)
    fp = _flat_from_named(k, pol, cri)
    (args, grads, metrics, st, keep), counts = S._paths(tc_engine, lambda: _run_fwdbwd(k, fp, mb, S._hp(S.ENT)))
    S._assert_update_path(counts, head_on_tc=True)

    def worst_distance():
        g64, norms, met = S._oracle64(*fp.state_dicts(), mb, S.ENT)
        ours = S._named_grads(k, grads)
        S._assert_losses(metrics.cpu().numpy(), met, mb["advantages"], m)
        return {n: S._dist(ours[n], ref) / norms[n] for n, ref in g64.items()}

    before = worst_distance()
    assert max(before.values()) <= 1e-5, before
    old = fp.flat.clone()
    if update == "clip_adam":
        st["lr"].fill_(1e-3)
        k.clip_adam(args)
    else:
        g = torch.Generator(device=DEV).manual_seed(5)
        for seg, shape in fp.shapes.items():
            if seg.startswith(("W1", "W2")):  # the weights the GEMMs read through the copies
                fp.view(fp.flat, seg).add_(0.01 * torch.randn(shape, generator=g, device=DEV))
    torch.cuda.synchronize()
    moved = float((fp.flat - old).norm() / old.norm())
    assert moved > 1e-4, moved
    grads.fill_(NAN)
    metrics.fill_(NAN)
    _, counts = S._paths(tc_engine, lambda: k.fwdbwd(args))
    S._assert_update_path(counts, head_on_tc=True)
    after = worst_distance()
    print(f"\n{update}: parameters moved {moved:.1e}; worst gradient distance to float64 before {max(before.values()):.2e}, "
          f"after {max(after.values()):.2e}")
    assert max(after.values()) <= 1e-5, after
