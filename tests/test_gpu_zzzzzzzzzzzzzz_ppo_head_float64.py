"""The PPO loss head inside rlx_ppo_minibatch_fwdbwd_f32, one case per kernel instance the dispatcher (launch_train_head / launch_head_wgrad,
csrc/ppo.cu) can pick, against float64 autograd of oracle/ppo_oracle.py, with proof of which instance ran.

Instances.  The train head is ppo_head_train_kernel<NCH, BF16> (act > 31 or odd hidden), ppo_head_train2_kernel<NCH, ACT_MAX, BF16>,
ppo_head_train3_kernel<H, ACT_MAX, BF16> (hidden 128 / 256 / 512), ppo_head_train4_kernel<H, NT> (head engine 2, fp32, shared memory <= 220
KB) or the GEMM head of csrc/ppo_head_gemm.cu (head engine 1, fp32, scratch <= m * 2H); its weight gradient is ppo_head_wgrad_kernel<8|32|64>,
ppo_head_wgrad3_kernel<4..32> or the wgmma GEMM.  `expected_head_path` mirrors those rules; the CPU test below enumerates every accepted
(act, hidden) and asserts that the case tables reach every instance it can produce, fp32 on each head engine and bf16, and that every case
is the only one to cover some instance or edge.  After every call the GPU tests read the library's record of what it launched
(rlx_debug_ppo_head_path) and compare it with the mirror: a silent fallback (engine 2 to train3, engine 1 to the fused head, bf16 to engine 0)
fails there, not in a tolerance.

Inputs.  Old log-probs are set from the float64 new log-probs so that every |ratio - 1| lies at least 1e-4 from the clip range, with rows on
both sides of it; the workspace, the gradient and the metrics start as float32 NaN, so an element nothing wrote, or a read of one, fails.

Bounds (fp32 mode, SIMT GEMM engine unless a case says otherwise), with g64 the float64 oracle's gradient at the same parameters and data:
  * per gradient tensor ||g - g64|| <= 1e-5 ||g64||, where for the two last-layer biases ||g64|| stands for the root-sum-square of their per-row
    terms when that is larger (test_gpu_zzzzzz_tc_ppo_shapes.py's _oracle64);
  * losses by test_gpu_parity.py's scale rules (pg_loss against the summand scale, approx_kl with a 1e-2 floor), each scaled by m / m_global;
  * the clip fraction exactly: the kernels count rows in fp32 (exact below 2^24) and multiply by the fp32 1 / m_global;
  * ESPO's ratio-delta metric (clip_range = inf): the mean and the lower median of |ratio - 1| within 1e-5 relative.
bf16 mode: test_gpu_bf16.py's stated tolerances against its autocast oracle (gradients 1e-2 of the norm, 5e-2 for the two last-layer biases,
bf16-valued weight and bias gradients, losses 1e-2 of their scale, clip fraction 0.01 + 2 / m).
Measured on an H100 80GB HBM3 (SXM, 700 W power limit): worst per-tensor distance 5.2e-6 of the norm on head engine 0, 8.9e-7 on engine 1,
2.4e-6 on engine 2, 1.4e-6 with the wgmma weight gradient; worst bf16 distance 4.0e-3; the whole file in 41-46 s.

Sorted after the other GPU files: a kernel fault takes the CUDA context with it, and then costs only this file.  Every fixture puts head engine
0, GEMM engine 0 and bf16 off back, because those are process-wide settings."""
import ctypes as C
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from test_gpu_bf16 import _grads_under_autocast, _is_bf16
from test_gpu_parity import _flat_from_named
from test_gpu_zzzzzz_tc_ppo_shapes import SUMMED_BIASES, _f64, _minibatch_case, _named_grads, _oracle64

DEV = "cuda"
NAMES = ("states", "actions", "log_probs", "advantages", "returns")
CLIP, CRITIC_COEF, MAX_NORM = 0.2, 0.5, 0.5
SXM_SMS = 132  # H100 SXM; the GPU tests read the real count

# ------------------------------------------------------------------------------------------ dispatcher mirror (ppo.cu)
TRAIN, TRAIN2, TRAIN3, TRAIN4, GEMM_HEAD = 0, 1, 2, 3, 4
WGRAD, WGRAD3, WGRAD_TC = 0, 1, 2


def _ceil(a, b):
    return -(-a // b)


def head_dims_ok(act, hidden):
    """head_dims_ok: act <= 64, hidden <= 1024, the train head's shared memory (head_smem_bytes) <= 200 KB."""
    smem = 4 * (act * hidden + hidden) + 4 * 8 * (2 * act + 5 + 2 * hidden)
    return 1 <= act <= 64 and 1 <= hidden <= 1024 and smem <= 200 * 1024


def head4_smem_floats(H, act, NT):
    tables = 2 * act * (H + 16) + H
    work = (H // 16) * 2 * NT * 32 * 4 + 8 * NT * 32 * 4 + 8 * 16
    return tables + max(work, 8 * (2 * act + 5 + 2 * H))


def head_gemm_scratch_floats(m, H, A):
    return m * (2 * A + 8) + (m // 256 + 2) * max(2 * H, 8)


def tc_supported(obs, H):
    return H % 128 == 0 and 128 <= H <= 1024 and obs % 4 == 0 and obs >= 32


def _nch(H):
    n = _ceil(H, 32)
    return 2 if n <= 2 else 4 if n <= 4 else 8 if n <= 8 else 16 if n <= 16 else 32


def _act_max(A):
    return 8 if A <= 8 else 16 if A <= 16 else 24 if A <= 24 else 31


def expected_head_path(obs, act, hidden, m, head_engine, gemm_engine, bf16):
    """What rlx_debug_ppo_head_path must report after one minibatch call: (train kernel, its two template arguments, BF16, wgrad kernel,
    its ACT_MAX)."""
    A, H, bf = act, hidden, int(bool(bf16))
    fast = A <= 31 and H % 2 == 0 and H <= 1024                              # fast_head_ok
    dh_ld = _ceil(A + 1, 4) * 4
    if fast and head_engine == 1 and not bf16 and head_gemm_scratch_floats(m, H, A) <= m * 2 * H:
        head = (GEMM_HEAD, 0, 0, 0)
    elif not fast:
        head = (TRAIN, _nch(H), 0, bf)
    else:
        vec = H in (128, 256, 512)
        nt4 = _ceil(dh_ld, 8)
        if vec and head_engine == 2 and not bf16 and nt4 <= 4 and head4_smem_floats(H, A, nt4) * 4 <= 220 * 1024:
            head = (TRAIN4, H, nt4, 0)
        elif vec:
            head = (TRAIN3, H, _act_max(A), bf)
        else:
            head = (TRAIN2, _nch(H), _act_max(A), bf)
    if not fast:
        wgrad = (WGRAD, 8 if A <= 8 else 32 if A <= 32 else 64)
    elif gemm_engine == 1 and tc_supported(obs, H):
        wgrad = (WGRAD_TC, 0)
    else:
        wgrad = (WGRAD3, next(am for am in (4, 8, 12, 16, 20, 24, 32) if A + 1 <= am or am == 32))
    return head + wgrad


def min_cta_iterations(kernel, m, sms):
    """Grid-stride iterations of the head CTA / warp that runs fewest: head_grid(m) CTAs of 8 warps; ppo_head_train_kernel takes one row per
    warp, train2 / train3 a pair of rows per warp, train4 one 128-row super tile per CTA (over min(ceil(m / 128), head_grid) CTAs)."""
    grid = min(_ceil(m, 16), 2 * sms)
    if kernel == TRAIN:
        return m // (8 * grid)
    if kernel in (TRAIN2, TRAIN3):
        return _ceil(m, 2) // (8 * grid)
    if kernel == TRAIN4:
        return _ceil(m, 128) // min(_ceil(m, 128), grid)
    return 0


# ------------------------------------------------------------------------------------------------------- cases
Case = namedtuple("Case", "obs act hidden m engine gemm mg ent", defaults=(0, 0, 1, 0.0))

FP32_CASES = [
    # ppo_head_train_kernel<NCH> (act > 31 or odd hidden) and ppo_head_wgrad_kernel
    Case(12, 64, 2, 7),             # <2>, wgrad<64>; widest act, narrowest hidden, m < 16
    Case(20, 33, 96, 4500),         # <4>; every warp runs two rows
    Case(16, 3, 255, 301),          # <8>, wgrad<8>; odd hidden
    Case(24, 63, 384, 1000),        # <16>
    Case(12, 1, 1023, 513),         # <32>; odd hidden, one action
    Case(16, 32, 33, 130),          # <2>, wgrad<32>; act 32 leaves the fast head
    # ppo_head_train2_kernel<NCH, ACT_MAX>
    Case(12, 8, 64, 257),
    Case(12, 24, 40, 333),
    Case(12, 31, 64, 129),          # value in lane 31
    Case(20, 4, 96, 8501),          # act 4: padding lanes of dh_ld 8; every warp runs two row pairs
    Case(20, 9, 96, 700, ent=0.01),
    Case(20, 23, 96, 1001),
    Case(20, 25, 96, 555),
    Case(16, 7, 192, 999),
    Case(16, 15, 130, 1025),
    Case(16, 17, 254, 640, mg=3),   # m_global = 3m: every term divided by the global count
    Case(16, 31, 192, 300),
    Case(24, 1, 384, 777),
    Case(24, 16, 300, 1000),
    Case(24, 24, 510, 511),
    Case(24, 28, 384, 1000),
    Case(12, 3, 640, 1000),
    Case(12, 12, 1024, 257),
    Case(12, 20, 640, 700),
    Case(12, 31, 1024, 1000),       # the widest fast head: 199 KB of the 200 KB gate
    # ppo_head_train3_kernel<H, ACT_MAX>
    Case(16, 8, 128, 1000),
    Case(16, 13, 128, 1001),
    Case(16, 24, 128, 9001),        # every warp runs two row pairs
    Case(16, 31, 128, 257),
    Case(24, 1, 256, 1000),
    Case(24, 16, 256, 999),
    Case(376, 17, 256, 32768),      # the benchmark's minibatch
    Case(24, 27, 256, 777),
    Case(32, 5, 512, 1000),
    Case(32, 9, 512, 513),
    Case(32, 19, 512, 1000),
    Case(32, 30, 512, 301),
    # head engine 2: ppo_head_train4_kernel<H, NT>
    Case(12, 1, 128, 70001, 2),     # every CTA runs two super tiles; partial last tile
    Case(12, 9, 128, 1000, 2),
    Case(12, 17, 128, 129, 2),
    Case(12, 31, 128, 1000, 2),
    Case(16, 4, 256, 1000, 2),
    Case(16, 15, 256, 333, 2),
    Case(16, 23, 256, 1000, 2),
    Case(16, 25, 256, 2049, 2),
    Case(24, 7, 512, 1000, 2),
    Case(24, 12, 512, 255, 2),
    Case(24, 20, 512, 1000, 2),
    Case(24, 24, 512, 1000, 2),     # over the 220 KB gate: train3<512, 24>
    # head engine 1: the GEMM head, and its scratch gate
    Case(24, 5, 128, 1000, 1),
    Case(12, 9, 8, 50, 1),          # scratch > m * 2H: the fused head
    # GEMM engine 1: the head weight gradient on the wgmma engine
    Case(32, 11, 128, 1000, gemm=1),
]

BF16_CASES = [
    Case(12, 64, 2, 200), Case(12, 32, 96, 300), Case(12, 3, 255, 301), Case(12, 63, 384, 400), Case(12, 1, 1023, 257),
    Case(12, 8, 64, 300), Case(12, 16, 62, 200), Case(12, 24, 40, 333), Case(12, 31, 64, 129),
    Case(12, 4, 96, 500), Case(12, 9, 96, 300), Case(12, 23, 96, 301), Case(12, 25, 96, 255),
    Case(12, 7, 192, 300), Case(12, 15, 130, 257), Case(12, 17, 254, 333), Case(12, 31, 192, 300),
    Case(12, 1, 384, 300), Case(12, 16, 300, 257), Case(12, 24, 510, 301), Case(12, 28, 384, 300),
    Case(12, 3, 640, 300), Case(12, 12, 1024, 257), Case(12, 20, 640, 301), Case(12, 31, 1024, 300),
    Case(12, 8, 128, 1000, 2),      # head engine 2 in bf16 mode: engine 0's kernel
    Case(12, 13, 128, 300), Case(12, 24, 128, 301), Case(12, 31, 128, 257),
    Case(12, 1, 256, 300), Case(12, 16, 256, 301, 1),  # head engine 1 in bf16 mode: engine 0's kernel
    Case(12, 17, 256, 1000), Case(12, 27, 256, 257),
    Case(12, 5, 512, 300), Case(12, 9, 512, 301), Case(12, 19, 512, 300), Case(12, 30, 512, 257),
]

EDGE_ACTS = (1, 3, 4, 7, 8, 9, 15, 16, 17, 23, 24, 25, 31, 32, 33, 63, 64)
EDGE_HIDDENS = (33, 255, 1023, 2, 96, 384, 640, 1024)


def _path(c, bf16):
    return expected_head_path(c.obs, c.act, c.hidden, c.m, c.engine, c.gemm, bf16)


def _features(c, bf16):
    """What one case covers: its train-head and weight-gradient instance, the edges it sits on, the fallbacks it proves."""
    p = _path(c, bf16)
    mode = "bf16" if bf16 else "fp32"
    f = {(mode, "train", p[:4]), (mode, "wgrad", p[4:])}
    if bf16:
        if c.engine:
            f.add(("bf16 on head engine", c.engine))
        return f
    f |= {("act", c.act), ("hidden", c.hidden)}
    if c.m % 2 and c.m < 16:
        f.add(("odd m < 16",))
    if p[0] == TRAIN4 and c.m % 128:
        f.add(("partial train4 super tile",))
    if min_cta_iterations(p[0], c.m, SXM_SMS) >= 2:
        f.add(("two grid-stride iterations", p[0]))
    if c.engine and p[0] != (GEMM_HEAD if c.engine == 1 else TRAIN4):
        f.add(("fallback of head engine", c.engine))
    if (c.obs, c.act, c.hidden, c.m) == (376, 17, 256, 32768):
        f.add(("bench",))
    if c.mg != 1:
        f.add(("m_global",))
    if c.ent:
        f.add(("entropy",))
    return f


def _reachable(bf16, head_engine, m_probe=(2, 7, 64, 255, 256, 1000, 32768, 70001)):
    """Every (train instance, wgrad instance) the mirror produces over act 1..64, hidden 1..1024 under head_dims_ok, on GEMM engine 0 (m enters
    only through the GEMM head's scratch gate)."""
    train, wgrad = set(), set()
    for act in range(1, 65):
        for hidden in range(1, 1025):
            if not head_dims_ok(act, hidden):
                continue
            for m in (m_probe if head_engine == 1 and not bf16 else m_probe[:1]):
                p = expected_head_path(32, act, hidden, m, head_engine, 0, bf16)
                train.add(p[:4])
                wgrad.add(p[4:])
    return train, wgrad


def test_case_tables_reach_every_instance_and_each_case_is_needed():
    covered = set()
    for c in FP32_CASES:
        covered |= _features(c, False)
    for c in BF16_CASES:
        covered |= _features(c, True)
    for bf16, engines in ((False, (0, 1, 2)), (True, (0, 1, 2))):
        mode = "bf16" if bf16 else "fp32"
        for e in engines:
            train, wgrad = _reachable(bf16, e)
            missing = {("train", p) for p in train if (mode, "train", p) not in covered}
            missing |= {("wgrad", p) for p in wgrad if (mode, "wgrad", p) not in covered}
            assert not missing, (mode, e, sorted(missing))
    # the wgmma weight gradient (GEMM engine 1) and the edges the tables are built around
    want = {("fp32", "wgrad", (WGRAD_TC, 0)), ("odd m < 16",), ("partial train4 super tile",), ("bench",), ("m_global",), ("entropy",),
            ("fallback of head engine", 1), ("fallback of head engine", 2), ("bf16 on head engine", 1), ("bf16 on head engine", 2)}
    want |= {("act", a) for a in EDGE_ACTS} | {("hidden", h) for h in EDGE_HIDDENS}
    want |= {("two grid-stride iterations", k) for k in (TRAIN, TRAIN2, TRAIN3, TRAIN4)}
    assert want <= covered, sorted(want - covered)
    # no case is redundant: each covers something no other case does
    tables = [(c, False) for c in FP32_CASES] + [(c, True) for c in BF16_CASES]
    for i, (c, bf16) in enumerate(tables):
        others = set()
        for j, (d, bf) in enumerate(tables):
            if j != i:
                others |= _features(d, bf)
        assert _features(c, bf16) - others, ("redundant case", c, bf16)
    for c, bf16 in tables:
        assert head_dims_ok(c.act, c.hidden) and c.m >= 2, c
        assert not bf16 or c.m <= 1000, c  # the autocast oracle runs on the CPU


def test_mirror_gates_at_their_edges():
    """Spot checks of the gates the mirror restates, at the values where they flip."""
    assert head_dims_ok(32, 1024) and not head_dims_ok(33, 1024)
    assert expected_head_path(32, 23, 512, 1000, 2, 0, 0)[:3] == (TRAIN4, 512, 3)
    assert expected_head_path(32, 24, 512, 1000, 2, 0, 0)[:3] == (TRAIN3, 512, 24)   # 251 KB of shared memory > 220 KB
    assert expected_head_path(32, 31, 256, 1000, 2, 0, 0)[:3] == (TRAIN4, 256, 4)
    assert expected_head_path(32, 5, 8, 50, 1, 0, 0)[0] == TRAIN2                     # scratch 1332 floats > m * 2H = 800
    assert expected_head_path(32, 5, 128, 50, 1, 0, 0)[0] == GEMM_HEAD
    assert expected_head_path(32, 5, 128, 1000, 1, 0, 1)[:4] == (TRAIN3, 128, 8, 1)  # bf16: engine 0's kernels
    assert expected_head_path(32, 31, 128, 1000, 0, 1, 0)[4:] == (WGRAD_TC, 0)
    assert expected_head_path(28, 31, 128, 1000, 0, 1, 0)[4:] == (WGRAD3, 32)         # obs 28: not on the tensor engine
    assert expected_head_path(32, 15, 64, 100, 0, 0, 0)[4:] == (WGRAD3, 16) and expected_head_path(32, 16, 64, 100, 0, 0, 0)[4:] == (WGRAD3, 20)
    assert min_cta_iterations(TRAIN4, 67456, SXM_SMS) == 1 and min_cta_iterations(TRAIN4, 67457, SXM_SMS) == 2


# --------------------------------------------------------------------------------------------------- inputs
def _inputs(c, dev, clip=CLIP):
    """_minibatch_case's parameters and minibatch, with the old log-probs set from the float64 new ones: ratio = 1 + u, |u| spread over
    [0.01, 0.45] and kept >= 1e-3 from the clip range, signs random."""
    pol, cri, mb = _minibatch_case(c.obs, c.act, c.hidden, c.m, dev)
    g = np.random.default_rng(c.m + 7)
    mag = g.permutation(np.linspace(0.01, 0.45, c.m))
    near = np.abs(mag - CLIP) < 1e-3
    mag[near] = CLIP + np.where(mag[near] < CLIP, -2e-3, 2e-3)
    u = mag * np.where(g.random(c.m) < 0.5, -1.0, 1.0)
    with torch.no_grad():
        lp64, _ = O.get_logprob_entropy(_f64(pol, dev), mb["states"].to(dev, torch.float64), mb["actions"].to(dev, torch.float64))
    lp64 = lp64.cpu()
    mb["log_probs"] = (lp64 - torch.log1p(torch.from_numpy(u))).float()
    ratio = torch.exp(lp64 - mb["log_probs"].double())
    dev_from_edge = (torch.abs(ratio - 1) - CLIP).abs()
    assert float(dev_from_edge.min()) >= 1e-4, float(dev_from_edge.min())
    return pol, cri, mb, ratio


# --------------------------------------------------------------------------------------------------- GPU runs
@pytest.fixture
def lib():
    from rl_x_b200 import _native as nt
    lib = nt.load()
    yield lib
    lib.rlx_set_head_engine(0)
    lib.rlx_set_gemm_engine(0)
    lib.rlx_set_autocast_bf16(0)


def _head_path(lib):
    out = (C.c_int32 * 6)()
    assert lib.rlx_debug_ppo_head_path(C.addressof(out)) == 0
    return tuple(out)


def _run(lib, c, pol, cri, mb, hp, bf16=False):
    """One rlx_ppo_minibatch_fwdbwd_f32 call with NaN-filled workspace, gradient and metrics: (named float64 gradients, metrics, path)."""
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    assert lib.rlx_set_head_engine(c.engine) == c.engine and lib.rlx_set_gemm_engine(c.gemm) == c.gemm
    assert lib.rlx_set_autocast_bf16(int(bf16)) == int(bf16)
    k = PpoKernels(c.obs, c.act, c.hidden)
    fp = _flat_from_named(k, pol, cri)
    m, P, ldx, nan = c.m, k.param_count, k.states_pitch(), float("nan")
    xs = torch.zeros(m, ldx, device=DEV)
    xs[:, :c.obs] = mb["states"].to(DEV)
    xs[:, c.obs] = 1.0
    d = {n: mb[n].to(DEV).contiguous() for n in NAMES[1:]}
    stats = torch.empty(1, 2, device=DEV)
    k.advantage_stats(d["advantages"], m, m, stats)
    grads, metrics = torch.full((P,), nan, device=DEV), torch.full((8,), nan, device=DEV)
    ws = k.minibatch_workspace(m, DEV)
    ws.view(torch.float32).fill_(nan)
    z = torch.zeros(P, device=DEV)
    args = k.minibatch_args(m=m, m_global=c.mg * m, states=xs, actions=d["actions"], log_probs=d["log_probs"], advantages=d["advantages"],
                            returns=d["returns"], adv_stats=stats, params=fp.flat, grads=grads, exp_avg=z, exp_avg_sq=z,
                            lr=torch.full((1,), 3e-4, device=DEV), step_count=torch.zeros(1, dtype=torch.int64, device=DEV), hp=hp,
                            metrics=metrics, workspace=ws, states_ld=ldx, states_ones_col=True)
    k.fwdbwd(args)
    torch.cuda.synchronize()
    return _named_grads(k, grads), metrics.cpu().numpy(), _head_path(lib), grads


def _assert_path(lib, c, path, bf16):
    want = _path(c, bf16)
    assert path == want, (c, "ran", path, "expected", want)
    if ("two grid-stride iterations", path[0]) in _features(c, bf16):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert min_cta_iterations(path[0], c.m, sms) >= 2, (c, sms)


def _grad_distances(g, g64, norms):
    return {n: float(np.linalg.norm(g[n] - ref)) / norms[n] for n, ref in g64.items()}


def _assert_grads(g, g64, norms):
    """The project's bar: ||g - g64|| <= 1e-5 ||g64|| per tensor (root-sum-square rule for the two last-layer biases: _oracle64)."""
    dist = _grad_distances(g, g64, norms)
    bad = {n: v for n, v in dist.items() if not v <= 1e-5}
    assert not bad, bad
    return dist


def _ref64(c, pol, cri, mb):
    """float64 gradients, norms and losses, divided by m_global as the kernels divide (the oracle takes means over the m rows)."""
    g64, norms, met = _oracle64(pol, cri, mb, c.ent)
    s = 1.0 / c.mg
    return {n: v * s for n, v in g64.items()}, {n: v * s for n, v in norms.items()}, {n: v * s for n, v in met.items()}


def _assert_losses(c, mm, met, adv, ratio):
    s = 1.0 / c.mg
    scale = s * float(torch.abs(adv - adv.mean()).mean() / adv.std())
    assert abs(mm[0] - met["pg_loss"]) <= 1e-5 * max(abs(met["pg_loss"]), scale), (mm[0], met["pg_loss"])
    assert abs(mm[1] - met["critic_loss"]) <= 1e-5 * abs(met["critic_loss"]), (mm[1], met["critic_loss"])
    assert abs(mm[2] - met["entropy_loss"]) <= 1e-5 * abs(met["entropy_loss"]), (mm[2], met["entropy_loss"])
    assert abs(mm[3] - met["approx_kl"]) <= 1e-5 * max(abs(met["approx_kl"]), 1e-2 * s), (mm[3], met["approx_kl"])
    count = int((torch.abs(ratio - 1) > CLIP).sum())
    assert 0 < count < c.m
    want = np.float32(count) * (np.float32(1.0) / np.float32(c.mg * c.m))
    assert mm[4] == want, (mm[4], want, count)
    assert mm[7] == c.m


WORST = {}


@pytest.mark.gpu
@pytest.mark.parametrize("c", FP32_CASES, ids=lambda c: f"{c.obs}-{c.act}-{c.hidden}-{c.m}-e{c.engine}g{c.gemm}")
def test_head_instance_vs_float64(lib, c):
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    pol, cri, mb, ratio = _inputs(c, DEV)
    g64, norms, met = _ref64(c, pol, cri, mb)
    g, mm, path, _ = _run(lib, c, pol, cri, mb, make_hparams(CLIP, c.ent, CRITIC_COEF, MAX_NORM))
    _assert_path(lib, c, path, False)
    dist = _assert_grads(g, g64, norms)
    key = f"head engine {c.engine}, GEMM engine {c.gemm}"
    worst = max(dist, key=dist.get)
    WORST[key] = max(WORST.get(key, (0.0, "")), (dist[worst], f"{worst} at {tuple(c)}"))
    print(f"\n{tuple(c)}: path {path}; worst distance {dist[worst]:.2e} ({worst}); worst so far on {key}: {WORST[key][0]:.2e} ({WORST[key][1]})")
    _assert_losses(c, mm, met, mb["advantages"], ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("c", BF16_CASES, ids=lambda c: f"{c.obs}-{c.act}-{c.hidden}-{c.m}-e{c.engine}")
def test_bf16_head_instance_vs_autocast_oracle(lib, c):
    """test_gpu_bf16.py's oracle and tolerances, at each bf16 instance."""
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    pol, cri, mb, _ = _inputs(c, DEV)
    L = O.Learner(pol, cri, clip_range=CLIP, entropy_coef=c.ent, critic_coef=CRITIC_COEF, bf16=True)
    gp, gc, met = _grads_under_autocast(L, mb)
    g, mm, path, _ = _run(lib, c, pol, cri, mb, make_hparams(CLIP, c.ent, CRITIC_COEF, MAX_NORM), bf16=True)
    _assert_path(lib, c, path, True)
    report = {}
    for name, ref in {**gp, **gc}.items():
        ours = torch.from_numpy(g[name]).float()
        report[name] = float(np.linalg.norm(g[name] - ref.double().numpy()) / max(float(np.linalg.norm(ref.double().numpy())), 1e-30))
        if name != "policy_logstd":
            assert _is_bf16(ours), name
    print(f"\n{tuple(c)} bf16: path {path}; worst distance {max(report.values()):.2e}")
    for name, dist in report.items():
        assert dist <= (5e-2 if name in SUMMED_BIASES else 1e-2), (name, report)
    scale = float(torch.abs(mb["advantages"] - mb["advantages"].mean()).mean() / mb["advantages"].std())
    assert abs(mm[0] - met["pg_loss"]) <= 1e-2 * max(abs(met["pg_loss"]), scale)
    assert abs(mm[1] - met["critic_loss"]) <= 1e-2 * abs(met["critic_loss"])
    assert abs(mm[3] - met["approx_kl"]) <= 1e-2 * max(abs(met["approx_kl"]), 1e-2)
    assert abs(mm[4] - met["clip_fraction"]) <= 0.01 + 2.0 / c.m


ESPO_CASE = Case(24, 5, 128, 1000)  # engine 1: the GEMM head (scratch 19 280 floats <= 256 000); engine 2: train4<128, 1>


@pytest.mark.gpu
@pytest.mark.parametrize("operator", ["mean", "median"])
@pytest.mark.parametrize("engine", [0, 1, 2])
def test_espo_ratio_delta_on_each_head_engine(lib, engine, operator):
    """ESPO's delta_calc_operator (hp.ratio_delta_metric 1 / 2, clip_range = inf): metrics[4] is the mean or the lower median (torch.median)
    of |ratio - 1| over the minibatch, whichever kernel computed the ratios."""
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    c = ESPO_CASE._replace(engine=engine)
    pol, cri, mb, ratio = _inputs(c, DEV)
    _, mm, path, _ = _run(lib, c, pol, cri, mb, make_hparams(float("inf"), 0.0, CRITIC_COEF, MAX_NORM, ratio_delta_metric=operator))
    assert path == _path(c, False) and path[0] == (TRAIN3, GEMM_HEAD, TRAIN4)[engine], path
    delta = torch.abs(ratio - 1)
    ref = float(delta.mean() if operator == "mean" else torch.median(delta))
    assert abs(float(mm[4]) - ref) <= 1e-5 * ref, (engine, operator, float(mm[4]), ref)


@pytest.mark.gpu
def test_call_without_rows_clears_the_record(lib):
    """m == 0 launches no head: the record reads -1 after such a call, not the previous call's kernels."""
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels, make_hparams
    c = Case(16, 8, 128, 1000)
    pol, cri, mb, _ = _inputs(c, DEV)
    _, _, path, _ = _run(lib, c, pol, cri, mb, make_hparams(CLIP, 0.0, CRITIC_COEF, MAX_NORM))
    assert path == _path(c, False)
    k = PpoKernels(c.obs, c.act, c.hidden)
    fp = _flat_from_named(k, pol, cri)
    P = k.param_count
    z = torch.zeros(P, device=DEV)
    args = k.minibatch_args(m=0, m_global=1, states=None, actions=None, log_probs=None, advantages=None, returns=None, adv_stats=None,
                            params=fp.flat, grads=torch.empty(P, device=DEV), exp_avg=z, exp_avg_sq=z, lr=torch.full((1,), 3e-4, device=DEV),
                            step_count=torch.zeros(1, dtype=torch.int64, device=DEV), hp=make_hparams(CLIP, 0.0, CRITIC_COEF, MAX_NORM),
                            metrics=torch.zeros(8, device=DEV), workspace=k.minibatch_workspace(0, DEV))
    k.fwdbwd(args)
    torch.cuda.synchronize()
    assert _head_path(lib) == (-1,) * 6


# ------------------------------------------------------------------------------------------ sensitivity control (CPU)
@pytest.mark.parametrize("c", [max(FP32_CASES, key=lambda c: c.m), max(FP32_CASES, key=lambda c: (c.hidden, c.m))],
                         ids=["largest-m", "widest-hidden"])
def test_comparison_sees_one_row_left_out(c):
    """_assert_grads passes the float64 gradient against itself and rejects the float64 gradient of the same minibatch with its last row left
    out, at the largest m and the widest hidden of the table: the 1e-5 bar resolves one missing row (or lane) there."""
    pol, cri, mb, _ = _inputs(c, "cpu")
    g64, norms, _ = _oracle64(pol, cri, mb, c.ent, dev="cpu")
    _assert_grads(g64, g64, norms)
    g_drop, _, _ = _oracle64(pol, cri, {n: v[:-1] for n, v in mb.items()}, c.ent, dev="cpu")
    dist = _grad_distances(g_drop, g64, norms)
    print(f"\n{tuple(c)}: distance of the gradient without row m - 1, per tensor: " + ", ".join(f"{n} {v:.1e}" for n, v in dist.items()))
    with pytest.raises(AssertionError):
        _assert_grads(g_drop, g64, norms)
