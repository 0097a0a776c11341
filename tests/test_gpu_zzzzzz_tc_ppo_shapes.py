"""The PPO update and rollout forward on the wgmma 3xTF32 engine at the network shapes `tc_supported` (gemm_tc.cu) sends to it besides
the benchmark's (hidden % 128 == 0, 128 <= hidden <= 1024, obs % 4 == 0, obs >= 32), against float64 autograd of oracle/ppo_oracle.py and
against the exact-fp32 SIMT engine on the same fp32 inputs.  The float64 reference runs on the GPU (ATen double kernels) to keep the
large shapes fast.

Each shape pins a coordinate the engine gets wrong only at some widths: batch-2 operands at column / row offsets (the net halves of H1 / dZ2,
W2 and its pre-split copies), split-K partials with a ragged last chain, the transposed dW1 | db1 store whose extra row goes to its own
buffer once per split, the head weight-gradient GEMM with M = dh_ld of 4 to 32, and tf32_split jobs of 2H x obs and 2 x H x H.

Proof of path.  `run_gemm` falls back to the SIMT engine without a word when the wgmma engine returns RLX_ERR_UNSUPPORTED, and a SIMT
result passes every numeric bound here.  So the tests read back which GEMM kernels each engine-1 call launched, from the library's
host-side launch counters (rlx_gemm_path_count): the tc_gemm_kernel instances by their template arguments, tf32_split_kernel, and no
sgemm_kernel.  (torch.profiler is not used for this: one of its sessions came back with no kernel record at all on an H100, so the exact
counts asserted here cannot rest on it.)  Outputs start as NaN, so an element no kernel wrote fails the numeric checks.

Bounds, per gradient tensor g, with g64 the float64 oracle's gradient at the same parameters and minibatch (for the two last-layer
biases, ||g64|| stands for the root-sum-square of their per-row terms where that is larger; see _oracle64):
  (i)  ||g - g64|| <= 1e-5 ||g64|| for both engines, the project's bar;
  (ii) ||g_tc - g64|| <= 2 ||g_simt - g64|| + F ||g64||.
Derivation of (ii).  Both engines run the same fp32 program except for the GEMMs, so g_tc - g64 = (g_simt - g64) + (E_tc - E_simt), where
E_x is the part of the gradient error that engine x's GEMM roundings cause.  E_simt is part of the SIMT engine's whole error:
||E_simt|| <= ||g_simt - g64|| (independent rounding errors do not cancel systematically), hence the factor 2.  test_gpu_tc_engine.py
bounds one 3xTF32 product at e(K) = 6e-7 + 3.2e-9 K of the output's norm, K the length of one accumulation chain; the update keeps each
chain <= 1024 rows (choose_splits), so a weight-gradient product has K <= min(m, 1024).  A gradient tensor depends on at most four
products: forward layer 1 (K = obs), forward layer 2 (K = hidden), the dX product (K = hidden) and its own weight-gradient product.  An
output error of relative size e in one of them reaches the gradient with a gain of order one (tanh' <= 1, the products downstream are
linear in it), so ||E_tc|| <= F ||g64|| with
    F = e(obs) + 2 e(hidden) + e(min(m, 1024)),
from 6.6e-6 at (32, 1, 128, 1000) to 1.3e-5 at (376, 17, 1024, 4096), where (i) is the tighter bound.  Single-pass TF32 (2^-11 per
operand, about 5e-4 per product) misses both.
Forward quantities: the per-element tolerances of test_gpu_parity.py's test_forward_vs_oracle.  Losses: its scale rules.

Sorted after the other GPU files: a kernel fault on a new shape takes the CUDA context with it, and then costs only this file."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from test_gpu_parity import _flat_from_named, _random_minibatch, _run_fwdbwd

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = ("states", "actions", "log_probs", "advantages", "returns")
CLIP, ENT, CRITIC_COEF, MAX_NORM = 0.2, 0.01, 0.5, 0.5

# (obs, act, hidden, m) on the tensor engine; dh_ld = act + 1 rounded up to 4 is the M of the head weight-gradient GEMM
TC_SHAPES = [
    (32, 1, 128, 1000),     # smallest accepted obs and hidden; one k-block in layer 1; dW1 M = 33; dh_ld = 4
    (124, 3, 128, 4099),    # the extra (db1) row inside an edge tile; ragged last split chain
    (128, 4, 384, 2048),    # the extra row alone in the second M tile (M = 129); hidden not a power of two; dh_ld = 8
    (380, 31, 512, 3000),   # M = 381; act at the fast_head_ok limit (dh_ld = 32)
    (64, 32, 256, 1500),    # act 32: the head wgrad leaves the tensor engine, the other GEMMs stay on it
    (376, 17, 1024, 4096),  # widest hidden: 2H = 2048, the largest tf32_split jobs
    (256, 8, 640, 33),      # m < 64: one split, a reduction of 33 rows (2 k-blocks, the second mostly zero fill)
    (1024, 6, 256, 8192),   # layer-1 K = 1024 (32 k-blocks); dW1 M = 1025 (9 tiles)
]
# shapes tc_supported rejects: engine 1 must run them on the SIMT engine alone
SIMT_SHAPES = [
    (28, 3, 128, 500),      # obs below 32
    (36, 3, 192, 500),      # hidden not a multiple of 128
]

# tc_gemm_kernel<A_KMAJ, B_KMAJ, EPI, BF16, TRANS, SPLIT_B> instances (EPI 0 none, 1 bias + tanh, 2 tanh')
FWD_PRESPLIT = (True, True, 1, False, False, True)   # update, layers 1 and 2: B = tf32_split's copies of W1cat / W2
DX_PRESPLIT = (True, True, 2, False, False, True)    # update, dZ1 = (dZ2 W2) * tanh': B = the copies of W2^T
DW = (False, False, 0, False, False, False)          # update, dW2 and the head's dW3 | dw3c
DW1_T = (False, False, 0, False, True, False)        # update, dW1 | db1 stored transposed
FWD_CONVERT = (True, True, 1, False, False, False)   # rollout / critic forward: B split by the converter warpgroup
# rlx_gemm_path_count slots after the 256 tc_gemm_kernel instances (include/rlx_b200.h)
GP_TF32_SPLIT, GP_SGEMM, GP_HEAD_WGRAD_SIMT, GP_SLOTS = 256, 257, 258, 259


@pytest.fixture(autouse=True)
def lib():
    """The native library; the GEMM engine is back at 0 (SIMT) after every test whatever it left."""
    from rl_x_b200 import _native as nt
    lib = nt.load()
    yield lib
    lib.rlx_set_gemm_engine(0)


def _engine(lib, engine):
    assert lib.rlx_set_gemm_engine(engine) == engine


def _kern(obs, act, hidden):
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(obs, act, hidden)


def _hp(ent):
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    return make_hparams(CLIP, ent, CRITIC_COEF, MAX_NORM)


def _f64(d, dev=DEV):
    return {n: v.detach().to(dev, torch.float64) for n, v in d.items()}


SUMMED_BIASES = ("policy_mean.4.bias", "critic.4.bias")


def _oracle64(pol, cri, mb, ent, dev=DEV):
    """oracle.Learner.grads in float64: (gradients as float64 numpy arrays by parameter name, the norm each is measured against, losses).

    The norm is ||g64||, except for the two last-layer biases: their gradients are sums of m signed per-row terms that largely cancel (the
    critic's is critic_coef * mean(value - return)), while every term carries the fp32 rounding of the forward pass.  Those errors add in
    quadrature, so they are measured against the root-sum-square of the terms when it is larger (the rule test_gpu_bf16.py applies to the
    same two tensors, and test_gpu_parity.py to pg_loss).  The shape that needs it is (32, 1, 128, 1000), where the root-sum-square is 60x
    / 100x ||g64||: there even plain fp32 autograd (the oracle on the CPU) sits at 1.05e-5 / 1.18e-5 of ||g64|| for the policy / critic
    bias, and the tensor engine's critic bias at 3.0e-5 (SIMT 5.7e-6; measured on an H100).  The test prints both distances of both
    engines.  The terms are the gradients of row-wise copies of the bias ([m, out]; F.linear adds a
    bias broadcast to its output), which sum to the gradient itself."""
    m = mb["states"].shape[0]
    pol64, cri64 = _f64(pol, dev), _f64(cri, dev)
    pol64["policy_mean.4.bias"] = pol64["policy_mean.4.bias"].expand(m, -1).clone()
    cri64["critic.4.bias"] = cri64["critic.4.bias"].expand(m, -1).clone()
    L = O.Learner(pol64, cri64, clip_range=CLIP, entropy_coef=ent, critic_coef=CRITIC_COEF)
    gp, gc, met = L.grads(*(mb[n].to(dev, torch.float64) for n in NAMES))
    g = {n: v.cpu().numpy() for n, v in {**gp, **gc}.items()}
    norms = {n: float(np.linalg.norm(v)) for n, v in g.items()}
    for n in SUMMED_BIASES:
        terms = g[n]
        g[n] = terms.sum(0)
        norms[n] = max(float(np.linalg.norm(g[n])), float(np.linalg.norm(np.sqrt((terms ** 2).sum(0)))))
    return g, {n: max(v, 1e-30) for n, v in norms.items()}, met


def _named_grads(k, grads):
    from rl_x_b200.algorithms.ppo.b200.ppo import FlatParameters
    gflat = FlatParameters(k, DEV)
    gflat.flat.copy_(grads)
    gpol, gcri = gflat.state_dicts()
    return {n: v.numpy().astype(np.float64) for n, v in {**gpol, **gcri}.items()}


def _minibatch_case(obs, act, hidden, m, dev=DEV):
    """Seeded parameters and minibatch as test_gpu_parity.py's test_minibatch_gradients_vs_oracle_autograd builds them: old log-probs near
    the policy's, so that the ratios straddle the clip range."""
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.9, seed=m)
    g = torch.Generator().manual_seed(m + 1)
    for w in list(pol.values()) + list(cri.values()):
        w.add_(0.02 * torch.randn(w.shape, generator=g))
    mb = _random_minibatch(obs, act, m, seed=m + 2)
    mb["log_probs"] = _logp64(pol, mb, dev) + 0.15 * torch.randn(m, generator=g)
    return pol, cri, mb


def _logp64(pol, mb, dev=DEV):
    with torch.no_grad():
        lp, _ = O.get_logprob_entropy(_f64(pol, dev), mb["states"].to(dev, torch.float64), mb["actions"].to(dev, torch.float64))
    return lp.float().cpu()


def _paths(lib, fn):
    """(fn(), launches of each GEMM path during fn) from the library's own counters (rlx_gemm_path_count): every launch is counted on the
    host where the library issues it, so the record is complete and the same on every run."""
    torch.cuda.synchronize()
    lib.rlx_reset_gemm_path_counts()
    out = fn()
    torch.cuda.synchronize()
    counts = {s: int(lib.rlx_gemm_path_count(s)) for s in range(GP_SLOTS)}
    return out, {s: c for s, c in counts.items() if c}


def _tc_instances(counts):
    """Launch counts of the tc_gemm_kernel instances, keyed by their template arguments (slot = A_KMAJ | B_KMAJ << 1 | EPI << 2 | BF16 << 5 |
    TRANS << 6 | SPLIT_B << 7)."""
    return {(bool(s & 1), bool(s & 2), (s >> 2) & 7, bool(s & 32), bool(s & 64), bool(s & 128)): c for s, c in counts.items() if s < 256}


def _assert_update_path(counts, head_on_tc):
    want = {FWD_PRESPLIT: 2, DX_PRESPLIT: 1, DW1_T: 1, DW: 2 if head_on_tc else 1}
    assert _tc_instances(counts) == want, (_tc_instances(counts), want, counts)
    assert counts.get(GP_TF32_SPLIT, 0) == 1, counts
    assert counts.get(GP_SGEMM, 0) == 0, counts
    # the head weight gradient: the second DW launch, or (act > 31, no fast head) the SIMT kernel of the generic head
    assert counts.get(GP_HEAD_WGRAD_SIMT, 0) == (0 if head_on_tc else 1), counts


def _run(k, lib, engine, pol, cri, mb, ent):
    """One minibatch forward + backward on `engine`: (named float64 gradients, metrics, GEMM path counts, flat gradient)."""
    _engine(lib, engine)
    fp = _flat_from_named(k, pol, cri)
    (_, grads, metrics, _, _), counts = _paths(lib, lambda: _run_fwdbwd(k, fp, mb, _hp(ent)))
    return _named_grads(k, grads), metrics.cpu().numpy(), counts, grads


def _assert_losses(mm, met, adv, m):
    """test_gpu_parity.py's scale rules: pg_loss is a mean of signed terms with a near-zero mean, so its norm is the summand scale."""
    scale = float(torch.abs(adv - adv.mean()).mean() / adv.std())
    assert abs(mm[0] - met["pg_loss"]) <= 1e-5 * max(abs(met["pg_loss"]), scale), (mm[0], met["pg_loss"])
    assert abs(mm[1] - met["critic_loss"]) <= 1e-5 * abs(met["critic_loss"]), (mm[1], met["critic_loss"])
    assert abs(mm[2] - met["entropy_loss"]) <= 1e-5 * abs(met["entropy_loss"]), (mm[2], met["entropy_loss"])
    assert abs(mm[3] - met["approx_kl"]) <= 1e-5 * max(abs(met["approx_kl"]), 1e-2), (mm[3], met["approx_kl"])
    assert abs(mm[4] - met["clip_fraction"]) <= 1.5 / m, (mm[4], met["clip_fraction"])  # a ratio within 1e-7 of the clip edge may flip
    assert mm[7] == m


def _dist(a, ref):
    return float(np.linalg.norm(a - ref))


def _gemm_err(K):
    """test_gpu_tc_engine.py's error model of one 3xTF32 product, relative to the output's norm, chains capped at 1024 rows."""
    return 6e-7 + 3.2e-9 * min(K, 1024)


# ------------------------------------------------------------------------------------------- minibatch fwd + bwd
@pytest.mark.parametrize("obs,act,hidden,m", TC_SHAPES)
def test_minibatch_on_tensor_engine_vs_float64(lib, obs, act, hidden, m):
    k = _kern(obs, act, hidden)
    pol, cri, mb = _minibatch_case(obs, act, hidden, m)
    g64, norms, met = _oracle64(pol, cri, mb, ENT)
    g_simt, mm_simt, paths_simt, _ = _run(k, lib, 0, pol, cri, mb, ENT)
    g_tc, mm_tc, paths_tc, _ = _run(k, lib, 1, pol, cri, mb, ENT)
    assert _tc_instances(paths_simt) == {} and paths_simt.get(GP_SGEMM, 0) > 0, paths_simt
    _assert_update_path(paths_tc, head_on_tc=act <= 31)
    floor = _gemm_err(obs) + 2 * _gemm_err(hidden) + _gemm_err(m)
    report = {}
    for name, ref in g64.items():
        n64 = norms[name]
        d_tc, d_simt = _dist(g_tc[name], ref), _dist(g_simt[name], ref)
        report[name] = (d_tc / n64, d_simt / n64)
        assert d_simt <= 1e-5 * n64, (name, "simt", d_simt / n64)
        assert d_tc <= 1e-5 * n64, (name, "tc", d_tc / n64)
        assert d_tc <= 2 * d_simt + floor * n64, (name, d_tc / n64, d_simt / n64, floor)
    worst_tc, worst_simt = max(v[0] for v in report.values()), max(v[1] for v in report.values())
    print(f"\n({obs}, {act}, {hidden}, {m}): worst distance to float64 / norm: tc {worst_tc:.2e}  simt {worst_simt:.2e}  (F = {floor:.2e})")
    for name in SUMMED_BIASES:  # the same two distances against the plain ||g64||
        ref, plain = g64[name], max(float(np.linalg.norm(g64[name])), 1e-30)
        print(f"  {name}: / ||g64||: tc {_dist(g_tc[name], ref) / plain:.2e}  simt {_dist(g_simt[name], ref) / plain:.2e};"
              f"  rss of terms / ||g64|| = {norms[name] / plain:.1f}")
    _assert_losses(mm_simt, met, mb["advantages"], m)
    _assert_losses(mm_tc, met, mb["advantages"], m)


@pytest.mark.parametrize("obs,act,hidden,m", SIMT_SHAPES)
def test_shapes_outside_the_tensor_engine_run_simt_only(lib, obs, act, hidden, m):
    """rlx_set_gemm_engine(1) is a preference: use_tc() keeps a shape tc_supported rejects on the SIMT engine, with no error, and the result
    is the SIMT engine's to the bit."""
    k = _kern(obs, act, hidden)
    pol, cri, mb = _minibatch_case(obs, act, hidden, m)
    g64, norms, met = _oracle64(pol, cri, mb, ENT)
    _, _, _, flat_simt = _run(k, lib, 0, pol, cri, mb, ENT)
    g_tc, mm_tc, paths, flat_tc = _run(k, lib, 1, pol, cri, mb, ENT)
    assert _tc_instances(paths) == {} and paths.get(GP_TF32_SPLIT, 0) == 0, paths
    assert paths.get(GP_SGEMM, 0) > 0, paths
    assert torch.equal(flat_tc, flat_simt)
    for name, ref in g64.items():
        assert _dist(g_tc[name], ref) <= 1e-5 * norms[name], (name, _dist(g_tc[name], ref) / norms[name])
    _assert_losses(mm_tc, met, mb["advantages"], m)


# --------------------------------------------------------------------------------------------- multi-minibatch epoch
@pytest.mark.parametrize("obs,act,hidden,mb", [(128, 4, 384, 2048), (380, 31, 512, 3000)])
def test_epoch_gradients_follow_the_weights(lib, obs, act, hidden, mb):
    """Three minibatches through rlx_ppo_update_epoch_f32 on the tensor engine, as test_one_epoch_at_bench_shape_vs_oracle runs them: before
    each step the oracle is evaluated in float64 at OUR current weights, so minibatch i's gradient must follow the weights Adam wrote at step
    i - 1 (pre-split copies that missed an update would not).  The same epoch as one call must then leave the same weights, Adam moments,
    metrics and last gradient, to the bit: it runs the same kernels in the same order."""
    nmb = 3
    B = mb * nmb
    _engine(lib, 1)
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, seed=obs)
    data = _random_minibatch(obs, act, B, seed=obs + 1)
    data["log_probs"] = _logp64(pol, data) + 0.1 * torch.randn(B, generator=torch.Generator().manual_seed(obs + 2))
    ldx = k.states_pitch()
    xs = torch.zeros(B, ldx, device=DEV)
    xs[:, :obs] = data["states"].to(DEV)
    xs[:, obs] = 1.0
    d = {n: data[n].to(DEV).contiguous() for n in NAMES[1:]}
    stats = torch.empty(nmb, 2, device=DEV)
    k.advantage_stats(d["advantages"], B, mb, stats)
    P = k.param_count

    def start():
        fp = _flat_from_named(k, pol, cri)
        st = dict(grads=torch.zeros(P, device=DEV), exp_avg=torch.zeros(P, device=DEV), exp_avg_sq=torch.zeros(P, device=DEV),
                  lr=torch.full((1,), 3e-4, device=DEV), step=torch.zeros(1, dtype=torch.int64, device=DEV),
                  metrics=torch.zeros(nmb, 8, device=DEV), ws=k.minibatch_workspace(mb, DEV))
        return fp, st

    def args(fp, st, i, rows):
        sl = slice(i * mb, i * mb + rows)
        return k.minibatch_args(m=0, m_global=1, states=xs[sl], actions=d["actions"][sl], log_probs=d["log_probs"][sl], advantages=d["advantages"][sl],
                                returns=d["returns"][sl], adv_stats=stats[i], params=fp.flat, grads=st["grads"], exp_avg=st["exp_avg"],
                                exp_avg_sq=st["exp_avg_sq"], lr=st["lr"], step_count=st["step"], hp=_hp(0.0), metrics=st["metrics"][i],
                                workspace=st["ws"], states_ld=ldx, states_ones_col=True)

    fp, st = start()
    report = []
    for i in range(nmb):
        sl = slice(i * mb, (i + 1) * mb)
        pol_now, cri_now = fp.state_dicts()
        g64, norms, met = _oracle64(pol_now, cri_now, {n: data[n][sl] for n in NAMES}, 0.0)
        _, paths = _paths(lib, lambda: k.update_epoch(args(fp, st, i, mb), mb, mb))  # one minibatch: forward, loss, backward, clip, Adam
        _assert_update_path(paths, head_on_tc=True)
        ours = _named_grads(k, st["grads"])
        dist = {n: _dist(ours[n], ref) / norms[n] for n, ref in g64.items()}
        report.append(max(dist.values()))
        assert max(dist.values()) <= 1e-5, (i, dist)
        _assert_losses(st["metrics"][i].cpu().numpy(), met, data["advantages"][sl], mb)
    print(f"\nepoch ({obs}, {act}, {hidden}, mb {mb}): worst gradient distance to float64 per minibatch: {report}")
    assert int(st["step"].item()) == nmb

    fp1, st1 = start()
    k.update_epoch(args(fp1, st1, 0, B), B, mb)
    torch.cuda.synchronize()
    assert int(st1["step"].item()) == nmb
    for key in ("grads", "exp_avg", "exp_avg_sq", "metrics"):
        assert torch.equal(st1[key], st[key]), key
    assert torch.equal(fp1.flat, fp.flat)


# ------------------------------------------------------------------------------------------------- rollout forward
@pytest.mark.parametrize("n", [1, 63, 4097])
@pytest.mark.parametrize("obs,act,hidden", [(32, 1, 128), (128, 4, 384), (376, 17, 1024)])
def test_rollout_forward_on_tensor_engine_vs_float64(lib, obs, act, hidden, n):
    """rlx_ppo_forward_f32 (explicit noise, then deterministic) and rlx_critic_forward_f32 on both engines against float64.  The rollout
    takes the converter instances (B split per tile): it has no pre-split copies."""
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.8, seed=obs + n)
    g = torch.Generator().manual_seed(n)
    for w in list(pol.values()) + list(cri.values()):
        w.add_(0.05 * torch.randn(w.shape, generator=g))  # non-zero biases / logstd
    x = torch.randn(n, obs, generator=g)
    noise = torch.randn(n, act, generator=g)
    low, high = torch.full((act,), -2.0), torch.full((act,), 0.5)
    dd = lambda t: t.to(DEV, torch.float64)
    with torch.no_grad():
        pol64, cri64 = _f64(pol), _f64(cri)
        a_ref, e_ref, lp_ref = (t.cpu() for t in O.get_action_logprob(pol64, dd(x), dd(noise), dd(low), dd(high)))
        v_ref = O.critic_value(cri64, dd(x)).reshape(-1).cpu()
        d_ref = O.get_deterministic_action(pol64, dd(x), dd(low), dd(high)).cpu()
    fp = _flat_from_named(k, pol, cri)
    ws = k.forward_workspace(n, DEV)
    xd, nd, lo, hi = x.to(DEV), noise.to(DEV), low.to(DEV), high.to(DEV)
    # 1e-5 relative to the scale of each quantity (elementwise: rtol on the value + the same fraction of the tensor's rms)
    tol = lambda ref: dict(rtol=1e-5, atol=1e-5 * float(ref.pow(2).mean().sqrt()))
    rel = lambda a, ref: float(np.linalg.norm(a.double().numpy() - ref.numpy()) / max(float(ref.norm()), 1e-30))
    for engine in (0, 1):
        _engine(lib, engine)
        a, e, d = (torch.full((n, act), float("nan"), device=DEV) for _ in range(3))
        lp, v, v2 = (torch.full((n,), float("nan"), device=DEV) for _ in range(3))

        def run():
            k.forward(fp.flat, xd, ws, noise=nd, act_low=lo, act_high=hi, action=a, env_action=e, logp=lp, value=v)
            k.forward(fp.flat, xd, ws, act_low=lo, act_high=hi, deterministic=True, env_action=d)
            k.critic_forward(fp.flat, xd, v2, ws)

        _, paths = _paths(lib, run)
        if engine == 1:
            assert _tc_instances(paths) == {FWD_CONVERT: 6}, paths  # 2 layers x 3 calls
            assert paths.get(GP_SGEMM, 0) == 0 and paths.get(GP_TF32_SPLIT, 0) == 0, paths
        else:
            assert _tc_instances(paths) == {} and paths.get(GP_SGEMM, 0) == 6, paths
        a, e, lp, v, d, v2 = (t.cpu() for t in (a, e, lp, v, d, v2))
        for ours, ref in ((a, a_ref), (e, e_ref), (lp, lp_ref), (v, v_ref), (d, d_ref)):
            np.testing.assert_allclose(ours.double().numpy(), ref.numpy(), **tol(ref), err_msg=f"engine {engine}")
        assert rel(a, a_ref) < 5e-6 and rel(v, v_ref) < 5e-6, (engine, rel(a, a_ref), rel(v, v_ref))
        assert torch.equal(v2, v)
