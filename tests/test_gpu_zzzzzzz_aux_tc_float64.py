"""The FastSAC and FastTD3 updates and acting kernels on both GEMM engines of `aux_gemm` (csrc/dual_build.cuh) against the project's own oracles
(oracle/fastsac_oracle.py, oracle/fasttd3_oracle.py) run in float64, at batches of one to thirty-two weight-gradient splits, with a count of
the GEMM kernels each call launched.

Why.  The golden batches of test_gpu_zzzz_fastsac.py / test_gpu_zzzzz_fasttd3.py have 16 rows and aux_gemm needs M, N >= 64, so they run the
SIMT engine whatever the switch says; their batch-1024 tests compare the engines with each other at one shape (one weight-gradient split).
Here every case runs both engines from the same state, in a NaN-filled workspace of exactly rlx_*_workspace_bytes and with NaN-filled
gradient buffers: an element no kernel wrote, or a pad column of the padded [s | a] pitch that a kernel read, fails the numeric checks.

Proof of path.  aux_gemm falls back to the SIMT engine without a word when the wgmma engine returns RLX_ERR_UNSUPPORTED.  This file restates
the gate (`on_tensor_engine`) and lists the GEMMs each entry point issues (`td3_gemms`, `sac_gemms`, written from fasttd3.cu, fastsac.cu and
c51_ops.cuh), derives how many launches each tc_gemm_kernel instance and the SIMT GEMM must show, and asserts equality with the library's
launch counters (rlx_gemm_path_count) around every call.  The table is what the code should do: both critics take the same path.  Critic 2
sits at q_params + nq with nq % 4 == nr_atoms % 4, so with 101 atoms none of its weights is 16-byte aligned in place; the plugins read it
through an aligned copy (c51_ops.cuh: aligned_params).  `in_place=True` derives what reading it in place would give: the host test below
shows that this is half of the critics' weight-operand GEMMs on the SIMT engine.

The ReLU flip.  FastTD3's networks are piecewise linear: a hidden unit whose pre-activation is within fp32 noise of zero takes opposite sides in
two computations, which switches that row's backward path through the unit (1e-3 of a critic's gradient for one unit, measured by
test_gpu_zzzzz_fasttd3.py).  The clipped double-Q selection (q1_next < q2_next, v1 < v2) is the same kind of discontinuity.  Instead of a wide
bar, the batches avoid it: about twice the rows are drawn, the float64 forward of every network the update differentiates through gives
each row's smallest |pre-activation| relative to the rms of its layer in that row, rows under RELU_MARGIN (and rows whose two values are closer than
VALUE_MARGIN) are dropped, and the first n survivors are the batch.  FastSAC (LayerNorm + SiLU) is smooth and needs no filter; it runs
with its default, the mean of the two values.

Bounds, per parameter tensor g of a network (never one norm over the concatenation, where a small tensor hides), g64 the float64 gradient:
  (i)  ||g - g64|| <= BAR ||g64|| on both engines;
  (ii) ||g_tc - g64|| <= 2 ||g_simt - g64|| + F ||g64||.
(ii) is test_gpu_zzzzzz_tc_ppo_shapes.py's: the engines run the same fp32 program except for the GEMMs, and one 3xTF32 product is within
e(K) = 6e-7 + 3.2e-9 K of its output's norm (test_gpu_tc_engine.py), K <= 1024 per accumulation chain.  A gradient tensor depends on a
chain of products whose errors reach it with a gain of order one (ReLU' and tanh' <= 1, LayerNorm and SiLU' of order one), so F is the sum
of e(K) over the chain.  Critic update: policy forward (4), target forward (4), online forward (4), input gradients (3), the weight
gradient (1).  Policy update: policy forward (4), critic forward (4), critic input gradients (4), policy input gradients (3), the weight
gradient (1).  That is 16 products, F = 2.5e-5 to 3.4e-5 (`_floor`; the 1024- and 512-wide layers weigh most).  Measured on an H100 (80 GB HBM3, 700 W): the
worst tensor of any case is 8.2e-6 on the SIMT engine and 1.0e-5 on the tensor engine (FastSAC: 4.1e-6 and 4.5e-6), so BAR = 2e-5 is the bound that bites and (ii) guards
the tensor engine where the SIMT engine happens to sit very close to float64 (the policy update: 5e-7 - 7e-7).  Linear-layer bias gradients are sums of n signed per-row terms that can
largely cancel while each term carries its own rounding: they are measured against the root-sum-square of the terms where that is larger
than ||g64|| (the rule of the PPO file).  After the AdamW step the parameters and the polyak targets are compared per network at PARAM_BAR:
Adam's first step is lr * g / (|g| + eps), the sign of g, so one element whose gradient is within rounding of zero moves by 2 lr whatever
the engine - a per-tensor bar on a 17-element zero-initialised bias would measure that element alone.

Sorted after the other GPU files: a kernel fault on a new shape takes the CUDA context with it, and then costs only this file."""
import collections
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import fastsac_oracle as FS
from oracle import fasttd3_oracle as TD

gpu = pytest.mark.gpu
DEV = "cuda"
RELU_MARGIN, VALUE_MARGIN = 1e-4, 1e-4
BAR, PARAM_BAR = 2e-5, 3e-5
LR = 3e-4

# ----------------------------------------------------------------------------------------------- the gate, restated
TC_NONE, TC_BIAS_TANH, TC_DTANH, TC_BIAS_RELU, TC_DRELU, TC_BIAS = range(6)   # gemm_tc_common.cuh: TcEpi
# (A_KMAJ, B_KMAJ, epilogue) of the fp32 tc_gemm_kernel instances tc_gemm_impl can launch without a pre-split B
INSTANCES = {(1, 1, TC_BIAS_TANH), (1, 1, TC_NONE), (1, 1, TC_BIAS_RELU), (1, 1, TC_BIAS), (1, 0, TC_DRELU), (1, 0, TC_DTANH), (1, 0, TC_NONE),
             (0, 0, TC_NONE)}
GP_SGEMM = 257          # rlx_gemm_path_count slot of the SIMT GEMM (common.cuh)
WGRAD_ROWS = 1024       # c51_ops.cuh: kWgradRows
TC_BK = 32              # gemm_tc_common.cuh: BK

# One GEMM as aux_gemm sees it.  a / b / c: offsets (in floats) of the operand bases from a 16-byte aligned allocation.
Gemm = collections.namedtuple("Gemm", "name a_kmaj b_kmaj epi M N K lda ldb ldc a b c splits split_c")


def on_tensor_engine(g):
    """aux_gemm's size gate, tc_gemm_impl's base / pitch / split checks, and the instances that exist."""
    gate = g.M >= 64 and g.N >= 64 and g.K >= 32
    bases = all(v % 4 == 0 for v in (g.a, g.b, g.c, g.lda, g.ldb, g.ldc))
    split = g.splits == 1 or (WGRAD_ROWS % TC_BK == 0 and g.split_c % 2 == 0)
    return gate and bases and split and (g.a_kmaj, g.b_kmaj, g.epi) in INSTANCES


def tc_slot(g):
    """common.cuh: tc_path_slot(a_kmaj, b_kmaj, epi, bf16 = 0, trans = 0, split_b = 0)."""
    return g.a_kmaj | g.b_kmaj << 1 | g.epi << 2


def derive_paths(gemms, engine):
    """{rlx_gemm_path_count slot: launches} a list of GEMMs must leave behind on `engine`."""
    want = collections.Counter()
    for g in gemms:
        want[tc_slot(g) if engine == 1 and on_tensor_engine(g) else GP_SGEMM] += 1
    return dict(want)


def _fwd(name, n, inp, out, epi, w, ldx=None, ldw=None, x=0):   # c51_ops.cuh: lin_fwd
    return Gemm(name, 1, 1, epi, n, out, inp, ldx or inp, ldw or inp, out, x, w, 0, 1, 0)


def _dx(name, n, inp, out, epi, w, ldw=None):                    # lin_bwd_input: dX[n, in] = dY[n, out] W[out, in]
    return Gemm(name, 1, 0, epi, n, inp, out, out, ldw or inp, inp, 0, w, 0, 1, 0)


def _dw(name, n, inp, out, ldx=None, ldc=None):                  # lin_bwd_weight: dW[out, in] = dY^T X, split over rows
    return Gemm(name, 0, 0, TC_NONE, out, inp, n, out, ldx or inp, ldc or inp, 0, 0, 0, -(-n // WGRAD_ROWS), (ldc or inp) * out)


def mlp_offsets(inp, widths, out):
    """fasttd3.cu: mlp_layout - weight, bias per layer, nothing rounded."""
    off, o = [], 0
    for w in tuple(widths) + (out,):
        off += [o, o + w * inp]
        o += w * inp + w
        inp = w
    return off + [o]


def sac_offsets(inp, widths, heads):
    """fastsac.cu: make_layout - Linear weight, bias, LayerNorm weight, bias per torso block, then (weight, bias) per head."""
    off, o = [], 0
    for w in widths:
        for sz in (w * inp, w, w, w):
            off.append(o)
            o += sz
        inp = w
    for h in heads:
        off += [o, o + h * inp]
        o += h * inp + h
    return off + [o]


def td3_gemms(obs, act, atoms, n, entry, in_place=False):
    """The GEMMs of rlx_fasttd3_{critic_update,policy_update,act}_f32 in issue order."""
    PW, QW = TD.POLICY_WIDTHS, TD.Q_WIDTHS
    po, qo = mlp_offsets(obs, PW, act), mlp_offsets(obs + act, QW, atoms)
    nq, pitch = qo[-1], -(-(obs + act) // 4) * 4

    def mlp_fwd(tag, off, widths, inp, out, head_epi, base, ldx, w1, ldw1):
        dims = (inp,) + tuple(widths)
        g = [_fwd(f"{tag}.fwd0", n, inp, widths[0], TC_BIAS_RELU, w1, ldx, ldw1)]
        g += [_fwd(f"{tag}.fwd{k}", n, dims[k], widths[k], TC_BIAS_RELU, base + off[2 * k]) for k in (1, 2)]
        return g + [_fwd(f"{tag}.fwd3", n, widths[2], out, head_epi, base + off[6])]

    def mlp_bwd(tag, off, widths, inp, out, base, ldx):
        g = [_dw(f"{tag}.dw3", n, widths[2], out), _dx(f"{tag}.dx3", n, widths[2], out, TC_DRELU, base + off[6])]
        for k in (2, 1, 0):
            if k > 0:
                g += [_dw(f"{tag}.dw{k}", n, widths[k - 1], widths[k]), _dx(f"{tag}.dx{k}", n, widths[k - 1], widths[k], TC_DRELU, base + off[2 * k])]
            else:
                g.append(_dw(f"{tag}.dw0", n, inp, widths[0], ldx, ldx))   # at the row pitch of X, reduced to the unpadded gradient afterwards
        return g

    pol_fwd = mlp_fwd("pol", po, PW, obs, act, TC_BIAS_TANH, 0, obs, po[0], obs)
    q_base = lambda q: q * nq % 4 if in_place else 0                       # aligned_params: an aligned copy when the block is not
    q_fwd = lambda q, tag: mlp_fwd(f"{tag}{q + 1}", qo, QW, obs + act, atoms, TC_BIAS, q_base(q), pitch, 0, pitch)   # layer 1: the staged padded copy
    if entry == "act":
        return pol_fwd
    if entry == "critic":
        g = pol_fwd + q_fwd(0, "qt") + q_fwd(1, "qt")
        for q in (0, 1):
            g += q_fwd(q, "q") + mlp_bwd(f"q{q + 1}", qo, QW, obs + act, atoms, q_base(q), pitch)
        return g
    g = pol_fwd + q_fwd(0, "q") + q_fwd(1, "q")
    for q in (0, 1):
        g.append(_dx(f"q{q + 1}.dx3", n, QW[2], atoms, TC_DRELU, q_base(q) + qo[6]))
        g += [_dx(f"q{q + 1}.dx{k}", n, QW[k - 1], QW[k], TC_DRELU, q_base(q) + qo[2 * k]) for k in (2, 1)]
        g.append(_dx(f"q{q + 1}.dx0_actions", n, act, QW[0], TC_NONE, q_base(q) + qo[0] + obs, obs + act))   # the action block of W1, read in place
    return g + mlp_bwd("pol", po, PW, obs, act, 0, obs)


def sac_gemms(obs, act, atoms, n, entry, in_place=False):
    """The GEMMs of rlx_fastsac_{critic_update,policy_update,act}_f32 in issue order."""
    PW, QW = FS.POLICY_WIDTHS, FS.Q_WIDTHS
    po, qo = sac_offsets(obs, PW, (act, act)), sac_offsets(obs + act, QW, (atoms,))
    nq = qo[-1]

    def torso_fwd(tag, off, widths, inp, base):
        dims = (inp,) + tuple(widths)
        return [_fwd(f"{tag}.fwd{k}", n, dims[k], widths[k], TC_BIAS, base + off[4 * k]) for k in range(3)]

    def torso_bwd(tag, off, widths, inp, base, dx0):
        dims, g = (inp,) + tuple(widths), []
        for k in (2, 1, 0):
            g.append(_dw(f"{tag}.dw{k}", n, dims[k], widths[k]))
            if k > 0 or dx0:
                g.append(_dx(f"{tag}.dx{k}", n, dims[k], widths[k], TC_NONE, base + off[4 * k]))
        return g

    pol_fwd = torso_fwd("pol", po, PW, obs, 0) + [_fwd("pol.mean", n, 128, act, TC_BIAS, po[12]), _fwd("pol.log_std", n, 128, act, TC_BIAS, po[14])]
    q_base = lambda q: q * nq % 4 if in_place else 0
    q_fwd = lambda q, tag: torso_fwd(f"{tag}{q + 1}", qo, QW, obs + act, q_base(q)) + [_fwd(f"{tag}{q + 1}.head", n, 192, atoms, TC_BIAS, q_base(q) + qo[12])]
    if entry == "act":
        return pol_fwd
    if entry == "critic":
        g = pol_fwd + q_fwd(0, "qt") + q_fwd(1, "qt")
        for q in (0, 1):
            g += q_fwd(q, "q") + [_dw(f"q{q + 1}.dw_head", n, 192, atoms), _dx(f"q{q + 1}.dx_head", n, 192, atoms, TC_NONE, q_base(q) + qo[12])]
            g += torso_bwd(f"q{q + 1}", qo, QW, obs + act, q_base(q), False)
        return g
    g = pol_fwd + q_fwd(0, "q") + q_fwd(1, "q")
    dims = (obs + act,) + tuple(QW)
    for q in (0, 1):
        g.append(_dx(f"q{q + 1}.dx_head", n, 192, atoms, TC_NONE, q_base(q) + qo[12]))
        g += [_dx(f"q{q + 1}.dx{k}", n, dims[k], QW[k], TC_NONE, q_base(q) + qo[4 * k]) for k in (2, 1, 0)]
    g += [_dw("pol.dw_mean", n, 128, act), _dw("pol.dw_log_std", n, 128, act), _dx("pol.dx_mean", n, 128, act, TC_NONE, po[12]),
          _dx("pol.dx_log_std", n, 128, act, TC_NONE, po[14])]
    return g + torso_bwd("pol", po, PW, obs, 0, False)


def _err(K):
    """test_gpu_tc_engine.py's error model of one 3xTF32 product, relative to the output's norm; accumulation chains are capped at 1024."""
    return 6e-7 + 3.2e-9 * min(K, 1024)


def _floor(gemms_of, obs, act, atoms, n, entry):
    """F of the module docstring for one update: e(K) summed over the 16 products a gradient tensor can depend on."""
    fwd, bwd = {}, {}
    for g in gemms_of(obs, act, atoms, n, entry):
        net = g.name.split(".")[0]
        (bwd if g.a_kmaj and not g.b_kmaj else fwd if g.a_kmaj else {}).setdefault(net, []).append(_err(g.K))
    chain = fwd["pol"] + fwd["q1"] + bwd["q1"] + [_err(n)]
    chain += fwd["qt1"] if entry == "critic" else bwd["pol"]
    return sum(chain)


# ------------------------------------------------------------------------------------------------- the two algorithms
class Td3:
    name, oracle, gemms = "fasttd3", TD, staticmethod(td3_gemms)
    # metrics slots compared with the oracle's: (slot, oracle key)
    critic_metrics, policy_metrics = ((0, "loss/q_loss"), (1, "q/q_min"), (2, "q/q_max"), (3, "gradients/critic_grad_norm")), \
        ((0, "loss/policy_loss"), (1, "gradients/policy_grad_norm"))
    critic_inputs = ("states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps", "smoothing_noise")
    policy_inputs = ("states",)
    hp = dict(gamma=0.97, tau=0.1, v_min=-10.0, v_max=10.0, se=0.2, sclip=0.5, wd=0.1)

    @staticmethod
    def leaves(net):
        return TD.leaves(net)

    @staticmethod
    def tensor_names(net):
        return [f"{k}.{'weight' if j == 0 else 'bias'}" for k in range(len(net)) for j in (0, 1)]

    @staticmethod
    def linear_bias(net):
        return [j == 1 for _ in net for j in (0, 1)]

    @staticmethod
    def rebuild(net, leaves):
        return [(leaves[2 * k], leaves[2 * k + 1]) for k in range(len(net))]

    @classmethod
    def learner(cls, nets, clipped, dtype, **_):
        h = cls.hp
        return TD.Learner(*nets, LR, h["wd"], h["gamma"], h["tau"], h["v_min"], h["v_max"], nets[1][-1][0].shape[0], h["se"], h["sclip"], bool(clipped), -1.0,
                          dtype=dtype)

    @staticmethod
    def critic_step(L, b):
        return L.critic_step(b["states"], b["next_states"], b["actions"], b["rewards"], b["dones"], b["truncations"], b["effective_n_steps"],
                             b["smoothing_noise"])

    @staticmethod
    def policy_step(L, b):
        return L.policy_step(b["states"])

    @staticmethod
    def noise_name():
        return "smoothing_noise"


class Sac:
    name, oracle, gemms = "fastsac", FS, staticmethod(sac_gemms)
    critic_metrics, policy_metrics = ((0, "loss/q_loss"), (1, "loss/entropy_loss"), (2, "q/q_min"), (3, "q/q_max"), (4, "entropy/entropy"),
                                      (5, "gradients/critic_grad_norm")), ((0, "loss/policy_loss"), (1, "entropy/alpha"), (2, "gradients/policy_grad_norm"))
    critic_inputs = ("states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps", "noise")
    policy_inputs = ("states", "noise")
    hp = dict(gamma=0.99, tau=0.1, v_min=-10.0, v_max=10.0, wd=0.1, b1=0.9, b2=0.95, alpha=0.05, lsmin=-5.0, lsmax=0.0)

    @staticmethod
    def leaves(net):
        return FS._leaves(net)

    @staticmethod
    def _heads(net):
        return [k for k in ("mean", "log_std", "head") if k in net]

    @classmethod
    def tensor_names(cls, net):
        names = [f"torso.{i // 2}.{'linear' if i % 2 == 0 else 'layernorm'}.{p}" for i in range(len(net["torso"])) for p in ("weight", "bias")]
        return names + [f"{k}.{p}" for k in cls._heads(net) for p in ("weight", "bias")]

    @classmethod
    def linear_bias(cls, net):
        return [i % 2 == 0 and j == 1 for i in range(len(net["torso"])) for j in (0, 1)] + [j == 1 for _ in cls._heads(net) for j in (0, 1)]

    @classmethod
    def rebuild(cls, net, leaves):
        nt = len(net["torso"])
        out = {"torso": [(leaves[2 * i], leaves[2 * i + 1]) for i in range(nt)]}
        for j, k in enumerate(cls._heads(net)):
            out[k] = (leaves[2 * nt + 2 * j], leaves[2 * nt + 2 * j + 1])
        return out

    @classmethod
    def learner(cls, nets, clipped, dtype, scale=None):
        h = cls.hp
        act, atoms = nets[0]["mean"][0].shape[0], nets[1]["head"][0].shape[0]
        return FS.Learner(*nets, scale, LR, h["wd"], (h["b1"], h["b2"]), h["gamma"], h["tau"], h["v_min"], h["v_max"], atoms, -float(act), h["alpha"],
                          h["lsmin"], h["lsmax"], bool(clipped), -1.0, dtype=dtype)

    @staticmethod
    def critic_step(L, b):
        return L.critic_and_entropy_step(b["states"], b["next_states"], b["actions"], b["rewards"], b["dones"], b["truncations"], b["effective_n_steps"],
                                         b["noise"])

    @staticmethod
    def policy_step(L, b):
        return L.policy_step(b["states"], b["noise"])

    @staticmethod
    def noise_name():
        return "noise"


def _init(algo, obs, act, atoms, seed):
    """The reference's initial networks, with FastSAC's zero-initialised heads moved off zero (a zero head makes the policy ignore its torso)."""
    pol, q1, q2 = algo.oracle.reference_init(obs, act, atoms, seed)
    if algo is Sac:
        g = torch.Generator().manual_seed(seed + 1)
        for k in ("mean", "log_std"):
            pol[k] = tuple(t + 0.05 * torch.randn(t.shape, generator=g) for t in pol[k])
    return pol, q1, q2


def _to(algo, net, device, dtype):
    return algo.rebuild(net, [t.detach().to(device, dtype) for t in algo.leaves(net)])


def _draw(algo, obs, act, rows, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    u = lambda *s: torch.rand(*s, generator=g)
    return {"states": r(rows, obs), "next_states": r(rows, obs), "actions": u(rows, act) * 2 - 1, "rewards": r(rows), "dones": (u(rows) < 0.05).float(),
            "truncations": (u(rows) < 0.02).float(), "effective_n_steps": torch.randint(1, 4, (rows,), generator=g).float(), algo.noise_name(): r(rows, act)}


def _relu_margin(net, x):
    """Float64 forward of a Linear-ReLU MLP: (per row, the smallest |pre-activation| of a hidden unit over the rms of that row's layer, so that
    a row's margin does not depend on which other rows are in the batch; the output)."""
    m = torch.full((x.shape[0],), float("inf"), dtype=x.dtype, device=x.device)
    for w, b in net[:-1]:
        z = F.linear(x, w, b)
        m = torch.minimum(m, z.abs().amin(1) / z.pow(2).mean(1).sqrt())
        x = F.relu(z)
    return m, F.linear(x, *net[-1])


def td3_margins(nets, b, clipped, device):
    """Per candidate row, in float64 at the weights `nets`: (critic-update margin, policy-update margin), each the pair (smallest relative
    |pre-activation| over the networks the update differentiates through, |difference| of the two values a clipped update selects between
    or inf)."""
    pol, q1, q2 = (_to(Td3, net, device, torch.float64) for net in nets)
    b = {k: v.to(device, torch.float64) for k, v in b.items()}
    inf = torch.full_like(b["rewards"], float("inf"))
    with torch.no_grad():
        xa = torch.cat([b["states"], b["actions"]], 1)
        relu_c = torch.minimum(_relu_margin(q1, xa)[0], _relu_margin(q2, xa)[0])
        L = Td3.learner((pol, q1, q2), clipped, torch.float64)
    Td3.critic_step(L, b)   # a throw-away learner: its per-row next values are the two sides of the critic's clipped selection
    with torch.no_grad():
        val_c = (L.next_values[0] - L.next_values[1]).abs() if clipped else inf
        mp, pre = _relu_margin(pol, b["states"])
        xp = torch.cat([b["states"], torch.tanh(pre)], 1)
        (m1, l1), (m2, l2) = _relu_margin(q1, xp), _relu_margin(q2, xp)
        support = torch.linspace(Td3.hp["v_min"], Td3.hp["v_max"], l1.shape[1], dtype=torch.float64, device=device)
        v1, v2 = (F.softmax(l1, 1) * support).sum(1), (F.softmax(l2, 1) * support).sum(1)
        relu_p, val_p = torch.minimum(mp, torch.minimum(m1, m2)), (v1 - v2).abs() if clipped else inf
    return (relu_c, val_c), (relu_p, val_p)


def _keep(b, margins, n):
    """The first n rows of b outside both margins."""
    relu, val = margins
    ok = ((relu > RELU_MARGIN) & (val > VALUE_MARGIN)).cpu()
    idx = torch.nonzero(ok).reshape(-1)
    assert idx.numel() >= n, f"only {idx.numel()} of {ok.numel()} candidate rows are outside the margins, {n} needed"
    return {k: v[idx[:n]].contiguous() for k, v in b.items()}


def make_batches(algo, nets, obs, act, n, seed, clipped, device):
    """(critic batch, policy batch) of n rows each.  FastTD3: margin-filtered at the weights `nets` (module docstring), and checked to be."""
    if algo is Sac:
        return _draw(algo, obs, act, n, seed), _draw(algo, obs, act, n, seed + 1)
    out = []
    for which, s in ((0, seed), (1, seed + 1)):
        cand = _draw(algo, obs, act, 2 * n + 64, s)
        kept = _keep(cand, td3_margins(nets, cand, clipped, device)[which], n)
        relu, val = td3_margins(nets, kept, clipped, device)[which]
        assert float(relu.min()) > RELU_MARGIN and float(val.min()) > VALUE_MARGIN, (float(relu.min()), float(val.min()))
        out.append(kept)
    return tuple(out)


def oracle_update(algo, nets, which, b, clipped, device, dtype=torch.float64, scale=None, rss=True):
    """One critic or policy step of the oracle's Learner in `dtype` on `device`: dict(grads, norms, params, targets, metrics), the tensors as
    float64 numpy arrays in flat-layout order ([q1 | q2] for the critic).  norms: ||g||, or for Linear biases the root-sum-square of the
    per-row terms where larger - from a second learner whose Linear biases are row-wise copies ([n, out]; F.linear adds a bias broadcast to
    its output), whose gradients are the terms."""
    n = b["states"].shape[0]
    b = {k: v.to(device, dtype) for k, v in b.items()}
    kw = dict(scale=scale.to(device, dtype)) if scale is not None else {}
    mine = (lambda L: algo.leaves(L.q1) + algo.leaves(L.q2)) if which == "critic" else (lambda L: algo.leaves(L.pol))
    step = algo.critic_step if which == "critic" else algo.policy_step
    L = algo.learner(tuple(_to(algo, net, device, dtype) for net in nets), clipped, dtype, **kw)
    metrics = step(L, b)
    np64 = lambda ts: [t.detach().double().cpu().numpy() for t in ts]
    grads = np64([p.grad for p in mine(L)])
    norms = [float(np.linalg.norm(g)) for g in grads]
    if rss:
        wide = []
        for net in nets:
            lv, mask = algo.leaves(_to(algo, net, device, dtype)), algo.linear_bias(net)
            wide.append(algo.rebuild(net, [t.expand(n, -1).clone() if m else t for t, m in zip(lv, mask)]))
        L2 = algo.learner(tuple(wide), clipped, dtype, **kw)
        step(L2, b)
        masks = (algo.linear_bias(nets[1]) + algo.linear_bias(nets[2])) if which == "critic" else algo.linear_bias(nets[0])
        for i, (p, m) in enumerate(zip(mine(L2), masks)):
            if m:
                terms = p.grad.detach().double()
                assert float((terms.sum(0).cpu() - torch.from_numpy(grads[i])).norm()) <= 1e-9 * max(norms[i], 1e-30) + 1e-30
                norms[i] = max(norms[i], float(terms.pow(2).sum(0).sqrt().norm()))
    out = dict(grads=grads, norms=[max(v, 1e-30) for v in norms], metrics=metrics, params=np64(mine(L)))
    if which == "critic":
        out["targets"] = np64(algo.leaves(L.q1t) + algo.leaves(L.q2t))
    return out


def _split(flat, like):
    """A flat float32 buffer cut into float64 arrays of the shapes of `like`."""
    out, o = [], 0
    for t in like:
        out.append(flat[o:o + t.size].astype(np.float64).reshape(t.shape))
        o += t.size
    assert o == flat.size
    return out


def _flat(algo, net):
    return np.concatenate([t.detach().numpy().reshape(-1) for t in algo.leaves(net)]).astype(np.float32)


# ------------------------------------------------------------------------------------------------- host-only tests
@pytest.mark.parametrize("atoms", [101, 100, 51])
def test_path_table_names_the_critic_2_alignment(atoms):
    """With every critic-2 weight read in place at q_params + nq, nq % 4 == nr_atoms % 4: at 101 atoms each forward / input-gradient GEMM whose B is
    such a weight would run SIMT (FastTD3 layers 2-4 - layer 1 is staged - and FastSAC layers 1-4, online and target), at 100 atoms none.  The
    table the device tests assert is the aligned one: both critics on the same instances."""
    for gemms_of, dims in ((td3_gemms, (376, 17, atoms, 8192)), (sac_gemms, (48, 12, atoms, 8192))):
        offs = mlp_offsets(dims[0] + dims[1], TD.Q_WIDTHS, atoms) if gemms_of is td3_gemms else sac_offsets(dims[0] + dims[1], FS.Q_WIDTHS, (atoms,))
        assert offs[-1] % 4 == atoms % 4 and all(o % 4 == 0 for o in offs[:-1])
        for entry in ("critic", "policy"):
            want, in_place = (derive_paths(gemms_of(*dims, entry, in_place=p), 1) for p in (False, True))
            by_name = {g.name: on_tensor_engine(g) for g in gemms_of(*dims, entry)}
            for q1_name, on in by_name.items():   # the table itself: critic 2 goes where critic 1 goes
                if q1_name.startswith(("q1.", "qt1.")):
                    assert by_name[q1_name.replace("1.", "2.", 1)] == on, q1_name
            lost = in_place.get(GP_SGEMM, 0) - want.get(GP_SGEMM, 0)
            if atoms % 4 == 0:
                assert lost == 0 and in_place == want
            else:
                moved = [g for g in gemms_of(*dims, entry, in_place=True) if g.name.startswith(("q2.", "qt2.")) and g.b % 4 and
                         on_tensor_engine(g._replace(b=0))]
                assert lost == len(moved) > 0, (entry, lost, len(moved))
    # FastTD3's default shape, critic update: 4 tensor GEMMs per forward (one of them the logits layer only when atoms % 4 == 0)
    t = derive_paths(td3_gemms(376, 17, atoms, 8192, "critic"), 1)
    relu_fwd = tc_slot(Gemm("", 1, 1, TC_BIAS_RELU, *[0] * 11))
    assert t[relu_fwd] == 3 * 5   # policy + 2 target + 2 online forwards, three hidden layers each
    assert (tc_slot(Gemm("", 1, 1, TC_BIAS, *[0] * 11)) in t) == (atoms == 100)


def test_gate_edges():
    g = _fwd("x", 64, 32, 64, TC_BIAS, 0)
    assert on_tensor_engine(g)
    for bad in (g._replace(M=63), g._replace(N=63), g._replace(K=31), g._replace(b=1), g._replace(lda=33), g._replace(ldc=66), g._replace(a_kmaj=0),
                _dw("w", 2048, 101, 64)):   # the last: split offset of C odd
        assert not on_tensor_engine(bad), bad
    assert on_tensor_engine(_dw("w", 40, 64, 64)) and not on_tensor_engine(_dw("w", 31, 64, 64))
    assert derive_paths([g, g._replace(M=8)], 1) == {tc_slot(g): 1, GP_SGEMM: 1} and derive_paths([g, g], 0) == {GP_SGEMM: 2}


@pytest.mark.parametrize("algo", [Td3, Sac], ids=["fasttd3", "fastsac"])
def test_float64_oracle_agrees_with_the_float32_oracle(algo):
    """The float64 learner is the same program as the pinned float32 one: on the first golden batch its gradients, metrics and stepped parameters
    agree to float32 accuracy, per tensor, and the per-row bias terms sum to the bias gradients."""
    import os
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"{algo.name}_update.npz")
    z = np.load(golden)
    obs, act, batch, atoms = int(z["meta"][1]), int(z["meta"][2]), int(z["meta"][3]), int(z["meta"][9])
    nets = _init(algo, obs, act, atoms, 5)
    scale = torch.full((act,), 0.8) if algo is Sac else None
    b = {k: torch.from_numpy(z[f"step0/{k}"][:batch]) for k in algo.critic_inputs[:-1]}
    b[algo.noise_name()] = torch.from_numpy(z["step0/smoothing_noise" if algo is Td3 else "step0/normals"][0])
    for which in ("critic", "policy"):
        r64 = oracle_update(algo, nets, which, b, True, "cpu", torch.float64, scale)
        r32 = oracle_update(algo, nets, which, b, True, "cpu", torch.float32, scale, rss=False)
        for g64, g32, nrm in zip(r64["grads"], r32["grads"], r64["norms"]):
            assert np.linalg.norm(g32 - g64) <= 2e-5 * nrm
        cat = lambda ts: np.concatenate([t.reshape(-1) for t in ts])   # Adam's first step is the sign of g: per network (module docstring)
        assert np.linalg.norm(cat(r32["params"]) - cat(r64["params"])) <= PARAM_BAR * np.linalg.norm(cat(r64["params"]))
        for key, v in r64["metrics"].items():
            assert abs(r32["metrics"][key] - v) <= 2e-5 * max(1.0, abs(v)), key


def test_margin_filter_drops_rows_near_a_kink():
    obs, act, atoms, n = 24, 6, 51, 64
    nets = _init(Td3, obs, act, atoms, 5)
    cand = _draw(Td3, obs, act, 2 * n + 64, 3)
    (relu, val), _ = td3_margins(nets, cand, True, "cpu")
    relu[0] = 0.5 * RELU_MARGIN   # a row with a unit inside the margin
    kept = _keep(cand, (relu, val), n)
    assert kept["states"].shape == (n, obs) and torch.equal(kept["states"][0], cand["states"][1])
    (relu_kept, val_kept), _ = td3_margins(nets, kept, True, "cpu")
    assert float(relu_kept.min()) > RELU_MARGIN and float(val_kept.min()) > VALUE_MARGIN
    with pytest.raises(AssertionError):
        _keep(cand, (torch.zeros_like(relu), val), n)


# ------------------------------------------------------------------------------------------------------ device side
@pytest.fixture
def lib():
    """The native library; the aux GEMM engine is back at 0 (SIMT) after every test whatever it left."""
    from rl_x_b200 import _native as nt
    lib = nt.load()
    try:
        yield lib
    finally:
        lib.rlx_set_aux_gemm_engine(0)


def _t(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).to(DEV).contiguous()


class _Device:
    """Flat buffers of one learner on the device and the update calls, every output NaN before the call that writes it."""

    def __init__(self, algo, lib, obs, act, atoms, n, nets, clipped, scale=None):
        from rl_x_b200 import _native as nt
        self.algo, self.lib, self.nt, self.n, self.dims, self.like = algo, lib, nt, n, (obs, act, atoms), nets
        self.P, self.Q = _t(_flat(algo, nets[0])), _t(np.concatenate([_flat(algo, nets[1]), _flat(algo, nets[2])]))
        self.QT = self.Q.clone()
        zl = torch.zeros_like
        self.gP, self.mP, self.vP, self.gQ, self.mQ, self.vQ = zl(self.P), zl(self.P), zl(self.P), zl(self.Q), zl(self.Q), zl(self.Q)
        self.lr, self.steps = _t([LR]), torch.zeros(3, dtype=torch.int64, device=DEV)
        h = algo.hp
        if algo is Td3:
            self.d, self.Args = nt.FastTd3Dims(obs, act, atoms), nt.FastTd3UpdateArgs
            self.hp = nt.FastTd3Hparams(h["gamma"], h["tau"], h["v_min"], h["v_max"], h["se"], h["sclip"], h["wd"], 0.9, 0.999, 1e-8, -1.0, float(clipped))
            self.nbytes = lib.rlx_fasttd3_workspace_bytes(C.byref(self.d), n)
            self.fns = dict(critic=lib.rlx_fasttd3_critic_update_f32, policy=lib.rlx_fasttd3_policy_update_f32)
        else:
            self.d, self.Args = nt.FastSacDims(obs, act, atoms), nt.FastSacUpdateArgs
            self.hp = nt.FastSacHparams(h["gamma"], h["tau"], h["v_min"], h["v_max"], -float(act), h["lsmin"], h["lsmax"], h["wd"], h["b1"], h["b2"], 1e-8,
                                        -1.0, float(clipped))
            self.nbytes = lib.rlx_fastsac_workspace_bytes(C.byref(self.d), n)
            self.fns = dict(critic=lib.rlx_fastsac_critic_update_f32, policy=lib.rlx_fastsac_policy_update_f32)
            self.scale, self.la, self.astate = _t(scale), _t([math.log(h["alpha"])]), torch.zeros(3, device=DEV)
        assert self.nbytes > 0 and self.nbytes % 4 == 0
        self.ws = torch.empty(self.nbytes // 4, device=DEV)   # exactly the size the library asks for

    def update(self, which, batch):
        a = self.Args()
        a.dims, a.n = self.d, self.n
        keep = {k: _t(batch[k]) for k in (self.algo.critic_inputs if which == "critic" else self.algo.policy_inputs)}
        for k, v in keep.items():
            assert v.shape[0] == self.n
            setattr(a, k, v.data_ptr())
        a.policy_params, a.policy_grads, a.policy_m, a.policy_v = self.P.data_ptr(), self.gP.data_ptr(), self.mP.data_ptr(), self.vP.data_ptr()
        a.q_params, a.q_grads, a.q_m, a.q_v, a.q_target_params = self.Q.data_ptr(), self.gQ.data_ptr(), self.mQ.data_ptr(), self.vQ.data_ptr(), self.QT.data_ptr()
        a.lr, a.steps, a.hp = self.lr.data_ptr(), self.steps.data_ptr(), self.hp
        if self.algo is Sac:
            a.action_scale, a.log_alpha, a.alpha_state = self.scale.data_ptr(), self.la.data_ptr(), self.astate.data_ptr()
        metrics = torch.full((8,), float("nan"), device=DEV)
        self.ws.fill_(float("nan"))
        (self.gQ if which == "critic" else self.gP).fill_(float("nan"))
        a.metrics, a.workspace, a.workspace_bytes = metrics.data_ptr(), self.ws.data_ptr(), self.nbytes
        self.nt.check(self.fns[which](C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), f"{self.algo.name} {which} update")
        torch.cuda.synchronize()
        return metrics.cpu().numpy()

    def nets(self):
        """(policy, q1, q2) at the current device weights, float32 on the CPU."""
        obs, act, atoms = self.dims
        like = self.like
        P, Q = self.P.cpu(), self.Q.cpu()
        out, srcs = [], (P, Q[:Q.numel() // 2], Q[Q.numel() // 2:])
        for net, src in zip(like, srcs):
            lv, o = [], 0
            for t in self.algo.leaves(net):
                lv.append(src[o:o + t.numel()].reshape(t.shape).clone())
                o += t.numel()
            assert o == src.numel()
            out.append(self.algo.rebuild(net, lv))
        return tuple(out)


def _counted(lib, engine, gemms, fn):
    """fn() on `engine` with the launches of every GEMM path asserted equal to the table derived from `gemms`."""
    from test_gpu_zzzzzz_tc_ppo_shapes import _paths
    assert lib.rlx_set_aux_gemm_engine(engine) == engine
    before = int(lib.rlx_aux_tc_gemm_count())
    out, counts = _paths(lib, fn)
    want = derive_paths(gemms, engine)
    assert counts == want, (f"engine {engine}: GEMM launches by path differ from the derived table", counts, want,
                            [(g.name, on_tensor_engine(g)) for g in gemms])
    assert int(lib.rlx_aux_tc_gemm_count()) - before == sum(c for s, c in want.items() if s != GP_SGEMM)
    return out, counts


def _check_update(algo, dev, ref, which, metrics, label, report, simt=None, floor=None, params=True):
    """Bounds (i) and (ii) of the module docstring on the gradient buffer, then metrics, stepped parameters and polyak targets."""
    names = [f"{net}.{t}" for net, src in (("q1", 1), ("q2", 2)) for t in algo.tensor_names(dev.like[src])] if which == "critic" else \
        [f"pol.{t}" for t in algo.tensor_names(dev.like[0])]
    grads = _split((dev.gQ if which == "critic" else dev.gP).cpu().numpy(), ref["grads"])
    dist = {}
    for name, g, g64, nrm in zip(names, grads, ref["grads"], ref["norms"]):
        assert np.isfinite(g).all(), (label, name, "an element was not written")
        dist[name] = float(np.linalg.norm(g - g64))
        assert dist[name] <= BAR * nrm, (label, name, dist[name] / nrm)
        if simt is not None:
            assert dist[name] <= 2 * simt[name] + floor * nrm, (label, name, dist[name] / nrm, simt[name] / nrm, floor)
    worst = max(zip(names, ref["norms"]), key=lambda kv: dist[kv[0]] / kv[1])
    report.append(f"{label}: worst {dist[worst[0]] / worst[1]:.2e} ({worst[0]})")
    for slot, key in (algo.critic_metrics if which == "critic" else algo.policy_metrics):
        assert abs(float(metrics[slot]) - ref["metrics"][key]) <= BAR * max(1.0, abs(ref["metrics"][key])), (label, key, metrics[slot], ref["metrics"][key])
    if params:
        pairs = [("params", dev.Q if which == "critic" else dev.P, ref["params"])] + ([("targets", dev.QT, ref["targets"])] if which == "critic" else [])
        for what, buf, want in pairs:
            got = _split(buf.cpu().numpy(), want)
            per_net = len(want) // 2 if which == "critic" else len(want)
            for i in range(0, len(want), per_net):
                a, r = np.concatenate([x.reshape(-1) for x in got[i:i + per_net]]), np.concatenate([x.reshape(-1) for x in want[i:i + per_net]])
                assert np.linalg.norm(a - r) <= PARAM_BAR * np.linalg.norm(r), (label, what, i, np.linalg.norm(a - r) / np.linalg.norm(r))
    return dist


def _case(algo, lib, obs, act, atoms, n, clipped, params=True):
    nets = _init(algo, obs, act, atoms, 3)
    scale = torch.linspace(0.5, 1.5, act) if algo is Sac else None
    cb, pb = make_batches(algo, nets, obs, act, n, 11, clipped, DEV)
    refs = {w: oracle_update(algo, nets, w, b, clipped, DEV, scale=scale) for w, b in (("critic", cb), ("policy", pb))}
    report, simt = [], {}
    for engine in (0, 1):
        for which, b in (("critic", cb), ("policy", pb)):
            dev = _Device(algo, lib, obs, act, atoms, n, nets, clipped, scale)   # each update from the initial state, where its reference is
            metrics, _ = _counted(lib, engine, algo.gemms(obs, act, atoms, n, which), lambda: dev.update(which, b))
            floor = _floor(algo.gemms, obs, act, atoms, n, which)
            label = f"{algo.name} ({obs}, {act}, {atoms}, {n}) {which} engine {engine}"
            d = _check_update(algo, dev, refs[which], which, metrics, label, report, simt.get(which) if engine else None, floor, params)
            if engine == 0:
                simt[which] = d
            else:
                report[-1] += f"  F = {floor:.2e}"
    print("\n" + "\n".join(report))


TD3_CASES = [
    (376, 17, 101, 8192, 1),   # the default network, eight full weight-gradient splits
    (376, 17, 101, 2500, 1),   # ragged last split (452 rows), n not a multiple of 32
    (376, 17, 101, 4099, 1),   # last split of 3 rows: one k-block, 29 of its 32 rows zero fill
    (376, 17, 101, 64, 1),     # one split, half a tile in M
    (376, 17, 101, 100, 0),    # M = 100: a ragged half tile; the mean of the two values instead of the clipped selection
    (376, 17, 101, 40, 1),     # forward and input gradients on SIMT (n < 64), weight gradients on the tensor engine (K = n >= 32)
    (375, 18, 101, 1024, 1),   # obs % 4 != 0: policy layer 1 on SIMT, Q layer 1 on the padded pitch (393 -> 396)
    (376, 17, 100, 1024, 1),   # atoms % 4 == 0: the logits layer (TC_BIAS), its dX with ragged K = 100 and its dW on the tensor engine
    (376, 17, 51, 1024, 1),    # atoms < 64
    (64, 64, 101, 1024, 1),    # act = 64: the tanh head and the action-block dX (B at a column offset of W1) on the tensor engine
]
SAC_CASES = [
    (48, 12, 101, 8192, 0),    # the default network and batch
    (48, 12, 101, 2500, 0),
    (48, 12, 101, 64, 0),
    (48, 12, 101, 100, 1),     # the clipped selection (FastSAC's default is the mean)
    (48, 12, 101, 40, 0),
    (47, 12, 101, 1024, 0),    # obs + act and obs not multiples of 4: both first layers on SIMT
    (48, 12, 104, 1024, 0),    # atoms % 4 == 0: the logits layer on the tensor engine
    (48, 12, 51, 1024, 0),
    (64, 64, 101, 1024, 0),    # act = 64: the heads and their gradients on the tensor engine
]


@gpu
@pytest.mark.parametrize("obs,act,atoms,n,clipped", TD3_CASES)
def test_fasttd3_update_vs_float64_on_both_engines(lib, obs, act, atoms, n, clipped):
    _case(Td3, lib, obs, act, atoms, n, clipped)


@gpu
def test_fasttd3_gradients_at_the_default_batch(lib):
    """Batch 32768, the plugin's default and the one profiles/bench_fasttd3.py times: 32 weight-gradient splits.  Gradients and metrics only."""
    _case(Td3, lib, 376, 17, 101, 32768, 1, params=False)


@gpu
@pytest.mark.parametrize("obs,act,atoms,n,clipped", SAC_CASES)
def test_fastsac_update_vs_float64_on_both_engines(lib, obs, act, atoms, n, clipped):
    _case(Sac, lib, obs, act, atoms, n, clipped)


@gpu
@pytest.mark.parametrize("algo,obs,act,atoms,n", [(Td3, 376, 17, 101, 2500), (Sac, 48, 12, 101, 2500)], ids=["fasttd3", "fastsac"])
def test_two_steps_follow_the_weights(lib, algo, obs, act, atoms, n):
    """critic, critic, policy - twice - on the tensor engine: before each call the float64 oracle is evaluated at the device's current weights and
    targets (for FastTD3 on a batch filtered at those weights), so a staged copy of a weight (FastTD3's padded layer 1, critic 2's aligned
    block) that missed an AdamW step would show in the next gradient."""
    nets = _init(algo, obs, act, atoms, 4)
    scale = torch.linspace(0.5, 1.5, act) if algo is Sac else None
    dev = _Device(algo, lib, obs, act, atoms, n, nets, algo is Td3, scale)
    report = []
    for step in range(2):
        for i, which in enumerate(("critic", "critic", "policy")):
            now = dev.nets()
            b = make_batches(algo, now, obs, act, n, 100 + 10 * step + i, algo is Td3, DEV)[0 if which == "critic" else 1]
            ref = _oracle_at(algo, dev, now, which, b, scale)
            metrics, _ = _counted(lib, 1, algo.gemms(obs, act, atoms, n, which), lambda: dev.update(which, b))
            _check_update(algo, dev, ref, which, metrics, f"{algo.name} step {step} {which} {i}", report, params=False)
    print("\n" + "\n".join(report))
    assert [int(v) for v in dev.steps.cpu()][:2] == ([4, 2] if algo is Td3 else [4, 4])


def _oracle_at(algo, dev, now, which, b, scale):
    """oracle_update at the device's current online weights `now`, target weights and (FastSAC) entropy coefficient."""
    tq = dev.QT.cpu()
    halves = (tq[:tq.numel() // 2], tq[tq.numel() // 2:])

    class AtDevice(algo):
        @classmethod
        def learner(cls, nets, clipped, dtype, **kw):
            L = super().learner(nets, clipped, dtype, **kw)
            with torch.no_grad():
                for tgt, src in zip((L.q1t, L.q2t), halves):
                    o = 0
                    for t in algo.leaves(tgt):
                        t.copy_(src[o:o + t.numel()].reshape(t.shape))
                        o += t.numel()
                if algo is Sac:
                    L.log_alpha.copy_(dev.la)
            return L

    return oracle_update(AtDevice, now, which, b, algo is Td3, DEV, scale=scale, rss=False)


@gpu
@pytest.mark.parametrize("n", [63, 64, 4097])
@pytest.mark.parametrize("algo,obs,act", [(Td3, 376, 17), (Sac, 48, 12), (Td3, 64, 64), (Sac, 64, 64)], ids=["fasttd3", "fastsac", "fasttd3_act64", "fastsac_act64"])
def test_acting_kernels_vs_float64_on_both_engines(lib, algo, obs, act, n):
    """rlx_fasttd3_act_f32 / rlx_fastsac_act_f32 into NaN outputs, noisy, against the oracle's acting function in float64."""
    from rl_x_b200 import _native as nt
    atoms = 101
    pol = _init(algo, obs, act, atoms, 6)[0]
    g = torch.Generator().manual_seed(n)
    pol = algo.rebuild(pol, [t + 0.05 * torch.randn(t.shape, generator=g) for t in algo.leaves(pol)])
    x, noise = torch.randn(n, obs, generator=g), torch.randn(n, act, generator=g)
    scales, sc = torch.rand(n, 1, generator=g) * 0.4 + 0.001, torch.linspace(0.5, 1.5, act)
    p64, dd = _to(algo, pol, DEV, torch.float64), lambda t: t.to(DEV, torch.float64)
    with torch.no_grad():
        if algo is Td3:
            ref = TD.act(p64, dd(x), dd(noise), dd(scales))[0].cpu()
        else:
            ref = FS.action_and_log_prob(p64, dd(x), dd(noise), dd(sc), Sac.hp["lsmin"], Sac.hp["lsmax"])[0].cpu()
    P, st = _t(_flat(algo, pol)), lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    dx, dn, ds, dsc = _t(x), _t(noise), _t(scales), _t(sc)
    for engine in (0, 1):
        action = torch.full((n, act), float("nan"), device=DEV)
        if algo is Td3:
            d = nt.FastTd3Dims(obs, act, atoms)
            nbytes = lib.rlx_fasttd3_workspace_bytes(C.byref(d), n)
            ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
            run = lambda: nt.check(lib.rlx_fasttd3_act_f32(C.byref(d), P.data_ptr(), dx.data_ptr(), dn.data_ptr(), ds.data_ptr(), None, None, 0, n,
                                                           action.data_ptr(), None, ws.data_ptr(), nbytes, st()), "rlx_fasttd3_act_f32")
        else:
            d = nt.FastSacDims(obs, act, atoms)
            nbytes = lib.rlx_fastsac_workspace_bytes(C.byref(d), n)
            ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
            run = lambda: nt.check(lib.rlx_fastsac_act_f32(C.byref(d), P.data_ptr(), dx.data_ptr(), dn.data_ptr(), dsc.data_ptr(), Sac.hp["lsmin"],
                                                           Sac.hp["lsmax"], n, action.data_ptr(), ws.data_ptr(), nbytes, st()), "rlx_fastsac_act_f32")
        _counted(lib, engine, algo.gemms(obs, act, atoms, n, "act"), run)
        got = action.cpu().double()
        assert torch.isfinite(got).all()
        np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=1e-5, atol=1e-5, err_msg=f"engine {engine}")
        assert float((got - ref).norm() / ref.norm()) <= 5e-6, (engine, float((got - ref).norm() / ref.norm()))
