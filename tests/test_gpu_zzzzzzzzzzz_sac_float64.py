"""The SAC update (rlx_sac_update_f32) and acting step (rlx_sac_act_f32) on both GEMM engines of `run_gemm` (csrc/gemm_dispatch.cuh) against
oracle/sac_oracle.py run in float64, with a count of the GEMM kernels each call launched.

Why.  SAC's default is the tensor engine (gemm_engine "auto" = rlx_set_gemm_engine(1)), and its GEMMs reach the wgmma kernels at shapes no
other caller gives them: the policy head with N = 2 act, one-row acting, ragged K at hidden widths that are not multiples of 32, and the
only batched (twin-Q) wgmma calls whose batch stride is a parameter block.  tc_gemm_impl turns such a stride into a TMA coordinate when it
is a whole number of rows of the weight's pitch (the operand's extent is then stretched across both nets, and an MN-major weight's K tail
reads the next parameters instead of TMA's zero fill), and otherwise runs the nets one launch each.  test_gpu_sac.py compares one shape
with the float32 oracle, where both first layers, the Q output layer and every weight gradient run on SIMT whatever the switch says.
Every case here runs both engines from the same state, in a NaN-filled workspace of exactly rlx_sac_workspace_bytes, with NaN-filled
g_policy / g_q / g_log_alpha and NaN-filled acting outputs: an element no kernel wrote fails the checks.

Proof of path.  run_gemm falls back to the SIMT engine without a word when the wgmma engine returns RLX_ERR_UNSUPPORTED.  This file lists
the GEMMs of one update and one act (`sac_gemms`, written from sac.cu: policy_forward, q_forward, layer_bwd_input, layer_bwd_weight),
restates run_gemm's gate (K >= 32, no rowsum) and tc_gemm_impl's checks (16-byte bases, pitches of 4 floats, an even batch stride of C,
`expressible` batch strides or the per-net loop, the instances that exist) in `tc_launches`, derives the launches of each tc_gemm_kernel
instance and of the SIMT GEMM (a looped batched GEMM is 2 launches, a coordinate-path one 1; weight gradients call launch_sgemm
directly and are always SIMT), and asserts equality with the library's counters (rlx_gemm_path_count) around every call.

Discontinuities.  The update differentiates through ReLU networks, the clipped double-Q selection min(q1, q2), the clamp of log_std and
tanh.  A row within fp32 noise of a ReLU kink, of a tie or of a clamp bound takes opposite sides in fp32 and float64, which moves that
row's gradient by O(1).  And where |u| is large, 1 - tanh(u)^2 has an fp32 rounding error of 2^-24 / (1 - t^2) relative to itself (6e-6 at
|u| = 3; at |u| ~ 9 it underflows to 0 and fp32 moves logp by about 0.05).  So eight times the rows are drawn, a first float64 pass
gives each candidate row its margins - the smallest |pre-activation| of any hidden unit relative to the rms of its layer in that row (the
policy on s' and on s; q1_target, q2_target on (s', a'); q1, q2 on (s, a); the updated q1, q2 on (s, pi(s))), |q1_target - q2_target| and
|q1 - q2| at the selections, the distance of the raw log_std to ls_min / ls_max, and max |u| - rows inside RELU_MARGIN / VALUE_MARGIN /
LS_MARGIN or beyond U_MAX are dropped, and the first n survivors are the batch.  The policy step runs through the *updated* critics, so the
batch changes what was filtered on: the final float64 pass checks every kept row is still beyond half of each margin.

Bounds, per parameter tensor g (never one norm over the concatenation, where a small tensor hides), g64 the float64 gradient:
  (i)  ||g - g64|| <= BAR ||g64|| on both engines;
  (ii) ||g_tc - g64|| <= 2 ||g_simt - g64|| + F ||g64||.
(ii) is test_gpu_zzzzzz_tc_ppo_shapes.py's: the engines run the same fp32 program except for the GEMMs, the SIMT engine's GEMM error is part
of its whole error (hence the factor 2), and one 3xTF32 product is within e(K) = 6e-7 + 3.2e-9 K of its output's norm
(test_gpu_tc_engine.py), K <= 1024 per accumulation chain.  A gradient tensor depends on a chain of products whose errors reach it with a gain
of order one (ReLU' and tanh' <= 1), so F is e(K) summed over that chain (`floor`): g_q - the policy forward on s' (3), the target and online
Q forwards (3 + 3), the critic's input gradients (2) and the weight gradient (1); g_policy - the policy forward (3), the Q forward (3), the
Q input gradients (3), the policy input gradients (2) and the weight gradient (1).  Linear-layer bias gradients are sums of n signed
per-row terms that can largely cancel while each term carries its own rounding: they are measured against the root-sum-square of the terms
where that is larger than ||g64||.  g_q is the critic gradient as it stands after q_loss.backward() (Learner.q_grads).  The nine metrics,
g_log_alpha and log_alpha are compared at BAR relative to max(1, |value|); the stepped parameters and the Polyak targets per network at
PARAM_BAR: Adam's first step is lr g / (|g| + eps), the sign of g, so an element whose gradient is within rounding of zero moves by up to
2 lr whatever the engine.  Measured on an H100 (80 GB HBM3, 700 W), the worst tensor of any case is 5.6e-7 on the SIMT engine and
4.3e-6 on the tensor engine; the pinned float32 oracle on the CPU sits at up to 6.4e-7 (the printed report, -s).

Sorted after the other GPU files: a kernel fault on a new shape takes the CUDA context with it, and then costs only this file."""
import collections
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sac_oracle as S

gpu = pytest.mark.gpu
DEV = "cuda"
RELU_MARGIN, VALUE_MARGIN, LS_MARGIN, U_MAX = 1e-4, 1e-4, 1e-4, 3.0
BAR, PARAM_BAR = 2e-5, 3e-5
f32 = lambda x: float(np.float32(x))   # every scalar the library and the oracle share is an fp32 value
LR, GAMMA, TAU, LOG_ALPHA0 = f32(3e-4), f32(0.99), f32(0.005), f32(-0.3)
LOW, HIGH = -2.0, 0.5

# ----------------------------------------------------------------------------------------------------- the layout, restated
POLICY_KEYS = ("torso.0.weight", "torso.0.bias", "torso.2.weight", "torso.2.bias", "mean.weight", "log_std.weight", "mean.bias", "log_std.bias")
POLICY_BIASES = ("torso.0.bias", "torso.2.bias", "mean.bias", "log_std.bias")
Q_BIASES = ("critic.0.bias", "critic.2.bias", "critic.4.bias")
Q_NETS = ("q1", "q2", "q1_target", "q2_target")


def shapes(O, A, H):
    """Tensor shapes by name: (policy, q)."""
    pol = {"torso.0.weight": (H, O), "torso.0.bias": (H,), "torso.2.weight": (H, H), "torso.2.bias": (H,), "mean.weight": (A, H),
           "log_std.weight": (A, H), "mean.bias": (A,), "log_std.bias": (A,)}
    q = {"critic.0.weight": (H, O + A), "critic.0.bias": (H,), "critic.2.weight": (H, H), "critic.2.bias": (H,), "critic.4.weight": (1, H),
         "critic.4.bias": (1,)}
    return pol, q


def layout(O, A, H):
    """sac.cu: sac_layout - (policy offsets, Pp, q offsets within one net, valid floats of one net, Pq = that rounded up to 64 floats)."""
    sp, sq = shapes(O, A, H)

    def offsets(keys, sh):
        off, o = {}, 0
        for k in keys:
            off[k] = o
            o += int(np.prod(sh[k]))
        return off, o
    (po, pp), (qo, nq) = offsets(POLICY_KEYS, sp), offsets(S.Q_KEYS, sq)
    return po, pp, qo, nq, -(-nq // 64) * 64


def workspace_bytes(O, A, H, B):
    """sac.cu: sac_plan - every buffer aligned to 256 bytes."""
    OA = O + A
    sizes = [B * OA, B * H, B * H, B * 2 * A, B * A, B, B, 2 * B * H, 2 * B * H, 2 * B, B, 2 * B, 2 * B * H, 2 * B * H, 2 * B * OA, B * 2 * A,
             B * H, B * H]
    max_w = max(2 * H * max(H, OA), 2 * A * H)
    sizes += [16 * 2 * max(max_w, H * max(H, O)), 16 * 2 * max(H, 2 * A), 8]
    return sum(-(-4 * n // 256) * 256 for n in sizes)


# ----------------------------------------------------------------------------------------------------- the gate, restated
TC_NONE, TC_BIAS_TANH, TC_DTANH, TC_BIAS_RELU, TC_DRELU, TC_BIAS = range(6)   # gemm_tc_common.cuh: TcEpi
# (A_KMAJ, B_KMAJ, epilogue) of the fp32 tc_gemm_kernel instances tc_gemm_impl can launch without a pre-split B
INSTANCES = {(1, 1, TC_BIAS_TANH), (1, 1, TC_NONE), (1, 1, TC_BIAS_RELU), (1, 1, TC_BIAS), (1, 0, TC_DRELU), (1, 0, TC_DTANH), (1, 0, TC_NONE),
             (0, 0, TC_NONE)}
GP_SGEMM = 257          # rlx_gemm_path_count slot of the SIMT GEMM (common.cuh)

# One GEMM as sac.cu issues it, in GemmP's terms.  a / b / c: offsets (floats) of the operand bases from a 16-byte aligned allocation;
# sA / sB / sC / sAux: batch strides; kind: fwd (layer_fwd), dx (layer_bwd_input) or dw (layer_bwd_weight).
Gemm = collections.namedtuple("Gemm", "name kind a_kmaj b_kmaj epi M N K lda ldb ldc a b c sA sB sC sAux batch")


def expressible(off, ld):
    """gemm_tc.cu: a batch stride that is a pure row or column offset of the operand's 2-D tensor becomes a TMA coordinate."""
    return off == 0 or off % ld == 0 or off < ld


def tc_launches(g):
    """tc_gemm_kernel launches of one GEMM on engine 1, 0 when it runs on SIMT: run_gemm's gate, then tc_gemm_impl's checks."""
    if g.kind == "dw" or g.K < 32:                        # layer_bwd_weight calls launch_sgemm (and has a rowsum); run_gemm: K >= 32
        return 0
    if any(v % 4 for v in (g.a, g.b, g.c, g.lda, g.ldb, g.ldc)):
        return 0
    if g.batch > 1 and g.sC % 2:                          # pairwise stores of C
        return 0
    if (g.a_kmaj, g.b_kmaj, g.epi) not in INSTANCES:
        return 0
    if g.batch > 1 and not (expressible(g.sA, g.lda) and expressible(g.sB, g.ldb)):
        return 0 if any(v % 4 for v in (g.sA, g.sB, g.sC, g.sAux)) else g.batch   # the per-net loop
    return 1


def tc_slot(g):
    """common.cuh: tc_path_slot(a_kmaj, b_kmaj, epi, bf16 = 0, trans = 0, split_b = 0)."""
    return g.a_kmaj | g.b_kmaj << 1 | g.epi << 2


def derive_paths(gemms, engine):
    """{rlx_gemm_path_count slot: launches} a list of GEMMs must leave behind on `engine`."""
    want = collections.Counter()
    for g in gemms:
        n = tc_launches(g) if engine == 1 else 0
        want[tc_slot(g) if n else GP_SGEMM] += n or 1
    return dict(want)


def sac_gemms(O, A, H, B, entry):
    """The GEMMs of rlx_sac_update_f32 (entry "update") or rlx_sac_act_f32 ("act") in issue order."""
    po, _, qo, _, Pq = layout(O, A, H)
    OA = O + A

    def fwd(name, lda, sA, w, sW, N, K, ldc, sC, batch, relu):                      # layer_fwd: C = act(A W^T + b)
        return Gemm(name, "fwd", 1, 1, TC_BIAS_RELU if relu else TC_BIAS, B, N, K, lda, K, ldc, 0, w, 0, sA, sW, sC, 0, batch)

    def dx(name, ldz, sZ, w, ldw, sW, relu, sAux, ldx, sX, Nout, Kin, batch):       # layer_bwd_input: dX = (dZ W) [* relu'(aux)]
        return Gemm(name, "dx", 1, 0, TC_DRELU if relu else TC_NONE, B, Kin, Nout, ldz, ldw, ldx, 0, w, 0, sZ, sW, sX, sAux, batch)

    def dw(name, Nout, Kin, batch):                                                  # layer_bwd_weight: dW = dZ^T X, always SIMT
        return Gemm(name, "dw", 0, 0, TC_NONE, Nout, Kin, B, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, batch)

    def policy(tag):
        return [fwd(f"{tag}.fwd1", O, 0, po["torso.0.weight"], 0, H, O, H, 0, 1, True),
                fwd(f"{tag}.fwd2", H, 0, po["torso.2.weight"], 0, H, H, H, 0, 1, True),
                fwd(f"{tag}.head", H, 0, po["mean.weight"], 0, 2 * A, H, 2 * A, 0, 1, False)]

    def q(tag, net0):
        base = net0 * Pq
        return [fwd(f"{tag}.fwd1", OA, 0, base + qo["critic.0.weight"], Pq, H, OA, H, B * H, 2, True),
                fwd(f"{tag}.fwd2", H, B * H, base + qo["critic.2.weight"], Pq, H, H, H, B * H, 2, True),
                fwd(f"{tag}.out", H, B * H, base + qo["critic.4.weight"], Pq, 1, H, 1, B, 2, False)]

    def q_dx(tag):
        return [dx(f"{tag}.dx3", 1, B, qo["critic.4.weight"], H, Pq, True, B * H, H, B * H, 1, H, 2),
                dx(f"{tag}.dx2", H, B * H, qo["critic.2.weight"], H, Pq, True, B * H, H, B * H, H, H, 2)]

    if entry == "act":
        return policy("pi")
    g = policy("pi_next") + q("qt", 2) + q("q", 0)
    qdx = q_dx("q")
    g += [dw("q.dw3", 1, H, 2), qdx[0], dw("q.dw2", H, H, 2), qdx[1], dw("q.dw1", H, OA, 2)]
    g += policy("pi") + q("q_pi", 0) + q_dx("q_pi")
    g.append(dx("q_pi.dx1", H, B * H, qo["critic.0.weight"], OA, Pq, False, 0, OA, B * OA, H, OA, 2))
    g += [dw("pi.dw_head", 2 * A, H, 1), dx("pi.dx_head", 2 * A, 0, po["mean.weight"], H, 0, True, 0, H, 0, 2 * A, H, 1),
          dw("pi.dw2", H, H, 1), dx("pi.dx2", H, 0, po["torso.2.weight"], H, 0, True, 0, H, 0, H, H, 1), dw("pi.dw1", H, O, 1)]
    return g


def _err(K):
    """test_gpu_tc_engine.py's error model of one 3xTF32 product, relative to the output's norm; accumulation chains are capped at 1024."""
    return 6e-7 + 3.2e-9 * min(K, 1024)


def floor(O, A, H, B):
    """F of the module docstring: {"critic": for g_q, "policy": for g_policy}."""
    g = {x.name: x for x in sac_gemms(O, A, H, B, "update")}
    splits = max(1, min(16, B // 256))                  # layer_bwd_weight: one accumulation chain is one split of the rows
    chain = -(-B // splits)
    crit = [n for n in g if n.split(".")[0] in ("pi_next", "qt") or n in ("q.fwd1", "q.fwd2", "q.out", "q.dx3", "q.dx2")]
    pol = [n for n in g if n.split(".")[0] == "q_pi" or n in ("pi.fwd1", "pi.fwd2", "pi.head", "pi.dx_head", "pi.dx2")]
    return {"critic": sum(_err(g[n].K) for n in crit) + _err(min(chain, B)), "policy": sum(_err(g[n].K) for n in pol) + _err(min(chain, B))}


# ----------------------------------------------------------------------------------------------------------- cases
# (obs, act, hidden, batch, clamp): clamp offsets log_std.bias so that part of the rows sit above ls_max and below ls_min
Case = collections.namedtuple("Case", "O A H B clamp")
CASES = {
    "default": Case(17, 6, 256, 4096, False),          # layer 1s on SIMT (K = 17, 23); Q layer 2 and its dX loop over the nets
    "split_1": Case(17, 6, 256, 511, False),           # layer_bwd_weight: one split
    "split_2": Case(17, 6, 256, 512, False),           # two splits
    "split_16_ragged": Case(17, 6, 256, 4097, False),  # 16 splits of 264 rows, the last of 137
    "m63": Case(17, 6, 256, 63, False),                # M under one tile
    "m129": Case(17, 6, 256, 129, False),              # one row into a second tile
    "m1": Case(17, 6, 256, 1, False),                  # a single-row update
    "first_layers_tc": Case(32, 8, 256, 1024, False),  # K = obs = 32, K = obs + act = 40; the dxa GEMM with N = 40
    "act16": Case(17, 16, 256, 1024, False),           # 2A = 32: the head's input gradient on the tensor engine
    "act1": Case(17, 1, 256, 1024, False),             # N = 2: the head on SIMT
    "act3": Case(17, 3, 256, 1024, False),             # N = 6: the head on SIMT
    "h64_coordinate": Case(17, 6, 64, 1024, False),    # Q layer 2: Pq % 64 == 0, the coordinate path
    "h64_all_coordinate": Case(28, 4, 64, 1024, False),  # every batched tensor GEMM on the coordinate path
    "h100_ragged": Case(17, 6, 100, 1024, False),      # ragged K and N
    "h1024": Case(17, 6, 1024, 256, False),            # 4H pre-activations per row: a fifth of the candidates pass the margins
    "h66_pitch": Case(17, 6, 66, 1024, False),         # pitch not a multiple of 4: no tensor launch on either engine
    "h36_k_tail": Case(4, 4, 36, 1024, False),         # coordinate path with a K tail of 4: the MN-major weights' tail reads the next net
    "log_std_clamped": Case(17, 6, 256, 1024, True),   # sac_policy_grad_kernel's in_range gating, both bounds
}


def _ls_bounds(case):
    return (-0.5, 0.5) if case.clamp else (-20.0, 2.0)


def _nets(case, seed):
    """(pol, q1, q2, q1_target, q2_target, adam): named float32 tensors with the reference's default initialisation, targets moved off the
    online nets (so that a wrong net read for the targets, or a wrong Polyak step, shows), and a mid-training Adam state (`_adam_state`)."""
    pol, q1, q2 = S.init_params(case.O, case.A, case.H, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    q1t, q2t = ({k: v + 0.02 * torch.randn(v.shape, generator=g) for k, v in q.items()} for q in (q1, q2))
    if case.clamp:
        off = torch.full((case.A,), 0.5)
        off[case.A // 2:] = -0.5
        pol["log_std.bias"] = pol["log_std.bias"] + off
    nets = (pol, q1, q2, q1t, q2t, None)
    return nets[:5] + (_adam_state(case, nets, seed + 2),)


ADAM_STEP0 = 100


def _adam_state(case, nets, seed):
    """Adam moments after ADAM_STEP0 steps, scaled per tensor by the rms of a gradient on a warm-up batch: exp_avg ~ 0.5 rms N(0, 1),
    exp_avg_sq ~ rms^2 U(1, 2).  From zero moments Adam's first step is lr times the sign of each gradient element, so the critics the
    policy step runs through would change by 2 lr wherever one row more or less flips the sign of an element, and the margins at the
    updated critics would depend on the batch at the 1e-3 level.  With these moments the step is a smooth function of the gradient, and
    the stepped parameters measure the gradient's error rather than its signs."""
    L = _learner(case, nets, torch.float64, "cpu")
    _update(L, _draw(case, 256, seed))
    g = torch.Generator().manual_seed(seed)

    def mv(grad):
        rms = max(float(grad.pow(2).mean().sqrt()), 1e-12)
        return (0.5 * rms * torch.randn(grad.shape, generator=g)).float(), (rms * rms * (1 + torch.rand(grad.shape, generator=g))).float()
    return {"pol": {k: mv(L.pol[k].grad) for k in POLICY_KEYS}, "q1": {k: mv(L.q_grads[0][k]) for k in S.Q_KEYS},
            "q2": {k: mv(L.q_grads[1][k]) for k in S.Q_KEYS}, "la": mv(L.log_alpha.grad)}


def _draw(case, rows, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    u = lambda *s: torch.rand(*s, generator=g)
    return {"states": r(rows, case.O), "next_states": r(rows, case.O), "actions": u(rows, case.A) * 2 - 1, "rewards": r(rows),
            "terminations": (u(rows) < 0.05).float(), "eps_next": r(rows, case.A), "eps_cur": r(rows, case.A)}


# ---------------------------------------------------------------------------------------------------- float64 oracle
def _learner(case, nets, dtype, device, wide=()):
    """oracle Learner over `nets`, with their Adam state where it is given; the Linear biases of the networks named in `wide` are row-wise
    copies ([n, out]; F.linear adds a bias broadcast to its output), so that their gradients are the per-row terms."""
    lo, hi = _ls_bounds(case)
    adam = nets[5]
    nets = list(nets[:5])
    for i, net in enumerate(("pol", "q", "q", "q", "q")):   # the targets too: Polyak steps them with the online nets' shapes
        if net in wide:
            nets[i] = {k: (v.expand(wide[net], -1) if k in POLICY_BIASES + Q_BIASES else v) for k, v in nets[i].items()}
    pol, q1, q2, q1t, q2t = nets
    L = S.Learner(pol, q1, q2, torch.full((case.A,), LOW), torch.full((case.A,), HIGH), lr=LR, gamma=GAMMA, tau=TAU, target_entropy=-float(case.A),
                  ls_min=lo, ls_max=hi, log_alpha=LOG_ALPHA0, q1_target=q1t, q2_target=q2t, dtype=dtype, device=device)
    if adam is not None:
        def put(opt, p, mv):
            opt.state[p] = {"step": torch.tensor(float(ADAM_STEP0)), "exp_avg": mv[0].to(device, dtype).clone(),
                            "exp_avg_sq": mv[1].to(device, dtype).clone()}
        for net, params, opt in (("pol", L.pol, L.popt), ("q1", L.q1, L.qopt), ("q2", L.q2, L.qopt)):
            if ("pol" if net == "pol" else "q") not in wide:
                for k, mv in adam[net].items():
                    put(opt, params[k], mv)
        put(L.aopt, L.log_alpha, adam["la"])
    return L


def _update(L, b):
    dt, dv = L.log_alpha.dtype, L.log_alpha.device
    b = {k: v.to(dv, dt) for k, v in b.items()}
    return L.update(b["states"], b["next_states"], b["actions"], b["rewards"], b["terminations"], b["eps_next"], b["eps_cur"])


def _mlp(layers, x):
    """Float64 forward of a Linear-ReLU MLP: (per row, the smallest |pre-activation| of a hidden unit over the rms of that row's layer, so that
    a row's margin does not depend on which other rows are in the batch; the output)."""
    m = torch.full((x.shape[0],), float("inf"), dtype=x.dtype, device=x.device)
    for w, b in layers[:-1]:
        z = F.linear(x, w, b)
        m = torch.minimum(m, z.abs().amin(1) / z.pow(2).mean(1).sqrt().clamp_min(1e-300))
        x = F.relu(z)
    return m, F.linear(x, *layers[-1])


def _pol_layers(p):
    return [(p["torso.0.weight"], p["torso.0.bias"]), (p["torso.2.weight"], p["torso.2.bias"]),
            (torch.cat([p["mean.weight"], p["log_std.weight"]]), torch.cat([p["mean.bias"], p["log_std.bias"]]))]


def _q_layers(q):
    return [(q[f"critic.{i}.weight"], q[f"critic.{i}.bias"]) for i in (0, 2, 4)]


def margins(case, nets, updated, b):
    """Per row, in float64: the margins of the module docstring (relu, tie, ls: larger is safer; u: max |u|, smaller is safer).  nets: the
    initial (pol, q1, q2, q1_target, q2_target); updated: (q1, q2) after the critic step."""
    lo, hi = _ls_bounds(case)
    A = case.A
    with torch.no_grad():
        dv = updated[0]["critic.0.weight"].device
        d = lambda t: t.detach().to(dv, torch.float64)
        pol, q1, q2, q1t, q2t = ({k: d(v) for k, v in net.items()} for net in nets[:5])
        q1n, q2n = ({k: d(v) for k, v in net.items()} for net in updated)
        b = {k: d(v) for k, v in b.items()}

        def policy(x, eps):
            m, head = _mlp(_pol_layers(pol), x)
            ls = head[:, A:]
            u = head[:, :A] + torch.exp(ls.clamp(lo, hi)) * eps
            return m, torch.tanh(u), torch.minimum((ls - lo).abs(), (ls - hi).abs()).amin(1), u.abs().amax(1)

        def twin(qa, qb, x, a):
            (m1, v1), (m2, v2) = _mlp(_q_layers(qa), torch.cat([x, a], 1)), _mlp(_q_layers(qb), torch.cat([x, a], 1))
            return torch.minimum(m1, m2), (v1 - v2).abs().reshape(-1)

        r1, a_next, ls1, u1 = policy(b["next_states"], b["eps_next"])
        r2, t1 = twin(q1t, q2t, b["next_states"], a_next)
        r3, _ = twin(q1, q2, b["states"], b["actions"])
        r4, a_cur, ls2, u2 = policy(b["states"], b["eps_cur"])
        r5, t2 = twin(q1n, q2n, b["states"], a_cur)
        relu = torch.stack([r1, r2, r3, r4, r5]).amin(0)
        return {"relu": relu, "tie": torch.minimum(t1, t2), "ls": torch.minimum(ls1, ls2), "u": torch.maximum(u1, u2)}


def outside(mg, frac=1.0):
    """Rows beyond frac times every margin."""
    return (mg["relu"] > frac * RELU_MARGIN) & (mg["tie"] > frac * VALUE_MARGIN) & (mg["ls"] > frac * LS_MARGIN) & (mg["u"] < U_MAX)


def make_batch(case, nets, n, seed, device):
    """n rows outside the margins, filtered on a float64 pass over 8n + 64 candidates."""
    return _filter(case, nets, _draw(case, 8 * n + 64, seed), n, device)


def _filter(case, nets, cand, n, device, rounds=40):
    """The first n rows of cand outside the margins.  The margins at the updated critics depend on the batch the critics were updated on
    (Adam's first step is lr times the sign of each gradient element), so the filter is run on its own result until every row of the batch
    is outside the margins of an update on exactly that batch; rows that fail are replaced by the next candidates."""
    def ok_rows(b):
        L = _learner(case, nets, torch.float64, device)
        _update(L, b)
        return outside(margins(case, nets, (L.q1, L.q2), b)).cpu()

    usable = ok_rows(cand)
    for _ in range(rounds):
        idx = torch.nonzero(usable).reshape(-1)
        assert idx.numel() >= n, f"only {idx.numel()} of {usable.numel()} candidate rows are outside the margins, {n} needed"
        b = {k: v[idx[:n]].contiguous() for k, v in cand.items()}
        ok = ok_rows(b)
        if bool(ok.all()):
            return b
        usable[idx[:n][~ok]] = False
    raise AssertionError(f"the margin filter did not settle in {rounds} rounds")


def oracle64(case, nets, b, device):
    """The float64 update on batch b: dict(grads {name: array}, norms {name: float}, metrics, params {net: {name: array}}, log_alpha,
    g_log_alpha), names "pol.<key>" / "q1.<key>" / "q2.<key>".  Asserts that every row of b is still beyond half of each margin."""
    n = b["states"].shape[0]
    L = _learner(case, nets, torch.float64, device)
    met = _update(L, b)
    mg = margins(case, nets, (L.q1, L.q2), b)
    assert bool(outside(mg, 0.5).all()), {k: float(v.amin() if k != "u" else v.amax()) for k, v in mg.items()}
    a = lambda t: t.detach().double().cpu().numpy()
    grads = {f"pol.{k}": a(L.pol[k].grad) for k in POLICY_KEYS}
    grads.update({f"{net}.{k}": a(g[k]) for net, g in zip(("q1", "q2"), L.q_grads) for k in S.Q_KEYS})
    norms = {k: float(np.linalg.norm(v)) for k, v in grads.items()}
    # per-row terms of the bias gradients: one learner with the policy's biases widened, one with the critics'
    Lp = _learner(case, nets, torch.float64, device, wide={"pol": n})
    _update(Lp, b)
    Lq = _learner(case, nets, torch.float64, device, wide={"q": n})
    _update(Lq, b)
    terms = {f"pol.{k}": Lp.pol[k].grad for k in POLICY_BIASES}
    terms.update({f"{net}.{k}": g[k] for net, g in zip(("q1", "q2"), Lq.q_grads) for k in Q_BIASES})
    for name, t in terms.items():
        t = t.detach().double()
        assert float((t.sum(0).cpu() - torch.from_numpy(grads[name])).norm()) <= 1e-9 * max(norms[name], 1e-30) + 1e-30, name
        norms[name] = max(norms[name], float(t.pow(2).sum(0).sqrt().norm()))
    params = {"pol": {k: a(L.pol[k]) for k in POLICY_KEYS}, "q1": {k: a(L.q1[k]) for k in S.Q_KEYS}, "q2": {k: a(L.q2[k]) for k in S.Q_KEYS},
              "q1_target": {k: a(L.q1t[k]) for k in S.Q_KEYS}, "q2_target": {k: a(L.q2t[k]) for k in S.Q_KEYS}}
    return dict(grads=grads, norms={k: max(v, 1e-30) for k, v in norms.items()}, metrics=met, params=params,
                log_alpha=float(L.log_alpha.detach()), g_log_alpha=float(L.log_alpha.grad))


# ------------------------------------------------------------------------------------------------------- host-only tests
@pytest.mark.parametrize("name", list(CASES))
def test_restated_layout_matches_the_library(name):
    from rl_x_b200 import _native as nt
    from rl_x_b200.algorithms.sac.b200.sac import POLICY_SEGMENTS, Q_SEGMENTS
    lib = nt.load()
    c = CASES[name]
    po, pp, qo, nq, pq = layout(c.O, c.A, c.H)
    assert int(lib.rlx_sac_policy_param_count(c.O, c.A, c.H)) == pp
    assert int(lib.rlx_sac_q_param_count(c.O, c.A, c.H)) == pq and pq % 64 == 0 and 0 <= pq - nq < 64
    assert qo["critic.4.bias"] + 1 == nq
    for B in (1, 63, c.B):
        assert int(lib.rlx_sac_workspace_bytes(c.O, c.A, c.H, B)) == workspace_bytes(c.O, c.A, c.H, B)
    assert tuple(k for k, _ in POLICY_SEGMENTS) == POLICY_KEYS and tuple(k for k, _ in Q_SEGMENTS) == tuple(S.Q_KEYS)   # the plugin's views agree


def _by_name(case, entry="update"):
    return {g.name: tc_launches(g) for g in sac_gemms(case.O, case.A, case.H, case.B, entry)}


def test_path_table_reaches_what_each_case_is_named_for():
    t = {name: _by_name(c) for name, c in CASES.items()}
    dflt = t["default"]
    # default (17, 6, 256): layer 1s on SIMT, Q layer 2 and its dX looped (Pq % 256 == 64), head on the tensor engine, its dX on SIMT
    assert dflt["q.fwd1"] == dflt["pi.fwd1"] == dflt["q_pi.dx1"] == 0 and dflt["q.fwd2"] == dflt["q.dx2"] == dflt["q_pi.dx2"] == 2
    assert dflt["pi.fwd2"] == dflt["pi.head"] == dflt["pi.dx2"] == 1 and dflt["pi.dx_head"] == 0
    for tab in t.values():    # weight gradients, the Q output layer (N = 1, ldc = 1) and its dX (K = 1) never reach the tensor engine
        assert all(v == 0 for k, v in tab.items() if ".dw" in k or k.endswith((".out", ".dx3")))
    for name in ("split_1", "split_2", "split_16_ragged", "m63", "m129", "m1", "log_std_clamped"):
        assert t[name] == dflt, name
    fl = t["first_layers_tc"]
    assert fl["pi.fwd1"] == 1 and fl["q.fwd1"] == fl["qt.fwd1"] == 2 and fl["q_pi.dx1"] == 2
    assert t["act16"]["pi.dx_head"] == 1 and t["act16"]["pi.head"] == 1
    assert t["act1"]["pi.head"] == t["act3"]["pi.head"] == t["act1"]["pi.dx_head"] == t["act3"]["pi.dx_head"] == 0
    assert t["h64_coordinate"]["q.fwd2"] == t["h64_coordinate"]["q.dx2"] == 1 and t["h64_coordinate"]["q.fwd1"] == 0
    batched = lambda tab: {k: v for k, v in tab.items() if k.split(".")[0] in ("q", "qt", "q_pi") and v}
    assert set(batched(t["h64_all_coordinate"]).values()) == {1} and "q_pi.dx1" in batched(t["h64_all_coordinate"])
    assert sum(t["h100_ragged"].values()) > 0 and sum(t["h1024"].values()) > 0
    assert sum(t["h66_pitch"].values()) == 0 and derive_paths(sac_gemms(17, 6, 66, 1024, "update"), 1) == \
        derive_paths(sac_gemms(17, 6, 66, 1024, "update"), 0)
    k36 = t["h36_k_tail"]
    assert k36["q.dx2"] == k36["q_pi.dx2"] == k36["q.fwd2"] == 1 and 36 % 32 and layout(4, 4, 36)[4] % 36 == 0
    # the acting step: one policy forward
    assert _by_name(CASES["default"], "act") == {"pi.fwd1": 0, "pi.fwd2": 1, "pi.head": 1}


@pytest.mark.parametrize("O,A,H,net_loop", [(17, 6, 256, True), (17, 6, 64, False), (28, 4, 64, False), (4, 4, 36, False), (32, 8, 256, True),
                                            (17, 6, 100, True), (17, 6, 1024, True)])
def test_loop_or_coordinate_per_shape(O, A, H, net_loop):
    """Q layer 2 and its input gradient: one launch for both nets when Pq is a whole number of rows of pitch H, one per net otherwise."""
    Pq = layout(O, A, H)[4]
    assert (Pq % H != 0) == net_loop
    t = _by_name(Case(O, A, H, 1024, False))
    assert t["q.fwd2"] == t["q.dx2"] == (2 if net_loop else 1)


def test_gate_edges():
    g = next(x for x in sac_gemms(32, 8, 256, 1024, "update") if x.name == "pi.fwd1")
    assert tc_launches(g) == 1
    assert tc_launches(g._replace(K=31)) == 0 and tc_launches(g._replace(K=32, lda=32, ldb=32)) == 1    # K < 32
    assert tc_launches(g._replace(ldc=66)) == 0 and tc_launches(g._replace(b=2)) == 0                 # pitch / base not a multiple of 4
    assert tc_launches(g._replace(N=1, ldc=1)) == 0                                                   # the Q output layer
    for A, on in ((1, 0), (2, 1), (3, 0), (6, 1)):                                                    # odd act: ldc = 2A not a multiple of 4
        head = next(x for x in sac_gemms(17, A, 256, 1024, "update") if x.name == "pi.head")
        assert tc_launches(head) == on, A
    q2 = next(x for x in sac_gemms(17, 6, 256, 1024, "update") if x.name == "q.fwd2")
    assert tc_launches(q2) == 2 and tc_launches(q2._replace(sB=256 * 283)) == 1 and tc_launches(q2._replace(sB=4 * 283 + 2)) == 0
    assert derive_paths([g, g._replace(K=8)], 1) == {tc_slot(g): 1, GP_SGEMM: 1} and derive_paths([g, g], 0) == {GP_SGEMM: 2}
    assert derive_paths([q2], 1) == {tc_slot(q2): 2}


def test_float64_oracle_agrees_with_the_float32_oracle():
    """The float64 learner is the same program as the pinned float32 one, and its critic gradient is the one before policy_loss.backward()."""
    case = Case(9, 3, 32, 64, False)
    nets = _nets(case, 1)
    b = _draw(case, 64, 2)
    L32, L64 = _learner(case, nets, torch.float32, "cpu"), _learner(case, nets, torch.float64, "cpu")
    m32, m64 = _update(L32, b), _update(L64, b)
    for k, v in m64.items():
        assert abs(m32[k] - v) <= 2e-5 * max(1.0, abs(v)), k
    for g32, g64 in zip(L32.q_grads, L64.q_grads):
        for k in S.Q_KEYS:
            assert float((g32[k].double() - g64[k]).norm()) <= 2e-5 * float(g64[k].norm()), k
    # q_grads is not what .grad holds at the end (the policy loss accumulated into it)
    assert not torch.equal(L64.q_grads[0]["critic.2.weight"], L64.q1["critic.2.weight"].grad)
    for k in POLICY_KEYS:
        assert float((L32.pol[k].double() - L64.pol[k]).norm()) <= PARAM_BAR * float(L64.pol[k].norm()), k
    assert L64.log_alpha.dtype == torch.float64 and L64.low.dtype == torch.float64


def test_margin_filter_drops_a_row_placed_on_a_kink():
    case = Case(9, 3, 32, 64, False)
    nets = _nets(case, 1)
    cand = _draw(case, 3 * 64 + 64, 3)
    # move row 0's state onto the kink of policy unit 5: its pre-activation becomes exactly zero
    w, b0 = nets[0]["torso.0.weight"][5].double(), nets[0]["torso.0.bias"][5].double()
    s = cand["states"][0].double()
    cand["states"][0] = (s - (w @ s + b0) / (w @ w) * w).float()
    L = _learner(case, nets, torch.float64, "cpu")
    _update(L, cand)
    mg = margins(case, nets, (L.q1, L.q2), cand)
    assert float(mg["relu"][0]) < RELU_MARGIN and bool(outside(mg)[1:].any())
    kept_idx = torch.nonzero(outside(mg)).reshape(-1)
    assert 0 not in kept_idx.tolist()
    kept = _filter(case, nets, cand, 64, "cpu")
    assert not (kept["states"] == cand["states"][0]).all(1).any()
    assert torch.equal(kept["states"][0], cand["states"][int(kept_idx[0])])
    oracle64(case, nets, kept, "cpu")    # the final pass's check holds on the kept rows


# ------------------------------------------------------------------------------------------------------------ device side
@pytest.fixture
def lib():
    """The native library; the GEMM engine is back at 0 (SIMT) after every test whatever it left."""
    from rl_x_b200 import _native as nt
    lib = nt.load()
    try:
        yield lib
    finally:
        lib.rlx_set_gemm_engine(0)


def _t(x):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).to(DEV).contiguous()


def _nan(n):
    return torch.full((n,), float("nan"), device=DEV)


class _Device:
    """The flat buffers of one SAC learner on the device and the update call, every output NaN before the call that writes it."""

    def __init__(self, lib, case, nets):
        from rl_x_b200 import _native as nt
        self.lib, self.nt, self.case = lib, nt, case
        po, self.Pp, self.qo, self.nq, self.Pq = layout(case.O, case.A, case.H)
        self.po = po
        lo, hi = _ls_bounds(case)
        self.d = nt.SacDims(case.O, case.A, case.H, lo, hi)
        P = torch.zeros(self.Pp)
        for k in POLICY_KEYS:
            P[po[k]:po[k] + nets[0][k].numel()] = nets[0][k].reshape(-1)
        Q = torch.zeros(4 * self.Pq)   # the per-net pads are zero, as the plugin allocates them
        for i, net in enumerate(nets[1:5]):
            for k in S.Q_KEYS:
                o = i * self.Pq + self.qo[k]
                Q[o:o + net[k].numel()] = net[k].reshape(-1)
        self.P, self.Q = P.to(DEV), Q.to(DEV)
        adam = nets[5]
        mv = [torch.zeros(self.Pp), torch.zeros(self.Pp), torch.zeros(2 * self.Pq), torch.zeros(2 * self.Pq)]
        for k in POLICY_KEYS:
            for j in (0, 1):
                mv[j][po[k]:po[k] + nets[0][k].numel()] = adam["pol"][k][j].reshape(-1)
        for i, net in enumerate(("q1", "q2")):
            for k in S.Q_KEYS:
                o = i * self.Pq + self.qo[k]
                for j in (0, 1):
                    mv[2 + j][o:o + nets[1][k].numel()] = adam[net][k][j].reshape(-1)
        self.mP, self.vP, self.mQ, self.vQ = (t.to(DEV) for t in mv)
        self.gP, self.gQ, self.gLA = _nan(self.Pp), _nan(2 * self.Pq), _nan(1)
        self.la, self.mLA, self.vLA = _t([LOG_ALPHA0]), adam["la"][0].to(DEV), adam["la"][1].to(DEV)
        self.lr, self.steps = _t([LR]), torch.full((3,), ADAM_STEP0, dtype=torch.int64, device=DEV)
        self.low, self.high = torch.full((case.A,), LOW, device=DEV), torch.full((case.A,), HIGH, device=DEV)

    def update(self, b, fill=float("nan")):
        """One rlx_sac_update_f32 on batch b; the workspace is exactly rlx_sac_workspace_bytes and NaN-filled, the gradient buffers and the
        metrics are filled with `fill` first.  Returns the metrics."""
        c, nt = self.case, self.nt
        B = b["states"].shape[0]
        nbytes = int(self.lib.rlx_sac_workspace_bytes(c.O, c.A, c.H, B))
        assert nbytes > 0 and nbytes % 4 == 0
        ws = _nan(nbytes // 4)
        for g in (self.gP, self.gQ, self.gLA):
            g.fill_(fill)
        metrics = _nan(nt.RLX_SAC_NMETRIC)
        keep = {k: _t(v) for k, v in b.items()}
        a = nt.SacUpdateArgs()
        a.dims, a.batch = self.d, B
        for name, t in [("policy", self.P), ("q", self.Q), ("log_alpha", self.la), ("states", keep["states"]), ("next_states", keep["next_states"]),
                        ("actions", keep["actions"]), ("rewards", keep["rewards"]), ("terminations", keep["terminations"]), ("eps_next", keep["eps_next"]),
                        ("eps_cur", keep["eps_cur"]), ("act_low", self.low), ("act_high", self.high), ("g_policy", self.gP), ("m_policy", self.mP),
                        ("v_policy", self.vP), ("g_q", self.gQ), ("m_q", self.mQ), ("v_q", self.vQ), ("g_log_alpha", self.gLA), ("m_log_alpha", self.mLA),
                        ("v_log_alpha", self.vLA), ("lr", self.lr), ("steps", self.steps), ("metrics", metrics), ("workspace", ws)]:
            setattr(a, name, t.data_ptr())
        a.gamma, a.tau, a.target_entropy = GAMMA, TAU, -float(c.A)
        a.adam_beta1, a.adam_beta2, a.adam_eps = 0.9, 0.999, 1e-8
        a.workspace_bytes = nbytes
        nt.check(self.lib.rlx_sac_update_f32(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "rlx_sac_update_f32")
        torch.cuda.synchronize()
        return metrics.cpu().numpy()

    def named(self, what):
        """{"<net>.<key>": float64 array} of a flat buffer: "grads" (g_policy, g_q) or "params" (policy, q: all four nets)."""
        sp, sq = shapes(self.case.O, self.case.A, self.case.H)
        P, Q = (self.gP, self.gQ) if what == "grads" else (self.P, self.Q)
        P, Q = P.cpu().double().numpy(), Q.cpu().double().numpy()
        out = {f"pol.{k}": P[self.po[k]:self.po[k] + int(np.prod(sp[k]))].reshape(sp[k]) for k in POLICY_KEYS}
        nets = ("q1", "q2") if what == "grads" else Q_NETS
        for i, net in enumerate(nets):
            for k in S.Q_KEYS:
                o = i * self.Pq + self.qo[k]
                out[f"{net}.{k}"] = Q[o:o + int(np.prod(sq[k]))].reshape(sq[k])
        return out

    def pads(self):
        """The per-net pads of g_q, m_q, v_q and the four nets."""
        pad = lambda t, nets: torch.stack([t[i * self.Pq + self.nq:(i + 1) * self.Pq] for i in range(nets)]).cpu()
        return {"g_q": pad(self.gQ, 2), "m_q": pad(self.mQ, 2), "v_q": pad(self.vQ, 2), "q": pad(self.Q, 4)}


def _counted(lib, engine, gemms, fn):
    """fn() on `engine` with the launches of every GEMM path asserted equal to the table derived from `gemms`."""
    from test_gpu_zzzzzz_tc_ppo_shapes import _paths, _tc_instances
    assert lib.rlx_set_gemm_engine(engine) == engine
    out, counts = _paths(lib, fn)
    want = derive_paths(gemms, engine)
    assert counts == want, (f"engine {engine}: GEMM launches by path differ from the derived table", _tc_instances(counts), counts, want,
                            [(g.name, tc_launches(g)) for g in gemms])
    return out, counts


def _check(dev, ref, metrics, fl, label, simt=None):
    """Bounds (i) and (ii) of the module docstring, metrics, temperature, stepped parameters and Polyak targets, and the pads.  Returns the
    gradient distances and a report line."""
    grads = dev.named("grads")
    dist = {}
    for name, g64 in ref["grads"].items():
        g, nrm = grads[name], ref["norms"][name]
        assert np.isfinite(g).all(), (label, name, "an element was not written")
        dist[name] = float(np.linalg.norm(g - g64))
        assert dist[name] <= BAR * nrm, (label, name, dist[name] / nrm)
        if simt is not None:
            F_ = fl["policy" if name.startswith("pol.") else "critic"]
            assert dist[name] <= 2 * simt[name] + F_ * nrm, (label, name, dist[name] / nrm, simt[name] / nrm, F_)
    from rl_x_b200 import _native as nt
    for i, key in enumerate(nt.SAC_METRIC_NAMES):
        v = ref["metrics"][key]
        assert abs(float(metrics[i]) - v) <= BAR * max(1.0, abs(v)), (label, key, float(metrics[i]), v)
    gla = float(dev.gLA.cpu()[0])
    assert abs(gla - ref["g_log_alpha"]) <= BAR * max(1.0, abs(ref["g_log_alpha"])), (label, "g_log_alpha", gla, ref["g_log_alpha"])
    la = float(dev.la.cpu()[0])
    assert abs(la - ref["log_alpha"]) <= PARAM_BAR * max(1.0, abs(ref["log_alpha"])), (label, "log_alpha", la, ref["log_alpha"])
    params = dev.named("params")
    for net, want in ref["params"].items():
        a = np.concatenate([params[f"{net}.{k}"].reshape(-1) for k in want])
        r = np.concatenate([v.reshape(-1) for v in want.values()])
        assert np.linalg.norm(a - r) <= PARAM_BAR * np.linalg.norm(r), (label, net, np.linalg.norm(a - r) / np.linalg.norm(r))
    for what, pad in dev.pads().items():
        assert bool((pad == 0).all()), (label, what, "pad not zero")
    worst = max(dist, key=lambda k: dist[k] / ref["norms"][k])
    return dist, f"{dist[worst] / ref['norms'][worst]:.2e} ({worst})"


def _f32_oracle_distance(case, nets, b, ref):
    """The pinned float32 oracle (CPU) on the same batch: its worst tensor distance to float64, the scale the bars sit on."""
    L = _learner(case, nets, torch.float32, "cpu")
    _update(L, b)
    g = {f"pol.{k}": L.pol[k].grad for k in POLICY_KEYS}
    g.update({f"{net}.{k}": q[k] for net, q in zip(("q1", "q2"), L.q_grads) for k in S.Q_KEYS})
    return max(float(np.linalg.norm(g[k].double().numpy() - v)) / ref["norms"][k] for k, v in ref["grads"].items())


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sac_update_vs_float64_on_both_engines(lib, name):
    case = CASES[name]
    nets = _nets(case, 3)
    b = make_batch(case, nets, case.B, 11, DEV)
    ref = oracle64(case, nets, b, DEV)
    fl = floor(case.O, case.A, case.H, case.B)
    gemms = sac_gemms(case.O, case.A, case.H, case.B, "update")
    simt, report, outs = None, [], []
    for engine in (0, 1):
        dev = _Device(lib, case, nets)     # each engine from the initial state, where the reference is
        metrics, _ = _counted(lib, engine, gemms, lambda: dev.update(b))
        dist, line = _check(dev, ref, metrics, fl, f"{name} engine {engine}", simt)
        report.append(f"engine {engine} worst {line}")
        outs.append(torch.cat([dev.gP, dev.gQ, dev.P, dev.Q, dev.la, dev.gLA]).cpu())
        if engine == 0:
            simt = dist
    if derive_paths(gemms, 1) == derive_paths(gemms, 0):
        assert torch.equal(outs[0], outs[1]), "no tensor GEMM on engine 1, yet the engines differ"
    f32 = _f32_oracle_distance(case, nets, b, ref)
    print(f"\n{name} {tuple(case)}: {'; '.join(report)}; float32 oracle {f32:.2e}; F = {fl['critic']:.2e} / {fl['policy']:.2e}")


@gpu
@pytest.mark.parametrize("engine", [0, 1])
def test_two_updates_do_not_depend_on_what_g_q_held(lib, engine):
    """g_q's per-net pad is written by no gradient kernel: two consecutive updates from a NaN-filled g_q leave the same result, to the bit,
    as from a zero-filled one - metrics finite, the pads of g_q, m_q, v_q and the four nets zero.  At (4, 4, 36) the tensor engine's
    input-gradient GEMMs read net 0's pad through their K tail, so a NaN there would reach the second update's outputs."""
    case = Case(4, 4, 36, 256, False)
    nets = _nets(case, 5)
    b1, b2 = (_draw(case, case.B, s) for s in (21, 22))
    runs = []
    for fill in (float("nan"), 0.0):
        dev = _Device(lib, case, nets)
        mets = []
        for b in (b1, b2):
            mets.append(_counted(lib, engine, sac_gemms(case.O, case.A, case.H, case.B, "update"), lambda: dev.update(b, fill))[0])
            assert np.isfinite(mets[-1][:9]).all(), (fill, mets[-1])
            for what, pad in dev.pads().items():
                assert bool((pad == 0).all()), (fill, what)
        runs.append((np.stack(mets), torch.cat([dev.gP, dev.gQ, dev.P, dev.Q, dev.mQ, dev.vQ, dev.la]).cpu()))
    assert np.array_equal(runs[0][0][:, :9], runs[1][0][:, :9]) and torch.equal(runs[0][1], runs[1][1])


@gpu
@pytest.mark.parametrize("n", [1, 7, 333, 4096])
@pytest.mark.parametrize("O,A,H", [(17, 6, 256), (32, 8, 256)])
def test_sac_act_vs_float64_on_both_engines(lib, O, A, H, n):
    """rlx_sac_act_f32 into NaN outputs, stochastic and deterministic, against the oracle's policy in float64.  logp is compared on the rows
    where max |u| <= U_MAX (beyond, fp32's 1 - tanh^2 is the error, not the kernel) and must be finite on all."""
    from rl_x_b200 import _native as nt
    case = Case(O, A, H, n, False)
    pol = _nets(case, 6)[0]
    g = torch.Generator().manual_seed(n)
    pol = {k: v + 0.05 * torch.randn(v.shape, generator=g) for k, v in pol.items()}
    x, eps = torch.randn(n, O, generator=g), torch.randn(n, A, generator=g)
    low, high = torch.full((A,), LOW), torch.full((A,), HIGH)
    d64 = lambda t: t.to(DEV, torch.float64)
    with torch.no_grad():
        p64 = {k: d64(v) for k, v in pol.items()}
        a_ref, s_ref, lp_ref = (t.cpu() for t in S.policy_get_action(p64, d64(x), d64(eps), d64(low), d64(high)))
        d_ref = S.policy_deterministic(p64, d64(x), d64(low), d64(high)).cpu()
        _, head = _mlp(_pol_layers(p64), d64(x))
        dt_ref = torch.tanh(head[:, :A]).cpu()
        u = head[:, :A] + torch.exp(head[:, A:].clamp(-20.0, 2.0)) * d64(eps)
        sane = (u.abs().amax(1) <= U_MAX).cpu()
    po, Pp = layout(O, A, H)[:2]
    P = torch.zeros(Pp)
    for k in POLICY_KEYS:
        P[po[k]:po[k] + pol[k].numel()] = pol[k].reshape(-1)
    P, dx, de, lo, hi = P.to(DEV), _t(x), _t(eps), low.to(DEV), high.to(DEV)
    dims = nt.SacDims(O, A, H, -20.0, 2.0)
    nbytes = int(lib.rlx_sac_workspace_bytes(O, A, H, n))
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    tol = lambda ref: dict(rtol=1e-5, atol=1e-5 * float(ref.pow(2).mean().sqrt()))
    for engine in (0, 1):
        ws = _nan(nbytes // 4)
        at, ea, lp, det_t, det_e = _nan(n * A), _nan(n * A), _nan(n), _nan(n * A), _nan(n * A)

        def run():
            nt.check(lib.rlx_sac_act_f32(C.byref(dims), P.data_ptr(), dx.data_ptr(), de.data_ptr(), n, lo.data_ptr(), hi.data_ptr(), 0, at.data_ptr(),
                                         ea.data_ptr(), lp.data_ptr(), ws.data_ptr(), nbytes, st()), "rlx_sac_act_f32")
            nt.check(lib.rlx_sac_act_f32(C.byref(dims), P.data_ptr(), dx.data_ptr(), None, n, lo.data_ptr(), hi.data_ptr(), 1, det_t.data_ptr(),
                                         det_e.data_ptr(), None, ws.data_ptr(), nbytes, st()), "rlx_sac_act_f32 deterministic")

        _counted(lib, engine, 2 * sac_gemms(O, A, H, n, "act"), run)
        at, ea, lp, det_t, det_e = (t.cpu().double() for t in (at, ea, lp, det_t, det_e))
        at, ea, det_t, det_e = (t.reshape(n, A) for t in (at, ea, det_t, det_e))
        assert all(bool(torch.isfinite(t).all()) for t in (at, ea, lp, det_t, det_e)), engine
        for ours, ref in ((at, a_ref), (ea, s_ref), (det_e, d_ref), (det_t, dt_ref)):
            np.testing.assert_allclose(ours.numpy(), ref.numpy(), **tol(ref), err_msg=f"engine {engine}")
        lp_ref1 = lp_ref.reshape(-1)
        assert n < 7 or int(sane.sum()) > n // 2
        if bool(sane.any()):
                np.testing.assert_allclose(lp[sane].numpy(), lp_ref1[sane].numpy(), **tol(lp_ref1[sane]), err_msg=f"engine {engine} logp")
        rel = float((at - a_ref).norm() / a_ref.norm())
        assert rel <= 5e-6, (engine, rel)
