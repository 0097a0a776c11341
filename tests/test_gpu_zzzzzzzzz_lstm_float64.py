"""The PPO+LSTM update (rlx_lstm_ppo_minibatch_fwdbwd_f32), the full minibatch step around it (rlx_gather_env_columns_f32,
rlx_mean_popstd_f32, rlx_optax_clip_adam_f32) and the acting step (rlx_lstm_step_f32, rlx_lstm_mask_carry_f32,
rlx_lstm_critic_forward_f32) against oracle/ppo_lstm_oracle.py run in float64, on both GEMM engines of `aux_gemm` and both recurrence
paths, with the launches of every GEMM path asserted around every call.

Why.  test_gpu_zzz_ppo_lstm.py compares with the float32 oracle at rtol 3e-4, and proves the tensor engine ran with one global count.  Here
every case runs from the same state in a NaN-filled workspace of exactly rlx_lstm_minibatch_workspace_bytes, into NaN-filled gradient buffers,
from a nonzero initial carry: an element no kernel wrote fails the numeric checks.

Proof of path.  aux_gemm falls back to the SIMT engine without a word when the wgmma engine returns RLX_ERR_UNSUPPORTED.  `fwdbwd_gemms`,
`step_gemms` and `critic_gemms` list the GEMMs of each entry point as lstm.cu issues them (operand offsets from the parameter layout, the
K-major copies and the workspace plan, restated below and checked against the library's own layout / workspace size in a host build), and
every call asserts the launches per tc_gemm_kernel instance and of the SIMT GEMM (test_gpu_zzzzzzz_aux_tc_float64.py's `_counted`), and the
change of rlx_lstm_persistent_launch_count: 2 where `seq_cfg` (restated) lets the one-launch recurrence run, else 0.  The table found a
defect: the K-major copies sat at the parameters' own offsets, so with FiLM and an odd act the copy of Wf was not 16-byte aligned and both
FiLM products ran on the SIMT engine (`in_place=True` restates that; test_table_edges shows it).

Bounds, per parameter segment g (never one norm over a whole network), g64 the float64 oracle's gradient:
  (i)  ||g - g64|| <= max(BAR N, K32 d32) on both engines, N = max(||g64||, root-sum-square of the per-row terms) for the segments that are
       sums over rows (Linear and LSTM biases, LayerNorm scales and biases; a sum of signed terms can cancel while each term keeps its own
       rounding), d32 = ||g32 - g64|| the distance of the float32 oracle (GPU, TF32 off) on the same inputs.
  (ii) ||g_tc - g64|| <= 2 ||g_simt - g64|| + F N.
Why d32.  Measured on an H100 (80 GB HBM3, 700 W), the float32 oracle on the same inputs sits at 7e-7 to 4.6e-6 of N (the largest at act 64,
on bh), the SIMT engine at up to 1.17e-5 and the tensor engine at up to 1.13e-5, both on that same segment; everywhere else both engines stay
under 4.5e-6.  The SIMT engine runs the same fp32 arithmetic as the float32 oracle in another order (a sequential FMA chain per output instead of
cuBLAS's blocked sums), so its distance is of the size of d32, not of a fixed constant: K32 = 4 bounds it with room for the order (the ratio is
2.5 where it decides).  The float32 oracle is itself checked against float64 at a small shape (test_float64_oracle_agrees_with_the_float32_oracle).
Derivation of (ii).  Both engines run the same fp32 program except the GEMMs, so g_tc - g64 = (g_simt - g64) + (E_tc - E_simt), E_x the part of
the error engine x's GEMMs cause; ||E_simt|| <= ||g_simt - g64||, hence the 2.  One 3xTF32 product is within e(K) = 6e-7 + 3.2e-9 min(K, 1024)
of its output's norm (test_gpu_tc_engine.py), and an output error reaches a gradient with a gain of order one (tanh', sigmoid' <= 1,
LayerNorm of order one, the recurrence contracting through the forget gate).  A segment depends on a subset of its network's forward and
input-gradient products plus its own weight-gradient product, so F = sum of e(K) over the network's forward and input-gradient products that
ran on the tensor engine + e(min(R, 1024)) (`_floor`, 7e-7 to 1.5e-5 here).  Single-pass TF32 (about 5e-4 per product) misses (i) and (ii).

The per-step and one-launch recurrences run the same arithmetic in the same order: gradients and metrics must agree bit for bit.

Sorted after the other GPU files: a kernel fault on a new shape takes the CUDA context with it, and then costs only this file."""
import contextlib
import ctypes as C
import math
import os
import time

import numpy as np
import pytest
import torch

from oracle import ppo_lstm_oracle as L
from test_gpu_zzzzzzz_aux_tc_float64 import (GP_SGEMM, INSTANCES, TC_BIAS, TC_BIAS_TANH, TC_DTANH, TC_NONE, Gemm, _counted, derive_paths,
                                             on_tensor_engine)
from test_lstm_emulation import CRITIC_SEGS, POLICY_SEGS, flatten_critic, flatten_policy

gpu = pytest.mark.gpu
DEV = "cuda"
OPT_FILM, OPT_SHARED = 1, 2              # RLX_LSTM_OPT_*
CLIP, ENT, CC, MAX_NORM, LR = 0.2, 0.01, 0.5, 0.5, 3e-4
BAR, K32, PARAM_BAR, NU_BAR = 1e-5, 4.0, 3e-5, 3e-5
WGRAD_ROWS = 1024                        # lstm.cu: kWgradRows
EPI = dict(none=TC_NONE, bias=TC_BIAS, bias_tanh=TC_BIAS_TANH, dtanh=TC_DTANH)   # lstm.cu's EPI_* as the tensor engine's epilogues

# segment indices of the flat layouts (lstm.cu: PSeg / CSeg)
(WE1, BE1, G1, N1, WE2, BE2, G2, N2, WI, WH, BH, GL, NL, WT1, BT1, WT2, BT2, WM, BM, LOGSTD, WF, BF) = range(22)
WC1, BC1, WC2, BC2, WC3, BC3 = range(6)


# ----------------------------------------------------------------------------------------------- lstm.cu, restated
def _up(x, a):
    return -(-x // a) * a


def layout(dims):
    """make_layout: (policy offsets [23], critic offsets [7]), nothing rounded."""
    O, A, H, E, Lh, opt = dims
    E2, TIW, F = (0 if opt & OPT_SHARED else E), (E if opt & OPT_FILM else E + Lh), (2 * E if opt & OPT_FILM else 0)
    ps = [O * E, E, E, E, O * E2, E2, E2, E2, E * 4 * Lh, Lh * 4 * Lh, 4 * Lh, Lh, Lh, TIW * H, H, H * H, H, H * A, A, A, Lh * F, F]
    cs = [O * H, H, H * H, H, H, 1]
    return [int(v) for v in np.concatenate([[0], np.cumsum(ps)])], [int(v) for v in np.concatenate([[0], np.cumsum(cs)])]


def kmajor(offs):
    """kmajor_layout: the same segments, each starting on a multiple of 4 floats."""
    out, o = [], 0
    for a, b in zip(offs[:-1], offs[1:]):
        o = _up(o, 4)
        out.append(o)
        o += b - a
    return out + [o]


def plan(dims, T, n):
    """plan(): workspace offsets in floats, and "total" in bytes."""
    O, A, H, E, Lh, opt = dims
    R, w, o = T * n, {}, 0
    film = 1 if opt & OPT_FILM else 0

    def take(name, cnt):
        nonlocal o
        w[name] = o
        o += _up(cnt, 64)
    for name, cnt in (("Z1", R * E), ("E1", R * E), ("Z2", R * E), ("TI", R * (E + Lh)), ("Gi", R * 4 * Lh), ("Gates", R * 4 * Lh), ("Call", R * Lh),
                      ("Hall", R * Lh), ("Hm", R * Lh), ("Cm", R * Lh), ("T1", R * H), ("T2", R * H), ("C1", R * H), ("C2", R * H), ("Mean", R * A),
                      ("V", R), ("dMean", R * A), ("dV", R), ("Terms", R * 4), ("dLs", R * A), ("dT2", R * H), ("dT1", R * H), ("dTI", R * (E + Lh)),
                      ("dHall", R * Lh), ("dG", R * 4 * Lh), ("dE1", R * E), ("dZ1", R * E), ("dZ2", R * E), ("dC2", R * H), ("dC1", R * H),
                      ("Gh", n * 4 * Lh), ("dHn", n * Lh), ("dCn", n * Lh), ("Small", 64), ("Stats1", R * 2), ("Stats2", R * 2), ("StatsL", R * 2)):
        take(name, cnt)
    take("Part", -(-R // WGRAD_ROWS) * max(O * E, E * 4 * Lh, Lh * 4 * Lh, (E + Lh) * H, H * H, H * A, O * H, H, Lh * 2 * E))
    take("Col", -(-R // 256) * max(8, H, 4 * Lh, 2 * E, 2 * Lh, A))
    take("WhT", 4 * Lh * Lh)
    for name, cnt in (("E2", R * E), ("LL", R * Lh), ("GB", R * 2 * E), ("dGB", R * 2 * E), ("dOL", R * E), ("dLL", R * Lh)):
        take(name, film * cnt)
    p, c = layout(dims)
    take("TP", kmajor(p)[-1])
    take("TC", kmajor(c)[-1])
    w["total"] = 4 * o
    return w


def seq_cfg(Lh, persistent=True):
    """seq_cfg: (envs per block, threads, shared bytes forward, backward, one-launch path taken)."""
    epb = max(1, 128 // Lh)
    smem_f, smem_b = 4 * (Lh * 4 * Lh + 2 * epb * Lh), 4 * (4 * Lh * Lh + 2 * epb * 4 * Lh)
    return epb, epb * Lh, smem_f, smem_b, bool(persistent) and epb * Lh <= 1024 and max(smem_f, smem_b) <= 200 * 1024


def fwdbwd_gemms(dims, T, n, in_place=False):
    """The GEMMs of rlx_lstm_ppo_minibatch_fwdbwd_f32 in issue order.  Offsets: workspace buffers from plan(), the K-major copies PT / TC at
    kmajor() (in_place: at the parameters' own offsets, the layout before the fix), the states X an allocation of their own."""
    O, A, H, E, Lh, opt = dims
    film, shared = opt & OPT_FILM, opt & OPT_SHARED
    R, EL = T * n, E + Lh
    TIW = E if film else EL
    p, c = layout(dims)
    kp, kc = (p, c) if in_place else (kmajor(p), kmajor(c))
    w = plan(dims, T, n)
    PT, CT = (lambda s: w["TP"] + kp[s]), (lambda s: w["TC"] + kc[s])
    X = 0
    LLp = w["LL"] if film else w["TI"] + E

    def fwd(name, x, ldx, wt, inp, out, epi, cc, ldc):             # dense_fwd_t
        return Gemm(name, 1, 1, EPI[epi], R, out, inp, ldx, inp, ldc, x, wt, cc, 1, 0)

    def dx(name, dy, ldy, wt, inp, out, epi, cc, ldc):             # dense_bwd_input_t
        return Gemm(name, 1, 0, EPI[epi], R, inp, out, ldy, inp, ldc, dy, wt, cc, 1, 0)

    def dw(name, x, ldx, dy, ldy, inp, out):                       # dense_bwd_weight: partials at Part, one per row split
        return Gemm(name, 0, 0, TC_NONE, inp, out, R, ldx, ldy, out, x, dy, w["Part"], -(-R // WGRAD_ROWS), inp * out)

    g = [fwd("fwd.WE1", X, O, PT(WE1), O, E, "bias", w["Z1"], E)]
    if not shared:
        g.append(fwd("fwd.WE2", X, O, PT(WE2), O, E, "bias", w["Z2"], E))
    g.append(fwd("fwd.WI", w["E1"], E, PT(WI), E, 4 * Lh, "none", w["Gi"], 4 * Lh))
    if film:
        g.append(fwd("fwd.WF", LLp, Lh, PT(WF), Lh, 2 * E, "bias", w["GB"], 2 * E))
    g += [fwd("fwd.WT1", w["TI"], TIW, PT(WT1), TIW, H, "bias_tanh", w["T1"], H), fwd("fwd.WT2", w["T1"], H, PT(WT2), H, H, "bias_tanh", w["T2"], H),
          fwd("fwd.WM", w["T2"], H, PT(WM), H, A, "bias", w["Mean"], A),
          fwd("fwd.WC1", X, O, CT(WC1), O, H, "bias_tanh", w["C1"], H), fwd("fwd.WC2", w["C1"], H, CT(WC2), H, H, "bias_tanh", w["C2"], H),
          fwd("fwd.WC3", w["C2"], H, CT(WC3), H, 1, "bias", w["V"], 1)]
    g += [dw("dw.WM", w["T2"], H, w["dMean"], A, H, A), dx("dx.WM", w["dMean"], A, PT(WM), H, A, "dtanh", w["dT2"], H),
          dw("dw.WT2", w["T1"], H, w["dT2"], H, H, H), dx("dx.WT2", w["dT2"], H, PT(WT2), H, H, "dtanh", w["dT1"], H),
          dw("dw.WT1", w["TI"], TIW, w["dT1"], H, TIW, H), dx("dx.WT1", w["dT1"], H, PT(WT1), TIW, H, "none", w["dTI"], TIW)]
    if film:
        g += [dw("dw.WF", LLp, Lh, w["dGB"], 2 * E, Lh, 2 * E), dx("dx.WF", w["dGB"], 2 * E, PT(WF), Lh, 2 * E, "none", w["dLL"], Lh)]
    if not shared:
        g.append(dw("dw.WE2", X, O, w["dZ2"], E, O, E))
    g += [dw("dw.WH", w["Hm"], Lh, w["dG"], 4 * Lh, Lh, 4 * Lh), dw("dw.WI", w["E1"], E, w["dG"], 4 * Lh, E, 4 * Lh),
          dx("dx.WI", w["dG"], 4 * Lh, PT(WI), E, 4 * Lh, "none", w["dE1"], E), dw("dw.WE1", X, O, w["dZ1"], E, O, E),
          dw("dw.WC3", w["C2"], H, w["dV"], 1, H, 1), dx("dx.WC3", w["dV"], 1, CT(WC3), H, 1, "dtanh", w["dC2"], H),
          dw("dw.WC2", w["C1"], H, w["dC2"], H, H, H), dx("dx.WC2", w["dC2"], H, CT(WC2), H, H, "dtanh", w["dC1"], H),
          dw("dw.WC1", X, O, w["dC1"], H, O, H)]
    return g


def _flax_fwd(name, rows, x, ldx, wofs, inp, out, epi, cc, ldc):   # dense_fwd: the kernel read in place, [in, out]
    return Gemm(name, 1, 0, EPI[epi], rows, out, inp, ldx, out, ldc, x, wofs, cc, 1, 0)


def critic_gemms(dims, rows):
    """critic_rows (rlx_lstm_critic_forward_f32, and the value of rlx_lstm_step_f32) on `rows` rows: x and out allocations of their own."""
    O, H = dims[0], dims[2]
    c, w = layout(dims)[1], plan(dims, 1, rows)
    return [_flax_fwd("critic.WC1", rows, 0, O, c[WC1], O, H, "bias_tanh", w["C1"], H),
            _flax_fwd("critic.WC2", rows, w["C1"], H, c[WC2], H, H, "bias_tanh", w["C2"], H),
            _flax_fwd("critic.WC3", rows, w["C2"], H, c[WC3], H, 1, "bias", 0, 1)]


def step_gemms(dims, n, value=True):
    """policy_one_step (+ critic_rows) of rlx_lstm_step_f32: obs and the carry h allocations of their own."""
    O, A, H, E, Lh, opt = dims
    film, shared = opt & OPT_FILM, opt & OPT_SHARED
    TIW = E if film else E + Lh
    p, w = layout(dims)[0], plan(dims, 1, n)
    f = lambda *a: _flax_fwd(a[0], n, *a[1:])
    g = [f("step.WE1", 0, O, p[WE1], O, E, "bias", w["Z1"], E)]
    if not shared:
        g.append(f("step.WE2", 0, O, p[WE2], O, E, "bias", w["Z2"], E))
    g += [f("step.WI", w["E1"], E, p[WI], E, 4 * Lh, "none", w["Gi"], 4 * Lh), f("step.WH", 0, Lh, p[WH], Lh, 4 * Lh, "none", w["Gh"], 4 * Lh)]
    if film:
        g.append(f("step.WF", w["LL"], Lh, p[WF], Lh, 2 * E, "bias", w["GB"], 2 * E))
    g += [f("step.WT1", w["TI"], TIW, p[WT1], TIW, H, "bias_tanh", w["T1"], H), f("step.WT2", w["T1"], H, p[WT2], H, H, "bias_tanh", w["T2"], H),
          f("step.WM", w["T2"], H, p[WM], H, A, "bias", w["Mean"], A)]
    return g + (critic_gemms(dims, n) if value else [])


def _e(K):
    """test_gpu_tc_engine.py's error model of one 3xTF32 product, relative to the output's norm; chains capped at 1024 rows."""
    return 6e-7 + 3.2e-9 * min(K, 1024)


def _floor(gemms, R):
    """F of the module docstring, per network: (policy, critic)."""
    f = {"W": 0.0, "C": 0.0}
    for g in gemms:
        if g.a_kmaj and on_tensor_engine(g):
            f["C" if g.name.split(".")[1].startswith("WC") else "W"] += _e(g.K)
    return f["W"] + _e(R), f["C"] + _e(R)


# ------------------------------------------------------------------------------------------------------ the oracle
def _params(dims, seed, wi_scale=1.0):
    O, A, H, E, Lh, opt = dims
    pol, cri = L.init_params(O, A, hidden=H, enc=E, lstm=Lh, std_dev=0.8, seed=seed, share_encoder=bool(opt & OPT_SHARED),
                             combine="film" if opt & OPT_FILM else "concat")
    g = torch.Generator().manual_seed(seed + 1)
    for tree in (pol, cri):
        for name, v in L.tree_leaves(tree):
            if name.endswith("bias") or name.endswith("scale"):
                v.add_(0.1 * torch.randn(v.shape, generator=g))
    for k in L.GATES:
        pol["lstm"]["i" + k]["kernel"].mul_(wi_scale)
    return pol, cri


def _to(tree, dtype, device):
    return L.tree_map(lambda v: v.detach().to(device, dtype), tree)


def _tree_from_leaves(tree, leaves):
    """A tree shaped like `tree` holding `leaves` in L.tree_leaves order."""
    it = iter(leaves)
    names = [nm for nm, _ in L.tree_leaves(tree)]
    out = {}
    for nm in names:
        node = out
        *path, last = nm.split(".")
        for k in path:
            node = node.setdefault(k, {})
        node[last] = next(it)
    return out


def _flat(tree, policy):
    return torch.cat([t.reshape(-1).to(torch.float64).cpu() for t in (flatten_policy(tree) if policy else flatten_critic(tree))])


def _segments(flat, offs):
    return [flat[a:b] for a, b in zip(offs[:-1], offs[1:])]


def _tree_from_flat(like, flat, policy):
    """Inverse of flatten_policy / flatten_critic: a tree shaped like `like` from a flat-layout vector."""
    leaves = L.tree_leaves(like)
    base = np.cumsum([0] + [v.numel() for _, v in leaves])
    index = _tree_from_leaves(like, [torch.arange(base[i], base[i + 1], dtype=torch.float64).reshape(v.shape) for i, (_, v) in enumerate(leaves)])
    pos = _flat(index, policy).long()
    vec = torch.empty(int(base[-1]), dtype=flat.dtype)
    vec[pos] = flat.cpu()
    return _tree_from_leaves(like, [vec[base[i]:base[i + 1]].reshape(v.shape) for i, (_, v) in enumerate(leaves)])


@contextlib.contextmanager
def _row_terms(rec):
    """While active, every Linear, LayerNorm and LSTM-cell call of the oracle adds a zero tensor of its output's shape to it: its gradient is the
    per-row terms of the bias (for LayerNorm also, times xhat, of the scale).  rec: [(leaf id, zero tensor, xhat or None)]."""
    dense0, ln0, cell0 = L.dense, L.layer_norm, L.lstm_cell

    def zero_like(y):
        return torch.zeros_like(y).requires_grad_(True)

    def dense(p, x):
        y = dense0(p, x)
        z = zero_like(y)
        rec.append((id(p["bias"]), z, None))
        return y + z

    def layer_norm(p, x):
        y = ln0(p, x)
        z = zero_like(y)
        with torch.no_grad():
            mean = x.mean(-1, keepdim=True)
            xhat = (x - mean) * torch.rsqrt(torch.clamp((x * x).mean(-1, keepdim=True) - mean * mean, min=0.0) + L.LN_EPS)
        rec.extend([(id(p["bias"]), z, None), (id(p["scale"]), z, xhat)])
        return y + z

    def lstm_cell(p, carry, x):
        p2 = dict(p)
        for k in L.GATES:
            b = p["h" + k]["bias"]
            z = torch.zeros(x.shape[0], b.shape[0], dtype=b.dtype, device=b.device, requires_grad=True)
            rec.append((id(b), z, None))
            p2["h" + k] = {"kernel": p["h" + k]["kernel"], "bias": b + z}
        return cell0(p2, carry, x)

    L.dense, L.layer_norm, L.lstm_cell = dense, layer_norm, lstm_cell
    try:
        yield rec
    finally:
        L.dense, L.layer_norm, L.lstm_cell = dense0, ln0, cell0


def oracle(pol, cri, mb, dtype, device, terms=True):
    """Learner.grads in `dtype` on `device` (TF32 off): (policy segments, critic segments, metrics, policy norms N, critic norms N) in the flat
    layout as float64 numpy arrays.  With terms, N is max(||g||, root-sum-square of the per-row terms) for the row sums (module docstring)."""
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        mbd = {k: (tuple(t.to(device, dtype) for t in v) if k == "init_carry" else v.to(device, dtype)) for k, v in mb.items()}
        lr = L.Learner(_to(pol, dtype, device), _to(cri, dtype, device), clip_range=CLIP, entropy_coef=ENT, critic_coef=CC)
        gp, gc, met = lr.grads(mbd)
        rss = {}
        if terms:
            rec = []
            adv = mbd["advantages"]
            with _row_terms(rec):
                loss, _ = L.loss_fn(lr.pol, lr.cri, mbd["states"], mbd["actions"], mbd["log_probs"], mbd["returns"],
                                    (adv - adv.mean()) / (adv.std(unbiased=False) + 1e-8), mbd["dones"], mbd["init_carry"], CLIP, ENT, CC)
                gz = torch.autograd.grad(loss, [z for _, z, _ in rec])
            sq, sums = {}, {}
            for (leaf, _, xhat), t in zip(rec, gz):
                t = (t if xhat is None else t * xhat).reshape(-1, t.shape[-1])
                sq[leaf] = sq.get(leaf, 0.0) + t.pow(2).sum(0)
                if xhat is None:
                    sums[leaf] = sums.get(leaf, 0.0) + t.sum(0)
            rss = {leaf: s.sqrt() for leaf, s in sq.items()}
            byid = dict(zip([id(v) for v in lr.pleaves + lr.cleaves], gp + gc))
            for leaf, s in sums.items():   # the bias terms sum to the oracle's own gradient
                assert float((s - byid[leaf]).norm()) <= 1e-9 * float(byid[leaf].norm()) + 1e-12
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32

    def flat(leaves, grads, policy):
        tree = lr.pol if policy else lr.cri
        g = _flat(_tree_from_leaves(tree, grads), policy).numpy()
        r = _flat(_tree_from_leaves(tree, [rss.get(id(v), torch.zeros_like(v)) for v in leaves]), policy).numpy()
        return g, r
    gpf, rpf = flat(lr.pleaves, gp, True)
    gcf, rcf = flat(lr.cleaves, gc, False)
    return gpf, gcf, rpf, rcf, met


# ------------------------------------------------------------------------------------------------ inputs of one case
def make_case(dims, T, n, seed, dones="rand", wi_scale=1.0):
    """Parameters and a minibatch: nonzero initial carry; old log-probs 0.15 (in log ratio) from the float64 policy's, kept 1e-3 away from the clip
    edges so that no row switches its PPO branch between two computations."""
    O, A, Lh = dims[0], dims[1], dims[4]
    pol, cri = _params(dims, seed, wi_scale)
    g = torch.Generator().manual_seed(seed + 2)
    r = lambda *s: torch.randn(*s, generator=g)
    dn = {"rand": (torch.rand(T, n, generator=g) < 0.2).float(), "none": torch.zeros(T, n), "all": torch.ones(T, n),
          "t0": torch.cat([torch.ones(1, n), torch.zeros(T - 1, n)]), "last": torch.cat([torch.zeros(T - 1, n), torch.ones(1, n)])}[dones]
    mb = dict(states=r(T, n, O), actions=r(T, n, A) * 0.8, returns=r(T, n), advantages=r(T, n), dones=dn, init_carry=(r(n, Lh) * 0.5, r(n, Lh) * 0.5))
    dev = DEV if torch.cuda.is_available() else "cpu"
    with torch.no_grad():
        p64 = _to(pol, torch.float64, dev)
        mean, logstd = L.forward_sequence(p64, mb["states"].to(dev, torch.float64), mb["dones"].to(dev, torch.float64),
                                          tuple(t.to(dev, torch.float64) for t in mb["init_carry"]))
        a = mb["actions"].to(dev, torch.float64)
        lp = (-0.5 * ((a - mean) / logstd.exp()) ** 2 - 0.5 * math.log(2 * math.pi) - logstd).sum(-1).cpu()
    delta = 0.15 * r(T, n).double()
    for edge in (math.log(1 - CLIP), math.log(1 + CLIP)):
        delta = torch.where((delta - edge).abs() < 1e-3, delta + 3e-3, delta)
    mb["log_probs"] = (lp - delta).float()
    return pol, cri, mb


def references(pol, cri, mb):
    """(float64 oracle, float32 oracle), both on the GPU when there is one."""
    dev = DEV if torch.cuda.is_available() else "cpu"
    return oracle(pol, cri, mb, torch.float64, dev), oracle(pol, cri, mb, torch.float32, dev, terms=False)


def _norms(g, r):
    return max(float(np.linalg.norm(g)), float(np.linalg.norm(r)), 1e-30)


# ------------------------------------------------------------------------------------------------------ host-only tests
BASE = (64, 8, 256, 128, 64, 0)   # BASELINE config 5: obs 64, act 8, hidden 256, enc 128, lstm 64


@pytest.fixture(scope="module")
def emu_layout(tmp_path_factory):
    """The host build of lstm.cu (test_lstm_emulation.py): its rlx_lstm_param_layout and rlx_lstm_minibatch_workspace_bytes."""
    import subprocess
    from conftest import emu_build_cmd
    from test_lstm_emulation import Dims, ROOT
    out = tmp_path_factory.mktemp("lstm_layout") / "liblstm_emu.so"
    subprocess.run(emu_build_cmd(out, os.path.join(ROOT, "rl_x_b200", "csrc", "lstm.cu")), check=True)
    lib = C.CDLL(str(out))
    lib.rlx_lstm_minibatch_workspace_bytes.restype = C.c_size_t
    lib.rlx_lstm_minibatch_workspace_bytes.argtypes = [C.POINTER(Dims), C.c_int64, C.c_int64]
    return lib, Dims


@pytest.mark.parametrize("dims,T,n", [(BASE, 128, 256), ((64, 17, 256, 128, 64, OPT_FILM), 32, 96), ((63, 33, 128, 64, 113, OPT_SHARED), 33, 100),
                                      ((64, 8, 128, 64, 48, OPT_FILM | OPT_SHARED), 5, 6)])
def test_restated_layout_and_plan_match_the_library(emu_layout, dims, T, n):
    lib, Dims = emu_layout
    d = Dims(*dims)
    poff, coff = (C.c_int64 * 23)(), (C.c_int64 * 7)()
    assert lib.rlx_lstm_param_layout(C.byref(d), poff, coff) == 0
    p, c = layout(dims)
    assert list(poff) == p and list(coff) == c
    assert lib.rlx_lstm_minibatch_workspace_bytes(C.byref(d), T, n) == plan(dims, T, n)["total"]


def _tc_names(gemms):
    return {g.name for g in gemms if on_tensor_engine(g)}


def test_table_edges():
    """Which products reach the tensor engine, at the edges of aux_gemm's gate and tc_gemm_impl's checks."""
    T, n = 16, 64
    base = _tc_names(fwdbwd_gemms(BASE, T, n))
    assert base == {"fwd.WE1", "fwd.WE2", "fwd.WI", "fwd.WT1", "fwd.WT2", "fwd.WC1", "fwd.WC2", "dw.WT2", "dx.WT2", "dw.WT1", "dx.WT1", "dw.WE2", "dw.WH",
                    "dw.WI", "dx.WI", "dw.WE1", "dw.WC2", "dx.WC2", "dw.WC1"}, base
    assert {(g.a_kmaj, g.b_kmaj, g.epi) for g in fwdbwd_gemms(BASE, T, n)} <= INSTANCES
    # act: 8 keeps the three WM products on SIMT; at 32 the input gradient (K = act) goes to the tensor engine; 33 leaves by the dMean pitch;
    # 64 (the dims_ok maximum) puts all three there
    wm = lambda act: _tc_names(g for g in fwdbwd_gemms((64, act, 256, 128, 64, 0), T, n) if g.name.endswith(".WM"))
    assert (wm(8), wm(32), wm(33), wm(64)) == (set(), {"dx.WM"}, set(), {"fwd.WM", "dx.WM", "dw.WM"})
    # obs not a multiple of 4: exactly the products reading the states X leave, by their pitch
    assert base - _tc_names(fwdbwd_gemms((63,) + BASE[1:], T, n)) == {"fwd.WE1", "fwd.WE2", "fwd.WC1", "dw.WE1", "dw.WE2", "dw.WC1"}
    # lstm 32: dW of Wh has M = 32
    assert base - _tc_names(fwdbwd_gemms(BASE[:4] + (32, 0), T, n)) == {"dw.WH"}
    # rows: below 64 the forward and input-gradient products leave (M = R); the weight gradients (K = R) stay down to 32 rows
    assert _tc_names(fwdbwd_gemms(BASE, 7, 9)) == {nm for nm in base if nm.startswith("dw.")}
    assert _tc_names(fwdbwd_gemms(BASE, 5, 6)) == set()
    # lstm 113: the torso input [OL | LL] has an odd pitch and so has Hm
    assert base - _tc_names(fwdbwd_gemms(BASE[:4] + (113, 0), T, n)) == {"fwd.WT1", "dw.WT1", "dx.WT1", "dw.WH"}
    # FiLM with an odd act: Wf sits at 2 mod 4 in the parameters; read at that offset, both FiLM products would run SIMT
    film = (64, 17, 256, 128, 64, OPT_FILM)
    p = layout(film)[0]
    assert p[WF] == 169890 and p[WF] % 4 == 2 and all(o % 4 == 0 for o in kmajor(p)[:-1] + kmajor(layout(film)[1])[:-1])
    assert _tc_names(fwdbwd_gemms(film, T, n)) - _tc_names(fwdbwd_gemms(film, T, n, in_place=True)) == {"fwd.WF", "dx.WF"}
    assert {"fwd.WF", "dx.WF", "dw.WF"} <= _tc_names(fwdbwd_gemms(film, T, n))
    # the table's counters: one slot per launch
    want = derive_paths(fwdbwd_gemms(BASE, T, n), 1)
    assert sum(want.values()) == len(fwdbwd_gemms(BASE, T, n)) and want[GP_SGEMM] == len(fwdbwd_gemms(BASE, T, n)) - len(base)
    assert derive_paths(fwdbwd_gemms(BASE, T, n), 0) == {GP_SGEMM: len(fwdbwd_gemms(BASE, T, n))}
    # acting step: only Wi / Wh (EPI_NONE, kernel read in place) have an instance; at n >= 64 they go to the tensor engine
    assert _tc_names(step_gemms(BASE, 64)) == {"step.WI", "step.WH"} and _tc_names(step_gemms(BASE, 63)) == set()
    assert _tc_names(critic_gemms(BASE, 4097)) == set()


def test_persistent_gate():
    """seq_cfg: envs per block, block size and the 200 KB shared-memory gate."""
    assert seq_cfg(32)[:2] == (4, 128) and seq_cfg(48)[:2] == (2, 96) and seq_cfg(64)[:2] == (2, 128) and seq_cfg(100)[:2] == (1, 100)
    assert seq_cfg(112) == (1, 112, 201600, 204288, True)
    assert seq_cfg(113)[2:] == (205208, 207920, False)   # both above 200 KB: the per-step path
    assert not seq_cfg(64, persistent=False)[4]


def test_float64_oracle_agrees_with_the_float32_oracle():
    """The float64 oracle is the same program as the float32 one: at a small FiLM shape every segment agrees to float32 accuracy, and the
    per-row terms sum to the bias gradients (asserted inside `oracle`)."""
    dims = (6, 3, 12, 8, 4, OPT_FILM)
    pol, cri, mb = make_case(dims, 9, 7, 5)
    gp64, gc64, rp, rc, m64 = oracle(pol, cri, mb, torch.float64, "cpu")
    gp32, gc32, _, _, m32 = oracle(pol, cri, mb, torch.float32, "cpu", terms=False)
    p, c = layout(dims)
    for a, b, r, offs in ((gp32, gp64, rp, p), (gc32, gc64, rc, c)):
        for x, y, t in zip(_segments(a, offs), _segments(b, offs), _segments(r, offs)):
            assert np.linalg.norm(x - y) <= 1e-5 * _norms(y, t)
    for k, v in m64.items():
        assert abs(m32[k] - v) <= 1e-5 * max(1.0, abs(v)), k


# ------------------------------------------------------------------------------------------------------ device side
@pytest.fixture
def lib():
    """The native library; the aux GEMM engine and the recurrence switch go back to the process defaults after every test."""
    from rl_x_b200 import _native as nt
    lib = nt.load()
    try:
        yield lib
    finally:
        lib.rlx_set_aux_gemm_engine(int(os.environ.get("RLX_AUX_GEMM_ENGINE", "0") == "1"))
        lib.rlx_set_lstm_persistent(int(os.environ.get("RLX_LSTM_PERSISTENT", "0") == "1"))


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _proven(lib, engine, persistent, gemms, launches, fn):
    """fn() with the GEMM path table and the change of the persistent launch count asserted."""
    assert lib.rlx_set_lstm_persistent(persistent) == persistent
    before = int(lib.rlx_lstm_persistent_launch_count())
    out, _ = _counted(lib, engine, gemms, fn)
    assert int(lib.rlx_lstm_persistent_launch_count()) - before == launches
    return out


class _Fwdbwd:
    """One learner's flat buffers on the device and the fwdbwd call: NaN workspace of exactly the size asked for, NaN gradients and metrics."""

    def __init__(self, lib, dims, T, n, P, Cc):
        from rl_x_b200 import _native as nt
        self.lib, self.nt, self.dims, self.T, self.n, self.P, self.Cc = lib, nt, dims, T, n, P, Cc
        self.d = nt.LstmDims(*dims)
        self.nbytes = int(lib.rlx_lstm_minibatch_workspace_bytes(C.byref(self.d), T, n))
        assert self.nbytes == plan(dims, T, n)["total"]
        self.ws = torch.empty(self.nbytes // 4, device=DEV)
        self.gP, self.gC, self.metrics = torch.empty_like(P), torch.empty_like(Cc), torch.empty(8, device=DEV)

    def __call__(self, mbd, stats):
        """mbd: device float32 tensors by LstmMinibatchArgs field name; stats: the [2] device advantage statistics."""
        for t in (self.ws, self.gP, self.gC, self.metrics):
            t.fill_(float("nan"))
        a = self.nt.LstmMinibatchArgs()
        a.dims, a.T, a.n_env = self.d, self.T, self.n
        for k, v in mbd.items():
            assert v.is_contiguous() and v.dtype == torch.float32
            setattr(a, k, v.data_ptr())
        a.adv_stats, a.policy_params, a.critic_params = stats.data_ptr(), self.P.data_ptr(), self.Cc.data_ptr()
        a.policy_grads, a.critic_grads, a.metrics = self.gP.data_ptr(), self.gC.data_ptr(), self.metrics.data_ptr()
        a.clip_range, a.entropy_coef, a.critic_coef = CLIP, ENT, CC
        a.workspace, a.workspace_bytes = self.ws.data_ptr(), self.nbytes
        self.nt.check(self.lib.rlx_lstm_ppo_minibatch_fwdbwd_f32(C.byref(a), _st()), "rlx_lstm_ppo_minibatch_fwdbwd_f32")
        torch.cuda.synchronize()
        return self.gP.cpu().clone(), self.gC.cpu().clone(), self.metrics.cpu().clone()


def _mb_dev(mb):
    out = {k: mb[k].to(DEV).contiguous() for k in ("states", "actions", "log_probs", "advantages", "returns", "dones")}
    out["init_c"], out["init_h"] = (t.to(DEV).contiguous() for t in mb["init_carry"])
    return out


METRICS = ("loss/policy_gradient_loss", "loss/critic_loss", "loss/entropy_loss", "policy_ratio/approx_kl", "policy_ratio/clip_fraction")


def _check(dims, R, got, ref64, ref32, label, simt=None, floors=None):
    """Bounds (i) and (ii) per segment and the metrics.  Returns ({segment: distance}, report line)."""
    gP, gC, metrics = got
    gp64, gc64, rp, rc, m64 = ref64
    gp32, gc32 = ref32[0], ref32[1]
    p, c = layout(dims)
    dist, worst, used = {}, (0.0, "", 0.0), 0.0
    for net, g, g64, r, g32, offs, names, fl in (("pol", gP, gp64, rp, gp32, p, POLICY_SEGS, floors and floors[0]),
                                                 ("cri", gC, gc64, rc, gc32, c, CRITIC_SEGS, floors and floors[1])):
        g = g.numpy().astype(np.float64)
        assert np.isfinite(g).all(), (label, net, "an element was not written")
        for x, y, t, z, name in zip(_segments(g, offs), _segments(g64, offs), _segments(r, offs), _segments(g32, offs), names):
            if y.size == 0:
                continue
            N, d32 = _norms(y, t), float(np.linalg.norm(z - y))
            key = f"{net}.{name}"
            dist[key] = d = float(np.linalg.norm(x - y))
            bound = max(BAR * N, K32 * d32)
            assert d <= bound, (label, key, "(i)", d / N, d32 / N)
            used = max(used, d / bound)
            if simt is not None:
                assert d <= 2 * simt[key] + fl * N, (label, key, "(ii)", d / N, simt[key] / N, fl)
            if d / N > worst[0]:
                worst = (d / N, key, d32 / N)
    for j, key in enumerate(METRICS):
        tol = 0.5 / R if key.endswith("clip_fraction") else BAR * max(1.0, abs(m64[key]))
        assert abs(float(metrics[j]) - m64[key]) <= tol, (label, key, float(metrics[j]), m64[key])
    assert float(metrics[7]) == R
    return dist, f"{label}: worst {worst[0]:.2e} ({worst[1]}; float32 oracle there {worst[2]:.2e}); bound (i) used up to {used:.2f}"


def _d32_worst(dims, ref64, ref32):
    p, c = layout(dims)
    w = 0.0
    for g64, r, g32, offs in ((ref64[0], ref64[2], ref32[0], p), (ref64[1], ref64[3], ref32[1], c)):
        for y, t, z in zip(_segments(g64, offs), _segments(r, offs), _segments(g32, offs)):
            if y.size:
                w = max(w, float(np.linalg.norm(z - y)) / _norms(y, t))
    return w


def run_case(lib, dims, T, n, dones="rand", wi_scale=1.0, seed=3):
    t0 = time.time()
    pol, cri, mb = make_case(dims, T, n, seed, dones, wi_scale)
    ref64, ref32 = references(pol, cri, mb)
    P, Cc = torch.cat(flatten_policy(pol)).to(DEV), torch.cat(flatten_critic(cri)).to(DEV)
    adv = mb["advantages"].double()
    stats = torch.tensor([float(adv.mean()), float(adv.std(unbiased=False))], dtype=torch.float32, device=DEV)
    call, mbd, R = _Fwdbwd(lib, dims, T, n, P, Cc), _mb_dev(mb), T * n
    gemms = fwdbwd_gemms(dims, T, n)
    fits = seq_cfg(dims[4])[4]
    floors = _floor(gemms, R)
    out, simt, report = {}, None, []
    for engine in (0, 1):
        for pers in (0, 1):
            out[engine, pers] = _proven(lib, engine, pers, gemms, 2 if pers and fits else 0, lambda: call(mbd, stats))
        for a, b in zip(out[engine, 0], out[engine, 1]):   # the two recurrences: same arithmetic in the same order
            assert torch.equal(a, b), (dims, T, n, engine, "per-step and one-launch recurrences differ")
        label = f"{dims} T={T} n={n} dones={dones}{' Wi x%g' % wi_scale if wi_scale != 1 else ''} engine {engine}"
        dist, line = _check(dims, R, out[engine, 0], ref64, ref32, label, simt, floors if engine else None)
        if engine == 0:
            simt = dist
        else:
            line += f"  F = {floors[0]:.2e} / {floors[1]:.2e}"
        report.append(line)
    report.append(f"  float32 oracle worst {_d32_worst(dims, ref64, ref32):.2e}; {time.time() - t0:.1f} s")
    print("\n" + "\n".join(report))
    return out, call, mbd, stats


# (dims, T, n, dones, Wi scale): each pins an edge
CASES = [
    pytest.param(BASE, 128, 256, "rand", 1.0, id="baseline_T128_n256"),                        # 32 weight-gradient splits, EPB 2
    pytest.param((64, 17, 256, 128, 64, OPT_FILM), 32, 96, "rand", 1.0, id="film_act17"),       # Wf at 2 mod 4 in the parameters
    pytest.param((64, 8, 256, 128, 64, OPT_FILM | OPT_SHARED), 32, 96, "rand", 1.0, id="film_shared"),
    pytest.param((64, 8, 256, 128, 64, OPT_SHARED), 32, 96, "rand", 1.0, id="concat_shared"),
    pytest.param((64, 32, 128, 64, 64, 0), 16, 100, "none", 1.0, id="act32"),                  # dx of Wm on the tensor engine
    pytest.param((64, 64, 128, 64, 64, 0), 16, 100, "rand", 1.0, id="act64"),                  # all three Wm products there
    pytest.param((63, 8, 128, 64, 64, 0), 16, 80, "rand", 1.0, id="obs63"),                    # X-operand products leave by pitch
    pytest.param((64, 8, 128, 64, 64, 0), 33, 100, "rand", 1.0, id="ragged_R3300"),             # 4 splits, the last of 228 rows
    pytest.param((64, 8, 128, 64, 64, 0), 7, 9, "rand", 1.0, id="R63"),                         # forwards SIMT, weight gradients tensor
    pytest.param((64, 8, 128, 64, 64, 0), 5, 6, "rand", 1.0, id="R30_all_simt"),
    pytest.param((64, 8, 128, 64, 32, 0), 16, 50, "rand", 1.0, id="lstm32_epb4"),              # n % 4 != 0: inactive slots in the last block
    pytest.param((64, 8, 128, 64, 48, 0), 16, 37, "rand", 1.0, id="lstm48_96threads"),
    pytest.param((64, 8, 128, 64, 100, 0), 16, 40, "rand", 1.0, id="lstm100_100threads"),
    pytest.param((64, 8, 128, 64, 112, 0), 8, 33, "rand", 1.0, id="lstm112_widest_one_launch"),
    pytest.param((64, 8, 128, 64, 113, 0), 8, 33, "rand", 1.0, id="lstm113_gate_fails"),
    pytest.param((64, 8, 128, 64, 64, 0), 1, 128, "rand", 1.0, id="T1"),                       # no carried gradient
    pytest.param((64, 8, 128, 64, 64, 0), 256, 64, "rand", 1.0, id="T256"),
    pytest.param((64, 8, 128, 64, 64, 0), 16, 64, "all", 1.0, id="dones_all"),                 # the carry resets every step
    pytest.param((64, 8, 128, 64, 64, 0), 16, 64, "t0", 1.0, id="dones_t0"),
    pytest.param((64, 8, 128, 64, 64, 0), 16, 64, "rand", 6.0, id="saturated_gates"),          # sigmoid / tanh near 0 and 1
]


@gpu
@pytest.mark.parametrize("dims,T,n,dones,wi_scale", CASES)
def test_fwdbwd_vs_float64_on_both_engines_and_recurrences(lib, dims, T, n, dones, wi_scale):
    run_case(lib, dims, T, n, dones, wi_scale)


@gpu
def test_done_at_the_last_step_has_no_effect(lib):
    """A done after the last step resets nothing inside the sequence: bit-identical results with and without it, on every path."""
    dims, T, n = (64, 8, 128, 64, 64, 0), 16, 64
    out, call, mbd, stats = run_case(lib, dims, T, n, "last")
    mbd = dict(mbd, dones=torch.zeros_like(mbd["dones"]))
    gemms = fwdbwd_gemms(dims, T, n)
    for (engine, pers), want in out.items():
        got = _proven(lib, engine, pers, gemms, 2 * pers, lambda: call(mbd, stats))
        assert all(torch.equal(a, b) for a, b in zip(got, want)), (engine, pers)


# ------------------------------------------------------------------------------------------ two full minibatch steps
def _moments_tree(like, leaves):
    return _tree_from_leaves(like, [t.detach() for t in leaves])


@gpu
@pytest.mark.parametrize("engine", [0, 1])
def test_two_minibatch_steps_follow_the_weights(lib, engine):
    """Gather (under a permutation) -> advantage statistics -> fwdbwd -> clip + Adam on both nets, twice, against Learner's minibatch step in
    float64.  Step 2's reference starts from the device's weights and Adam moments after step 1, so a step that reached the parameters but not
    the moments, or the reverse, shows.  Gradients per segment at (i); parameters per network at PARAM_BAR (Adam's first step is lr times the
    sign of g: an element whose gradient is within rounding of zero moves by 2 lr whatever the engine, so not per segment); Adam moments per
    network, mu at the gradient bar (it is linear in the clipped gradient) and nu at NU_BAR: besides twice the gradient's error, the kernel's
    1 - beta2 in float32 is 1.3e-5 off 0.001 (measured 1.3e-5 to 1.5e-5 on an H100)."""
    from rl_x_b200 import _native as nt
    dims, T, n = BASE, 32, 64
    Nenv = 2 * n
    pol, cri, roll = make_case(dims, T, Nenv, 7)
    perm = torch.randperm(Nenv, generator=torch.Generator().manual_seed(8))
    P, Cc = torch.cat(flatten_policy(pol)).to(DEV), torch.cat(flatten_critic(cri)).to(DEV)
    state = dict(P=P, Cc=Cc, mP=torch.zeros_like(P), vP=torch.zeros_like(P), mC=torch.zeros_like(Cc), vC=torch.zeros_like(Cc),
                 sP=torch.zeros(1, dtype=torch.int64, device=DEV), sC=torch.zeros(1, dtype=torch.int64, device=DEV))
    src = {k: roll[k].to(DEV).contiguous() for k in ("states", "actions", "log_probs", "advantages", "returns", "dones")}
    src["init_c"], src["init_h"] = (t.to(DEV).contiguous() for t in roll["init_carry"])
    widths = dict(states=dims[0], actions=dims[1], log_probs=1, advantages=1, returns=1, dones=1, init_c=dims[4], init_h=dims[4])
    call = _Fwdbwd(lib, dims, T, n, P, Cc)
    gemms = fwdbwd_gemms(dims, T, n)
    lr_dev = torch.tensor([LR], device=DEV)
    p, c = layout(dims)
    report = []
    for step in range(2):
        idx = perm[step * n:(step + 1) * n].contiguous()
        idx_dev = idx.to(DEV)
        # the reference at the device's current weights and moments
        now_p = _tree_from_flat(pol, state["P"].cpu().double(), True)
        now_c = _tree_from_flat(cri, state["Cc"].cpu().double(), False)
        mb = {k: roll[k][:, idx] for k in ("states", "actions", "log_probs", "returns", "advantages", "dones")}
        mb["init_carry"] = tuple(t[idx] for t in roll["init_carry"])
        ref64, ref32 = references(now_p, now_c, mb)
        ref = L.Learner(_to(now_p, torch.float64, DEV), _to(now_c, torch.float64, DEV), lr=LR, clip_range=CLIP, entropy_coef=ENT, critic_coef=CC,
                        max_grad_norm=MAX_NORM)
        for opt, like, m, v, s, pol_net in ((ref.popt, ref.pol, state["mP"], state["vP"], state["sP"], True),
                                            (ref.copt, ref.cri, state["mC"], state["vC"], state["sC"], False)):
            opt.mu = [t.to(DEV) for _, t in L.tree_leaves(_tree_from_flat(like, m.cpu().double(), pol_net))]
            opt.nu = [t.to(DEV) for _, t in L.tree_leaves(_tree_from_flat(like, v.cpu().double(), pol_net))]
            opt.count = int(s.item())
        mbd64 = {k: (tuple(t.to(DEV, torch.float64) for t in v) if k == "init_carry" else v.to(DEV, torch.float64)) for k, v in mb.items()}
        gp, gc, met = ref.grads(mbd64)   # Learner.minibatch_step, written out to keep the gradients
        norm_p, norm_c = ref.popt.step(gp), ref.copt.step(gc)
        assert max(norm_p, norm_c) >= MAX_NORM, "the clip branch of the optimiser is not exercised"
        # the device: gather, statistics, fwdbwd, two optimiser steps - every call with its path table
        mbd = {k: _nan(T, n, widths[k]).squeeze(-1) if widths[k] == 1 else _nan(T, n, widths[k]) for k in ("states", "actions", "log_probs", "advantages",
                                                                                                             "returns", "dones")}
        mbd["init_c"], mbd["init_h"] = _nan(n, dims[4]), _nan(n, dims[4])
        for k, dst in mbd.items():
            rows = 1 if k.startswith("init") else T
            _proven(lib, engine, 1, [], 0, lambda: nt.check(lib.rlx_gather_env_columns_f32(src[k].data_ptr(), idx_dev.data_ptr(), rows, Nenv, n, widths[k],
                                                                                            dst.data_ptr(), _st()), "gather"))
            want = roll[k][:, idx] if not k.startswith("init") else roll["init_carry"][0 if k == "init_c" else 1][idx]
            assert torch.equal(dst.cpu(), want), k
        stats, sws = _nan(2), _nan(T * n + 2 * (-(-T * n // 256)) + 8)
        _proven(lib, engine, 1, [], 0, lambda: nt.check(lib.rlx_mean_popstd_f32(mbd["advantages"].data_ptr(), T * n, stats.data_ptr(), sws.data_ptr(), _st()),
                                                        "mean_popstd"))
        a64 = mb["advantages"].double()
        assert abs(float(stats[0]) - float(a64.mean())) <= 2e-6 * float(a64.std()) and abs(float(stats[1]) / float(a64.std(unbiased=False)) - 1) <= 2e-6
        got = _proven(lib, engine, 1, gemms, 2, lambda: call(mbd, stats))
        _check(dims, T * n, got, ref64, ref32, f"step {step} engine {engine}")
        norms = _nan(2)
        for j, (prm, g, m, v, s, nel) in enumerate(((state["P"], call.gP, state["mP"], state["vP"], state["sP"], P.numel()),
                                                    (state["Cc"], call.gC, state["mC"], state["vC"], state["sC"], Cc.numel()))):
            ows = _nan(nel // 1024 + 8)
            _proven(lib, engine, 1, [], 0, lambda: nt.check(lib.rlx_optax_clip_adam_f32(prm.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), nel,
                                                                                          lr_dev.data_ptr(), s.data_ptr(), MAX_NORM, 0.9, 0.999, 1e-8,
                                                                                          norms[j:].data_ptr(), ows.data_ptr(), _st()), "optax"))
        torch.cuda.synchronize()
        for j, (want_n, net) in enumerate(((norm_p, "policy"), (norm_c, "critic"))):
            assert abs(float(norms[j]) - want_n) <= BAR * want_n, (net, float(norms[j]), want_n)
        assert int(state["sP"]) == int(state["sC"]) == step + 1
        for what, dev_t, ref_t, bar in (("params", state["P"], ref.pol, PARAM_BAR), ("mu", state["mP"], _moments_tree(ref.pol, ref.popt.mu), BAR),
                                        ("nu", state["vP"], _moments_tree(ref.pol, ref.popt.nu), NU_BAR),
                                        ("params", state["Cc"], ref.cri, PARAM_BAR), ("mu", state["mC"], _moments_tree(ref.cri, ref.copt.mu), BAR),
                                        ("nu", state["vC"], _moments_tree(ref.cri, ref.copt.nu), NU_BAR)):
            is_pol = dev_t.numel() == P.numel()
            want = _flat(ref_t, is_pol).numpy()
            have = dev_t.cpu().double().numpy()
            rel = float(np.linalg.norm(have - want) / np.linalg.norm(want))
            assert rel <= bar, (step, engine, what, "policy" if is_pol else "critic", rel)
            report.append(f"step {step} engine {engine} {what} {'policy' if is_pol else 'critic'}: {rel:.2e}")
    print("\n" + "\n".join(report))


# ----------------------------------------------------------------------------------------------------- acting step
@gpu
@pytest.mark.parametrize("n", [63, 64, 4097])
@pytest.mark.parametrize("noise,clip_rescale", [(True, True), (False, False), (True, False)], ids=["noise_clip", "deterministic", "noise_noclip"])
def test_acting_step_vs_float64_on_both_engines(lib, n, noise, clip_rescale):
    """rlx_lstm_step_f32 for three steps with rlx_lstm_mask_carry_f32 between them, against get_action_and_value in float64 at the device's carry
    of each step; then rlx_lstm_critic_forward_f32 against critic_value.  Every output starts as NaN."""
    from rl_x_b200 import _native as nt
    dims = BASE
    O, A, Lh = dims[0], dims[1], dims[4]
    pol, cri = _params(dims, 11)
    g = torch.Generator().manual_seed(n)
    low, high = torch.linspace(-2.0, -0.5, A), torch.linspace(0.5, 2.0, A)
    P, Cc = torch.cat(flatten_policy(pol)).to(DEV), torch.cat(flatten_critic(cri)).to(DEV)
    p64, c64 = _to(pol, torch.float64, DEV), _to(cri, torch.float64, DEV)
    d = nt.LstmDims(*dims)
    nbytes = int(lib.rlx_lstm_minibatch_workspace_bytes(C.byref(d), 1, n))
    assert nbytes == plan(dims, 1, n)["total"]
    ws = torch.empty(nbytes // 4, device=DEV)
    dd = lambda t: t.to(DEV, torch.float64)
    close = lambda got, want, what: (np.testing.assert_allclose(got.cpu().double().numpy(), want.cpu().numpy(), rtol=1e-5, atol=1e-5, err_msg=what),
                                     _rel_ok(got, want, what))
    for engine in (0, 1):
        c, h = (torch.randn(n, Lh, generator=g) * 0.5).to(DEV), (torch.randn(n, Lh, generator=g) * 0.5).to(DEV)
        for t in range(3):
            obs = torch.randn(n, O, generator=g)
            eps = torch.randn(n, A, generator=g) if noise else torch.zeros(n, A)
            with torch.no_grad():
                proc, act, val, logp, (nc, nh) = L.get_action_and_value(p64, c64, dd(obs), (dd(c), dd(h)), dd(eps), dd(low), dd(high), clip_rescale)
            out = dict(action=_nan(n, A), env_action=_nan(n, A), logp=_nan(n), value=_nan(n))
            obs_d, eps_d, low_d, high_d = obs.to(DEV), eps.to(DEV), low.to(DEV), high.to(DEV)
            a = nt.LstmStepArgs()
            a.dims, a.n = d, n
            a.obs, a.c, a.h = obs_d.data_ptr(), c.data_ptr(), h.data_ptr()
            a.noise = eps_d.data_ptr() if noise else None
            a.policy_params, a.critic_params, a.act_low, a.act_high, a.clip_rescale = P.data_ptr(), Cc.data_ptr(), low_d.data_ptr(), high_d.data_ptr(), int(clip_rescale)
            a.action, a.env_action, a.logp, a.value = (out[k].data_ptr() for k in ("action", "env_action", "logp", "value"))
            ws.fill_(float("nan"))
            a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
            _proven(lib, engine, 0, step_gemms(dims, n), 0, lambda: nt.check(lib.rlx_lstm_step_f32(C.byref(a), _st()), "rlx_lstm_step_f32"))
            for k, want in (("action", act), ("env_action", proc), ("logp", logp), ("value", val)):
                close(out[k], want, f"engine {engine} step {t} {k}")
            close(c, nc, f"engine {engine} step {t} c")
            close(h, nh, f"engine {engine} step {t} h")
            done = (torch.rand(n, generator=g) < 0.3).float().to(DEV)
            _proven(lib, engine, 0, [], 0, lambda: nt.check(lib.rlx_lstm_mask_carry_f32(c.data_ptr(), h.data_ptr(), done.data_ptr(), n, Lh, _st()), "mask"))
            keep = (1 - done).unsqueeze(1)
            close(c, nc * keep.double(), f"engine {engine} step {t} masked c")
            close(h, nh * keep.double(), f"engine {engine} step {t} masked h")
        x = torch.randn(n, O, generator=g)
        vout = _nan(n)
        ws.fill_(float("nan"))
        x_d = x.to(DEV)
        _proven(lib, engine, 0, critic_gemms(dims, n), 0,
                lambda: nt.check(lib.rlx_lstm_critic_forward_f32(C.byref(d), Cc.data_ptr(), x_d.data_ptr(), n, vout.data_ptr(), ws.data_ptr(), nbytes, _st()),
                                 "critic_forward"))
        with torch.no_grad():
            close(vout, L.critic_value(c64, dd(x)).reshape(-1), f"engine {engine} critic_forward")


def _rel_ok(got, want, what):
    got = got.cpu().double()
    want = want.cpu()
    assert torch.isfinite(got).all(), what
    assert float((got - want).norm()) <= 5e-6 * max(float(want.norm()), 1e-30), (what, float((got - want).norm() / want.norm()))
