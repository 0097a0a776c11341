"""GPU parity tests: every CUDA entry point (called through the C-ABI via ctypes) against the CPU oracle on the same
seeded inputs, and against the golden vectors captured from the executed reference.

Tolerances (north_star: <= 1e-5 relative fp32 on losses/advantages, bit-exact on index work):
  * GAE, gather, shuffles: bit-exact.
  * per-element forward quantities (log-prob, value, actions): rtol 1e-5 (+ atol 1e-6 near zero).
  * reduced scalars (losses): |delta| <= 1e-5 * max(|ref|, mean|summand|) — pg_loss is a mean of signed terms with
    near-zero mean (SURVEY.md §7 hard part a), so the norm is the summand scale.
  * gradients: ||g - g_ref|| <= 1e-5 * ||g_ref|| per tensor.
"""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["simt", "tcgen05"])
def gemm_engine(request):
    """Every test runs once per GEMM engine (shapes the wgmma engine, selected as "tcgen05", does not cover fall back to the SIMT engine)."""
    from rl_x_b200 import _native as nt
    lib = nt.load()
    lib.rlx_set_gemm_engine(1 if request.param == "tcgen05" else 0)
    yield request.param
    lib.rlx_set_gemm_engine(0)

DEV = "cuda"


def _kern(obs, act, hidden):
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(obs, act, hidden)


def _flat_from_named(k, pol, cri):
    from rl_x_b200.algorithms.ppo.b200.ppo import FlatParameters
    fp = FlatParameters(k, DEV)
    fp.load_named({**{n: torch.as_tensor(v) for n, v in pol.items()}, **{n: torch.as_tensor(v) for n, v in cri.items()}})
    return fp


def _t(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in d.items()}


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


# ------------------------------------------------------------------------------------------------------------ GAE
# (130, 9601) and (65, 16384): more than 2 CTAs per SM -> the 64-step-tile instantiation, with a ragged last tile
@pytest.mark.parametrize("T,N", [(1, 1), (5, 3), (128, 4096), (129, 33), (300, 100), (64, 31), (130, 9601), (65, 16384)])
@pytest.mark.parametrize("shortcut", [False, True])
@pytest.mark.parametrize("tma", [True, False])
def test_gae_bit_exact_vs_oracle(T, N, shortcut, tma):
    """tma=True: tiles staged by cp.async.bulk.tensor where alignment allows (N % 4 == 0), ordinary loads elsewhere; False: ordinary loads always."""
    k = _kern(8, 2, 32)
    k.lib.rlx_set_gae_tma(1 if tma else 0)
    g = torch.Generator().manual_seed(T * 1000 + N)
    r = torch.randn(T, N, generator=g)
    term = (torch.rand(T, N, generator=g) < 0.1).float()
    if shortcut:
        vall = torch.randn(T + 1, N, generator=g)
        v, nv = vall[:T].contiguous(), vall[1:].contiguous()
    else:
        v, nv = torch.randn(T, N, generator=g), torch.randn(T, N, generator=g)
    adv_ref, ret_ref = O.gae(r, term, v, nv, 0.99, 0.95)
    adv, ret = torch.empty(T, N, device=DEV), torch.empty(T, N, device=DEV)
    if shortcut:
        k.gae(r.to(DEV), term.to(DEV), v.to(DEV), 0.99, 0.95, adv, ret, last_value=nv[T - 1].contiguous().to(DEV))
    else:
        k.gae(r.to(DEV), term.to(DEV), v.to(DEV), 0.99, 0.95, adv, ret, next_values=nv.to(DEV))
    k.lib.rlx_set_gae_tma(1)
    assert np.array_equal(adv.cpu().numpy(), adv_ref.numpy())
    assert np.array_equal(ret.cpu().numpy(), ret_ref.numpy())


def test_gae_bit_exact_vs_reference_golden(golden):
    g = golden
    k = _kern(g.obs, g.act, g.hidden)
    for it in range(g.iterations):
        nv = torch.from_numpy(g[f"iter{it}/next_values"])  # the critic output the reference fed into its GAE (ppo.py:253-254)
        adv, ret = torch.empty(g.T, g.N, device=DEV), torch.empty(g.T, g.N, device=DEV)
        k.gae(torch.from_numpy(g[f"iter{it}/rewards"]).to(DEV), torch.from_numpy(g[f"iter{it}/terminations"]).to(DEV),
              torch.from_numpy(g[f"iter{it}/values"]).to(DEV), g.gamma, g.gae_lambda, adv, ret, next_values=nv.to(DEV))
        assert np.array_equal(adv.cpu().numpy(), g[f"iter{it}/advantages"])
        assert np.array_equal(ret.cpu().numpy(), g[f"iter{it}/returns"])


def test_gae_empty_and_errors():
    k = _kern(8, 2, 32)
    e = torch.empty(0, 4, device=DEV)
    k.gae(e, e, e, 0.99, 0.95, e, e, last_value=torch.zeros(4, device=DEV))  # T == 0 is a no-op
    x = torch.zeros(3, 4, device=DEV)
    with pytest.raises(RuntimeError, match="next_values or last_value"):
        k.gae(x, x, x, 0.99, 0.95, x.clone(), x.clone())


# -------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("obs,act,hidden,n", [(11, 3, 64, 37), (376, 17, 256, 4096), (376, 17, 256, 130), (20, 40, 96, 65), (7, 1, 8, 1)])
def test_forward_vs_oracle(obs, act, hidden, n):
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.8, seed=obs + n)
    g = torch.Generator().manual_seed(n)
    for w in pol.values():
        w.add_(0.05 * torch.randn(w.shape, generator=g))  # non-zero biases / logstd
    for w in cri.values():
        w.add_(0.05 * torch.randn(w.shape, generator=g))
    x = torch.randn(n, obs, generator=g)
    noise = torch.randn(n, act, generator=g)
    low, high = torch.full((act,), -2.0), torch.full((act,), 0.5)
    with torch.no_grad():
        a_ref, e_ref, lp_ref = O.get_action_logprob(pol, x, noise, low, high)
        v_ref = O.critic_value(cri, x).reshape(-1)
        d_ref = O.get_deterministic_action(pol, x, low, high)
    fp = _flat_from_named(k, pol, cri)
    ws = k.forward_workspace(n, DEV)
    a, e, lp, v = (torch.empty(n, act, device=DEV), torch.empty(n, act, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV))
    k.forward(fp.flat, x.to(DEV), ws, noise=noise.to(DEV), act_low=low.to(DEV), act_high=high.to(DEV), action=a, env_action=e, logp=lp, value=v)
    # 1e-5 relative to the scale of each quantity (elementwise: rtol on the value + the same fraction of the tensor's rms)
    tol = lambda ref: dict(rtol=1e-5, atol=1e-5 * float(ref.pow(2).mean().sqrt()))
    np.testing.assert_allclose(a.cpu().numpy(), a_ref.numpy(), **tol(a_ref))
    np.testing.assert_allclose(e.cpu().numpy(), e_ref.numpy(), **tol(e_ref))
    np.testing.assert_allclose(lp.cpu().numpy(), lp_ref.numpy(), **tol(lp_ref))
    np.testing.assert_allclose(v.cpu().numpy(), v_ref.numpy(), **tol(v_ref))
    assert _rel(a.cpu().numpy(), a_ref.numpy()) < 5e-6 and _rel(v.cpu().numpy(), v_ref.numpy()) < 5e-6
    d = torch.empty(n, act, device=DEV)
    k.forward(fp.flat, x.to(DEV), ws, act_low=low.to(DEV), act_high=high.to(DEV), deterministic=True, env_action=d)
    np.testing.assert_allclose(d.cpu().numpy(), d_ref.numpy(), **tol(d_ref))
    v2 = torch.empty(n, device=DEV)
    k.critic_forward(fp.flat, x.to(DEV), v2, ws)
    assert torch.equal(v2, v)


def test_teacher_forced_forward_vs_reference_golden(golden):
    """values / log_probs stored by the reference during its rollout, reproduced from its states/actions/initial weights."""
    g = golden
    k = _kern(g.obs, g.act, g.hidden)
    pol, cri = g.params("init")
    fp = _flat_from_named(k, pol, cri)
    states = torch.from_numpy(g["iter0/states"]).reshape(-1, g.obs)
    actions = torch.from_numpy(g["iter0/actions"]).reshape(-1, g.act)
    with torch.no_grad():
        mean = O.policy_mean(_t(pol), states)
    std = torch.exp(torch.from_numpy(pol["policy_logstd"]))
    noise = (actions - mean) / std
    n = states.shape[0]
    ws = k.forward_workspace(n, DEV)
    lp, v, a = torch.empty(n, device=DEV), torch.empty(n, device=DEV), torch.empty(n, g.act, device=DEV)
    low = torch.full((g.act,), g.act_low, device=DEV)
    high = torch.full((g.act,), g.act_high, device=DEV)
    e = torch.empty(n, g.act, device=DEV)
    k.forward(fp.flat, states.to(DEV), ws, noise=noise.to(DEV), act_low=low, act_high=high, action=a, env_action=e, logp=lp, value=v)
    np.testing.assert_allclose(v.cpu().numpy(), g["iter0/values"].reshape(-1), rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(a.cpu().numpy(), actions.numpy(), rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(lp.cpu().numpy(), g["iter0/log_probs"].reshape(-1), rtol=1e-5, atol=2e-5)
    np.testing.assert_allclose(e.cpu().numpy()[:g.N], g["env_actions"][0], rtol=1e-5, atol=2e-6)


def test_philox_noise_is_standard_normal_and_reproducible():
    k = _kern(16, 8, 32)
    pol, cri = O.init_params(16, 8, 32, seed=0)
    fp = _flat_from_named(k, pol, cri)
    n = 1 << 16
    x = torch.zeros(n, 16, device=DEV)
    ws = k.forward_workspace(n, DEV)
    lo, hi = torch.full((8,), -1.0, device=DEV), torch.full((8,), 1.0, device=DEV)
    a1, a2, a3 = (torch.empty(n, 8, device=DEV) for _ in range(3))
    k.forward(fp.flat, x, ws, rng_seed=7, rng_offset=3, act_low=lo, act_high=hi, action=a1)
    k.forward(fp.flat, x, ws, rng_seed=7, rng_offset=3, act_low=lo, act_high=hi, action=a2)
    k.forward(fp.flat, x, ws, rng_seed=7, rng_offset=4, act_low=lo, act_high=hi, action=a3)
    assert torch.equal(a1, a2) and not torch.equal(a1, a3)
    z = a1.double()  # mean 0 (zero obs, zero bias), std exp(0) = 1
    assert abs(float(z.mean())) < 5e-3 and abs(float(z.std()) - 1.0) < 5e-3
    assert abs(float((z ** 4).mean()) - 3.0) < 0.1
    assert abs(float(torch.corrcoef(torch.stack([z[:, 0], z[:, 1]]))[0, 1])) < 0.02


# ------------------------------------------------------------------------------------------ gather / stats / store
@pytest.mark.parametrize("obs,act", [(376, 17), (11, 3)])
def test_gather_bit_exact(obs, act):
    k = _kern(obs, act, 32)
    B = 5000
    g = torch.Generator().manual_seed(1)
    src = [torch.randn(B, obs, generator=g), torch.randn(B, act, generator=g), torch.randn(B, generator=g), torch.randn(B, generator=g),
           torch.randn(B, generator=g)]
    perm = torch.randperm(B, generator=g)
    dst = [torch.empty_like(s, device=DEV) for s in src]
    k.gather(perm.to(DEV), *[s.to(DEV) for s in src], *dst)
    for s, d in zip(src, dst):
        assert torch.equal(d.cpu(), s[perm])
    sub = perm[:777].contiguous()
    dst2 = [torch.zeros(777, *s.shape[1:], device=DEV) for s in src]
    k.gather(sub.to(DEV), *[s.to(DEV) for s in src], *dst2)
    for s, d in zip(src, dst2):
        assert torch.equal(d.cpu(), s[sub])


def test_advantage_stats_vs_torch():
    k = _kern(8, 2, 32)
    count, mb = 10000, 3000  # last minibatch short (1000)
    adv = torch.randn(count, generator=torch.Generator().manual_seed(2)) * 3 + 0.5
    stats = torch.empty(4, 2, device=DEV)
    k.advantage_stats(adv.to(DEV), count, mb, stats)
    for i in range(4):
        chunk = adv[i * mb:(i + 1) * mb]
        np.testing.assert_allclose(stats[i].cpu().numpy(), [chunk.mean().item(), chunk.std().item()], rtol=2e-6, atol=1e-7)


def test_rollout_store():
    k = _kern(12, 2, 32)
    n = 1000
    g = torch.Generator().manual_seed(3)
    reward, nxt = torch.randn(n, generator=g), torch.randn(n, 12, generator=g)
    term, trunc = torch.rand(n, generator=g) < 0.3, torch.rand(n, generator=g) < 0.2
    rr, tr, nd = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, 12, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int64, device=DEV)
    for _ in range(2):
        k.rollout_store(reward.to(DEV), term.to(DEV), trunc.to(DEV), nxt.to(DEV), rr, tr, nd, cnt)
    assert torch.equal(rr.cpu(), reward) and torch.equal(tr.cpu(), term.float()) and torch.equal(nd.cpu(), nxt)
    assert int(cnt.item()) == 2 * int((term | trunc).sum())


# ------------------------------------------------------------------------------------------- minibatch fwd + bwd
def _random_minibatch(obs, act, m, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(states=torch.randn(m, obs, generator=g), actions=torch.randn(m, act, generator=g) * 0.7,
                log_probs=-1.0 - 0.3 * torch.rand(m, generator=g) * act, advantages=torch.randn(m, generator=g) * 2 + 0.3,
                returns=torch.randn(m, generator=g))


def _run_fwdbwd(k, fp, mbatch, hp, m_global=None):
    m = mbatch["states"].shape[0]
    P = k.param_count
    d = {n: v.to(DEV).contiguous() for n, v in mbatch.items()}
    ldx = k.states_pitch()  # padded pitch + constant-one column, as the plugin's gather produces it
    xs = torch.zeros(m, ldx, device=DEV)
    xs[:, :k.obs_dim] = d["states"]
    xs[:, k.obs_dim] = 1.0
    d["states"] = xs
    stats = torch.empty(1, 2, device=DEV)
    k.advantage_stats(d["advantages"], m, m, stats)
    grads, metrics = torch.zeros(P, device=DEV), torch.zeros(8, device=DEV)
    st = dict(exp_avg=torch.zeros(P, device=DEV), exp_avg_sq=torch.zeros(P, device=DEV), lr=torch.full((1,), 3e-4, device=DEV),
              step=torch.zeros(1, dtype=torch.int64, device=DEV))
    ws = k.minibatch_workspace(m, DEV)
    args = k.minibatch_args(m=m, m_global=m_global or m, states=d["states"], actions=d["actions"], log_probs=d["log_probs"],
                            advantages=d["advantages"], returns=d["returns"], adv_stats=stats, params=fp.flat, grads=grads,
                            exp_avg=st["exp_avg"], exp_avg_sq=st["exp_avg_sq"], lr=st["lr"], step_count=st["step"], hp=hp,
                            metrics=metrics, workspace=ws, states_ld=ldx, states_ones_col=True)
    k.fwdbwd(args)
    return args, grads, metrics, st, (d, stats, ws)


@pytest.mark.parametrize("obs,act,hidden,m,ent", [(11, 3, 64, 40, 0.01), (376, 17, 256, 1000, 0.0), (376, 17, 256, 4099, 0.02), (24, 33, 96, 257, 0.0),
                                                 (5, 2, 8, 1, 0.0), (376, 17, 256, 32768, 0.0)])  # last: the bench's own minibatch (BASELINE configs[1])
def test_minibatch_gradients_vs_oracle_autograd(obs, act, hidden, m, ent):
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.9, seed=m)
    g = torch.Generator().manual_seed(m + 1)
    for w in list(pol.values()) + list(cri.values()):
        w.add_(0.02 * torch.randn(w.shape, generator=g))
    mb = _random_minibatch(obs, act, m, seed=m + 2)
    if m > 1:
        with torch.no_grad():  # make old log-probs consistent with the policy so that ratios sit around 1 and straddle the clip range
            lp, _ = O.get_logprob_entropy(pol, mb["states"], mb["actions"])
        mb["log_probs"] = lp + 0.15 * torch.randn(m, generator=g)
    L = O.Learner(pol, cri, clip_range=0.2, entropy_coef=ent, critic_coef=0.5)
    if m > 1:
        gp, gc, met = L.grads(mb["states"], mb["actions"], mb["log_probs"], mb["advantages"], mb["returns"])
    fp = _flat_from_named(k, pol, cri)
    args, grads, metrics, st, keep = _run_fwdbwd(k, fp, mb, make_hparams(0.2, ent, 0.5, 0.5))
    torch.cuda.synchronize()
    if m == 1:
        assert torch.isnan(grads).any()  # std of a single advantage is NaN in the reference too (torch.std, ppo.py:134)
        return
    gflat = fp.__class__(k, DEV)
    gflat.flat.copy_(grads)
    gpol, gcri = gflat.state_dicts()
    for name, ref in {**gp, **gc}.items():
        ours = (gpol if name in gpol else gcri)[name].numpy()
        assert _rel(ours, ref.numpy()) <= 1e-5, (name, _rel(ours, ref.numpy()))
    mm = metrics.cpu().numpy()
    scale = float(torch.abs(mb["advantages"] - mb["advantages"].mean()).mean() / mb["advantages"].std())
    assert abs(mm[0] - met["pg_loss"]) <= 1e-5 * max(abs(met["pg_loss"]), scale)
    assert abs(mm[1] - met["critic_loss"]) <= 1e-5 * abs(met["critic_loss"])
    assert abs(mm[2] - met["entropy_loss"]) <= 1e-5 * abs(met["entropy_loss"])
    assert abs(mm[3] - met["approx_kl"]) <= 1e-5 * max(abs(met["approx_kl"]), 1e-2)
    assert abs(mm[4] - met["clip_fraction"]) <= 1.5 / m  # a ratio within 1e-7 of the clip edge may flip
    assert mm[7] == m


def test_clip_adam_step_vs_oracle():
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    obs, act, hidden, m = 23, 4, 64, 300
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, seed=11)
    L = O.Learner(pol, cri, lr=1e-3, clip_range=0.2, entropy_coef=0.0, critic_coef=0.5, max_grad_norm=0.5)
    fp = _flat_from_named(k, pol, cri)
    hp = make_hparams(0.2, 0.0, 0.5, 0.5)
    state = None
    for step in range(3):
        mb = _random_minibatch(obs, act, m, seed=100 + step)
        ref = L.minibatch_step(mb["states"], mb["actions"], mb["log_probs"], mb["advantages"], mb["returns"])
        args, grads, metrics, st, keep = _run_fwdbwd(k, fp, mb, hp)
        if state is None:
            state = st
            state["lr"].fill_(1e-3)
        args.exp_avg, args.exp_avg_sq = state["exp_avg"].data_ptr(), state["exp_avg_sq"].data_ptr()
        args.lr, args.step_count = state["lr"].data_ptr(), state["step"].data_ptr()
        k.clip_adam(args)
        torch.cuda.synchronize()
        mm = metrics.cpu().numpy()
        assert abs(mm[5] - ref["policy_grad_norm"]) <= 1e-5 * ref["policy_grad_norm"]
        assert abs(mm[6] - ref["critic_grad_norm"]) <= 1e-5 * ref["critic_grad_norm"]
        pol_now, cri_now = fp.state_dicts()
        for name in O.POLICY_KEYS:
            np.testing.assert_allclose(pol_now[name].numpy(), L.pol[name].detach().numpy(), rtol=1e-5, atol=2e-7, err_msg=f"{name} step {step}")
        for name in O.CRITIC_KEYS:
            np.testing.assert_allclose(cri_now[name].numpy(), L.cri[name].detach().numpy(), rtol=1e-5, atol=2e-7, err_msg=f"{name} step {step}")
    assert int(state["step"].item()) == 3


# ------------------------------------------------------------------------------- whole update vs the reference
def test_update_epochs_vs_reference_golden(golden):
    """From the reference's initial weights, rollout batch and recorded permutations: after the full update (epochs x
    minibatches, incl. a short last minibatch and LR annealing in the `small` fixture) weights, Adam moments and the logged
    losses match what the reference produced."""
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    from rl_x_b200 import _native as nt
    g = golden
    k = _kern(g.obs, g.act, g.hidden)
    pol, cri = g.params("init")
    fp = _flat_from_named(k, pol, cri)
    P, B = k.param_count, g.B
    hp = make_hparams(g.clip_range, g.entropy_coef, g.critic_coef, g.max_grad_norm)
    exp_avg, exp_avg_sq = torch.zeros(P, device=DEV), torch.zeros(P, device=DEV)
    grads = torch.zeros(P, device=DEV)
    lr, step = torch.zeros(1, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    nmb = -(-B // g.mb)
    ws = k.minibatch_workspace(min(g.mb, B), DEV)
    rng = nt.Pcg64Generator(g.seed)
    for it in range(g.iterations):
        lr.fill_(g.lr_at(it))
        src = [torch.from_numpy(g[f"iter{it}/{n}"]).reshape((B,) + g[f"iter{it}/{n}"].shape[2:]).to(DEV).contiguous()
               for n in ["states", "actions", "log_probs", "advantages", "returns"]]
        ldx = k.states_pitch()
        dst = [torch.empty(B, ldx, device=DEV)] + [torch.empty_like(s) for s in src[1:]]
        metrics = torch.zeros(g.epochs * nmb, 8, device=DEV)
        stats = torch.empty(nmb, 2, device=DEV)
        idx = np.arange(B)
        for e in range(g.epochs):
            rng.shuffle(idx)
            assert np.array_equal(idx, g.perms(it)[e])
            k.gather(torch.from_numpy(idx).to(DEV), *src, *dst, out_states_ld=ldx)
            assert torch.equal(dst[0][:, g.obs], torch.ones(B, device=DEV)) and torch.equal(dst[0][:, :g.obs], src[0][torch.from_numpy(idx).to(DEV)])
            k.advantage_stats(dst[3], B, g.mb, stats)
            args = k.minibatch_args(m=0, m_global=1, states=dst[0], actions=dst[1], log_probs=dst[2], advantages=dst[3], returns=dst[4],
                                    adv_stats=stats, params=fp.flat, grads=grads, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq, lr=lr,
                                    step_count=step, hp=hp, metrics=metrics[e * nmb], workspace=ws, states_ld=ldx, states_ones_col=True)
            k.update_epoch(args, B, g.mb)
        torch.cuda.synchronize()
        pol_ref, cri_ref = g.params(f"iter{it}")
        pol_now, cri_now = fp.state_dicts()
        for name, v in {**pol_ref, **cri_ref}.items():
            ours = (pol_now if name in pol_now else cri_now)[name].numpy()
            assert _rel(ours, v) <= 1e-5, (it, name, _rel(ours, v))
            # elementwise: Adam normalises the step, so a gradient component near zero can move a weight by a fraction of
            # one lr-sized step differently; bound that by 10 % of a step
            np.testing.assert_allclose(ours, v, rtol=1e-4, atol=0.1 * g.lr, err_msg=f"iter {it} {name}")
        m = metrics.cpu().numpy()
        for col, name, floor in [(0, "loss/policy_gradient_loss", 0.5), (1, "loss/critic_loss", 0.0), (2, "loss/entropy_loss", 0.0),
                                 (4, "policy_ratio/clip_fraction", 1.0), (5, "gradients/policy_grad_norm", 0.0),
                                 (6, "gradients/critic_grad_norm", 0.0)]:
            ref = float(g[f"metric/{name}"][it])
            assert abs(float(m[:, col].mean()) - ref) <= 1e-5 * max(abs(ref), floor), (it, name, float(m[:, col].mean()), ref)
        ref_kl = float(g["metric/policy_ratio/approx_kl"][it])
        assert abs(float(m[-nmb:, 3].mean()) - ref_kl) <= 1e-5 * max(abs(ref_kl), 1e-2)
        if f"iter{it}/policy_opt/policy_logstd/exp_avg" in g.z.files:
            mom = fp.__class__(k, DEV)
            mom.flat.copy_(exp_avg)
            mp, _ = mom.state_dicts()
            for name in O.POLICY_KEYS:
                assert _rel(mp[name].numpy(), g[f"iter{it}/policy_opt/{name}/exp_avg"]) <= 1e-4, name
    assert int(step.item()) == g.iterations * g.epochs * nmb


def test_one_epoch_at_bench_shape_vs_oracle():
    """BASELINE configs[1] update shape (obs 376, act 17, hidden 256, minibatch 32768): one epoch of 4 minibatches through
    rlx_ppo_update_epoch_f32 (the split-K chains, dW reductions and head grids are those of the benchmark; only the batch is 4x shorter so
    that the CPU oracle finishes in seconds), checked minibatch by minibatch:
      (a) kernel parity where the number is quoted: the flat gradient of minibatch k against the oracle's autograd evaluated AT THE SAME
          WEIGHTS (ours, before the step), 1e-5 of the norm per tensor, and the logged losses;
      (b) the trajectory: weights after the 4 steps against the oracle's own 4-step run.  A PPO policy step moves the ratios of the
          following minibatch, so the two trajectories separate faster than the per-step error: the bound is on the update, not 1e-5."""
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    obs, act, hidden, mb, nmb = 376, 17, 256, 32768, 4
    B = mb * nmb
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, seed=1)
    g = torch.Generator().manual_seed(5)
    data = _random_minibatch(obs, act, B, seed=6)
    with torch.no_grad():
        lp, _ = O.get_logprob_entropy(pol, data["states"], data["actions"])
    data["log_probs"] = lp + 0.1 * torch.randn(B, generator=g)
    names = ("states", "actions", "log_probs", "advantages", "returns")
    L = O.Learner(pol, cri, lr=3e-4, clip_range=0.2, entropy_coef=0.0, critic_coef=0.5, max_grad_norm=0.5)
    fp = _flat_from_named(k, pol, cri)
    P = k.param_count
    ldx = k.states_pitch()
    xs = torch.zeros(B, ldx, device=DEV)
    xs[:, :obs] = data["states"].to(DEV)
    xs[:, obs] = 1.0
    d = {n: v.to(DEV).contiguous() for n, v in data.items() if n != "states"}
    stats, metrics = torch.empty(nmb, 2, device=DEV), torch.zeros(nmb, 8, device=DEV)
    k.advantage_stats(d["advantages"], B, mb, stats)
    exp_avg, exp_avg_sq, grads = torch.zeros(P, device=DEV), torch.zeros(P, device=DEV), torch.zeros(P, device=DEV)
    lr, step = torch.full((1,), 3e-4, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    ws = k.minibatch_workspace(mb, DEV)
    hp = make_hparams(0.2, 0.0, 0.5, 0.5)
    report = []
    for i in range(nmb):
        sl = slice(i * mb, (i + 1) * mb)
        # the oracle at OUR current weights
        pol_now, cri_now = fp.state_dicts()
        Lk = O.Learner(pol_now, cri_now, clip_range=0.2, entropy_coef=0.0, critic_coef=0.5)
        gp, gc, met = Lk.grads(*(data[n][sl] for n in names))
        args = k.minibatch_args(m=0, m_global=1, states=xs[sl], actions=d["actions"][sl], log_probs=d["log_probs"][sl], advantages=d["advantages"][sl],
                                returns=d["returns"][sl], adv_stats=stats[i], params=fp.flat, grads=grads, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq, lr=lr,
                                step_count=step, hp=hp, metrics=metrics[i], workspace=ws, states_ld=ldx, states_ones_col=True)
        k.update_epoch(args, mb, mb)  # one minibatch: forward, loss, backward, clip, Adam
        torch.cuda.synchronize()
        gflat = fp.__class__(k, DEV)
        gflat.flat.copy_(grads)
        gpol, gcri = gflat.state_dicts()
        worst = max(_rel((gpol if n in gpol else gcri)[n].numpy(), ref.numpy()) for n, ref in {**gp, **gc}.items())
        report.append(worst)
        for n, ref in {**gp, **gc}.items():
            ours = (gpol if n in gpol else gcri)[n].numpy()
            assert _rel(ours, ref.numpy()) <= 1e-5, (i, n, _rel(ours, ref.numpy()))
        mm = metrics[i].cpu().numpy()
        assert abs(mm[0] - met["pg_loss"]) <= 1e-5 * max(abs(met["pg_loss"]), 0.5) and abs(mm[1] - met["critic_loss"]) <= 1e-5 * abs(met["critic_loss"])
        assert abs(mm[3] - met["approx_kl"]) <= 1e-5 * max(abs(met["approx_kl"]), 1e-2) and abs(mm[4] - met["clip_fraction"]) <= 2.0 / mb
        L.minibatch_step(*(data[n][sl] for n in names))  # the oracle's own trajectory
    print("bench-shape epoch: worst per-tensor gradient distance per minibatch (same weights on both sides):", report)
    assert int(step.item()) == nmb
    pol_now, cri_now = fp.state_dicts()
    traj = {}
    for name in list(O.POLICY_KEYS) + list(O.CRITIC_KEYS):
        ours = (pol_now if name in pol_now else cri_now)[name].numpy()
        ref = (L.pol if name in L.pol else L.cri)[name].detach().numpy()
        init = (pol if name in pol else cri)[name].numpy()
        traj[name] = float(np.linalg.norm(ours - ref) / max(np.linalg.norm(ref - init), 1e-30))  # distance relative to the UPDATE
        assert float(np.abs(ours - ref).max()) <= 0.6 * nmb * 3e-4, (name, float(np.abs(ours - ref).max()))
    print("bench-shape epoch: |ours - oracle trajectory| / |oracle update| after 4 steps:", traj)
    assert max(traj.values()) <= 2e-2, traj


@pytest.mark.parametrize("m", [1, 2, 7, 40, 4099, 32768])
def test_ratio_delta_median_is_torch_median(m):
    """hp.ratio_delta_metric = 2 (ESPO delta_calc_operator = "median", espo.py:59-60): metrics[4] = torch.median(|ratio - 1|), i.e. the LOWER
    median sorted[(m - 1) // 2], selected on the device from the per-row values the loss kernel leaves behind."""
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    obs, act, hidden = (24, 5, 128) if m < 1000 else (376, 17, 256)
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.9, seed=m)
    mb = _random_minibatch(obs, act, m, seed=m + 2)
    with torch.no_grad():
        lp, _ = O.get_logprob_entropy(pol, mb["states"], mb["actions"])
    mb["log_probs"] = lp + 0.15 * torch.randn(m, generator=torch.Generator().manual_seed(m))
    fp = _flat_from_named(k, pol, cri)
    if m == 1:
        mb["advantages"] = torch.zeros(1)  # the advantage normalisation of a single row is NaN; the ratio is not
    args, grads, metrics, st, keep = _run_fwdbwd(k, fp, mb, make_hparams(float("inf"), 0.0, 0.5, 0.5, ratio_delta_metric="median"))
    torch.cuda.synchronize()
    with torch.no_grad():
        lp_new, _ = O.get_logprob_entropy(pol, mb["states"], mb["actions"])
        dev = torch.abs(torch.exp(lp_new - mb["log_probs"]) - 1)
    ref = float(torch.median(dev))
    ours = float(metrics[4])
    # the kernel's ratios differ from the oracle's by fp32 rounding, so the selected element may be a neighbour in the sorted order
    srt = torch.sort(dev).values
    kth = (m - 1) // 2
    lo, hi = float(srt[max(kth - 2, 0)]), float(srt[min(kth + 2, m - 1)])
    assert abs(ours - ref) <= 2e-5 * max(ref, 1e-3) or (lo - 1e-6 <= ours <= hi + 1e-6), (ours, ref, lo, hi)


def test_library_reports_kernel_launches():
    from rl_x_b200 import _native as nt
    lib = nt.load()
    lib.rlx_reset_launch_count()
    k = _kern(8, 2, 32)
    x = torch.zeros(4, 8, device=DEV)
    k.gae(x[:, :4].contiguous(), x[:, :4].contiguous(), x[:, :4].contiguous(), 0.99, 0.95, torch.empty(4, 4, device=DEV),
          torch.empty(4, 4, device=DEV), last_value=torch.zeros(4, device=DEV))
    assert lib.rlx_launch_count() == 1


# ------------------------------------------------------------------------------------- multi-GPU helpers on one GPU
def test_segment_moments_reproduce_minibatch_mean_and_unbiased_std():
    """rlx_segment_moments_f32 (sharded advantage statistics): with one rank the two passes give torch's mean / std(ddof=1) of every
    ragged segment (ppo.py:133-134)."""
    k = _kern(8, 2, 32)
    g = torch.Generator().manual_seed(4)
    counts = [1000, 1, 37, 4096, 2]
    x = (torch.randn(sum(counts), generator=g) * 3 + 0.5).to(DEV)
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int64, device=DEV)
    gc = torch.tensor(counts, dtype=torch.float32, device=DEV)
    sums, ssq = torch.empty(len(counts), device=DEV), torch.empty(len(counts), device=DEV)
    k.segment_moments(x, offsets, None, None, sums)
    k.segment_moments(x, offsets, sums, gc, ssq)
    mean, std = (sums / gc).cpu(), torch.sqrt(ssq / (gc - 1)).cpu()
    o = 0
    for i, c in enumerate(counts):
        seg = x[o:o + c].cpu()
        o += c
        assert abs(float(mean[i]) - float(seg.mean())) <= 1e-6 * max(1.0, abs(float(seg.mean())))
        if c > 1:
            assert abs(float(std[i]) - float(seg.std())) <= 2e-6 * float(seg.std())
        else:
            assert torch.isnan(std[i])  # like torch.std of one element


def test_peer_comm_world_of_one_is_a_copy():
    """rlx_comm_* with a single rank: no peers to map, the all-reduce kernel returns the staged buffer (covers create / stage /
    double-buffered slots / destroy on a one-GPU box; the multi-rank protocol is tests/dist_check_comm.py)."""
    from rl_x_b200.algorithms.ppo.b200.kernels import PeerComm

    class OneRank:
        @staticmethod
        def get_rank():
            return 0

        @staticmethod
        def get_world_size():
            return 1

        class ReduceOp:
            MIN = None

        @staticmethod
        def all_gather(out, t):
            out[0].copy_(t)

        @staticmethod
        def all_reduce(t, op=None):
            return None

    n = 1003
    comm = PeerComm(OneRank, n, torch.device(DEV))
    out = torch.empty(n, device=DEV)
    for i in range(5):
        src = torch.arange(n, device=DEV, dtype=torch.float32) * (i + 1)
        comm.stage(src)
        comm.allreduce_sum(out)
        assert torch.equal(out, src)
    comm.stage(src, 10)
    comm.allreduce_sum(out, 10)
    with pytest.raises(RuntimeError):
        comm.allreduce_sum(out, n + 1)
    comm.close()
