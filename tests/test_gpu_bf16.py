"""bf16-autocast mode of the PPO path on the GPU (rlx_set_autocast_bf16; the reference's default `bf16_mixed_precision_training`,
rl_x/algorithms/ppo/pytorch/ppo.py:98-107,123,155,208,253; SURVEY.md §8 f3) against oracle/ppo_oracle.py's autocast variant, which is
pinned to a CPU-autocast run of the executed reference (tests/golden/ppo_small_bf16.npz, tests/test_oracle_vs_reference.py).

Stated tolerance.  Every tensor autocast keeps in bf16 carries a rounding of relative size 2^-9 (half a bf16 ulp); two implementations
that accumulate a GEMM in a different order round a fraction of those elements to neighbouring bf16 values.  Hence: index work and the
mixed-precision GAE bit-exact; bf16-valued forward quantities within 2 bf16 ulps per element (2^-7 relative) and 2e-3 of the tensor norm;
gradients within 1e-2 of the norm per tensor; losses within 1e-2 of their summand scale.  (The fp32 path's bar stays 1e-5.)"""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True, params=["simt", "tcgen05"])
def bf16_mode(request):
    from rl_x_b200 import _native as nt
    lib = nt.load()
    lib.rlx_set_gemm_engine(1 if request.param == "tcgen05" else 0)
    lib.rlx_set_autocast_bf16(1)
    yield request.param
    lib.rlx_set_autocast_bf16(0)
    lib.rlx_set_gemm_engine(0)


def _kern(obs, act, hidden):
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(obs, act, hidden)


def _flat(k, pol, cri):
    from rl_x_b200.algorithms.ppo.b200.ppo import FlatParameters
    fp = FlatParameters(k, DEV)
    fp.load_named({**{n: torch.as_tensor(v) for n, v in pol.items()}, **{n: torch.as_tensor(v) for n, v in cri.items()}})
    return fp


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _is_bf16(t):
    return torch.equal(t, t.bfloat16().float())


def test_bf16_gae_bit_exact_vs_reference_golden():
    """calculate_gae_advantages_and_returns_mixed_precision (ppo.py:98-107): `gamma * next_values` is a bf16 product, the scan is fp32."""
    from conftest import Golden
    g = Golden("small_bf16")
    k = _kern(g.obs, g.act, g.hidden)
    for it in range(g.iterations):
        adv, ret = torch.empty(g.T, g.N, device=DEV), torch.empty(g.T, g.N, device=DEV)
        k.gae(torch.from_numpy(g[f"iter{it}/rewards"]).to(DEV), torch.from_numpy(g[f"iter{it}/terminations"]).to(DEV),
              torch.from_numpy(g[f"iter{it}/values"]).to(DEV), g.gamma, g.gae_lambda, adv, ret, next_values=torch.from_numpy(g[f"iter{it}/next_values"]).to(DEV))
        assert np.array_equal(adv.cpu().numpy(), g[f"iter{it}/advantages"]) and np.array_equal(ret.cpu().numpy(), g[f"iter{it}/returns"])


@pytest.mark.parametrize("obs,act,hidden,n", [(11, 3, 64, 108), (376, 17, 256, 4096), (24, 5, 128, 300), (32, 1, 128, 1000), (128, 4, 384, 2048)])
def test_bf16_forward_vs_oracle(obs, act, hidden, n):
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.8, seed=obs + n)
    g = torch.Generator().manual_seed(n)
    for w in list(pol.values()) + list(cri.values()):
        w.add_(0.05 * torch.randn(w.shape, generator=g))
    x, noise = torch.randn(n, obs, generator=g), torch.randn(n, act, generator=g)
    low, high = torch.full((act,), -2.0), torch.full((act,), 0.5)
    fp = _flat(k, pol, cri)
    ws = k.forward_workspace(n, DEV)
    a, e, lp, v = (torch.empty(n, act, device=DEV), torch.empty(n, act, device=DEV), torch.empty(n, device=DEV), torch.empty(n, device=DEV))
    k.forward(fp.flat, x.to(DEV), ws, noise=noise.to(DEV), act_low=low.to(DEV), act_high=high.to(DEV), action=a, env_action=e, logp=lp, value=v)
    d = torch.empty(n, act, device=DEV)
    k.forward(fp.flat, x.to(DEV), ws, act_low=low.to(DEV), act_high=high.to(DEV), deterministic=True, env_action=d)
    a, e, lp, v, d = a.cpu(), e.cpu(), lp.cpu(), v.cpu(), d.cpu()
    assert _is_bf16(a) and _is_bf16(v)  # Normal(bf16 loc, fp32 scale).sample() and the critic's Linear output are bf16 tensors
    with torch.no_grad(), O.autocast_bf16(True):
        mean = O.policy_mean(pol, x)
        v_ref = O.critic_value(cri, x).reshape(-1)
        d_ref = O.get_deterministic_action(pol, x, low, high)
        # the rollout's log-prob is evaluated on the bf16 sample (here: OUR sample, fed to the oracle)
        lp_ref, _ = O.get_logprob_entropy(pol, x, a.bfloat16())
        clipped = torch.clip(a.bfloat16(), -1, 1)
        e_ref = low + (0.5 * (clipped + 1.0) * (high - low))
    assert mean.dtype == torch.bfloat16 and v_ref.dtype == torch.bfloat16
    ulp2 = lambda ref: dict(rtol=2.0 ** -7, atol=2.0 ** -7 * float(ref.float().pow(2).mean().sqrt()))
    np.testing.assert_allclose(v.numpy(), v_ref.float().numpy(), **ulp2(v_ref))
    assert _rel(v.numpy(), v_ref.float().numpy()) <= 2e-3
    # deterministic env action = low + 0.5 * (clip(mean) + 1) * (high - low): 2 ulps of a clipped bf16 mean (|mean| <= 1: 2 * 2^-8) scaled by
    # (high - low) / 2; relative to the env action itself the bound would be meaningless near its zero crossing
    np.testing.assert_allclose(d.numpy(), d_ref.float().numpy(), rtol=0, atol=2 * 2.0 ** -8 * float((high - low).max()) / 2 * 1.01)
    np.testing.assert_allclose(e.numpy(), e_ref.float().numpy(), rtol=1e-6, atol=1e-6)          # same bf16 sample in, same fp32 arithmetic out
    # the sample itself: loc + scale * eps through at::normal's in-place chain on a bf16 tensor (3 roundings), with OUR mean
    std = torch.exp(pol["policy_logstd"]).expand(n, act)
    t = (noise.bfloat16() * std).bfloat16().float()
    chain = (t + mean.float()).bfloat16().float()
    # the mean may sit 2 bf16 ulps from the oracle's (as checked on v / d above) and the sum is rounded once more: 4 ulps of the LARGER
    # summand - where loc and scale * eps cancel, an ulp of the mean is many ulps of the small sum
    # plus the absolute noise every mean carries whatever its own size: it is a dot product over bf16 activations that differ by ulps
    # between the two implementations (the same floor the assert on d uses: 2 bf16 ulps of the tensor's rms)
    tol = 2.0 ** -6 * torch.maximum(mean.float().abs(), t.abs()) + 2.0 ** -7 * float(mean.float().pow(2).mean().sqrt())
    worst = float(((a - chain).abs() / tol).max())
    assert worst <= 1.0, worst
    # log-prob of that sample: the oracle's mean may sit one bf16 ulp from ours -> (a - mean)/sigma^2 * ulp(mean) per action dimension
    np.testing.assert_allclose(lp.numpy(), lp_ref.float().numpy(), rtol=1e-2, atol=2e-2 * act ** 0.5)


def _grads_under_autocast(L, mb):
    """oracle.Learner.grads with the two loss functions under autocast, as Learner.minibatch_step runs them (ppo.py:123,155)."""
    L.popt.zero_grad()
    L.copt.zero_grad()
    with O.autocast_bf16(True):
        loss, pg, ent, kl, cf = O.policy_loss(L.pol, mb["states"], mb["actions"], mb["log_probs"], mb["advantages"], L.clip_range, L.entropy_coef)
    loss.backward()
    with O.autocast_bf16(True):
        closs = O.critic_loss(L.cri, mb["states"], mb["returns"], L.critic_coef)
    closs.backward()
    gp = {n: L.pol[n].grad.clone() for n in O.POLICY_KEYS}
    gc = {n: L.cri[n].grad.clone() for n in O.CRITIC_KEYS}
    return gp, gc, dict(pg_loss=pg.item(), critic_loss=closs.item(), approx_kl=kl.item(), clip_fraction=cf.item())


@pytest.mark.parametrize("obs,act,hidden,m,ent", [(11, 3, 64, 40, 0.01), (376, 17, 256, 4096, 0.0), (376, 17, 256, 32768, 0.0), (24, 5, 128, 1000, 0.02),
                                                 (32, 1, 128, 1000, 0.0), (128, 4, 384, 2048, 0.01)])  # the last two on the wgmma engine's BF16 instances
def test_bf16_minibatch_gradients_vs_oracle_autograd(obs, act, hidden, m, ent):
    from rl_x_b200.algorithms.ppo.b200.kernels import make_hparams
    from test_gpu_parity import _random_minibatch, _run_fwdbwd
    k = _kern(obs, act, hidden)
    pol, cri = O.init_params(obs, act, hidden, std_dev=0.9, seed=m)
    g = torch.Generator().manual_seed(m + 1)
    for w in list(pol.values()) + list(cri.values()):
        w.add_(0.02 * torch.randn(w.shape, generator=g))
    mb = _random_minibatch(obs, act, m, seed=m + 2)
    with torch.no_grad():
        lp, _ = O.get_logprob_entropy(pol, mb["states"], mb["actions"])
    mb["log_probs"] = lp + 0.15 * torch.randn(m, generator=g)
    L = O.Learner(pol, cri, clip_range=0.2, entropy_coef=ent, critic_coef=0.5, bf16=True)
    gp, gc, met = _grads_under_autocast(L, mb)
    fp = _flat(k, pol, cri)
    args, grads, metrics, st, keep = _run_fwdbwd(k, fp, mb, make_hparams(0.2, ent, 0.5, 0.5))
    torch.cuda.synchronize()
    gflat = fp.__class__(k, DEV)
    gflat.flat.copy_(grads)
    gpol, gcri = gflat.state_dicts()
    report = {}
    for name, ref in {**gp, **gc}.items():
        ours = (gpol if name in gpol else gcri)[name]
        report[name] = _rel(ours.numpy(), ref.numpy())
        if name != "policy_logstd":
            assert _is_bf16(ours), name  # weight / bias gradients leave the bf16 ops as bf16 tensors; logstd's is fp32
    print("bf16 gradient distances:", report)
    # 1e-2 of the norm per tensor.  The last layer's bias gradients are sums of m signed bf16 terms that largely cancel (a scalar for the
    # critic): their bf16 noise is measured against the root-sum-square of the terms, i.e. sqrt(m) * |term| * 2^-9, not against the small sum
    for name, dist in report.items():
        assert dist <= (5e-2 if name in ("critic.4.bias", "policy_mean.4.bias") else 1e-2), (name, report)
    mm = metrics.cpu().numpy()
    scale = float(torch.abs(mb["advantages"] - mb["advantages"].mean()).mean() / mb["advantages"].std())
    assert abs(mm[0] - met["pg_loss"]) <= 1e-2 * max(abs(met["pg_loss"]), scale)
    assert abs(mm[1] - met["critic_loss"]) <= 1e-2 * abs(met["critic_loss"])
    assert abs(mm[3] - met["approx_kl"]) <= 1e-2 * max(abs(met["approx_kl"]), 1e-2)
    assert abs(mm[4] - met["clip_fraction"]) <= 0.01 + 2.0 / m


def test_bf16_plugin_reproduces_the_reference_run():
    """PPO(bf16_mixed_precision_training=True).train() on the replayed env stream of the reference's bf16 run (golden `small_bf16`):
    stored values are bf16 tensors within 2 ulps of the reference's, the mixed-precision advantages follow, and after the update the
    weights stay within the bf16 noise of the reference's (the update distance is stated relative to the size of the update)."""
    from conftest import Golden
    from rl_x_b200.algorithms.ppo.b200.ppo import PPO
    from test_gpu_train import ReplayEnv, _config, _reference_noise
    g = Golden("small_bf16")
    env = ReplayEnv(g, "TORCH")
    model = PPO(_config(g, engine="auto", bf16_mixed_precision_training=True), env, env, "/tmp/rlx_test_bf16", None)
    assert model.bf16_mixed_precision_training
    eps = _reference_noise(g)
    calls = {"n": 0}

    def draw(step):
        i = calls["n"]
        calls["n"] += 1
        return eps[i]

    model._draw_noise = draw
    logged, snaps = [], []
    model.log = lambda name, value, step: logged.append((name, float(value), int(step)))
    orig = model.start_logging

    def start_logging(step):
        b = model.batch
        snaps.append(dict(adv=b.advantages.cpu().numpy().copy(), val=b.values.cpu().numpy().copy(), act=b.actions.cpu().numpy().copy(), sd=model.params.state_dicts()))
        orig(step)

    model.start_logging = start_logging
    model.train()
    assert len(snaps) == g.iterations
    s0 = snaps[0]
    assert _is_bf16(torch.from_numpy(s0["val"])) and _is_bf16(torch.from_numpy(s0["act"]))
    np.testing.assert_allclose(s0["val"], g["iter0/values"], rtol=2.0 ** -7, atol=2.0 ** -7 * float(np.sqrt(np.mean(g["iter0/values"] ** 2))))
    assert _rel(s0["adv"], g["iter0/advantages"]) <= 1e-2
    pol0, cri0 = g.params("init")
    for it, s in enumerate(snaps):
        pol_ref, cri_ref = g.params(f"iter{it}")
        pol, cri = s["sd"]
        for name, v in {**pol_ref, **cri_ref}.items():
            ours = (pol if name in pol else cri)[name].numpy()
            start = (pol0 if name in pol0 else cri0)[name]
            dist = float(np.linalg.norm(ours - v) / max(np.linalg.norm(v - start), 1e-30))  # relative to the update since the start
            assert dist <= 0.25, (it, name, dist)
            assert _rel(ours, v) <= 5e-3 or np.linalg.norm(v) < 1e-2, (it, name, _rel(ours, v))
    for n in ("loss/critic_loss", "gradients/critic_grad_norm", "policy/std_dev"):
        ours = [v for m, v, _ in logged if m == n]
        np.testing.assert_allclose(ours, g[f"metric/{n}"], rtol=5e-2, err_msg=n)
