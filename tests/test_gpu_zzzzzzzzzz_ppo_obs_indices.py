"""PPO / ESPO with observation index sets on the GPU: the embedded layer-1 matrix (ppo_embed_w1_kernel) and the folded layer-1 gradient
(ppo_grad_reduce_kernel's column map) against float64 autograd of the index-selecting oracle (tests/obs_indices_oracle.py), on both GEMM
engines; explicit identity sets against NULL ones to the bit; the plugin against the executed reference's run
(tests/golden/ppo_obs_indices.npz); bf16-autocast mode, ESPO and checkpoints.

Bounds are the other GPU files': ||g - g64|| <= 1e-5 ||g64|| per gradient tensor (test_gpu_zzzzzz_tc_ppo_shapes.py, whose proof-of-path
counters are reused: the wgmma shapes must launch the pre-split tc_gemm_kernel instances and no SIMT GEMM), test_gpu_bf16.py's for bf16,
test_gpu_train.py's for the plugin run.  Sorted after the other GPU files."""
import numpy as np
import pytest
import torch

from conftest import Golden
from oracle import ppo_oracle as O
import obs_indices_oracle as X
from test_gpu_parity import _random_minibatch, _run_fwdbwd
from test_gpu_zzzzzz_tc_ppo_shapes import (FWD_CONVERT, GP_SGEMM, SUMMED_BIASES, _assert_losses, _assert_update_path, _dist, _f64, _hp,
                                           _paths, _tc_instances)

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = ("states", "actions", "log_probs", "advantages", "returns")
CLIP, ENT, CRITIC_COEF = 0.2, 0.01, 0.5


@pytest.fixture(autouse=True)
def lib():
    from rl_x_b200 import _native as nt
    lib = nt.load()
    yield lib
    lib.rlx_set_gemm_engine(0)
    lib.rlx_set_autocast_bf16(0)


def _sets(obs, P, C, seed):
    r = np.random.default_rng(seed)
    return r.permutation(obs)[:P].astype(np.int64), r.permutation(obs)[:C].astype(np.int64)


def _kern(obs, act, hidden, pidx=None, cidx=None):
    from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels
    return PpoKernels(obs, act, hidden, pidx, cidx)


def _flat(k, pol, cri):
    from rl_x_b200.algorithms.ppo.b200.ppo import FlatParameters
    fp = FlatParameters(k, DEV)
    fp.load_named({**{n: torch.as_tensor(v) for n, v in pol.items()}, **{n: torch.as_tensor(v) for n, v in cri.items()}})
    return fp


def _named(k, flat):
    from rl_x_b200.algorithms.ppo.b200.ppo import FlatParameters
    f = FlatParameters(k, DEV)
    f.flat.copy_(flat[:k.param_count])
    p, c = f.state_dicts()
    return {n: v.numpy().astype(np.float64) for n, v in {**p, **c}.items()}


def _case(obs, act, hidden, m, pidx, cidx):
    pol, cri = X.init_params(obs, act, hidden, std_dev=0.9, seed=m, policy_idx=pidx, critic_idx=cidx)
    g = torch.Generator().manual_seed(m + 1)
    for w in list(pol.values()) + list(cri.values()):
        w.add_(0.02 * torch.randn(w.shape, generator=g))
    mb = _random_minibatch(obs, act, m, seed=m + 2)
    with torch.no_grad():
        lp, _ = X.get_logprob_entropy(_f64(pol), mb["states"].to(DEV, torch.float64), mb["actions"].to(DEV, torch.float64), pidx)
    mb["log_probs"] = lp.float().cpu() + 0.15 * torch.randn(m, generator=g)
    return pol, cri, mb


def _oracle64(pol, cri, mb, pidx, cidx):
    """float64 gradients of the index-selecting oracle, with test_gpu_zzzzzz_tc_ppo_shapes.py's norm rule for the two last-layer biases."""
    m = mb["states"].shape[0]
    pol64, cri64 = _f64(pol), _f64(cri)
    pol64["policy_mean.4.bias"] = pol64["policy_mean.4.bias"].expand(m, -1).clone()
    cri64["critic.4.bias"] = cri64["critic.4.bias"].expand(m, -1).clone()
    L = X.Learner(pol64, cri64, pidx, cidx, clip_range=CLIP, entropy_coef=ENT, critic_coef=CRITIC_COEF)
    gp, gc, met = L.grads(*(mb[n].to(DEV, torch.float64) for n in NAMES))
    g = {n: v.cpu().numpy() for n, v in {**gp, **gc}.items()}
    norms = {n: float(np.linalg.norm(v)) for n, v in g.items()}
    for n in SUMMED_BIASES:
        terms = g[n]
        g[n] = terms.sum(0)
        norms[n] = max(float(np.linalg.norm(g[n])), float(np.linalg.norm(np.sqrt((terms ** 2).sum(0)))))
    return g, {n: max(v, 1e-30) for n, v in norms.items()}, met


# ------------------------------------------------------------------------------------------------------------ forward
FWD_SHAPES = [(376, 17, 256, 188, 376), (40, 4, 128, 23, 33)]


@pytest.mark.parametrize("obs,act,hidden,P,C", FWD_SHAPES)
@pytest.mark.parametrize("n", [63, 4096])
@pytest.mark.parametrize("engine", [0, 1])
def test_forward_vs_float64(lib, obs, act, hidden, P, C, n, engine):
    pidx, cidx = _sets(obs, P, C, obs + P)
    k = _kern(obs, act, hidden, pidx, cidx)
    pol, cri = X.init_params(obs, act, hidden, std_dev=0.7, seed=n, policy_idx=pidx, critic_idx=cidx)
    fp = _flat(k, pol, cri)
    g = torch.Generator().manual_seed(n)
    obs_t, noise = torch.randn(n, obs, generator=g), torch.randn(n, act, generator=g)
    low, high = -torch.ones(act) * 1.5, torch.ones(act)
    lib.rlx_set_gemm_engine(engine)
    ws = k.forward_workspace(n, DEV)
    out = {s: torch.full(shape, float("nan"), device=DEV) for s, shape in
           (("action", (n, act)), ("env_action", (n, act)), ("logp", (n,)), ("value", (n,)), ("det", (n, act)), ("critic", (n,)))}
    x, nz = obs_t.to(DEV), noise.to(DEV)

    def run():
        k.forward(fp.flat, x, ws, noise=nz, act_low=low.to(DEV), act_high=high.to(DEV), action=out["action"], env_action=out["env_action"],
                  logp=out["logp"], value=out["value"])
        k.forward(fp.flat, x, ws, act_low=low.to(DEV), act_high=high.to(DEV), deterministic=True, env_action=out["det"])
        k.critic_forward(fp.flat, x, out["critic"], ws)
    _, counts = _paths(lib, run)
    if engine == 1:
        assert set(_tc_instances(counts)) == {FWD_CONVERT} and counts.get(GP_SGEMM, 0) == 0, counts
    else:
        assert _tc_instances(counts) == {} and counts.get(GP_SGEMM, 0) > 0, counts
    x64, n64 = obs_t.double(), noise.double()
    p64, c64 = {a: b.double() for a, b in pol.items()}, {a: b.double() for a, b in cri.items()}
    with torch.no_grad():
        a64, ea64, lp64 = X.get_action_logprob(p64, x64, n64, low.double(), high.double(), True, pidx)
        v64 = X.critic_value(c64, x64, cidx).reshape(-1)
        det64 = X.get_deterministic_action(p64, x64, low.double(), high.double(), True, pidx)
    for name, ours, ref, tol in (("action", out["action"], a64, 2e-5), ("env_action", out["env_action"], ea64, 2e-5), ("value", out["value"], v64, 2e-5),
                                 ("critic", out["critic"], v64, 2e-5), ("det", out["det"], det64, 2e-5), ("logp", out["logp"], lp64, 1e-4 * act)):
        np.testing.assert_allclose(ours.cpu().double().numpy(), ref.numpy(), rtol=1e-5, atol=tol, err_msg=name)


# ------------------------------------------------------------------------------------------------ minibatch fwd + bwd
# (obs, act, hidden, m, P, C): the locomotion shape; the golden's; a policy narrower than 32 columns with a ragged m; obs off the 4-float
# grid (the wgmma engine declines the network: SIMT alone); the benchmark's minibatch
MB_SHAPES = [(376, 17, 256, 4096, 188, 376), (40, 4, 128, 1000, 23, 33), (64, 3, 128, 777, 20, 64), (42, 3, 128, 500, 30, 21),
             (376, 17, 256, 32768, 188, 376)]


@pytest.mark.parametrize("obs,act,hidden,m,P,C", MB_SHAPES)
def test_minibatch_gradients_vs_float64_on_both_engines(lib, obs, act, hidden, m, P, C):
    pidx, cidx = _sets(obs, P, C, m)
    k = _kern(obs, act, hidden, pidx, cidx)
    pol, cri, mb = _case(obs, act, hidden, m, pidx, cidx)
    g64, norms, met = _oracle64(pol, cri, mb, pidx, cidx)
    on_tc = obs % 4 == 0 and obs >= 32 and hidden % 128 == 0
    for engine in (0, 1):
        lib.rlx_set_gemm_engine(engine)
        fp = _flat(k, pol, cri)
        (_, grads, metrics, _, _), counts = _paths(lib, lambda: _run_fwdbwd(k, fp, mb, _hp(ENT)))
        if engine == 1 and on_tc:
            _assert_update_path(counts, head_on_tc=act <= 31)
        else:
            assert _tc_instances(counts) == {} and counts.get(GP_SGEMM, 0) > 0, counts
        ours = _named(k, grads)
        assert ours["policy_mean.0.weight"].shape == (hidden, P) and ours["critic.0.weight"].shape == (hidden, C)
        worst = 0.0
        for name, ref in g64.items():
            d = _dist(ours[name], ref) / norms[name]
            worst = max(worst, d)
            assert d <= 1e-5, (engine, name, d)
        print(f"\n({obs}, {act}, {hidden}, {m}, P={P}, C={C}) engine {engine}: worst distance / norm {worst:.2e}")
        _assert_losses(metrics.cpu().numpy(), met, mb["advantages"], m)


# --------------------------------------------------------------------------------- explicit identity == NULL, bit for bit
@pytest.mark.parametrize("obs,act,hidden,m", [(376, 17, 256, 4096), (11, 3, 64, 40)])
@pytest.mark.parametrize("engine", [0, 1])
@pytest.mark.parametrize("bf16", [0, 1])
def test_explicit_identity_sets_are_bit_identical_to_null(lib, obs, act, hidden, m, engine, bf16):
    """arange(obs_dim) passed as both index arrays takes the embed + fold path; it must give the NULL path's gradients, metrics, weights and
    Adam moments to the bit - the embedded matrix IS W1cat and the fold maps every column onto itself."""
    ident = np.arange(obs)
    k0, k1 = _kern(obs, act, hidden), _kern(obs, act, hidden, ident, ident)
    assert k1.dims.policy_idx and k1.dims.critic_idx and k0.param_count == k1.param_count
    pol, cri, mb = _case(obs, act, hidden, m, None, None)
    lib.rlx_set_gemm_engine(engine)
    lib.rlx_set_autocast_bf16(bf16)
    res = []
    for k in (k0, k1):
        fp = _flat(k, pol, cri)
        args, grads, metrics, st, keep = _run_fwdbwd(k, fp, mb, _hp(ENT))
        k.clip_adam(args)
        v = torch.zeros(m, device=DEV)
        k.critic_forward(fp.flat, keep[0]["states"][:, :obs].contiguous(), v, k.forward_workspace(m, DEV))
        torch.cuda.synchronize()
        res.append((grads.clone(), metrics.clone(), fp.flat.clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone(), v))
    for a, b, what in zip(res[0], res[1], ("gradient", "metrics", "weights", "exp_avg", "exp_avg_sq", "values")):
        assert torch.equal(a, b), what


# ---------------------------------------------------------------------------------------------- bf16-autocast mode
@pytest.mark.parametrize("obs,act,hidden,m,P,C", [(376, 17, 256, 4096, 188, 376), (40, 4, 128, 1000, 23, 33)])
@pytest.mark.parametrize("engine", [0, 1])
def test_bf16_minibatch_gradients_vs_oracle_autocast(lib, obs, act, hidden, m, P, C, engine):
    from test_gpu_bf16 import _is_bf16, _rel
    pidx, cidx = _sets(obs, P, C, m + 1)
    k = _kern(obs, act, hidden, pidx, cidx)
    pol, cri, mb = _case(obs, act, hidden, m, pidx, cidx)
    L = X.Learner(pol, cri, pidx, cidx, clip_range=CLIP, entropy_coef=ENT, critic_coef=CRITIC_COEF, bf16=True)
    L.popt.zero_grad()
    L.copt.zero_grad()
    with O.autocast_bf16(True):
        loss, pg, ent, kl, cf = O.policy_loss(L.pol, X.select(mb["states"], pidx), mb["actions"], mb["log_probs"], mb["advantages"], CLIP, ENT)
    loss.backward()
    with O.autocast_bf16(True):
        closs = O.critic_loss(L.cri, X.select(mb["states"], cidx), mb["returns"], CRITIC_COEF)
    closs.backward()
    ref = {n: L.pol[n].grad.numpy() for n in O.POLICY_KEYS}
    ref.update({n: L.cri[n].grad.numpy() for n in O.CRITIC_KEYS})
    lib.rlx_set_gemm_engine(engine)
    lib.rlx_set_autocast_bf16(1)
    fp = _flat(k, pol, cri)
    args, grads, metrics, st, keep = _run_fwdbwd(k, fp, mb, _hp(ENT))
    torch.cuda.synchronize()
    ours = _named(k, grads)
    report = {n: _rel(ours[n], r) for n, r in ref.items()}
    print("bf16 gradient distances:", report)
    for n, d in report.items():
        if n != "policy_logstd":
            assert _is_bf16(torch.from_numpy(ours[n]).float()), n
        assert d <= (5e-2 if n in SUMMED_BIASES else 1e-2), (n, report)
    mm = metrics.cpu().numpy()
    assert abs(mm[1] - closs.item()) <= 1e-2 * abs(closs.item())


# ------------------------------------------------------------------------------------------------ plugin: golden run
def _reference_noise(g, pidx):
    out = []
    for it in range(g.iterations):
        pol, _ = g.params("init" if it == 0 else f"iter{it - 1}")
        pol = {k: torch.from_numpy(v) for k, v in pol.items()}
        states = torch.from_numpy(g[f"iter{it}/states"]).reshape(-1, g.obs)
        with torch.no_grad():
            mean = X.policy_mean(pol, states, pidx)
        eps = (torch.from_numpy(g[f"iter{it}/actions"]).reshape(-1, g.act) - mean) / torch.exp(pol["policy_logstd"])
        out.append(eps.reshape(g.T, g.N, g.act))
    return torch.cat(out).to(DEV).contiguous()


@pytest.fixture(scope="module")
def golden_idx():
    return Golden("obs_indices")


def _indexed_env(g, interface, as_tensor=False):
    from test_gpu_train import ReplayEnv
    env = ReplayEnv(g, interface)
    env.policy_observation_indices = torch.from_numpy(g["policy_idx"]) if as_tensor else g["policy_idx"]
    env.critic_observation_indices = list(g["critic_idx"]) if as_tensor else g["critic_idx"]
    return env


@pytest.mark.parametrize("interface", ["TORCH", "NUMPY"])
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_plugin_reproduces_the_reference_run(golden_idx, interface, engine):
    from rl_x_b200.algorithms.ppo.b200.ppo import PPO
    from test_gpu_train import _config
    g = golden_idx
    env = _indexed_env(g, interface, as_tensor=interface == "TORCH")
    model = PPO(_config(g, engine=engine), env, env, "/tmp/rlx_test_run_idx", None)
    assert model.kernels.policy_in_dim == 23 and model.kernels.critic_in_dim == 33
    eps = _reference_noise(g, g["policy_idx"])
    calls = {"n": 0}

    def draw(step):
        calls["n"] += 1
        return eps[calls["n"] - 1]
    model._draw_noise = draw
    model.log = lambda *a, **k: None
    snaps = []
    orig = model.start_logging

    def start_logging(step):
        b = model.batch
        snaps.append(dict(adv=b.advantages.cpu().numpy().copy(), ret=b.returns.cpu().numpy().copy(), sd=model.params.state_dicts()))
        orig(step)
    model.start_logging = start_logging
    model.train()
    assert calls["n"] == g.T * g.iterations and len(snaps) == g.iterations
    np.testing.assert_allclose(torch.stack(env.actions).numpy(), g["env_actions"], rtol=1e-4, atol=5e-6)
    relnorm = lambda a, b: float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b.astype(np.float64)), 1e-30))
    for it, s in enumerate(snaps):
        bar = 1e-5 if it == 0 else 1e-4
        for key, name in (("adv", "advantages"), ("ret", "returns")):
            assert relnorm(s[key], g[f"iter{it}/{name}"]) <= bar, (it, name)
        pol, cri = s["sd"]
        pol_ref, cri_ref = g.params(f"iter{it}")
        for name, v in {**pol_ref, **cri_ref}.items():
            ours = (pol if name in pol else cri)[name].numpy()
            assert ours.shape == v.shape, name
            assert float(np.linalg.norm(ours - v) / np.linalg.norm(v)) <= 2e-5, (it, name)


def test_plugin_gae_and_index_stream_bit_exact_when_teacher_forced(golden_idx):
    """With the reference's stored values and next_values, the plugin's GAE kernel gives the reference's advantages / returns to the bit,
    and its permutation stream is the reference's (index sets change neither)."""
    from rl_x_b200.algorithms.ppo.b200.ppo import PPO
    from rl_x_b200 import _native as nt
    from test_gpu_train import _config
    g = golden_idx
    env = _indexed_env(g, "TORCH")
    model = PPO(_config(g), env, env, "/tmp/rlx_test_run_idx", None)
    k = model.kernels
    for it in range(g.iterations):
        r, te, v = (torch.from_numpy(g[f"iter{it}/{n}"]).to(DEV).contiguous() for n in ("rewards", "terminations", "values"))
        nv = torch.from_numpy(g[f"iter{it}/next_values"]).to(DEV).contiguous()
        adv, ret = torch.empty_like(r), torch.empty_like(r)
        k.gae(r, te, v, g.gamma, g.gae_lambda, adv, ret, next_values=nv)
        assert np.array_equal(adv.cpu().numpy(), g[f"iter{it}/advantages"]) and np.array_equal(ret.cpu().numpy(), g[f"iter{it}/returns"])
    rng = nt.Pcg64Generator(g.seed)
    for it in range(g.iterations):
        idx = np.arange(g.B)
        for e in range(g.epochs):
            rng.shuffle(idx)
            assert np.array_equal(idx, g[f"perm/{it * g.epochs + e}"])


# --------------------------------------------------------------------------------------------------------------- ESPO
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_espo_with_index_sets_matches_the_espo_oracle(golden_idx, engine):
    """ESPO inherits the index sets from PPO: one update pass on the golden run's first rollout, teacher-forced, against the ESPO oracle
    with the same sets and the same Generator.choice draws."""
    from rl_x_b200.algorithms.espo.b200.espo import ESPO
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.espo.b200.default_config import get_config
    g = golden_idx
    env = _indexed_env(g, "TORCH")
    a = get_config("espo.b200")
    a.nr_steps, a.minibatch_size, a.max_epochs, a.nr_hidden_units, a.total_timesteps = g.T, g.mb, 4, g.hidden, g.N * g.T
    a.std_dev, a.entropy_coef, a.learning_rate, a.gamma, a.gae_lambda, a.gemm_engine = g.std_dev, g.entropy_coef, g.lr, g.gamma, g.gae_lambda, engine
    cfg = ConfigDict(algorithm=a, environment=ConfigDict(seed=g.seed, nr_envs=g.N),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    model = ESPO(cfg, env, env, "/tmp/rlx_test_run_idx_espo", None)
    assert model.kernels.policy_in_dim == 23 and model.kernels.critic_in_dim == 33
    eps = _reference_noise(g, g["policy_idx"])
    calls = {"n": 0}

    def draw(step):
        calls["n"] += 1
        return eps[calls["n"] - 1]
    model._draw_noise = draw
    model.log = lambda *a, **k: None
    snap = {}
    orig = model.start_logging

    def start_logging(step):
        b = model.batch
        snap.update({n: getattr(b, n).cpu().clone() for n in ("states", "actions", "log_probs", "advantages", "returns")})
        orig(step)
    model.start_logging = start_logging
    model.train()
    pol, cri = g.params("init")
    L = X.EspoLearner(_t(pol), _t(cri), g["policy_idx"], g["critic_idx"], lr=cfg.algorithm.learning_rate, entropy_coef=cfg.algorithm.entropy_coef,
                      critic_coef=cfg.algorithm.critic_coef, max_grad_norm=cfg.algorithm.max_grad_norm, max_ratio_delta=cfg.algorithm.max_ratio_delta)
    T = g.T
    batch = O.flatten({"states": snap["states"][:T], "actions": snap["actions"], "log_probs": snap["log_probs"], "advantages": snap["advantages"],
                       "returns": snap["returns"]})
    rng = np.random.default_rng(g.seed)
    metrics = L.update(batch, lambda: rng.choice(g.B, size=cfg.algorithm.minibatch_size, replace=False), cfg.algorithm.max_epochs)
    assert len(metrics) >= 1
    p_sd, c_sd = model.params.state_dicts()
    for name, v in {**L.pol, **L.cri}.items():
        ours = (p_sd if name in p_sd else c_sd)[name].numpy()
        ref = v.detach().numpy()
        assert float(np.linalg.norm(ours - ref) / np.linalg.norm(ref)) <= 2e-5, name


def _t(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in d.items()}


# --------------------------------------------------------------------------------------------------------- checkpoints
def test_checkpoint_round_trip_and_reference_checkpoint(golden_idx, tmp_path, monkeypatch):
    """save() writes [H, P] / [H, C] first layers with the reference's keys and Adam numbering, load() restores them exactly; the best.model
    the reference's own save() wrote at the end of the golden run loads onto the flat layout, and training continues from it."""
    import os
    from rl_x_b200 import _native as nt
    from rl_x_b200.algorithms.ppo.b200.ppo import CRITIC_PARAM_ORDER, POLICY_PARAM_ORDER, PPO
    from test_gpu_train import _config
    g = golden_idx
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ck_path = os.path.join(root, "tests", "golden", "ppo_obs_indices_ref_checkpoint.model")
    ck = torch.load(ck_path, weights_only=False)
    cfg = _config(g)
    cfg.runner.load_model = ck_path
    cfg.runner.save_model = True
    env = _indexed_env(g, "TORCH")
    model = PPO.load(cfg, env, env, str(tmp_path / "run"), None, set())
    last = f"iter{g.iterations - 1}"
    pol, cri = g.params(last)
    for tag, keys, ref in (("policy", nt.POLICY_KEYS, pol), ("critic", nt.CRITIC_KEYS, cri)):
        for name, seg in keys.items():
            assert np.array_equal(model.params.view(model.params.flat, seg).cpu().numpy(), ref[name]), name
        # Adam states arrive where the reference's optimisers had them (parameter i of the reference is order[i])
        order = POLICY_PARAM_ORDER if tag == "policy" else CRITIC_PARAM_ORDER
        for i, name in enumerate(order):
            st = ck[f"{tag}_optimizer_state_dict"]["state"][i]
            assert torch.equal(model.params.view(model.exp_avg, keys[name]).cpu(), st["exp_avg"]), name
            assert torch.equal(model.params.view(model.exp_avg_sq, keys[name]).cpu(), st["exp_avg_sq"]), name
    step = int(model.adam_step.item())
    assert step == g.iterations * g.epochs * (g.B // g.mb)
    model.save()
    mine = torch.load(str(tmp_path / "run" / "models" / "best.model"), weights_only=False)
    for sd in ("policy_state_dict", "critic_state_dict"):
        assert list(mine[sd]) == list(ck[sd])
        for key in ck[sd]:
            assert torch.equal(mine[sd][key], ck[sd][key]), key
    for od in ("policy_optimizer_state_dict", "critic_optimizer_state_dict"):
        for i, s in ck[od]["state"].items():
            assert torch.equal(mine[od]["state"][i]["exp_avg"], s["exp_avg"]) and torch.equal(mine[od]["state"][i]["exp_avg_sq"], s["exp_avg_sq"]), i
    # round trip of our own file, then a continued run
    cfg2 = _config(g)
    cfg2.runner.load_model = str(tmp_path / "run" / "models" / "best.model")
    model2 = PPO.load(cfg2, env, env, str(tmp_path / "run2"), None, set())
    assert torch.equal(model2.params.flat, model.params.flat) and torch.equal(model2.exp_avg_sq, model.exp_avg_sq)
    env.t = 0
    model2.log = lambda *a, **k: None
    model2.train()
    assert int(model2.adam_step.item()) > step and torch.isfinite(model2.params.flat).all()
    # a checkpoint for other index sets is refused
    env_other = _indexed_env(g, "TORCH")
    env_other.policy_observation_indices = g["policy_idx"][:20]
    with pytest.raises((ValueError, RuntimeError)):
        PPO.load(cfg2, env_other, env_other, str(tmp_path / "run3"), None, set())
