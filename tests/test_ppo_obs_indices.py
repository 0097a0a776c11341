"""PPO / ESPO with the env's policy / critic observation index sets (asymmetric actor-critic), the parts that need no GPU: the CPU oracle
against the executed reference (tests/golden/ppo_obs_indices.npz, make_golden_ppo_obs_indices.py), initial weights, the reference-layout
state dicts and checkpoints, the C-ABI layout and the plugin's host-side validation."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, Golden
from oracle import ppo_oracle as O
import obs_indices_oracle as X


@pytest.fixture(scope="module")
def g():
    return Golden("obs_indices")


def _t(d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in d.items()}


def _idx(g):
    return g["policy_idx"], g["critic_idx"]


def _ref_checkpoint():
    """best.model written by the reference's own save() at the end of the golden run (make_golden_ppo_obs_indices.py)."""
    return torch.load(os.path.join(GOLDEN_DIR, "ppo_obs_indices_ref_checkpoint.model"), weights_only=False)


# parameter numbering of the reference's optimisers (torch.optim.Adam(module.parameters()), ppo.py:83-84)
_REF_ORDER = {"policy": ("policy_logstd", "policy_mean.0.weight", "policy_mean.0.bias", "policy_mean.2.weight", "policy_mean.2.bias",
                         "policy_mean.4.weight", "policy_mean.4.bias"),
              "critic": ("critic.0.weight", "critic.0.bias", "critic.2.weight", "critic.2.bias", "critic.4.weight", "critic.4.bias")}


def test_golden_index_sets_are_asymmetric(g):
    p, c = _idx(g)
    assert (len(p), len(c), g.obs) == (23, 33, 40)
    assert len(set(p)) == len(p) and len(set(c)) == len(c)
    assert not np.array_equal(p, np.sort(p)) and not np.array_equal(c, np.sort(c))  # permuted, not just subsets
    assert set(p) & set(c) and set(c) - set(p)                                       # overlap + privileged critic columns
    pol, cri = g.params("init")
    assert pol["policy_mean.0.weight"].shape == (g.hidden, 23) and cri["critic.0.weight"].shape == (g.hidden, 33)


def test_oracle_gae_values_and_log_probs_match_reference(g):
    pidx, cidx = _idx(g)
    for it in range(g.iterations):
        pol, cri = g.params("init" if it == 0 else f"iter{it - 1}")
        with torch.no_grad():
            nv_oracle = X.critic_value(_t(cri), torch.from_numpy(g[f"iter{it}/next_states"]), cidx).squeeze(-1)
            states = torch.from_numpy(g[f"iter{it}/states"]).reshape(-1, g.obs)
            logp, _ = X.get_logprob_entropy(_t(pol), states, torch.from_numpy(g[f"iter{it}/actions"]).reshape(-1, g.act), pidx)
            v = X.critic_value(_t(cri), states, cidx).reshape(-1)
        nv = torch.from_numpy(g[f"iter{it}/next_values"])
        np.testing.assert_allclose(nv_oracle.numpy(), nv.numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(logp.numpy(), g[f"iter{it}/log_probs"].reshape(-1), rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(v.numpy(), g[f"iter{it}/values"].reshape(-1), rtol=1e-5, atol=2e-6)
        adv, ret = O.gae(torch.from_numpy(g[f"iter{it}/rewards"]), torch.from_numpy(g[f"iter{it}/terminations"]),
                         torch.from_numpy(g[f"iter{it}/values"]), nv, g.gamma, g.gae_lambda)
        assert np.array_equal(adv.numpy(), g[f"iter{it}/advantages"]) and np.array_equal(ret.numpy(), g[f"iter{it}/returns"])


def test_shuffle_stream_is_unchanged_by_index_sets(g):
    rng, k = O.Pcg64Py(g.seed), 0
    for it in range(g.iterations):
        idx = list(range(g.B))
        for _ in range(g.epochs):
            O.pcg64_shuffle_py(rng, idx)
            assert idx == g[f"perm/{k}"].tolist()
            k += 1


def test_oracle_update_matches_reference(g):
    pidx, cidx = _idx(g)
    pol, cri = g.params("init")
    L = X.Learner(_t(pol), _t(cri), pidx, cidx, lr=g.lr, clip_range=g.clip_range, entropy_coef=g.entropy_coef, critic_coef=g.critic_coef,
                  max_grad_norm=g.max_grad_norm)
    torch.set_num_threads(1)
    for it in range(g.iterations):
        L.set_lr(g.lr_at(it))
        batch = {k: torch.from_numpy(g[f"iter{it}/{k}"]) for k in ["states", "actions", "log_probs", "advantages", "returns"]}
        metrics = L.update(O.flatten(batch), g.perms(it), g.mb)
        pol_ref, cri_ref = g.params(f"iter{it}")
        for k, v in {**pol_ref, **cri_ref}.items():
            ours = (L.pol if k in pol_ref else L.cri)[k].detach().numpy()
            np.testing.assert_allclose(ours, v, rtol=1e-5, atol=1e-7, err_msg=k)
        for name, key in [("loss/policy_gradient_loss", "pg_loss"), ("loss/critic_loss", "critic_loss"), ("policy_ratio/approx_kl", "approx_kl"),
                          ("policy_ratio/clip_fraction", "clip_fraction"), ("gradients/policy_grad_norm", "policy_grad_norm"),
                          ("gradients/critic_grad_norm", "critic_grad_norm"), ("loss/entropy_loss", "entropy_loss")]:
            vals = [m[key] for m in metrics]
            if key == "approx_kl":
                vals = vals[-(-(-g.B // g.mb)):]
            ours, ref = float(np.mean(vals)), float(g[f"metric/{name}"][it])
            assert abs(ours - ref) <= 1e-5 * max(1.0, abs(ref)), (name, ours, ref)
    # both Adam states after the run: the reference's own best.model of the same run holds them (its optimisers number the parameters in
    # module.parameters() order: policy_logstd first)
    ck = _ref_checkpoint()
    for opt, keys, tag in ((L.popt, O.POLICY_KEYS, "policy"), (L.copt, O.CRITIC_KEYS, "critic")):
        st, ref = opt.state_dict()["state"], ck[f"{tag}_optimizer_state_dict"]["state"]
        for i, k in enumerate(keys):
            j = _REF_ORDER[tag].index(k)
            np.testing.assert_allclose(st[i]["exp_avg"].numpy(), ref[j]["exp_avg"].numpy(), rtol=1e-4, atol=1e-9, err_msg=k)
            np.testing.assert_allclose(st[i]["exp_avg_sq"].numpy(), ref[j]["exp_avg_sq"].numpy(), rtol=1e-4, atol=1e-12, err_msg=k)


def test_espo_oracle_with_index_sets_is_the_espo_oracle_on_selected_columns(g):
    """ESPO's networks are PPO's (espo.py:84-92): with index sets its update equals the unchanged ESPO oracle run on explicitly
    index-selected copies of the states - the policy on states[:, policy_idx], the critic on states[:, critic_idx]."""
    from oracle import espo_oracle as E
    pidx, cidx = _idx(g)
    pol, cri = g.params("init")
    batch = O.flatten({k: torch.from_numpy(g[f"iter0/{k}"]) for k in ["states", "actions", "log_probs", "advantages", "returns"]})
    torch.set_num_threads(1)
    kw = dict(lr=g.lr, entropy_coef=g.entropy_coef, critic_coef=g.critic_coef, max_grad_norm=g.max_grad_norm, max_ratio_delta=1e9)
    ours = X.EspoLearner(_t(pol), _t(cri), pidx, cidx, **kw)
    rng = np.random.default_rng(7)
    draws = [rng.choice(g.B, size=g.mb, replace=False) for _ in range(3)]
    it = iter(draws)
    m_ours = ours.update(batch, lambda: next(it), 3)
    # the same draws through two plain ESPO learners, each fed explicitly index-selected states: one whose policy reads
    # states[:, policy_idx], one whose critic reads states[:, critic_idx] (the other net of each is a stand-in of the right width)
    H = g.hidden
    pol_learner = E.Learner(_t(pol), {**_t(cri), "critic.0.weight": torch.zeros(H, len(pidx))}, **kw)
    cri_learner = E.Learner({**_t(pol), "policy_mean.0.weight": torch.zeros(H, len(cidx))}, _t(cri), **kw)
    for learner, cols in ((pol_learner, pidx), (cri_learner, cidx)):
        it = iter(draws)
        learner.update({**batch, "states": batch["states"][:, torch.as_tensor(cols)]}, lambda: next(it), 3)
    for k in O.POLICY_KEYS:
        assert torch.equal(ours.pol[k], pol_learner.pol[k]), k
    for k in O.CRITIC_KEYS:
        assert torch.equal(ours.cri[k], cri_learner.cri[k]), k
    assert len(m_ours) == 3


def test_init_reference_parameters_equal_the_reference_initial_weights(g):
    from rl_x_b200.algorithms.ppo.b200.ppo import init_reference_parameters
    pidx, cidx = _idx(g)
    ours = init_reference_parameters(g.obs, g.act, g.hidden, g.std_dev, g.seed, len(pidx), len(cidx))
    pol, cri = g.params("init")
    for k, v in {**pol, **cri}.items():
        assert np.array_equal(ours[k].numpy(), v), k
    # identity sets (None) keep today's shapes and values
    base = init_reference_parameters(g.obs, g.act, g.hidden, g.std_dev, g.seed)
    same = init_reference_parameters(g.obs, g.act, g.hidden, g.std_dev, g.seed, g.obs, g.obs)
    assert all(torch.equal(base[k], same[k]) for k in base) and base["critic.0.weight"].shape == (g.hidden, g.obs)


# ------------------------------------------------------------------------------------------------ flat layout / checkpoints
class _HostLayout:
    """The parts of PpoKernels that FlatParameters uses, from the library's layout query (which reads no index values)."""

    def __init__(self, obs, act, hidden, pidx, cidx):
        from rl_x_b200 import _native as nt
        self._keep = [np.ascontiguousarray(pidx, np.int32), np.ascontiguousarray(cidx, np.int32)]
        d = nt.PpoDims(obs, act, hidden, len(pidx), len(cidx), self._keep[0].ctypes.data, self._keep[1].ctypes.data)
        self.obs_dim, self.act_dim, self.hidden, self.policy_in_dim, self.critic_in_dim = obs, act, hidden, len(pidx), len(cidx)
        self.param_count = int(nt.load().rlx_ppo_param_count(C.byref(d)))
        self.offsets, self.is_critic = nt.ppo_layout(obs, act, hidden, d)

    def segment_shapes(self):
        from rl_x_b200 import _native as nt
        return nt.segment_shapes(self.obs_dim, self.act_dim, self.hidden, self.policy_in_dim, self.critic_in_dim)


def test_layout_carries_the_reference_parameter_shapes(g):
    from rl_x_b200 import _native as nt
    pidx, cidx = _idx(g)
    k = _HostLayout(g.obs, g.act, g.hidden, pidx, cidx)
    H, A = g.hidden, g.act
    assert k.param_count == H * 23 + H * 33 + 2 * H + 2 * H * H + 2 * H + A * H + H + A + 1 + A
    sizes = np.diff(k.offsets)
    assert sizes[0] == H * 23 and sizes[1] == H * 33 and list(k.is_critic) == [0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0]
    ident = nt.ppo_layout(g.obs, A, H)[0]
    assert np.array_equal(np.diff(ident)[2:], sizes[2:])  # everything after layer 1 is today's layout


def test_c_abi_refuses_inconsistent_index_fields():
    from rl_x_b200 import _native as nt
    lib = nt.load()
    idx = np.arange(5, dtype=np.int32)
    cases = [((40, 4, 64, 0, 0, idx.ctypes.data, None), "policy_in_dim must be in"),
             ((40, 4, 64, 41, 0, idx.ctypes.data, None), "policy_in_dim must be in"),
             ((40, 4, 64, 0, 39, None, None), "critic_in_dim must be 0 or obs_dim"),
             ((40, 4, 64, 0, -1, None, idx.ctypes.data), "critic_in_dim must be in")]
    for args, msg in cases:
        d = nt.PpoDims(*args)
        assert lib.rlx_ppo_param_count(C.byref(d)) < 0
        assert msg in nt.last_error(), nt.last_error()
    for ok in [(40, 4, 64), (40, 4, 64, 40, 40, None, None), (40, 4, 64, 5, 40, idx.ctypes.data, None)]:
        assert lib.rlx_ppo_param_count(C.byref(nt.PpoDims(*ok))) > 0


def test_state_dicts_load_strictly_into_the_reference_modules(g):
    """Built from the flat buffer, the state dicts and Adam states load (strict load_state_dict, optimizer.load_state_dict, as the reference's
    load() does, ppo.py:447-450) into the reference's own PPO (staged in oracle/_ref) built for an env with these index sets, and its
    ContinuousFlatValuesPolicy / FlatValuesCritic then compute what the oracle computes."""
    from oracle import make_ref
    if not make_ref.available():
        pytest.skip("oracle/_ref not staged (python oracle/make_ref.py)")
    from oracle import ref_arm
    from rl_x_b200 import _native as nt
    from rl_x_b200.algorithms.ppo.b200.ppo import CRITIC_PARAM_ORDER, POLICY_PARAM_ORDER, FlatParameters
    os.environ["TORCHDYNAMO_DISABLE"] = "1"
    refppo = ref_arm.import_reference()
    from rl_x.algorithms.ppo.pytorch.default_config import get_config
    pidx, cidx = _idx(g)
    k = _HostLayout(g.obs, g.act, g.hidden, pidx, cidx)
    fp = FlatParameters(k, "cpu")
    pol, cri = g.params(f"iter{g.iterations - 1}")
    fp.load_named({**pol, **cri})
    gen = torch.Generator().manual_seed(0)
    m1, m2 = torch.randn(k.param_count, generator=gen), torch.rand(k.param_count, generator=gen)
    a = get_config("ppo.pytorch")
    a.device, a.bf16_mixed_precision_training, a.nr_steps, a.nr_epochs, a.minibatch_size, a.nr_hidden_units = "cpu", False, g.T, g.epochs, g.mb, g.hidden
    cfg = ref_arm._ConfigDict(algorithm=a, environment=ref_arm._ConfigDict(seed=0, nr_envs=g.N),
                              runner=ref_arm._ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False))
    env = ref_arm.SyntheticTorchEnv(g.N, g.obs, g.act)
    env.policy_observation_indices, env.critic_observation_indices = pidx, cidx
    model = refppo.PPO(cfg, env, env, "/tmp/rlx_obs_indices_interop", None)
    p_sd, c_sd = fp.state_dicts()
    model.policy.load_state_dict(p_sd, strict=True)
    model.critic.load_state_dict(c_sd, strict=True)
    model.policy_optimizer.load_state_dict(fp.adam_state_dict(POLICY_PARAM_ORDER, nt.POLICY_KEYS, m1, m2, 5, 3e-4))
    model.critic_optimizer.load_state_dict(fp.adam_state_dict(CRITIC_PARAM_ORDER, nt.CRITIC_KEYS, m1, m2, 5, 3e-4))
    for net, opt, keys in ((model.policy, model.policy_optimizer, nt.POLICY_KEYS), (model.critic, model.critic_optimizer, nt.CRITIC_KEYS)):
        for name, p in net.named_parameters():
            seg = keys[name.replace("_orig_mod.", "")]
            assert torch.equal(opt.state[p]["exp_avg"], fp.view(m1, seg)), name
    x = torch.from_numpy(g[f"iter{g.iterations - 1}/states"][0])
    with torch.no_grad():
        assert torch.equal(model.critic.get_value(x), X.critic_value(_t(cri), x, cidx))
        assert torch.equal(model.policy.get_deterministic_action(x), X.get_deterministic_action(
            _t(pol), x, torch.as_tensor(env.single_action_space.low), torch.as_tensor(env.single_action_space.high), True, pidx))


def test_reference_checkpoint_maps_onto_the_flat_layout(g):
    """best.model written by the reference's own save() at the end of the golden run: [H, P] / [H, C] first layers, Adam states numbered
    as the reference's optimisers number them (policy_logstd first); save-side dicts reproduce the file."""
    from rl_x_b200 import _native as nt
    from rl_x_b200.algorithms.ppo.b200.ppo import CRITIC_PARAM_ORDER, POLICY_PARAM_ORDER, FlatParameters
    ck = _ref_checkpoint()
    pidx, cidx = _idx(g)
    k = _HostLayout(g.obs, g.act, g.hidden, pidx, cidx)
    fp = FlatParameters(k, "cpu")
    m, v = torch.zeros(k.param_count), torch.zeros(k.param_count)
    fp.load_named({**ck["policy_state_dict"], **ck["critic_state_dict"]})
    sp = fp.load_adam_state(ck["policy_optimizer_state_dict"], POLICY_PARAM_ORDER, nt.POLICY_KEYS, m, v)
    sc = fp.load_adam_state(ck["critic_optimizer_state_dict"], CRITIC_PARAM_ORDER, nt.CRITIC_KEYS, m, v)
    assert sp == sc == g.iterations * g.epochs * (g.B // g.mb)
    assert tuple(ck["policy_optimizer_state_dict"]["state"][0]["exp_avg"].shape) == (1, g.act)  # policy_logstd is parameter 0
    assert fp.view(fp.flat, "W1p").shape == (g.hidden, 23) and fp.view(fp.flat, "W1c").shape == (g.hidden, 33)
    last = f"iter{g.iterations - 1}"
    pol, cri = g.params(last)
    for key, seg in {**nt.POLICY_KEYS, **nt.CRITIC_KEYS}.items():
        ref = pol[key] if key in pol else cri[key]
        assert np.array_equal(fp.view(fp.flat, seg).numpy(), ref), key
        tag = "policy" if key in pol else "critic"
        st = ck[f"{tag}_optimizer_state_dict"]["state"][_REF_ORDER[tag].index(key)]
        assert torch.equal(fp.view(m, seg), st["exp_avg"]) and torch.equal(fp.view(v, seg), st["exp_avg_sq"]), key
    p_sd, c_sd = fp.state_dicts()
    for key, t in {**p_sd, **c_sd}.items():
        src = ck["policy_state_dict"] if key in ck["policy_state_dict"] else ck["critic_state_dict"]
        assert torch.equal(t, src[key]), key
    popt = fp.adam_state_dict(POLICY_PARAM_ORDER, nt.POLICY_KEYS, m, v, sp, 3e-4)
    for i in ck["policy_optimizer_state_dict"]["state"]:
        assert torch.equal(popt["state"][i]["exp_avg_sq"], ck["policy_optimizer_state_dict"]["state"][i]["exp_avg_sq"]), i


# ------------------------------------------------------------------------------------------------------- plugin validation
BAD_SETS = [
    ("out of range", lambda obs: np.array([0, 1, obs])),
    ("negative", lambda obs: np.array([0, -1, 2])),
    ("duplicate", lambda obs: np.array([0, 3, 3])),
    ("empty", lambda obs: np.array([], dtype=np.int64)),
    ("2-D", lambda obs: np.arange(4).reshape(2, 2)),
    ("float dtype", lambda obs: np.array([0.0, 1.0, 2.0])),
]


@pytest.mark.parametrize("algo", ["ppo.b200", "espo.b200"])
@pytest.mark.parametrize("attr", ["policy_observation_indices", "critic_observation_indices"])
@pytest.mark.parametrize("case", [c[0] for c in BAD_SETS])
def test_bad_index_sets_are_refused_before_any_device_work(algo, attr, case, monkeypatch):
    from rl_x_b200.algorithms.algorithm_manager import get_algorithm_model_class
    from rl_x_b200.runner.runner import Runner
    import rl_x_b200.algorithms.ppo.b200.ppo as ppo_mod
    r = Runner(argv=[f"--algorithm.name={algo}", "--environment.nr_envs=8"])
    env, eval_env = r._create_train_and_eval_env(r._config)
    obs = env.single_observation_space.shape[0]
    setattr(env, attr, dict(BAD_SETS)[case](obs))

    def no_device(*a, **k):
        raise AssertionError("device work before the index sets were validated")
    monkeypatch.setattr(ppo_mod, "PpoKernels", no_device)
    monkeypatch.setattr(torch.cuda, "current_device", no_device)
    with pytest.raises(ValueError, match=attr):
        get_algorithm_model_class(algo)(r._config, env, eval_env, "/tmp/x", None)


def test_valid_index_sets_pass_validation_and_identity_means_none():
    from rl_x_b200 import _native as nt
    assert nt.observation_indices("p", None, 10) is None
    assert nt.observation_indices("p", np.arange(10), 10) is None
    assert nt.observation_indices("p", list(range(10)), 10) is None
    assert nt.observation_indices("p", torch.arange(10), 10) is None
    assert np.array_equal(nt.observation_indices("p", torch.tensor([3, 1, 2]), 10), [3, 1, 2])
    assert np.array_equal(nt.observation_indices("p", np.arange(10)[::-1], 10), np.arange(10)[::-1])  # a permutation is not the identity
    assert nt.observation_indices("p", np.array([4], dtype=np.int32), 10).dtype == np.int64
