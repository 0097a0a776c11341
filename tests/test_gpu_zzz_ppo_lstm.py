"""PPO+LSTM path on the GPU (rl_x_b200/csrc/lstm.cu through librlx_b200.so) against oracle/ppo_lstm_oracle.py.

The same sources are validated in host emulation (tests/test_lstm_emulation.py), including the FiLM / shared-encoder options and the
one-launch-per-step recurrence."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import ppo_lstm_oracle as L
from test_lstm_emulation import CRITIC_SEGS, POLICY_SEGS, flatten_critic, flatten_policy

pytestmark = pytest.mark.gpu
DEV = "cuda"


OPT_FILM, OPT_SHARED = 1, 2   # RLX_LSTM_OPT_*


def _perturbed(obs, act, hid, enc, lstm, seed, options=0):
    pol, cri = L.init_params(obs, act, hidden=hid, enc=enc, lstm=lstm, std_dev=0.8, seed=seed, share_encoder=bool(options & OPT_SHARED),
                             combine="film" if options & OPT_FILM else "concat")
    for tree in (pol, cri):
        for name, v in L.tree_leaves(tree):
            if name.endswith("bias") or name.endswith("scale"):
                v.add_(0.1 * torch.randn_like(v))
    return pol, cri


# last case: BASELINE.json configs[4] shapes — obs 64, act 8, seq_len 128, one minibatch of 32768 rows = 256 envs, reference widths
# (ppo_lstm/flax/default_config.py: lstm_hidden_dim 64, obs_encoding_dim 128, nr_hidden_units 256)
@pytest.mark.parametrize("T,n,obs,act,hid,enc,lstm,options", [
    (7, 5, 6, 2, 12, 8, 4, 0), (33, 40, 5, 2, 8, 8, 4, 0), (16, 24, 64, 8, 256, 128, 64, 0), (128, 256, 64, 8, 256, 128, 64, 0),
    # lstm_obs_combine_method = "film" / share_lstm_obs_encoder (policy.py:51-59, 99-125)
    (7, 5, 6, 2, 12, 8, 4, OPT_FILM), (7, 5, 6, 2, 12, 8, 4, OPT_SHARED), (33, 40, 5, 2, 8, 8, 4, OPT_FILM | OPT_SHARED),
    (16, 24, 64, 8, 256, 128, 64, OPT_FILM), (16, 24, 64, 8, 256, 128, 64, OPT_FILM | OPT_SHARED)])
def test_lstm_fwdbwd_matches_oracle_autograd(T, n, obs, act, hid, enc, lstm, options):
    from rl_x_b200 import _native as nt
    lib = nt.load()
    torch.manual_seed(T * 100 + n)
    pol, cri = _perturbed(obs, act, hid, enc, lstm, T, options)
    states, actions = torch.randn(T, n, obs), torch.randn(T, n, act)
    log_probs, adv, ret = torch.randn(T, n) * 0.1 - 2.5, torch.randn(T, n), torch.randn(T, n)
    dones = (torch.rand(T, n) < 0.2).float()
    init = (torch.randn(n, lstm) * 0.5, torch.randn(n, lstm) * 0.5)
    clip, ent, cc = 0.2, 0.01, 0.5
    learner = L.Learner(pol, cri, clip_range=clip, entropy_coef=ent, critic_coef=cc)
    gp_ref, gc_ref, metrics_ref = learner.grads(dict(states=states, actions=actions, log_probs=log_probs, returns=ret, advantages=adv, dones=dones,
                                                     init_carry=init))
    gp_tree = dict(zip([nm for nm, _ in L.tree_leaves(learner.pol)], gp_ref))
    gc_tree = dict(zip([nm for nm, _ in L.tree_leaves(learner.cri)], gc_ref))

    def grad_seg(name):
        if name in ("Wi", "Wh"):
            return torch.cat([gp_tree[f"lstm.{name[1].lower()}{k}.kernel"] for k in L.GATES], dim=1)
        if name == "bh":
            return torch.cat([gp_tree[f"lstm.h{k}.bias"] for k in L.GATES])
        if name in ("Wf", "bf"):
            leaf = "kernel" if name == "Wf" else "bias"
            return (torch.cat([gp_tree[f"lstm_film_gamma.{leaf}"], gp_tree[f"lstm_film_beta.{leaf}"]], dim=-1) if options & OPT_FILM
                    else torch.zeros(0))
        return gp_tree.get(name, torch.zeros(0))   # obs_encoder.* are absent with a shared encoder

    d = nt.LstmDims(obs, act, hid, enc, lstm, options)
    P = torch.cat(flatten_policy(pol)).to(DEV)
    Cc = torch.cat(flatten_critic(cri)).to(DEV)
    poff, coff = (C.c_int64 * (nt.RLX_LSTM_POLICY_NSEG + 1))(), (C.c_int64 * (nt.RLX_LSTM_CRITIC_NSEG + 1))()
    nt.check(lib.rlx_lstm_param_layout(C.byref(d), poff, coff), "layout")
    gP, gC = torch.full_like(P, float("nan")), torch.full_like(Cc, float("nan"))
    stats = torch.tensor([float(adv.mean()), float(adv.std(unbiased=False))], device=DEV)
    metrics = torch.zeros(8, device=DEV)
    nbytes = lib.rlx_lstm_minibatch_workspace_bytes(C.byref(d), T, n)
    ws = torch.zeros(nbytes // 4 + 64, device=DEV)
    dev = {k: v.contiguous().to(DEV) for k, v in dict(states=states, actions=actions, log_probs=log_probs, advantages=adv, returns=ret, dones=dones,
                                                      init_c=init[0], init_h=init[1]).items()}
    a = nt.LstmMinibatchArgs()
    a.dims, a.T, a.n_env = d, T, n
    for k, v in dev.items():
        setattr(a, k, v.data_ptr())
    a.adv_stats, a.policy_params, a.critic_params = stats.data_ptr(), P.data_ptr(), Cc.data_ptr()
    a.policy_grads, a.critic_grads, a.metrics = gP.data_ptr(), gC.data_ptr(), metrics.data_ptr()
    a.clip_range, a.entropy_coef, a.critic_coef = clip, ent, cc
    a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    nt.check(lib.rlx_lstm_ppo_minibatch_fwdbwd_f32(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "fwdbwd")
    gP, gC, metrics = gP.cpu().numpy(), gC.cpu().numpy(), metrics.cpu().numpy()
    assert np.isfinite(gP).all() and np.isfinite(gC).all()
    scale = max(max(float(grad_seg(nm).abs().max()) for nm in POLICY_SEGS if grad_seg(nm).numel()), 1.0)
    for i, name in enumerate(POLICY_SEGS):
        np.testing.assert_allclose(gP[poff[i]:poff[i + 1]], grad_seg(name).numpy().reshape(-1), rtol=3e-4, atol=3e-6 * scale, err_msg=name)
    for i, name in enumerate(CRITIC_SEGS):
        np.testing.assert_allclose(gC[coff[i]:coff[i + 1]], gc_tree[name].numpy().reshape(-1), rtol=3e-4, atol=3e-6, err_msg=name)
    for j, key in enumerate(["loss/policy_gradient_loss", "loss/critic_loss", "loss/entropy_loss", "policy_ratio/approx_kl", "policy_ratio/clip_fraction"]):
        assert abs(float(metrics[j]) - metrics_ref[key]) <= 3e-5 * max(1.0, abs(metrics_ref[key])), key


def _plugin_run(combine="concat", share=False, graph=False, iterations=2):
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.ppo_lstm.b200.default_config import get_config
    from rl_x_b200.algorithms.ppo_lstm.b200.ppo_lstm import PPO_LSTM
    from rl_x_b200.environments.synthetic.box.create_env import create_train_and_eval_env
    from rl_x_b200.environments.synthetic.box.default_config import get_config as env_config
    N, T = 16, 8
    e = env_config("synthetic.box")
    e.nr_envs, e.obs_dim, e.act_dim, e.seed = N, 12, 3, 7
    a = get_config("ppo_lstm.b200")
    a.nr_steps, a.minibatch_size, a.nr_epochs, a.total_timesteps = T, 4 * T, 2, iterations * N * T
    a.nr_hidden_units, a.obs_encoding_dim, a.lstm_hidden_dim, a.learning_rate = 32, 16, 8, 1e-3
    a.lstm_obs_combine_method, a.share_lstm_obs_encoder, a.use_cuda_graph = combine, share, graph
    cfg = ConfigDict(algorithm=a, environment=e, runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    env, _ = create_train_and_eval_env(cfg)
    model = PPO_LSTM(cfg, env, env, "/tmp/rlx_test_lstm_opts", None)
    logged = []
    model.log = lambda name, value, step: logged.append((name, float(value)))
    model.train()
    torch.cuda.synchronize()
    return model, logged


@pytest.mark.parametrize("combine,share", [("film", False), ("concat", True), ("film", True)])
def test_lstm_plugin_options_train(combine, share):
    """lstm_obs_combine_method / share_lstm_obs_encoder through the plugin: finite metrics, every live parameter segment moves, the segments
    the option removes are empty."""
    model, logged = _plugin_run(combine, share)
    assert all(np.isfinite(v) for n_, v in logged if not n_.startswith("time/"))
    pol, _ = model.named_parameters()
    assert pol["Wf"].numel() == (8 * 2 * 16 if combine == "film" else 0) and pol["We2"].numel() == (0 if share else 12 * 16)
    fresh, _ = _plugin_run(combine, share, iterations=0)
    pol0, _ = fresh.named_parameters()
    for name in ("We1", "Wi", "Wh", "Wt1", "Wm") + (("Wf",) if combine == "film" else ()) + (() if share else ("We2",)):
        assert float((pol[name] - pol0[name]).abs().max()) > 1e-6, name


def test_lstm_plugin_cuda_graph_replay_equals_eager_launches():
    """use_cuda_graph replays each minibatch update as one captured graph: same kernels in the same order on the same buffers, no atomics,
    so three iterations leave bit-identical weights, Adam moments and logged metrics."""
    eager, log_e = _plugin_run(graph=False, iterations=3)
    replay, log_r = _plugin_run(graph=True, iterations=3)
    assert replay._graph is not None and eager._graph is None
    for name in ("policy_params", "critic_params", "policy_mu", "policy_nu", "critic_mu", "critic_nu"):
        assert torch.equal(getattr(eager, name), getattr(replay, name)), name
    keep = lambda log: [(n_, v) for n_, v in log if n_.split("/")[0] in ("loss", "gradients", "policy_ratio", "lr")]
    assert keep(log_e) == keep(log_r)


def test_lstm_suite_in_a_subprocess_with_dense_layers_on_the_tensor_engine(tmp_path):
    """rlx_set_aux_gemm_engine(1): every dense layer of the update with at least half a tile per output dimension runs on the wgmma 3xTF32
    engine (forward and input-gradient products on K-major copies of the kernels), the heads stay on the SIMT engine.  The whole file -
    oracle parity at the config-5 shape included - must pass that way, and must actually have used the tensor engine."""
    from conftest import run_suite_with_switches
    rc, tail, tc, _ = run_suite_with_switches(__file__, tmp_path, tensor_engine=True)
    assert rc == 0, tail
    assert tc > 0, f"the tensor engine was never used ({tc})"


def test_lstm_suite_in_a_subprocess_with_the_one_launch_recurrence(tmp_path):
    """rlx_set_lstm_persistent(1): the recurrence of every update as ONE block-cooperative launch per direction (recurrent kernel in shared
    memory, a barrier per step).  Bit-identical to the per-step path in emulation (and race-free under ThreadSanitizer); on the device the
    whole file must pass that way and the path must have run."""
    from conftest import run_suite_with_switches
    rc, tail, _, pers = run_suite_with_switches(__file__, tmp_path, persistent=True)
    assert rc == 0, tail
    assert pers > 0, f"the one-launch recurrence never ran ({pers})"


@pytest.mark.skipif(os.environ.get("RLX_LSTM_PERSISTENT") != "1", reason="runs inside the one-launch-recurrence subprocess (previous test)")
def test_lstm_one_launch_recurrence_equals_per_step_recurrence_bit_for_bit():
    """Same arithmetic in the same order: gradients and metrics of one update at the config-5 widths (lstm 64: the recurrent kernel takes
    64 KB of shared memory) must not differ in a single bit between the two recurrence paths."""
    from rl_x_b200 import _native as nt
    lib = nt.load()
    T, n, obs, act, hid, enc, lstm = 32, 50, 64, 8, 256, 128, 64     # 50 envs: the last block has inactive threads
    torch.manual_seed(3)
    pol, cri = _perturbed(obs, act, hid, enc, lstm, 5)
    d = nt.LstmDims(obs, act, hid, enc, lstm, 0)
    P, Cc = torch.cat(flatten_policy(pol)).to(DEV), torch.cat(flatten_critic(cri)).to(DEV)
    adv = torch.randn(T, n)
    dev = {k: v.contiguous().to(DEV) for k, v in dict(
        states=torch.randn(T, n, obs), actions=torch.randn(T, n, act), log_probs=torch.randn(T, n) * 0.1 - 2.5, advantages=adv, returns=torch.randn(T, n),
        dones=(torch.rand(T, n) < 0.2).float(), init_c=torch.randn(n, lstm) * 0.5, init_h=torch.randn(n, lstm) * 0.5).items()}
    stats = torch.tensor([float(adv.mean()), float(adv.std(unbiased=False))], device=DEV)
    nbytes = lib.rlx_lstm_minibatch_workspace_bytes(C.byref(d), T, n)
    out = {}
    for persistent in (0, 1):
        assert lib.rlx_set_lstm_persistent(persistent) == persistent
        before = int(lib.rlx_lstm_persistent_launch_count())
        gP, gC, metrics = torch.full_like(P, float("nan")), torch.full_like(Cc, float("nan")), torch.zeros(8, device=DEV)
        ws = torch.full((nbytes // 4 + 64,), float("nan"), device=DEV)
        a = nt.LstmMinibatchArgs()
        a.dims, a.T, a.n_env = d, T, n
        for k, v in dev.items():
            setattr(a, k, v.data_ptr())
        a.adv_stats, a.policy_params, a.critic_params = stats.data_ptr(), P.data_ptr(), Cc.data_ptr()
        a.policy_grads, a.critic_grads, a.metrics = gP.data_ptr(), gC.data_ptr(), metrics.data_ptr()
        a.clip_range, a.entropy_coef, a.critic_coef = 0.2, 0.01, 0.5
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        nt.check(lib.rlx_lstm_ppo_minibatch_fwdbwd_f32(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "fwdbwd")
        torch.cuda.synchronize()
        out[persistent] = (gP.cpu(), gC.cpu(), metrics.cpu(), int(lib.rlx_lstm_persistent_launch_count()) - before)
    lib.rlx_set_lstm_persistent(1)   # the subprocess's setting
    assert out[0][3] == 0 and out[1][3] == 2
    assert torch.isfinite(out[1][0]).all() and all(torch.equal(x, y) for x, y in zip(out[0][:3], out[1][:3]))


def test_lstm_plugin_trains_on_synthetic_env():
    """PPO_LSTM.train() through the plugin surface: two iterations on the synthetic Box env, finite metrics, parameters move, the rollout
    step agrees with the oracle's get_action_and_value on the trained weights."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.ppo_lstm.b200.default_config import get_config
    from rl_x_b200.algorithms.ppo_lstm.b200.ppo_lstm import PPO_LSTM
    from test_gpu_train import _Space, _props
    N, T, obs, act = 8, 16, 12, 3

    class Env:
        general_properties = _props("TORCH")
        single_observation_space = _Space((obs,))
        single_action_space = _Space((act,), np.full(act, -1.0, np.float32), np.full(act, 1.0, np.float32))
        gen = torch.Generator(device=DEV).manual_seed(3)

        def reset(self):
            return torch.randn(N, obs, device=DEV, generator=self.gen), {}

        def step(self, action):
            return (torch.randn(N, obs, device=DEV, generator=self.gen), torch.randn(N, device=DEV, generator=self.gen),
                    torch.rand(N, device=DEV, generator=self.gen) < 0.1, torch.zeros(N, dtype=torch.bool, device=DEV), {})

        def get_logging_info_dict(self, info):
            return {}

        def close(self):
            pass

    a = get_config("ppo_lstm.b200")
    a.nr_steps, a.minibatch_size, a.nr_epochs, a.total_timesteps = T, 4 * T, 2, 2 * N * T
    a.nr_hidden_units, a.obs_encoding_dim, a.lstm_hidden_dim, a.learning_rate = 32, 16, 8, 1e-3
    cfg = ConfigDict(algorithm=a, environment=ConfigDict(seed=5, nr_envs=N),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    env = Env()
    model = PPO_LSTM(cfg, env, env, "/tmp/rlx_test_lstm", None)
    before = model.policy_params.clone()
    logged = []
    model.log = lambda name, value, step: logged.append((name, float(value)))
    model.train()
    assert all(np.isfinite(v) for n_, v in logged if not n_.startswith("time/"))
    assert len([1 for n_, _ in logged if n_ == "loss/critic_loss"]) == 2
    assert float((model.policy_params - before).abs().max()) > 1e-5
    # rollout step vs oracle on the trained weights
    pol_named, cri_named = model.named_parameters()
    E, Lh = 16, 8
    p = {k: v.cpu() for k, v in pol_named.items()}
    c = {k: v.cpu() for k, v in cri_named.items()}
    pol = {"lstm_obs_encoder_dense": {"kernel": p["We1"].view(obs, E), "bias": p["be1"]}, "lstm_obs_encoder_ln": {"scale": p["g1"], "bias": p["n1"]},
           "obs_encoder_dense": {"kernel": p["We2"].view(obs, E), "bias": p["be2"]}, "obs_encoder_ln": {"scale": p["g2"], "bias": p["n2"]},
           "lstm": {}, "lstm_ln": {"scale": p["gl"], "bias": p["nl"]},
           "torso_dense1": {"kernel": p["Wt1"].view(E + Lh, 32), "bias": p["bt1"]}, "torso_dense2": {"kernel": p["Wt2"].view(32, 32), "bias": p["bt2"]},
           "mean_head": {"kernel": p["Wm"].view(32, act), "bias": p["bm"]}, "policy_logstd": p["logstd"].view(1, act)}
    Wi, Wh, bh = p["Wi"].view(E, 4 * Lh), p["Wh"].view(Lh, 4 * Lh), p["bh"]
    for j, k in enumerate(L.GATES):
        pol["lstm"]["i" + k] = {"kernel": Wi[:, j * Lh:(j + 1) * Lh]}
        pol["lstm"]["h" + k] = {"kernel": Wh[:, j * Lh:(j + 1) * Lh], "bias": bh[j * Lh:(j + 1) * Lh]}
    cri = {"Dense_0": {"kernel": c["Wc1"].view(obs, 32), "bias": c["bc1"]}, "Dense_1": {"kernel": c["Wc2"].view(32, 32), "bias": c["bc2"]},
           "Dense_2": {"kernel": c["Wc3"].view(32, 1), "bias": c["bc3"]}}
    o, noise = torch.randn(N, obs), torch.randn(N, act)
    carry = (torch.randn(N, Lh) * 0.3, torch.randn(N, Lh) * 0.3)
    with torch.no_grad():
        proc, action, value, logp, nxt = L.get_action_and_value(pol, cri, o, carry, noise, torch.full((act,), -1.0), torch.full((act,), 1.0))
    z = lambda *s: torch.zeros(*s, device=DEV)
    cc_, hh_ = carry[0].to(DEV).contiguous(), carry[1].to(DEV).contiguous()
    out_a, out_e, out_lp, out_v = z(N, act), z(N, act), z(N), z(N)
    model._step(o.to(DEV), cc_, hh_, noise.to(DEV), out_a, out_e, out_lp, out_v)
    np.testing.assert_allclose(out_a.cpu().numpy(), action.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(out_e.cpu().numpy(), proc.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(out_lp.cpu().numpy(), logp.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(out_v.cpu().numpy(), value.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(hh_.cpu().numpy(), nxt[1].numpy(), rtol=1e-4, atol=1e-5)
