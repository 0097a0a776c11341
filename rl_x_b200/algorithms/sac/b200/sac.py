"""SAC with the reference's plugin surface (rl_x/algorithms/sac/pytorch/sac.py), executed by the sm_90a library.

Per environment step the reference does: act -> env.step -> replay add (host numpy) -> sample (2x rng.integers, 5 fancy-index gathers,
5 H2D copies) -> critic_loss_fn -> Polyak loop over parameters -> policy_and_entropy_loss_fn -> 10 .item() syncs (sac.py:180-259).
Here the replay ring lives on the device, the index stream is the same PCG64 stream (bit-exact), the rows are gathered by one kernel,
and target / twin-Q update / Polyak / actor / temperature are ONE native call (rlx_sac_update_f32); metrics stay on the device and are
read back only when the reference would log them (every `logging_frequency` steps).
"""
import ctypes as C
import logging
import os
import time
from collections import deque

import numpy as np
import torch
import torch.nn as nn

from rl_x_b200 import _native as nt
from rl_x_b200.algorithms.sac.b200.general_properties import GeneralProperties
from rl_x_b200.algorithms.sac.b200.replay_buffer import ReplayBuffer
from rl_x_b200.environments.types import DataInterfaceType, require_identity_observation_indices, same_member

rlx_logger = logging.getLogger("rl_x")

POLICY_SEGMENTS = [("torso.0.weight", "H,O"), ("torso.0.bias", "H"), ("torso.2.weight", "H,H"), ("torso.2.bias", "H"), ("mean.weight", "A,H"),
                   ("log_std.weight", "A,H"), ("mean.bias", "A"), ("log_std.bias", "A")]
Q_SEGMENTS = [("critic.0.weight", "H,OA"), ("critic.0.bias", "H"), ("critic.2.weight", "H,H"), ("critic.2.bias", "H"), ("critic.4.weight", "1,H"),
              ("critic.4.bias", "1")]
Q_NETS = ("q1", "q2", "q1_target", "q2_target")
# nn.Module.parameters() order of the reference modules = the numbering inside their torch.optim.Adam state dicts (sac.py:75-77)
POLICY_PARAM_ORDER = ("torso.0.weight", "torso.0.bias", "torso.2.weight", "torso.2.bias", "mean.weight", "mean.bias", "log_std.weight", "log_std.bias")
Q_PARAM_ORDER = tuple(k for k, _ in Q_SEGMENTS)


def _adam_state_dict(views_m, views_v, step, lr):
    """torch.optim.Adam.state_dict() layout over an ordered list of (exp_avg view, exp_avg_sq view) pairs."""
    state = {i: {"step": torch.tensor(float(step)), "exp_avg": m.detach().cpu().clone(), "exp_avg_sq": v.detach().cpu().clone()}
             for i, (m, v) in enumerate(zip(views_m, views_v))}
    group = {"lr": lr, "betas": (0.9, 0.999), "eps": 1e-08, "weight_decay": 0, "amsgrad": False, "maximize": False, "foreach": None,
             "capturable": False, "differentiable": False, "fused": None, "decoupled_weight_decay": False, "params": list(range(len(state)))}
    return {"state": state, "param_groups": [group]}


def checkpoint_dict(config_algorithm, pol, qs, log_alpha, optimizer_views, steps, lr):
    """The reference's `best.model` dictionary (sac.py:381-396) from named tensors: `pol` {key: tensor}, `qs` {net: {key: tensor}} for the four
    Q networks, `optimizer_views` {"policy" | "q" | "entropy": (exp_avg views, exp_avg_sq views)} in the reference's parameter numbering,
    `steps` (policy, q, entropy).  Module state_dicts in parameters() order, the three torch.optim.Adam state dicts, and log_alpha as an
    nn.Parameter like the reference's own entry: its load() assigns it to a registered parameter (sac.py:410), which refuses plain tensors."""
    ov = optimizer_views
    return {"config_algorithm": config_algorithm, "policy_state_dict": {k: pol[k] for k in POLICY_PARAM_ORDER}, "q1_state_dict": qs["q1"],
            "q2_state_dict": qs["q2"], "q1_target_state_dict": qs["q1_target"], "q2_target_state_dict": qs["q2_target"],
            "log_alpha": torch.nn.Parameter(torch.as_tensor(log_alpha).detach().cpu().clone().reshape(1)),
            "policy_optimizer_state_dict": _adam_state_dict(*ov["policy"], steps[0], lr),
            "q_optimizer_state_dict": _adam_state_dict(*ov["q"], steps[1], lr),
            "entropy_optimizer_state_dict": _adam_state_dict(*ov["entropy"], steps[2], lr)}


def _load_adam_state(osd, views_m, views_v, what):
    step = 0
    for i, (m, v) in enumerate(zip(views_m, views_v)):
        if i not in osd["state"]:
            continue
        st = osd["state"][i]
        if tuple(st["exp_avg"].shape) != tuple(m.shape):
            raise ValueError(f"{what} optimizer state {i}: exp_avg has shape {tuple(st['exp_avg'].shape)}, expected {tuple(m.shape)}")
        m.copy_(torch.as_tensor(st["exp_avg"], dtype=torch.float32))
        v.copy_(torch.as_tensor(st["exp_avg_sq"], dtype=torch.float32))
        step = max(step, int(float(st["step"])))
    return step


def _shape(spec, O, A, H):
    d = {"H": H, "O": O, "A": A, "OA": O + A, "1": 1}
    return tuple(d[x] for x in spec.split(","))


def init_reference_parameters(obs_dim, act_dim, hidden, seed):
    """Same RNG stream and construction order as the reference (torch.manual_seed(seed), sac.py:65; Policy then q1, q2, q1_target,
    q2_target with default nn.Linear init, targets then copied from the online nets: policy.py:34-43, critic.py:14-22)."""
    torch.manual_seed(seed)
    pol = {}
    for name, lin in [("torso.0", nn.Linear(obs_dim, hidden)), ("torso.2", nn.Linear(hidden, hidden)), ("mean", nn.Linear(hidden, act_dim)),
                      ("log_std", nn.Linear(hidden, act_dim))]:
        pol[name + ".weight"], pol[name + ".bias"] = lin.weight.detach().clone(), lin.bias.detach().clone()

    def qnet():
        d = {}
        for i, lin in zip((0, 2, 4), (nn.Linear(obs_dim + act_dim, hidden), nn.Linear(hidden, hidden), nn.Linear(hidden, 1))):
            d[f"critic.{i}.weight"], d[f"critic.{i}.bias"] = lin.weight.detach().clone(), lin.bias.detach().clone()
        return d

    q1, q2, _, _ = qnet(), qnet(), qnet(), qnet()
    return pol, q1, q2


class SacKernels:
    def __init__(self, obs_dim, act_dim, hidden, log_std_min, log_std_max):
        self.lib = nt.load()
        self.O, self.A, self.H = int(obs_dim), int(act_dim), int(hidden)
        self.dims = nt.SacDims(self.O, self.A, self.H, float(log_std_min), float(log_std_max))
        self.Pp = int(self.lib.rlx_sac_policy_param_count(self.O, self.A, self.H))
        self.Pq = int(self.lib.rlx_sac_q_param_count(self.O, self.A, self.H))

    def workspace(self, batch, device):
        n = int(self.lib.rlx_sac_workspace_bytes(self.O, self.A, self.H, int(batch)))
        return torch.empty(max(n, 16), dtype=torch.uint8, device=device)

    def policy_views(self, flat):
        out, o = {}, 0
        for key, spec in POLICY_SEGMENTS:
            shp = _shape(spec, self.O, self.A, self.H)
            n = int(np.prod(shp))
            out[key] = flat[o:o + n].view(shp)
            o += n
        assert o == self.Pp
        return out

    def q_views(self, flat):
        out = {}
        for i, net in enumerate(Q_NETS):
            o = i * self.Pq
            d = {}
            for key, spec in Q_SEGMENTS:
                shp = _shape(spec, self.O, self.A, self.H)
                n = int(np.prod(shp))
                d[key] = flat[o:o + n].view(shp)
                o += n
            out[net] = d
        return out

    def act(self, policy, obs, eps, low, high, ws, *, deterministic=False, action_tanh=None, env_action=None, logp=None):
        p = lambda t: t.data_ptr() if t is not None else None
        nt.check(self.lib.rlx_sac_act_f32(C.byref(self.dims), policy.data_ptr(), obs.data_ptr(), p(eps), obs.shape[0], low.data_ptr(), high.data_ptr(),
                                          int(bool(deterministic)), p(action_tanh), p(env_action), p(logp), ws.data_ptr(), ws.numel(),
                                          torch.cuda.current_stream().cuda_stream), "rlx_sac_act_f32")

    def update(self, args):
        nt.check(self.lib.rlx_sac_update_f32(C.byref(args), torch.cuda.current_stream().cuda_stream), "rlx_sac_update_f32")


class SAC:
    def __init__(self, config, train_env, eval_env, run_path, writer):
        self.config = config
        self.train_env, self.eval_env, self.writer = train_env, eval_env, writer
        self.save_model = config.runner.save_model
        self.save_path = os.path.join(run_path, "models")
        self.track_console, self.track_tb, self.track_wandb = config.runner.track_console, config.runner.track_tb, config.runner.track_wandb
        self.seed = config.environment.seed
        a = config.algorithm
        self.total_timesteps, self.nr_envs = a.total_timesteps, config.environment.nr_envs
        self.learning_rate, self.anneal_learning_rate = a.learning_rate, a.anneal_learning_rate
        self.buffer_size, self.learning_starts, self.batch_size = a.buffer_size, a.learning_starts, a.batch_size
        self.tau, self.gamma = a.tau, a.gamma
        self.logging_frequency, self.evaluation_frequency, self.evaluation_episodes = a.logging_frequency, a.evaluation_frequency, a.evaluation_episodes
        if a.get("bf16_mixed_precision_training", False):
            raise ValueError("rl_x_b200 SAC implements the reference's fp32 path; set algorithm.bf16_mixed_precision_training=False.")
        require_identity_observation_indices(self.train_env, "SAC")  # policy.py:13,46 / q_network.py:10,37
        if a.device != "gpu" or not torch.cuda.is_available():
            raise RuntimeError("rl_x_b200 SAC needs a CUDA device (algorithm.device=gpu); there is no CPU fallback.")
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.rng = nt.Pcg64Generator(self.seed)  # np.random.default_rng(self.seed), sac.py:64

        os_shape, as_shape = self.train_env.single_observation_space.shape, self.train_env.single_action_space.shape
        if len(os_shape) != 1 or len(as_shape) != 1:
            raise ValueError("rl_x_b200 SAC supports flat observations and flat continuous actions only.")
        self.os_shape, self.as_shape = tuple(os_shape), tuple(as_shape)
        O, A = int(os_shape[0]), int(as_shape[0])
        self.k = SacKernels(O, A, a.nr_hidden_units, a.log_std_min, a.log_std_max)
        self.k.lib.rlx_set_gemm_engine({"simt": 0, "tcgen05": 1, "auto": 1}[a.get("gemm_engine", "auto")])
        self.env_as_low = np.broadcast_to(np.asarray(torch.as_tensor(self.train_env.single_action_space.low).cpu(), dtype=np.float32).reshape(-1), (A,)).copy()
        self.env_as_high = np.broadcast_to(np.asarray(torch.as_tensor(self.train_env.single_action_space.high).cpu(), dtype=np.float32).reshape(-1), (A,)).copy()
        self.d_low, self.d_high = torch.from_numpy(self.env_as_low).to(self.device), torch.from_numpy(self.env_as_high).to(self.device)
        self.target_entropy = -float(A) if a.target_entropy == "auto" else float(a.target_entropy)  # entropy_coefficient.py:17-21

        z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=self.device)
        self.policy, self.q = z(self.k.Pp), z(4 * self.k.Pq)
        self.log_alpha = z(1)
        pol, q1, q2 = init_reference_parameters(O, A, a.nr_hidden_units, self.seed)
        self.load_named(pol, q1, q2, q1, q2)
        self.g_policy, self.m_policy, self.v_policy = z(self.k.Pp), z(self.k.Pp), z(self.k.Pp)
        self.g_q, self.m_q, self.v_q = z(2 * self.k.Pq), z(2 * self.k.Pq), z(2 * self.k.Pq)
        self.g_la, self.m_la, self.v_la = z(1), z(1), z(1)
        self.lr_dev = torch.full((1,), float(self.learning_rate), dtype=torch.float32, device=self.device)
        self.steps = z(3, torch.int64)
        self.metrics = z(nt.RLX_SAC_NMETRIC)
        self.metric_sums = z(nt.RLX_SAC_NMETRIC)
        self.ws = self.k.workspace(max(self.batch_size, self.nr_envs), self.device)
        self.eps = torch.zeros(2, self.batch_size, A, device=self.device)
        self.is_torch_data_interface = same_member(self.train_env.general_properties.data_interface_type, DataInterfaceType.TORCH)
        self.use_cuda_graph = bool(a.get("use_cuda_graph", True))
        self._graph = None
        self.replay_buffer = None
        if self.save_model:
            os.makedirs(self.save_path)
            self.best_mean_return = -np.inf

    # ------------------------------------------------------------------------------------------------- parameters
    def load_named(self, pol, q1, q2, q1t, q2t):
        strip = lambda d: {k.replace("_orig_mod.", ""): v for k, v in d.items()}
        pv = self.k.policy_views(self.policy)
        for key, v in strip(pol).items():
            pv[key].copy_(torch.as_tensor(v, dtype=torch.float32).reshape(pv[key].shape))
        qv = self.k.q_views(self.q)
        for net, d in zip(Q_NETS, (q1, q2, q1t, q2t)):
            for key, v in strip(d).items():
                qv[net][key].copy_(torch.as_tensor(v, dtype=torch.float32).reshape(qv[net][key].shape))

    def state_dicts(self):
        pol = {k: v.detach().cpu().clone() for k, v in self.k.policy_views(self.policy).items()}
        qs = {net: {k: v.detach().cpu().clone() for k, v in d.items()} for net, d in self.k.q_views(self.q).items()}
        return pol, qs

    # ---------------------------------------------------------------------------------------------------- pieces
    def _draw_eps(self, shape_rows):
        """Standard-normal draws of normal.rsample() (policy.py:56); tests override this to teacher-force the reference's draws."""
        return torch.randn(shape_rows, self.k.A, device=self.device)

    def _update_args(self, batch):
        s, ns, ac, r, t = batch
        a = nt.SacUpdateArgs()
        a.dims, a.batch = self.k.dims, s.shape[0]
        eps_next, eps_cur = self._draw_eps(s.shape[0]), self._draw_eps(s.shape[0])
        self._eps_keep = (eps_next, eps_cur)
        for name, tns in [("policy", self.policy), ("q", self.q), ("log_alpha", self.log_alpha), ("states", s), ("next_states", ns), ("actions", ac),
                          ("rewards", r), ("terminations", t), ("eps_next", eps_next), ("eps_cur", eps_cur), ("act_low", self.d_low), ("act_high", self.d_high),
                          ("g_policy", self.g_policy), ("m_policy", self.m_policy), ("v_policy", self.v_policy), ("g_q", self.g_q), ("m_q", self.m_q),
                          ("v_q", self.v_q), ("g_log_alpha", self.g_la), ("m_log_alpha", self.m_la), ("v_log_alpha", self.v_la), ("lr", self.lr_dev),
                          ("steps", self.steps), ("metrics", self.metrics), ("workspace", self.ws)]:
            setattr(a, name, tns.data_ptr())
        a.gamma, a.tau, a.target_entropy = float(self.gamma), float(self.tau), float(self.target_entropy)
        a.adam_beta1, a.adam_beta2, a.adam_eps = 0.9, 0.999, 1e-8
        a.workspace_bytes = self.ws.numel()
        return a

    def update(self, batch):
        """One optimisation step of the reference loop (sac.py:219-259) on a sampled batch.

        The ~58 kernels of an update (noise draws, fused update, metric accumulation) only touch static buffers, so they are
        captured ONCE into a CUDA graph and replayed per step: the update is launch-latency-bound at batch 4096 (SURVEY §8 a15).
        Eager launches are used when the noise hook is overridden (tests) or `use_cuda_graph` is off."""
        eager = (not self.use_cuda_graph or getattr(self._draw_eps, "__func__", None) is not SAC._draw_eps or self.replay_buffer is None
                 or self.replay_buffer._out is None or batch[0] is not self.replay_buffer._out[0])
        if eager:
            self.k.update(self._update_args(batch))
            self.metric_sums += self.metrics
            return
        if self._graph is None:
            # warm-up on a side stream (first-touch allocations, cudaFuncSetAttribute, TMA descriptor encoding), then capture
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._graph_update(batch)
            torch.cuda.current_stream().wait_stream(side)
            self._graph = torch.cuda.CUDAGraph()
            before = int(self.k.lib.rlx_launch_count())
            with torch.cuda.graph(self._graph):
                self._graph_update(batch)
            self._graph_launches = int(self.k.lib.rlx_launch_count()) - before  # kernels of this library inside one replay
            return  # the capture pass is not an update; the warm-up pass was
        self._graph.replay()
        self.k.lib.rlx_add_launch_count(self._graph_launches)

    def _graph_update(self, batch):
        self.eps.normal_()
        self._static_eps = (self.eps[0], self.eps[1])
        saved = self._draw_eps
        it = iter(self._static_eps)
        self._draw_eps = lambda n: next(it)
        try:
            self.k.update(self._update_args(batch))
        finally:
            self._draw_eps = saved
        self.metric_sums += self.metrics

    def _act(self, state, deterministic=False):
        obs = state if torch.is_tensor(state) else torch.from_numpy(np.ascontiguousarray(state, dtype=np.float32))
        obs = obs.to(self.device, torch.float32).contiguous()
        n = obs.shape[0]
        a_t, a_env = torch.empty(n, self.k.A, device=self.device), torch.empty(n, self.k.A, device=self.device)
        eps = None if deterministic else self._draw_eps(n)
        self.k.act(self.policy, obs, eps, self.d_low, self.d_high, self.ws, deterministic=deterministic, action_tanh=a_t, env_action=a_env)
        return a_t, a_env

    def current_learning_rate(self):
        if not self.anneal_learning_rate:
            return self.learning_rate
        total = max(int((self.total_timesteps - self.learning_starts) // self.nr_envs), 1)  # LinearLR total_iters, sac.py:80-82
        return self.learning_rate * (1.0 - min(self.nr_updates, total) / total)

    # ----------------------------------------------------------------------------------------------------- train
    def train(self):
        self._begin_training()
        while self.global_step < self.total_timesteps:
            self._train_step()

    def _begin_training(self):
        """Everything SAC.train() does before its while loop (sac.py:162-178)."""
        self.set_train_mode()
        self.replay_buffer = ReplayBuffer(int(self.buffer_size), self.nr_envs, self.os_shape, self.as_shape, self.rng, self.device)
        self.saving_return_buffer = deque(maxlen=100 * self.nr_envs)
        self.state, _ = self.train_env.reset()
        self.global_step, self.nr_updates, self.nr_episodes = 0, 0, 0
        self.time_metrics_collection, self.step_info_collection = {}, {}
        self.updates_since_log = 0
        self.prev_saving_end_time = None
        self.logging_time_prev = None

    def _train_step(self):
        """One pass of the reference's while-loop body (sac.py:180-348): act, env.step, replay add, sample, update, eval/save/log."""
        env, replay_buffer, state = self.train_env, self.replay_buffer, self.state
        start_time = time.time()
        if self.logging_time_prev:  # sac.py:183-184
            self.time_metrics_collection.setdefault("time/logging_time_prev", []).append(self.logging_time_prev)
        dones_this_rollout = 0
        # Acting (sac.py:187-196)
        if self.global_step < self.learning_starts:
            processed_action = np.array([env.single_action_space.sample() for _ in range(self.nr_envs)], dtype=np.float32)
            action = (processed_action - self.env_as_low) / (self.env_as_high - self.env_as_low) * 2.0 - 1.0
            step_action = torch.from_numpy(processed_action).to(self.device) if self.is_torch_data_interface else processed_action
        else:
            action, env_action = self._act(state)
            step_action = env_action if self.is_torch_data_interface else env_action.cpu().numpy()
        next_state, reward, terminated, truncated, info = env.step(step_action)
        done = terminated | truncated
        if self.is_torch_data_interface:
            actual_next_state = next_state  # auto-reset torch envs hand out the post-reset observation (same caveat as ppo.py:224-226)
            dones_this_rollout = int(done.sum().item())
        else:
            actual_next_state = next_state.copy()
            for i in np.nonzero(done)[0]:
                actual_next_state[i] = np.array(env.get_final_observation_at_index(info, int(i)))
                self.saving_return_buffer.append(env.get_final_info_value_at_index(info, "episode_return", int(i)))
                dones_this_rollout += 1
        for key, info_value in env.get_logging_info_dict(info).items():
            self.step_info_collection.setdefault(key, []).extend(info_value)
        replay_buffer.add(state, actual_next_state, action, reward, terminated)
        self.state = next_state
        self.global_step += self.nr_envs
        global_step = self.global_step
        self.nr_episodes += dones_this_rollout
        acting_end_time = time.time()
        self.time_metrics_collection.setdefault("time/acting_time", []).append(acting_end_time - start_time)

        should_learning_start = global_step > self.learning_starts
        should_evaluate = global_step % self.evaluation_frequency == 0 and self.evaluation_frequency != -1
        should_try_to_save = should_learning_start and self.save_model and dones_this_rollout > 0
        should_log = global_step % self.logging_frequency == 0

        if should_learning_start:
            self.lr_dev.fill_(self.current_learning_rate())
            self.update(replay_buffer.sample(self.batch_size))
            self.nr_updates += 1
            self.updates_since_log += 1
        optimizing_end_time = time.time()
        self.time_metrics_collection.setdefault("time/optimizing_time", []).append(optimizing_end_time - acting_end_time)

        evaluation_metrics = {}
        if should_evaluate:
            evaluation_metrics = self._evaluate()
        evaluating_end_time = time.time()
        self.time_metrics_collection.setdefault("time/evaluating_time", []).append(evaluating_end_time - optimizing_end_time)

        if should_try_to_save and len(self.saving_return_buffer) > 0:
            mean_return = np.mean(self.saving_return_buffer)
            if mean_return > self.best_mean_return:
                self.best_mean_return = mean_return
                self.save()
        saving_end_time = time.time()
        if self.prev_saving_end_time:
            self.time_metrics_collection.setdefault("time/sps", []).append(self.nr_envs / (saving_end_time - self.prev_saving_end_time))
        self.prev_saving_end_time = saving_end_time
        self.time_metrics_collection.setdefault("time/saving_time", []).append(saving_end_time - evaluating_end_time)

        if should_log:
            self.start_logging(global_step)
            combined = {}
            for info_name, values in self.step_info_collection.items():
                group = "rollout" if info_name in ["episode_return", "episode_length"] else "env_info"
                mean_value = np.mean(values)
                if mean_value == mean_value:
                    combined[f"{group}/{info_name}"] = mean_value
            combined.update({k: np.mean(v) for k, v in evaluation_metrics.items()})
            combined.update({"steps/nr_env_steps": global_step, "steps/nr_updates": self.nr_updates, "steps/nr_episodes": self.nr_episodes})
            combined.update({k: np.mean(v) for k, v in self.time_metrics_collection.items()})
            if self.updates_since_log > 0:  # the one device->host read of the optimisation metrics (means since the last log, sac.py:334-337)
                sums = (self.metric_sums / self.updates_since_log).cpu().numpy()
                combined.update({name: float(sums[i]) for i, name in enumerate(nt.SAC_METRIC_NAMES)})
                combined["lr/learning_rate"] = self.current_learning_rate()
                self.metric_sums.zero_()
                self.updates_since_log = 0
            for key, value in combined.items():
                self.log(f"{key}", value, global_step)
            self.time_metrics_collection, self.step_info_collection = {}, {}
            self.end_logging()
        self.logging_time_prev = time.time() - saving_end_time  # sac.py:347-348

    def _evaluate(self):
        """ref: sac.py:264-283."""
        self.set_eval_mode()
        eval_state, _ = self.eval_env.reset()
        n, out = 0, {"eval/episode_return": [], "eval/episode_length": []}
        while n < self.evaluation_episodes:
            _, env_action = self._act(eval_state, deterministic=True)
            eval_state, r, term, trunc, info = self.eval_env.step(env_action if self.is_torch_data_interface else env_action.cpu().numpy())
            for i, d in enumerate(np.asarray((term | trunc).cpu() if torch.is_tensor(term) else (term | trunc))):
                if d and n < self.evaluation_episodes:
                    n += 1
                    out["eval/episode_return"].append(self.eval_env.get_final_info_value_at_index(info, "episode_return", i))
                    out["eval/episode_length"].append(self.eval_env.get_final_info_value_at_index(info, "episode_length", i))
        self.set_train_mode()
        return out

    def test(self, episodes):
        """ref: sac.py:419-432."""
        self.set_eval_mode()
        for i in range(episodes):
            done, episode_return = False, 0
            state, _ = self.eval_env.reset()
            while not done:
                _, env_action = self._act(state, deterministic=True)
                state, reward, terminated, truncated, info = self.eval_env.step(env_action if self.is_torch_data_interface else env_action.cpu().numpy())
                d = terminated | truncated
                done = bool(d.any()) if hasattr(d, "any") else bool(d)
                episode_return += reward
            rlx_logger.info(f"Episode {i + 1} - Return: {episode_return}")

    # -------------------------------------------------------------------------------------------- logging / ckpt
    def log(self, name, value, step):
        if self.track_wandb:
            self.wandb_log_cache[name] = value
        if self.track_tb:
            self.writer.add_scalar(name, value, step)
        if self.track_console:
            self.log_console(name, value)

    def log_console(self, name, value):
        value = np.format_float_positional(value, trim="-")
        rlx_logger.info(f"│ {name.ljust(30)}│ {str(value).ljust(14)[:14]} │")

    def start_logging(self, step):
        if self.track_wandb:
            self.wandb_log_cache = {"global_step": int(step)}
        if self.track_console:
            rlx_logger.info("┌" + "─" * 31 + "┬" + "─" * 16 + "┐")
        else:
            rlx_logger.info(f"Step: {step}")

    def end_logging(self, wandb_commit=True):
        if self.track_wandb:
            import wandb
            wandb.log(self.wandb_log_cache, commit=wandb_commit)
        if self.track_console:
            rlx_logger.info("└" + "─" * 31 + "┴" + "─" * 16 + "┘")

    def _optimizer_views(self):
        """(exp_avg views, exp_avg_sq views) per reference optimiser, in the reference's parameter numbering: policy (sac.py:75),
        q1 then q2 (sac.py:76), log_alpha (sac.py:77)."""
        pm, pv = self.k.policy_views(self.m_policy), self.k.policy_views(self.v_policy)
        Pq = self.k.Pq

        def q_pair(flat):
            out = []
            for net in range(2):
                o = net * Pq  # per-net stride (padded to 256 bytes in the flat layout)
                for key, spec in Q_SEGMENTS:
                    shp = _shape(spec, self.k.O, self.k.A, self.k.H)
                    n = int(np.prod(shp))
                    out.append(flat[o:o + n].view(shp))
                    o += n
            return out

        return {"policy": ([pm[k] for k in POLICY_PARAM_ORDER], [pv[k] for k in POLICY_PARAM_ORDER]),
                "q": (q_pair(self.m_q), q_pair(self.v_q)),
                "entropy": ([self.m_la.view(1)], [self.v_la.view(1)])}

    def save(self):
        """Checkpoint with the reference's keys and optimizer layout (sac.py:381-396): module state_dicts in parameters() order, log_alpha,
        and the three torch.optim.Adam state dicts, so that either side's load() accepts the other's file."""
        pol, qs = self.state_dicts()
        steps = [int(x) for x in self.steps.cpu().tolist()]  # policy, q, entropy
        torch.save(checkpoint_dict(self.config.algorithm, pol, qs, self.log_alpha, self._optimizer_views(), steps, float(self.lr_dev.item())),
                   self.save_path + "/best.model")

    def load(config, train_env, eval_env, run_path, writer, explicitly_set_algorithm_params):
        ck = torch.load(config.runner.load_model, weights_only=False)
        for key, value in ck["config_algorithm"].items():
            if f"algorithm.{key}" not in explicitly_set_algorithm_params and key in config.algorithm and key not in ("name", "device", "bf16_mixed_precision_training", "compile_mode"):
                config.algorithm[key] = value
        model = SAC(config, train_env, eval_env, run_path, writer)
        model.load_named(ck["policy_state_dict"], ck["q1_state_dict"], ck["q2_state_dict"], ck["q1_target_state_dict"], ck["q2_target_state_dict"])
        model.log_alpha.copy_(torch.as_tensor(ck["log_alpha"]).detach().reshape(1))
        ov = model._optimizer_views()
        steps = [_load_adam_state(ck[f"{name}_optimizer_state_dict"], *ov[name], name) if f"{name}_optimizer_state_dict" in ck else 0
                 for name in ("policy", "q", "entropy")]
        if "optimizer_flat" in ck:  # files written by earlier versions of this build
            for k, v in ck["optimizer_flat"].items():
                getattr(model, k).copy_(v)
        else:
            model.steps.copy_(torch.tensor(steps, dtype=torch.int64))
        return model

    def set_train_mode(self):
        self.training = True

    def set_eval_mode(self):
        self.training = False

    def general_properties():
        return GeneralProperties
