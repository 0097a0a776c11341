"""FastTD3 on the GPU — mirrors rl_x/algorithms/fasttd3/pytorch/fasttd3.py (constructor, train(), test(), logging keys), fp32 path.

Host side: Python/PyTorch for device memory and the TORCH-interface environment; every compute step is a C-ABI call (include/rlx_b200.h):

    acting       observation_normalizer.normalize + policy.get_action (fasttd3.py:262-264)      rlx_fastsac_normalize_f32, rlx_fasttd3_act_f32
    replay       ReplayBuffer.add / sample (replay_buffer.py, FastSAC's file)                    fastsac.b200 ReplayBuffer (rlx_replay_sample_nstep_f32)
    update       critic_loss_fn + polyak (fasttd3.py:139-225, 316-320)                          rlx_fasttd3_critic_update_f32
                 policy_loss_fn (fasttd3.py:104-136)                                             rlx_fasttd3_policy_update_f32

Parameters are initialised exactly like the reference (the same torch modules built in the same order under torch.manual_seed(seed),
fasttd3.py:81-85) and live in the library's flat layout; the acting noise, smoothing noise and per-environment exploration scales are
torch.randn / torch.rand on the device, drawn in the reference's order.  The env's policy_observation_indices /
critic_observation_indices (policy.py:12,52, q_network.py:10,39) are validated on the host and passed to the library as device int32
arrays: the policy's first layer is [512, P] and each Q network's [1024, C + act], the reference's shapes; the replay buffer and the
observation normaliser stay full-width.  Not built: bf16 autocast.  GPU tests: tests/test_gpu_zzzzz_fasttd3.py,
tests/test_gpu_zzzzzzzzzzzzz_fasttd3_obs_indices.py; the same sources are checked in host emulation (tests/test_fasttd3_emulation.py,
tests/test_fasttd3_obs_indices.py).
"""
import ctypes as C
import logging
import os
import time

import numpy as np
import torch

from rl_x_b200 import _native as nt
from rl_x_b200.algorithms.fastsac.b200.replay_buffer import ReplayBuffer

rlx_logger = logging.getLogger("rl_x")
POLICY_WIDTHS, Q_WIDTHS = (512, 256, 128), (1024, 512, 256)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def reference_init(obs, act, nr_atoms, seed, policy_in=None, critic_in=None):
    """FastTD3.__init__'s parameter values (fasttd3.py:81-85, policy.py:33-48, critic.py:17-22): same torch modules, construction order and
    seed.  Returns the flat policy vector and the flat q1 | q2 vector in the layout of include/rlx_b200.h (torch state_dict order).
    policy_in / critic_in: the lengths of the observation index sets (None = obs), the fan-ins of the first layers (policy.py:30,
    q_network.py:24)."""
    policy_in = obs if policy_in is None else policy_in
    critic_in = obs if critic_in is None else critic_in
    torch.manual_seed(seed)

    def mlp(inp, widths, out):
        layers, last = [], inp
        for w in tuple(widths) + (out,):
            layers.append(torch.nn.Linear(last, w))
            last = w
        return layers

    def flat(layers):
        return torch.cat([t.detach().reshape(-1) for lyr in layers for t in (lyr.weight, lyr.bias)])

    pol = mlp(policy_in, POLICY_WIDTHS, act)
    torch.nn.init.normal_(pol[-1].weight, 0.0, 0.01)
    torch.nn.init.constant_(pol[-1].bias, 0.0)
    qs = [flat(mlp(critic_in + act, Q_WIDTHS, nr_atoms)) for _ in range(4)]   # q1, q2, then the targets, which consume the generator too
    return flat(pol), torch.cat(qs[:2])


class FastTD3:
    def __init__(self, config, train_env, eval_env, run_path, writer):
        self.config = config
        self.train_env = train_env
        self.eval_env = eval_env
        self.writer = writer

        self.save_model = config.runner.save_model
        self.save_path = os.path.join(run_path, "models")
        self.track_console = config.runner.track_console
        self.track_tb = config.runner.track_tb
        self.track_wandb = config.runner.track_wandb
        self.seed = config.environment.seed
        a = config.algorithm
        self.total_timesteps = a.total_timesteps
        self.nr_envs = config.environment.nr_envs
        self.learning_rate = a.learning_rate
        self.anneal_learning_rate = a.anneal_learning_rate
        self.batch_size = a.batch_size
        self.buffer_size_per_env = a.buffer_size_per_env
        self.learning_starts = a.learning_starts
        self.n_steps = a.n_steps
        self.gamma = a.gamma
        self.noise_std_min = a.noise_std_min
        self.noise_std_max = a.noise_std_max
        self.nr_critic_updates_per_policy_update = a.nr_critic_updates_per_policy_update
        self.nr_policy_updates_per_step = a.nr_policy_updates_per_step
        self.action_clipping_and_rescaling = a.action_clipping_and_rescaling
        self.enable_observation_normalization = a.enable_observation_normalization
        self.logging_frequency = a.logging_frequency
        self.evaluation_frequency = a.evaluation_frequency
        self.save_frequency = a.save_frequency
        self.horizon = self.train_env.horizon

        if self.logging_frequency % self.nr_envs != 0:
            raise ValueError("The logging frequency must be a multiple of the number of environments.")
        if self.save_frequency != -1 and self.save_frequency % self.nr_envs != 0:
            raise ValueError("The save frequency must be a multiple of the number of environments.")
        if a.get("bf16_mixed_precision_training", False):
            raise NotImplementedError("rl_x_b200 FastTD3 implements the reference's fp32 path; set algorithm.bf16_mixed_precision_training=False.")
        # the networks' input columns (policy.py:12,52 / q_network.py:10,39): validated on the host before any device work; None = identity
        obs = int(self.train_env.single_observation_space.shape[0])
        self.policy_observation_indices = nt.observation_indices(
            "policy_observation_indices", getattr(self.train_env, "policy_observation_indices", None), obs)
        self.critic_observation_indices = nt.observation_indices(
            "critic_observation_indices", getattr(self.train_env, "critic_observation_indices", None), obs)
        if a.device != "gpu" or not torch.cuda.is_available():
            raise RuntimeError("rl_x_b200 FastTD3 needs a CUDA device (algorithm.device=gpu); there is no CPU fallback.")
        self.device = torch.device("cuda", torch.cuda.current_device())
        rlx_logger.info(f"Using device: {self.device}")

        self.lib = nt.load()
        engine = a.get("gemm_engine", "auto")   # dense layers: exact-fp32 SIMT, or the 3xTF32 wgmma engine ("tcgen05") where it covers the product
        if engine not in ("auto", "simt", "tcgen05"):
            raise ValueError("algorithm.gemm_engine must be auto, simt or tcgen05")
        if engine != "auto":
            self.lib.rlx_set_aux_gemm_engine(1 if engine == "tcgen05" else 0)
        act = int(np.prod(self.train_env.single_action_space.shape))
        self.dims = nt.FastTd3Dims(obs, act, int(a.nr_atoms))
        # device copies of the index sets, kept alive for as long as self.dims points at them
        self._idx = {}
        for k, ind in (("policy", self.policy_observation_indices), ("critic", self.critic_observation_indices)):
            if ind is not None:
                self._idx[k] = torch.as_tensor(ind, dtype=torch.int32).to(self.device).contiguous()
                setattr(self.dims, f"{k}_in_dim", int(ind.size))
                setattr(self.dims, f"{k}_idx", self._idx[k].data_ptr())
        self.policy_in = obs if self.policy_observation_indices is None else int(self.policy_observation_indices.size)
        self.critic_in = obs if self.critic_observation_indices is None else int(self.critic_observation_indices.size)
        poff, qoff = (C.c_int64 * (nt.RLX_FASTTD3_POLICY_NSEG + 1))(), (C.c_int64 * (nt.RLX_FASTTD3_Q_NSEG + 1))()
        nt.check(self.lib.rlx_fasttd3_param_layout(C.byref(self.dims), poff, qoff), "rlx_fasttd3_param_layout")
        self.policy_offsets, self.q_offsets = list(poff), list(qoff)

        self.rng = np.random.default_rng(self.seed)
        policy, q = reference_init(obs, act, int(a.nr_atoms), self.seed, self.policy_in, self.critic_in)   # torch.manual_seed(self.seed) inside, as fasttd3.py:81
        assert policy.numel() == self.policy_offsets[-1] and q.numel() == 2 * self.q_offsets[-1]
        dev = self.device
        self.policy_params, self.q_params = policy.to(dev).contiguous(), q.to(dev).contiguous()
        self.q_target_params = self.q_params.clone()
        zl = torch.zeros_like
        self.policy_grads, self.policy_m, self.policy_v = zl(self.policy_params), zl(self.policy_params), zl(self.policy_params)
        self.q_grads, self.q_m, self.q_v = zl(self.q_params), zl(self.q_params), zl(self.q_params)
        self.steps = torch.zeros(2, dtype=torch.int64, device=dev)
        self.lr_dev = torch.full((1,), float(self.learning_rate), dtype=torch.float32, device=dev)
        self.lr_step = 0
        # torch.optim.AdamW defaults (fasttd3.py:88-89 passes lr and weight_decay only)
        self.hp = nt.FastTd3Hparams(float(a.gamma), float(a.tau), float(a.v_min), float(a.v_max), float(a.smoothing_epsilon), float(a.smoothing_clip_value),
                                    float(a.weight_decay), 0.9, 0.999, 1e-8, float(a.max_grad_norm), 1.0 if a.clipped_double_q_learning else 0.0)
        sp = self.train_env.single_action_space
        self.act_low = torch.as_tensor(np.asarray(sp.low, dtype=np.float32)).reshape(-1).to(dev).contiguous()
        self.act_high = torch.as_tensor(np.asarray(sp.high, dtype=np.float32)).reshape(-1).to(dev).contiguous()
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.norm_mean, self.norm_var, self.norm_std = z(obs), torch.ones(obs, device=dev), torch.ones(obs, device=dev)
        self.norm_count = torch.zeros(1, dtype=torch.int64, device=dev)
        self._ws = {}
        if self.save_model:
            os.makedirs(self.save_path)

    # --------------------------------------------------------------------------------------------------- kernels
    def current_learning_rate(self):
        if not self.anneal_learning_rate:
            return self.learning_rate
        total_iters = (self.total_timesteps // self.nr_envs) - self.learning_starts   # LinearLR(1 -> 0), fasttd3.py:91-93
        return self.learning_rate * (1.0 - min(self.lr_step, total_iters) / max(total_iters, 1))

    def _workspace(self, n):
        if n not in self._ws:
            nbytes = int(self.lib.rlx_fasttd3_workspace_bytes(C.byref(self.dims), int(n)))
            self._ws[n] = (torch.zeros(nbytes // 4 + 64, dtype=torch.float32, device=self.device), nbytes)
        return self._ws[n]

    def normalize(self, x, update):
        """ObservationNormalizer.normalize (observation_normalizer.py:20-27; the same module as FastSAC's)."""
        if not self.enable_observation_normalization:
            return x
        x = x.contiguous()
        n, obs = x.shape
        out = torch.empty_like(x)
        ws = torch.empty(4 * obs * (n // 256 + 2), dtype=torch.float32, device=self.device)
        nt.check(self.lib.rlx_fastsac_normalize_f32(x.data_ptr(), n, obs, self.norm_mean.data_ptr(), self.norm_var.data_ptr(), self.norm_std.data_ptr(),
                                                    self.norm_count.data_ptr(), 1 if (update and self.training) else 0, 1e-8, out.data_ptr(),
                                                    ws.data_ptr(), _stream()), "rlx_fastsac_normalize_f32")
        return out

    def draw_noise_scales(self):
        """torch.rand(nr_envs, 1) * (max - min) + min (fasttd3.py:241, 274-278)."""
        return torch.rand(self.nr_envs, 1, device=self.device) * (self.noise_std_max - self.noise_std_min) + self.noise_std_min

    def get_action(self, normalized_state, noise_scales=None):
        """Policy.get_action (policy.py:57-66): (action, processed_action); noise_scales None: deterministic."""
        n = normalized_state.shape[0]
        ws, nbytes = self._workspace(n)
        action = torch.empty(n, self.dims.act_dim, dtype=torch.float32, device=self.device)
        env_action = torch.empty_like(action) if self.action_clipping_and_rescaling else None
        noise, scales = None, None
        if noise_scales is not None:
            noise = torch.randn(n, self.dims.act_dim, device=self.device)
            scales = noise_scales.reshape(-1).contiguous()
        nt.check(self.lib.rlx_fasttd3_act_f32(C.byref(self.dims), self.policy_params.data_ptr(), normalized_state.contiguous().data_ptr(),
                                              nt.ptr(noise), nt.ptr(scales), self.act_low.data_ptr(), self.act_high.data_ptr(),
                                              1 if self.action_clipping_and_rescaling else 0, n, action.data_ptr(), nt.ptr(env_action), ws.data_ptr(),
                                              nbytes, _stream()), "rlx_fasttd3_act_f32")
        return action, (env_action if env_action is not None else action)

    def _update_args(self, n, metrics):
        ws, nbytes = self._workspace(n)
        a = nt.FastTd3UpdateArgs()
        a.dims, a.n = self.dims, n
        a.policy_params, a.policy_grads, a.policy_m, a.policy_v = (t.data_ptr() for t in (self.policy_params, self.policy_grads, self.policy_m, self.policy_v))
        a.q_params, a.q_grads, a.q_m, a.q_v = (t.data_ptr() for t in (self.q_params, self.q_grads, self.q_m, self.q_v))
        a.q_target_params = self.q_target_params.data_ptr()
        a.lr, a.steps, a.hp = self.lr_dev.data_ptr(), self.steps.data_ptr(), self.hp
        a.metrics, a.workspace, a.workspace_bytes = metrics.data_ptr(), ws.data_ptr(), nbytes
        return a

    def critic_update(self, s, ns, actions, rewards, dones, truncations, eff, metrics):
        n = s.shape[0]
        noise = torch.randn(n, self.dims.act_dim, device=self.device)   # torch.randn_like(actions), fasttd3.py:143
        a = self._update_args(n, metrics)
        for name, t in (("states", s), ("next_states", ns), ("actions", actions), ("rewards", rewards), ("dones", dones), ("truncations", truncations),
                        ("effective_n_steps", eff), ("smoothing_noise", noise)):
            assert t.is_contiguous()
            setattr(a, name, t.data_ptr())
        nt.check(self.lib.rlx_fasttd3_critic_update_f32(C.byref(a), _stream()), "rlx_fasttd3_critic_update_f32")

    def policy_update(self, s, metrics):
        a = self._update_args(s.shape[0], metrics)
        assert s.is_contiguous()
        a.states = s.data_ptr()
        nt.check(self.lib.rlx_fasttd3_policy_update_f32(C.byref(a), _stream()), "rlx_fasttd3_policy_update_f32")

    # ----------------------------------------------------------------------------------------------------- train
    def train(self):
        self.set_train_mode()
        env = self.train_env
        replay_buffer = ReplayBuffer(self.buffer_size_per_env, self.nr_envs, env.single_observation_space.shape, env.single_action_space.shape,
                                     self.n_steps, self.gamma, self.device)
        npu, ncu, B = self.nr_policy_updates_per_step, self.nr_critic_updates_per_policy_update, self.batch_size
        cm, pm = torch.zeros(8, device=self.device), torch.zeros(8, device=self.device)
        state, _ = env.reset()
        state = state.to(self.device, torch.float32)
        noise_scales = self.draw_noise_scales()
        global_step = 0
        nr_updates = 0
        nr_episodes = 0
        time_metrics_collection, step_info_collection, optimization_metrics_collection, evaluation_metrics_collection = {}, {}, {}, {}
        steps_metrics = {}
        prev_saving_end_time = None
        logging_time_prev = None

        while global_step < self.total_timesteps:
            start_time = time.time()
            if logging_time_prev:
                time_metrics_collection.setdefault("time/logging_time_prev", []).append(logging_time_prev)

            # Acting (fasttd3.py:260-282)
            action, processed_action = self.get_action(self.normalize(state, update=False), noise_scales)
            next_state, reward, terminated, truncated, info = env.step(processed_action)
            done = terminated | truncated
            dones_this_rollout = int(done.sum().item())
            for key, info_value in env.get_logging_info_dict(info).items():
                step_info_collection.setdefault(key, []).extend(info_value)
            next_state = next_state.to(self.device, torch.float32)
            replay_buffer.add(state, next_state, action, reward.to(self.device, torch.float32), done.to(self.device, torch.float32),
                              truncated.to(self.device, torch.float32))
            noise_scales = torch.where(done.to(self.device)[:, None], self.draw_noise_scales(), noise_scales)
            state = next_state
            global_step += self.nr_envs
            nr_episodes += dones_this_rollout
            acting_end_time = time.time()
            time_metrics_collection.setdefault("time/acting_time", []).append(acting_end_time - start_time)

            should_learning_start = global_step > self.learning_starts * self.nr_envs
            should_optimize = should_learning_start
            should_evaluate = global_step % self.evaluation_frequency == 0 and self.evaluation_frequency != -1
            should_try_to_save = should_learning_start and self.save_model and dones_this_rollout > 0 and self.save_frequency != -1 and global_step % self.save_frequency == 0
            should_log = global_step % self.logging_frequency == 0

            # Optimizing (fasttd3.py:297-341)
            if should_optimize:
                self.lr_dev.fill_(self.current_learning_rate())
                total = npu * ncu * B
                ts, tns, ta, tr, td, ttr, teff = replay_buffer.sample(total)
                ts = self.normalize(ts, update=True).view(npu, ncu, B, -1)
                tns = self.normalize(tns, update=True).view(npu, ncu, B, -1)
                ta = ta.view(npu, ncu, B, -1)
                tr, td, ttr, teff = (t.view(npu, ncu, B) for t in (tr, td, ttr, teff))
                for i in range(npu):
                    for j in range(ncu):
                        self.critic_update(ts[i, j], tns[i, j], ta[i, j], tr[i, j], td[i, j], ttr[i, j], teff[i, j], cm)
                        nr_updates += 1
                    self.policy_update(ts[i, -1], pm)
                    c, p = cm.cpu().numpy(), pm.cpu().numpy()
                    optimization_metrics = {
                        "gradients/policy_grad_norm": p[1], "gradients/critic_grad_norm": c[3], "loss/q_loss": c[0], "loss/policy_loss": p[0],
                        "lr/learning_rate": self.current_learning_rate(), "q/q_max": c[2], "q/q_min": c[1]}
                    for key, value in optimization_metrics.items():
                        optimization_metrics_collection.setdefault(key, []).append(float(value))
                if self.anneal_learning_rate:
                    self.lr_step += 1
            optimizing_end_time = time.time()
            time_metrics_collection.setdefault("time/optimizing_time", []).append(optimizing_end_time - acting_end_time)

            # Evaluating (fasttd3.py:348-364)
            if should_evaluate:
                self.set_eval_mode()
                eval_state, _ = self.eval_env.reset()
                for _ in range(self.horizon):
                    _, eval_action = self.get_action(self.normalize(eval_state.to(self.device, torch.float32), update=False))
                    eval_state, _, _, _, eval_info = self.eval_env.step(eval_action)
                    eval_logging_info = self.eval_env.get_logging_info_dict(eval_info)
                    for k_ in ("episode_return", "episode_length"):
                        if k_ in eval_logging_info:
                            evaluation_metrics_collection.setdefault(f"eval/{k_}", []).extend(eval_logging_info[k_])
                self.set_train_mode()
            evaluating_end_time = time.time()
            time_metrics_collection.setdefault("time/evaluating_time", []).append(evaluating_end_time - optimizing_end_time)

            if should_try_to_save:
                self.save()
            saving_end_time = time.time()
            if prev_saving_end_time:
                time_metrics_collection.setdefault("time/sps", []).append(self.nr_envs / (saving_end_time - prev_saving_end_time))
            prev_saving_end_time = saving_end_time
            time_metrics_collection.setdefault("time/saving_time", []).append(saving_end_time - evaluating_end_time)

            # Logging (fasttd3.py:382-413)
            if should_log:
                self.start_logging(global_step)
                steps_metrics["steps/nr_env_steps"] = global_step
                steps_metrics["steps/nr_critic_updates"] = nr_updates
                steps_metrics["steps/nr_policy_updates"] = nr_updates // ncu
                steps_metrics["steps/nr_episodes"] = nr_episodes
                rollout_info_metrics, env_info_metrics = {}, {}
                for info_name, vals in step_info_collection.items():
                    metric_group = "rollout" if info_name in ["episode_return", "episode_length"] else "env_info"
                    mean_value = np.mean(vals)
                    if mean_value == mean_value:
                        (rollout_info_metrics if metric_group == "rollout" else env_info_metrics)[f"{metric_group}/{info_name}"] = mean_value
                mean = lambda coll: {key: np.mean(value) for key, value in coll.items()}
                combined = {**rollout_info_metrics, **mean(evaluation_metrics_collection), **env_info_metrics, **steps_metrics, **mean(time_metrics_collection),
                            **mean(optimization_metrics_collection)}
                for key, value in combined.items():
                    self.log(f"{key}", value, global_step)
                time_metrics_collection, step_info_collection, optimization_metrics_collection, evaluation_metrics_collection = {}, {}, {}, {}
                self.end_logging()
            logging_end_time = time.time()
            logging_time_prev = logging_end_time - saving_end_time

    # ------------------------------------------------------------------------------------------------ test / io
    def test(self, episodes):
        rlx_logger.info("Testing runs infinitely. The episodes parameter is ignored.")
        self.set_eval_mode()
        state, _ = self.eval_env.reset()
        while True:   # as the reference (fasttd3.py:485-497)
            _, action = self.get_action(self.normalize(state.to(self.device, torch.float32), update=False))
            state, _, _, _, _ = self.eval_env.step(action)

    # ------------------------------------------------------------------------------------------------ checkpoints
    # The reference's file layout and state_dict key names (fasttd3.py:449-482), so that models move between the two implementations.
    def _named(self, flat, net):
        """flat parameter-like vector -> {state_dict key: tensor} for "policy" or one Q network."""
        act, atoms = self.dims.act_dim, self.dims.nr_atoms
        widths, inp, out, prefix = (POLICY_WIDTHS, self.policy_in, act, "policy") if net == "policy" else (Q_WIDTHS, self.critic_in + act, atoms, "critic")
        shapes, last = [], inp
        for k, w in enumerate(tuple(widths) + (out,)):
            shapes += [(f"{prefix}.{2 * k}.weight", (w, last)), (f"{prefix}.{2 * k}.bias", (w,))]
            last = w
        named, o = {}, 0
        for name, shape in shapes:
            n = int(np.prod(shape))
            named[name] = flat[o:o + n].view(shape)
            o += n
        assert o == flat.numel()
        return named

    def _adamw_state(self, m, v, step, named_like):
        state, o = {}, 0
        for i, (name, t) in enumerate(named_like.items()):
            n = t.numel()
            state[i] = {"step": torch.tensor(float(step)), "exp_avg": m[o:o + n].view(t.shape).cpu().clone(), "exp_avg_sq": v[o:o + n].view(t.shape).cpu().clone()}
            o += n
        group = {"lr": self.current_learning_rate(), "betas": (self.hp.adam_beta1, self.hp.adam_beta2), "eps": 1e-08, "weight_decay": self.hp.weight_decay,
                 "amsgrad": False, "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None,
                 "decoupled_weight_decay": True, "params": list(range(len(state)))}
        return {"state": state, "param_groups": [group]}

    def save(self):
        nq = self.q_offsets[-1]
        cpu = lambda d: {k: v.detach().cpu().clone() for k, v in d.items()}
        steps = self.steps.cpu().tolist()
        pol = self._named(self.policy_params, "policy")
        q1, q2 = self._named(self.q_params[:nq], "q"), self._named(self.q_params[nq:], "q")
        q_both = {**{"q1." + k: v for k, v in q1.items()}, **{"q2." + k: v for k, v in q2.items()}}   # q1's parameters numbered before q2's
        torch.save({
            "config_algorithm": self.config.algorithm,
            "policy_state_dict": cpu(pol),
            "q1_state_dict": cpu(q1), "q2_state_dict": cpu(q2),
            "q1_target_state_dict": cpu(self._named(self.q_target_params[:nq], "q")), "q2_target_state_dict": cpu(self._named(self.q_target_params[nq:], "q")),
            "policy_optimizer_state_dict": self._adamw_state(self.policy_m, self.policy_v, steps[1], pol),
            "q_optimizer_state_dict": self._adamw_state(self.q_m, self.q_v, steps[0], q_both),
            "observation_normalizer_state_dict": {"running_mean": self.norm_mean.cpu().view(1, -1).clone(), "running_var": self.norm_var.cpu().view(1, -1).clone(),
                                                  "running_std_dev": self.norm_std.cpu().view(1, -1).clone(), "count": self.norm_count.cpu()[0].clone()},
        }, os.path.join(self.save_path, "latest.model"))

    @classmethod
    def load(cls, config, train_env, eval_env, run_path, writer, explicitly_set_algorithm_params):
        ck = torch.load(config.runner.load_model, weights_only=False)
        for key, value in ck["config_algorithm"].items():
            if f"algorithm.{key}" not in explicitly_set_algorithm_params and key in config.algorithm and key not in ("name", "device", "bf16_mixed_precision_training", "compile_mode"):
                config.algorithm[key] = value
        model = cls(config, train_env, eval_env, run_path, writer)
        nq = model.q_offsets[-1]

        def fill(flat, net, sd):
            for name, dst in model._named(flat, net).items():
                src = sd[name] if name in sd else sd["_orig_mod." + name]   # torch.compile'd reference modules prefix their keys
                dst.copy_(torch.as_tensor(src, dtype=torch.float32).reshape(dst.shape))

        def fill_moments(m, v, named_like, osd):
            o, step = 0, 0.0
            for i, t in enumerate(named_like.values()):
                n = t.numel()
                if i in osd["state"]:
                    m[o:o + n].copy_(osd["state"][i]["exp_avg"].reshape(-1))
                    v[o:o + n].copy_(osd["state"][i]["exp_avg_sq"].reshape(-1))
                    step = max(step, float(osd["state"][i]["step"]))
                o += n
            return int(step)

        fill(model.policy_params, "policy", ck["policy_state_dict"])
        fill(model.q_params[:nq], "q", ck["q1_state_dict"]); fill(model.q_params[nq:], "q", ck["q2_state_dict"])
        fill(model.q_target_params[:nq], "q", ck["q1_target_state_dict"]); fill(model.q_target_params[nq:], "q", ck["q2_target_state_dict"])
        pol = model._named(model.policy_params, "policy")
        q_both = {**{"q1." + k: v for k, v in model._named(model.q_params[:nq], "q").items()},
                  **{"q2." + k: v for k, v in model._named(model.q_params[nq:], "q").items()}}
        steps = [fill_moments(model.q_m, model.q_v, q_both, ck["q_optimizer_state_dict"]),
                 fill_moments(model.policy_m, model.policy_v, pol, ck["policy_optimizer_state_dict"])]
        model.steps.copy_(torch.tensor(steps, dtype=torch.int64))
        n = ck["observation_normalizer_state_dict"]
        if "running_mean" in n:
            model.norm_mean.copy_(n["running_mean"].reshape(-1)); model.norm_var.copy_(n["running_var"].reshape(-1))
            model.norm_std.copy_(n["running_std_dev"].reshape(-1)); model.norm_count.fill_(int(n["count"]))
        return model

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

    def set_train_mode(self):
        self.training = True

    def set_eval_mode(self):
        self.training = False

    def general_properties():
        from rl_x_b200.algorithms.fasttd3.b200.general_properties import GeneralProperties
        return GeneralProperties
