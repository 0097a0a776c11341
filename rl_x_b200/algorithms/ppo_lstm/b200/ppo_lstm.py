"""PPO with an LSTM policy on the GPU — mirrors rl_x/algorithms/ppo_lstm/flax/ppo_lstm.py (constructor, train(), test(), logging keys).

The reference is JAX/Flax; here the host side is Python/PyTorch (device memory, streams) and every compute step is a call into the
C-ABI library (include/rlx_b200.h, "PPO + LSTM path"):

    acting      get_action_and_value (ppo_lstm.py:107-118)         -> rlx_lstm_step_f32 + rlx_lstm_mask_carry_f32
    advantages  calculate_gae_advantages (ppo_lstm.py:121-138)      -> rlx_lstm_critic_forward_f32 + rlx_gae_f32
    update      update / minibatch_update (ppo_lstm.py:141-231)     -> rlx_gather_env_columns_f32, rlx_mean_popstd_f32,
                                                                       rlx_lstm_ppo_minibatch_fwdbwd_f32, rlx_optax_clip_adam_f32 x2

Differences that follow from the missing JAX runtime (all explicit): parameters are initialised with the same initialiser families
from a torch generator (not jax.random), the action noise is torch.randn on the device, and the per-epoch env permutations come from
the library's PCG64 stream — so runs are not seed-for-seed comparable with the reference; checkpoints are torch files with named
tensors instead of Orbax trees.  GPU tests: tests/test_gpu_zzz_ppo_lstm.py; the same sources are checked in host emulation (tests/test_lstm_emulation.py).
"""
import ctypes as C
import logging
import math
import os
import time
from collections import deque

import numpy as np
import torch

from rl_x_b200 import _native as nt
from rl_x_b200.environments.types import DataInterfaceType, require_identity_observation_indices, same_member

rlx_logger = logging.getLogger("rl_x")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def init_parameters(dims, std_dev, seed):
    """Initialiser families of Policy.setup / Critic (policy.py:47-70, critic.py:22-30): orthogonal(sqrt 2) dense kernels, zero biases,
    LayerNorm scale 1 / bias 0, LSTM input kernels lecun-normal and recurrent kernels orthogonal, mean head orthogonal(0.01), critic head
    orthogonal(1), log-std = log(std_dev); FiLM gamma / beta layers orthogonal(sqrt 2) (policy.py:57-59).  Returns {segment name: tensor}
    for both trees ([in, out] kernels); segments an option removes (obs_encoder with a shared encoder, FiLM layers with "concat") are empty."""
    g = torch.Generator().manual_seed(int(seed))
    O, A, H, E, L = dims.obs_dim, dims.act_dim, dims.hidden, dims.enc_dim, dims.lstm_dim
    film, shared = bool(dims.options & nt.RLX_LSTM_OPT_FILM), bool(dims.options & nt.RLX_LSTM_OPT_SHARED_ENCODER)

    def orth(i, o, gain):
        w = torch.empty(o, i)
        torch.nn.init.orthogonal_(w, gain=gain, generator=g)
        return w.t().contiguous()

    s2 = math.sqrt(2.0)
    E2 = 0 if shared else E
    pol = {"We1": orth(O, E, s2), "be1": torch.zeros(E), "g1": torch.ones(E), "n1": torch.zeros(E),
           "We2": orth(O, E, s2) if not shared else torch.zeros(0), "be2": torch.zeros(E2), "g2": torch.ones(E2), "n2": torch.zeros(E2),
           "Wi": torch.cat([torch.randn(E, L, generator=g) / math.sqrt(E) for _ in range(4)], dim=1),
           "Wh": torch.cat([orth(L, L, 1.0) for _ in range(4)], dim=1), "bh": torch.zeros(4 * L),
           "gl": torch.ones(L), "nl": torch.zeros(L),
           "Wf": torch.cat([orth(L, E, s2), orth(L, E, s2)], dim=1) if film else torch.zeros(0), "bf": torch.zeros(2 * E if film else 0),
           "Wt1": orth(E if film else E + L, H, s2), "bt1": torch.zeros(H), "Wt2": orth(H, H, s2), "bt2": torch.zeros(H),
           "Wm": orth(H, A, 0.01), "bm": torch.zeros(A), "logstd": torch.full((A,), math.log(std_dev))}
    cri = {"Wc1": orth(O, H, s2), "bc1": torch.zeros(H), "Wc2": orth(H, H, s2), "bc2": torch.zeros(H), "Wc3": orth(H, 1, 1.0), "bc3": torch.zeros(1)}
    return pol, cri


class PPO_LSTM:
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
        self.nr_steps = a.nr_steps
        self.nr_epochs = a.nr_epochs
        self.minibatch_size = a.minibatch_size
        self.gamma = a.gamma
        self.gae_lambda = a.gae_lambda
        self.clip_range = a.clip_range
        self.entropy_coef = a.entropy_coef
        self.critic_coef = a.critic_coef
        self.max_grad_norm = a.max_grad_norm
        self.std_dev = a.std_dev
        self.lstm_hidden_dim = a.lstm_hidden_dim
        self.action_clipping_and_rescaling = a.action_clipping_and_rescaling
        self.evaluation_frequency = a.evaluation_frequency
        self.evaluation_episodes = a.evaluation_episodes
        self.use_cuda_graph = bool(a.get("use_cuda_graph", False))  # replay the minibatch update as one CUDA graph (same kernels, same order)
        self.batch_size = self.nr_envs * self.nr_steps
        self.nr_updates = int(self.total_timesteps // self.batch_size)                 # ppo_lstm.py:55
        self.nr_minibatches = self.batch_size // self.minibatch_size                  # ppo_lstm.py:56
        self.nr_minibatch_envs = self.minibatch_size // self.nr_steps                 # ppo_lstm.py:57

        if self.evaluation_frequency % (self.nr_steps * self.nr_envs) != 0 and self.evaluation_frequency != -1:
            raise ValueError("Evaluation frequency must be a multiple of the number of steps and environments.")
        if self.minibatch_size % self.nr_steps != 0:
            raise ValueError("Minibatch size must be a multiple of nr_steps for PPO_LSTM.")
        if a.lstm_obs_combine_method not in ("concat", "film"):
            raise ValueError("lstm_obs_combine_method must be 'concat' or 'film' (policy.py:99-105)")
        if self.nr_minibatches < 1 or self.nr_minibatch_envs * self.nr_minibatches != self.nr_envs:
            # the reference reshapes nr_epochs permutations of arange(nr_envs) to (nr_epochs * nr_minibatches, nr_minibatch_envs), ppo_lstm.py:189-191
            raise ValueError("nr_envs must equal nr_minibatches * (minibatch_size // nr_steps)")
        require_identity_observation_indices(self.train_env, "PPO_LSTM")  # policy.py:14,79,87 / critic.py
        if a.device != "gpu" or not torch.cuda.is_available():
            raise RuntimeError("rl_x_b200 PPO_LSTM needs a CUDA device (algorithm.device=gpu); there is no CPU fallback.")
        self.device = torch.device("cuda", torch.cuda.current_device())
        rlx_logger.info(f"Using device: {self.device}")

        self.os_shape = self.train_env.single_observation_space.shape
        self.as_shape = self.train_env.single_action_space.shape
        if len(self.os_shape) != 1 or len(self.as_shape) != 1:
            raise ValueError("rl_x_b200 PPO_LSTM supports flat observations and flat continuous actions only.")
        self.lib = nt.load()
        engine = a.get("gemm_engine", "auto")   # dense layers: exact-fp32 SIMT, or the 3xTF32 wgmma engine ("tcgen05") where it covers the product
        if engine not in ("auto", "simt", "tcgen05"):
            raise ValueError("algorithm.gemm_engine must be auto, simt or tcgen05")
        if engine != "auto":
            self.lib.rlx_set_aux_gemm_engine(1 if engine == "tcgen05" else 0)
        options = (nt.RLX_LSTM_OPT_FILM if a.lstm_obs_combine_method == "film" else 0) | (nt.RLX_LSTM_OPT_SHARED_ENCODER if a.share_lstm_obs_encoder else 0)
        self.dims = nt.LstmDims(int(self.os_shape[0]), int(self.as_shape[0]), int(a.nr_hidden_units), int(a.obs_encoding_dim), int(a.lstm_hidden_dim),
                                options)
        poff, coff = (C.c_int64 * (nt.RLX_LSTM_POLICY_NSEG + 1))(), (C.c_int64 * (nt.RLX_LSTM_CRITIC_NSEG + 1))()
        nt.check(self.lib.rlx_lstm_param_layout(C.byref(self.dims), poff, coff), "rlx_lstm_param_layout")
        self.policy_offsets, self.critic_offsets = list(poff), list(coff)
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)
        self.policy_params, self.critic_params = z(self.policy_offsets[-1]), z(self.critic_offsets[-1])
        pol, cri = init_parameters(self.dims, self.std_dev, self.seed)
        self.load_named(pol, cri)
        self.policy_grads, self.critic_grads = torch.zeros_like(self.policy_params), torch.zeros_like(self.critic_params)
        self.policy_mu, self.policy_nu = torch.zeros_like(self.policy_params), torch.zeros_like(self.policy_params)
        self.critic_mu, self.critic_nu = torch.zeros_like(self.critic_params), torch.zeros_like(self.critic_params)
        self.policy_step = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.critic_step = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.lr_dev = z(1)
        self.opt_count = 0  # optimiser steps taken (optax `count`), drives the linear schedule of ppo_lstm.py:78-81

        self.rng = nt.Pcg64Generator(self.seed)
        torch.manual_seed(self.seed)
        low = np.asarray(self.train_env.single_action_space.low, dtype=np.float32).reshape(-1)
        high = np.asarray(self.train_env.single_action_space.high, dtype=np.float32).reshape(-1)
        A = self.dims.act_dim
        self.act_low = torch.from_numpy(np.broadcast_to(low, (A,)).copy()).to(self.device)
        self.act_high = torch.from_numpy(np.broadcast_to(high, (A,)).copy()).to(self.device)
        self.is_torch_data_interface = same_member(self.train_env.general_properties.data_interface_type, DataInterfaceType.TORCH)

        if self.save_model:
            os.makedirs(self.save_path)
            self.best_mean_return = -np.inf
            self.best_model_file_name = "best.model"

    # ------------------------------------------------------------------------------------------------ parameters
    def named_parameters(self):
        pol = {n: self.policy_params[self.policy_offsets[i]:self.policy_offsets[i + 1]] for i, n in enumerate(nt.LSTM_POLICY_SEGMENTS)}
        cri = {n: self.critic_params[self.critic_offsets[i]:self.critic_offsets[i + 1]] for i, n in enumerate(nt.LSTM_CRITIC_SEGMENTS)}
        return pol, cri

    def load_named(self, pol, cri):
        p, c = self.named_parameters()
        for name, v in pol.items():
            p[name].copy_(torch.as_tensor(v, dtype=torch.float32).reshape(-1))
        for name, v in cri.items():
            c[name].copy_(torch.as_tensor(v, dtype=torch.float32).reshape(-1))

    def current_learning_rate(self):
        """ref: linear_schedule (ppo_lstm.py:78-81): a function of the optimiser step count."""
        if not self.anneal_learning_rate:
            return self.learning_rate
        fraction = 1.0 - (self.opt_count // (self.nr_minibatches * self.nr_epochs)) / max(self.nr_updates, 1)
        return self.learning_rate * fraction

    # --------------------------------------------------------------------------------------------------- kernels
    def _workspace(self, T, n):
        key = (int(T), int(n))
        cache = self.__dict__.setdefault("_ws_cache", {})
        if key not in cache:
            nbytes = int(self.lib.rlx_lstm_minibatch_workspace_bytes(C.byref(self.dims), key[0], key[1]))
            cache[key] = (torch.zeros(nbytes // 4 + 64, dtype=torch.float32, device=self.device), nbytes)
        return cache[key]

    def _step(self, obs, c, h, noise, action, env_action, logp, value):
        n = obs.shape[0]
        ws, nbytes = self._workspace(1, n)
        a = nt.LstmStepArgs()
        a.dims, a.n = self.dims, n
        a.obs, a.c, a.h = obs.data_ptr(), c.data_ptr(), h.data_ptr()
        a.noise = noise.data_ptr() if noise is not None else None
        a.policy_params = self.policy_params.data_ptr()
        a.critic_params = self.critic_params.data_ptr() if value is not None else None
        a.act_low, a.act_high, a.clip_rescale = self.act_low.data_ptr(), self.act_high.data_ptr(), 1 if self.action_clipping_and_rescaling else 0
        a.action, a.env_action = action.data_ptr(), env_action.data_ptr()
        a.logp = logp.data_ptr() if logp is not None else None
        a.value = value.data_ptr() if value is not None else None
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        nt.check(self.lib.rlx_lstm_step_f32(C.byref(a), _stream()), "rlx_lstm_step_f32")

    def _to_dev(self, x, dtype=torch.float32):
        if torch.is_tensor(x):
            return x.to(self.device, dtype).contiguous()
        return torch.as_tensor(np.asarray(x)).to(self.device, dtype).contiguous()

    # ----------------------------------------------------------------------------------------------------- train
    def train(self):
        self.set_train_mode()
        T, N, L, dev = self.nr_steps, self.nr_envs, self.dims.lstm_dim, self.device
        obs_d, act_d = self.dims.obs_dim, self.dims.act_dim
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        states, next_states, actions = z(T, N, obs_d), z(T, N, obs_d), z(T, N, act_d)
        rewards, values, terminations, dones, log_probs, advantages, returns = (z(T, N) for _ in range(7))
        next_values = z(T, N)
        carry_c, carry_h = z(N, L), z(N, L)                      # policy.initialize_carry (policy.py:73-75)
        init_c, init_h = z(N, L), z(N, L)
        env_action = z(N, act_d)
        n_mb = self.nr_minibatch_envs
        mb = dict(states=z(T, n_mb, obs_d), actions=z(T, n_mb, act_d), log_probs=z(T, n_mb), advantages=z(T, n_mb), returns=z(T, n_mb),
                  dones=z(T, n_mb), init_c=z(n_mb, L), init_h=z(n_mb, L))
        adv_stats, stats_ws = z(2), z(T * n_mb + 2 * (T * n_mb // 256 + 1) + 8)
        idx_dev = torch.zeros(n_mb, dtype=torch.int64, device=dev)
        nr_mb_total = self.nr_epochs * self.nr_minibatches
        metrics_dev, norms_dev = z(nr_mb_total, 8), z(nr_mb_total, 2)
        opt_ws = z(max(self.policy_params.numel(), self.critic_params.numel()) // 1024 + 8)
        ws_mb, ws_mb_bytes = self._workspace(T, n_mb)
        rows_per_call = min(T * N, 32768)  # next-value pass in row blocks: the workspace is sized per call
        ws_all, ws_all_bytes = self._workspace(1, rows_per_call)

        mb_args = nt.LstmMinibatchArgs()
        mb_args.dims, mb_args.T, mb_args.n_env = self.dims, T, n_mb
        for name in ("states", "actions", "log_probs", "advantages", "returns", "dones", "init_c", "init_h"):
            setattr(mb_args, name, mb[name].data_ptr())
        mb_args.adv_stats = adv_stats.data_ptr()
        mb_args.policy_params, mb_args.critic_params = self.policy_params.data_ptr(), self.critic_params.data_ptr()
        mb_args.policy_grads, mb_args.critic_grads = self.policy_grads.data_ptr(), self.critic_grads.data_ptr()
        mb_args.clip_range, mb_args.entropy_coef, mb_args.critic_coef = float(self.clip_range), float(self.entropy_coef), float(self.critic_coef)
        mb_args.workspace, mb_args.workspace_bytes = ws_mb.data_ptr(), ws_mb_bytes
        metrics_stage, norms_stage = z(8), z(2)   # fixed targets of the captured update (copied to row k of metrics_dev / norms_dev)
        self._graph = None

        def minibatch_update(metrics_row, norms_row):
            """minibatch_update (ppo_lstm.py:193-222) on the envs listed in idx_dev: gather their columns, advantage statistics, loss +
            gradients, clip + Adam for both trees.  Every pointer is fixed for the life of train() except the two result rows."""
            for name, src, width in (("states", states, obs_d), ("actions", actions, act_d), ("log_probs", log_probs, 1),
                                     ("advantages", advantages, 1), ("returns", returns, 1), ("dones", dones, 1)):
                nt.check(self.lib.rlx_gather_env_columns_f32(src.data_ptr(), idx_dev.data_ptr(), T, N, n_mb, width, mb[name].data_ptr(), _stream()),
                         "rlx_gather_env_columns_f32")
            for name, src in (("init_c", init_c), ("init_h", init_h)):
                nt.check(self.lib.rlx_gather_env_columns_f32(src.data_ptr(), idx_dev.data_ptr(), 1, N, n_mb, L, mb[name].data_ptr(), _stream()),
                         "rlx_gather_env_columns_f32")
            nt.check(self.lib.rlx_mean_popstd_f32(mb["advantages"].data_ptr(), T * n_mb, adv_stats.data_ptr(), stats_ws.data_ptr(), _stream()),
                     "rlx_mean_popstd_f32")
            mb_args.metrics = metrics_row.data_ptr()
            nt.check(self.lib.rlx_lstm_ppo_minibatch_fwdbwd_f32(C.byref(mb_args), _stream()), "rlx_lstm_ppo_minibatch_fwdbwd_f32")
            for params, grads, mu, nu, step, col in ((self.policy_params, self.policy_grads, self.policy_mu, self.policy_nu, self.policy_step, 0),
                                                     (self.critic_params, self.critic_grads, self.critic_mu, self.critic_nu, self.critic_step, 1)):
                nt.check(self.lib.rlx_optax_clip_adam_f32(params.data_ptr(), grads.data_ptr(), mu.data_ptr(), nu.data_ptr(), params.numel(),
                                                          self.lr_dev.data_ptr(), step.data_ptr(), float(self.max_grad_norm), 0.9, 0.999, 1e-8,
                                                          norms_row[col:].data_ptr(), opt_ws.data_ptr(), _stream()), "rlx_optax_clip_adam_f32")

        saving_return_buffer = deque(maxlen=100 * self.nr_envs)
        state, _ = self.train_env.reset()
        state = self._to_dev(state)
        global_step = 0
        nr_updates = 0
        nr_episodes = 0
        steps_metrics = {}
        prev_saving_end_time = None
        logging_time_prev = None
        env = self.train_env

        while global_step < self.total_timesteps:
            start_time = time.time()
            time_metrics = {}
            if logging_time_prev:
                time_metrics["time/logging_time_prev"] = logging_time_prev

            # Acting (ppo_lstm.py:274-304)
            dones_this_rollout = 0
            dones_on_device = torch.zeros((), dtype=torch.float32, device=dev)  # TORCH envs: counted on the device, read back once per rollout
            step_info_collection = {}
            init_c.copy_(carry_c)
            init_h.copy_(carry_h)
            for step in range(T):
                states[step].copy_(state)
                noise = torch.randn(N, act_d, device=dev)
                self._step(states[step], carry_c, carry_h, noise, actions[step], env_action, log_probs[step], values[step])
                act_out = env_action if self.is_torch_data_interface else env_action.cpu().numpy()
                next_state, reward, terminated, truncated, info = env.step(act_out)
                done = terminated | truncated
                done_dev = self._to_dev(done)
                nt.check(self.lib.rlx_lstm_mask_carry_f32(carry_c.data_ptr(), carry_h.data_ptr(), done_dev.data_ptr(), N, L, _stream()),
                         "rlx_lstm_mask_carry_f32")
                state = self._to_dev(next_state)
                next_states[step].copy_(state)
                if not self.is_torch_data_interface:
                    done_np = np.asarray(done)
                    for i in np.nonzero(done_np)[0]:
                        next_states[step, int(i)] = self._to_dev(np.array(env.get_final_observation_at_index(info, int(i)), dtype=np.float32))
                        saving_return_buffer.append(env.get_final_info_value_at_index(info, "episode_return", int(i)))
                        dones_this_rollout += 1
                else:
                    dones_on_device += done_dev.sum()   # no per-step host synchronisation
                for key, info_value in env.get_logging_info_dict(info).items():
                    step_info_collection.setdefault(key, []).extend(info_value)
                rewards[step].copy_(self._to_dev(reward))
                terminations[step].copy_(self._to_dev(terminated))
                dones[step].copy_(done_dev)
                global_step += N
            dones_this_rollout += int(dones_on_device.item())
            nr_episodes += dones_this_rollout
            acting_end_time = time.time()
            time_metrics["time/acting_time"] = acting_end_time - start_time

            # Calculating advantages and returns (ppo_lstm.py:121-138)
            flat_next, flat_nv = next_states.view(T * N, obs_d), next_values.view(T * N)
            for r0 in range(0, T * N, rows_per_call):
                r1 = min(T * N, r0 + rows_per_call)
                nt.check(self.lib.rlx_lstm_critic_forward_f32(C.byref(self.dims), self.critic_params.data_ptr(), flat_next[r0:r1].data_ptr(), r1 - r0,
                                                              flat_nv[r0:r1].data_ptr(), ws_all.data_ptr(), ws_all_bytes, _stream()),
                         "rlx_lstm_critic_forward_f32")
            nt.check(self.lib.rlx_gae_f32(rewards.data_ptr(), terminations.data_ptr(), values.data_ptr(), next_values.data_ptr(), None, T, N,
                                          float(self.gamma), float(self.gae_lambda), advantages.data_ptr(), returns.data_ptr(), _stream()), "rlx_gae_f32")
            calc_adv_return_end_time = time.time()
            time_metrics["time/calc_adv_and_return_time"] = calc_adv_return_end_time - acting_end_time

            # Optimizing (ppo_lstm.py:141-231)
            k = 0
            for epoch in range(self.nr_epochs):
                perm = np.arange(N)
                self.rng.shuffle(perm)  # one independent env permutation per epoch (ppo_lstm.py:189-191)
                for m in range(self.nr_minibatches):
                    idx_dev.copy_(torch.from_numpy(perm[m * n_mb:(m + 1) * n_mb]))
                    lr_used = self.current_learning_rate()
                    self.lr_dev.fill_(lr_used)
                    if not self.use_cuda_graph:
                        minibatch_update(metrics_dev[k], norms_dev[k])
                    else:
                        # every launch of a minibatch update works on fixed buffers (the env indices and the learning rate are device-side
                        # inputs written just above), so the ~400 launches are captured once and replayed: the recurrence is a chain of
                        # small dependent kernels and eager launches leave the device idle between them
                        if self._graph is None:
                            minibatch_update(metrics_stage, norms_stage)   # the first update runs eagerly (it also warms every kernel up) ...
                            self._graph = torch.cuda.CUDAGraph()
                            before = int(self.lib.rlx_launch_count())
                            with torch.cuda.graph(self._graph, capture_error_mode="thread_local"):   # ... then recorded (recording executes nothing)
                                minibatch_update(metrics_stage, norms_stage)
                            self._graph_launches = int(self.lib.rlx_launch_count()) - before
                        else:
                            self._graph.replay()
                            self.lib.rlx_add_launch_count(self._graph_launches)
                        metrics_dev[k].copy_(metrics_stage)
                        norms_dev[k].copy_(norms_stage)
                    self.opt_count += 1
                    k += 1
            m_host, n_host = metrics_dev.cpu().numpy(), norms_dev.cpu().numpy()  # the iteration's only device->host metric transfer
            optimization_metrics = {
                "loss/policy_gradient_loss": m_host[:, 0].mean(), "loss/critic_loss": m_host[:, 1].mean(), "loss/entropy_loss": m_host[:, 2].mean(),
                "policy_ratio/approx_kl": m_host[:, 3].mean(), "policy_ratio/clip_fraction": m_host[:, 4].mean(),
                "gradients/policy_grad_norm": n_host[:, 0].mean(), "gradients/critic_grad_norm": n_host[:, 1].mean(),
                "lr/learning_rate": lr_used,  # hyperparams["learning_rate"] of the last optimiser step (ppo_lstm.py:226)
                "v_value/explained_variance": float(1 - torch.var(returns - values, unbiased=False) / (torch.var(returns, unbiased=False) + 1e-8)),
                "policy/std_dev": float(torch.exp(self.named_parameters()[0]["logstd"]).mean()),
            }
            nr_updates += self.nr_epochs * self.nr_minibatches
            optimizing_end_time = time.time()
            time_metrics["time/optimizing_time"] = optimizing_end_time - calc_adv_return_end_time

            # Evaluating (ppo_lstm.py:319-343)
            evaluation_metrics = {}
            if global_step % self.evaluation_frequency == 0 and self.evaluation_frequency != -1:
                evaluation_metrics = self._evaluate()
            evaluating_end_time = time.time()
            time_metrics["time/evaluating_time"] = evaluating_end_time - optimizing_end_time

            # Saving
            if self.save_model and dones_this_rollout > 0 and len(saving_return_buffer) > 0:
                mean_return = np.mean(saving_return_buffer)
                if mean_return > self.best_mean_return:
                    self.best_mean_return = mean_return
                    self.save()
            saving_end_time = time.time()
            if prev_saving_end_time:
                time_metrics["time/sps"] = int((self.nr_steps * self.nr_envs) / (saving_end_time - prev_saving_end_time))
            prev_saving_end_time = saving_end_time
            time_metrics["time/saving_time"] = saving_end_time - evaluating_end_time

            # Logging (ppo_lstm.py:363-388)
            self.start_logging(global_step)
            steps_metrics["steps/nr_env_steps"] = global_step
            steps_metrics["steps/nr_updates"] = nr_updates
            steps_metrics["steps/nr_episodes"] = nr_episodes
            rollout_info_metrics, env_info_metrics = {}, {}
            for info_name, vals in step_info_collection.items():
                metric_group = "rollout" if info_name in ["episode_return", "episode_length"] else "env_info"
                metric_dict = rollout_info_metrics if metric_group == "rollout" else env_info_metrics
                mean_value = np.mean(vals)
                if mean_value == mean_value:
                    metric_dict[f"{metric_group}/{info_name}"] = mean_value
            combined = {**rollout_info_metrics, **evaluation_metrics, **env_info_metrics, **steps_metrics, **time_metrics, **optimization_metrics}
            for key, value in combined.items():
                self.log(f"{key}", value, global_step)
            self.end_logging()
            logging_end_time = time.time()
            logging_time_prev = logging_end_time - saving_end_time

    # ------------------------------------------------------------------------------------------------ eval / test
    def _deterministic_rollout(self, episodes):
        """ref: the evaluation loop (ppo_lstm.py:319-343) / test (:470-489): get_deterministic_action with the carry reset on done."""
        env = self.eval_env
        state, _ = env.reset()
        state = self._to_dev(state)
        n, L, act_d = state.shape[0], self.dims.lstm_dim, self.dims.act_dim
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)
        c, h, action, env_action = z(n, L), z(n, L), z(n, act_d), z(n, act_d)
        out = {"eval/episode_return": [], "eval/episode_length": []}
        finished = 0
        while finished < episodes:
            self._step(state, c, h, None, action, env_action, None, None)
            act_out = env_action if self.is_torch_data_interface else env_action.cpu().numpy()
            state, _, terminated, truncated, info = env.step(act_out)
            state = self._to_dev(state)
            done = terminated | truncated
            done_dev = self._to_dev(done)
            nt.check(self.lib.rlx_lstm_mask_carry_f32(c.data_ptr(), h.data_ptr(), done_dev.data_ptr(), n, L, _stream()), "rlx_lstm_mask_carry_f32")
            for i in np.nonzero(done_dev.cpu().numpy() > 0)[0]:
                finished += 1
                out["eval/episode_return"].append(env.get_final_info_value_at_index(info, "episode_return", int(i)))
                out["eval/episode_length"].append(env.get_final_info_value_at_index(info, "episode_length", int(i)))
                if finished == episodes:
                    break
        return out

    def _evaluate(self):
        self.set_eval_mode()
        metrics = {k: np.mean(v) for k, v in self._deterministic_rollout(self.evaluation_episodes).items()}
        self.set_train_mode()
        return metrics

    def test(self, episodes):
        self.set_eval_mode()
        out = self._deterministic_rollout(episodes)
        for i, r in enumerate(out["eval/episode_return"]):
            rlx_logger.info(f"Episode {i + 1} - Return: {r}")

    # ----------------------------------------------------------------------------------------------- checkpointing
    def save(self):
        """Named flat tensors + optimiser moments (the reference writes an Orbax tree, ppo_lstm.py:431-449; Orbax is not in this image)."""
        pol, cri = self.named_parameters()
        torch.save({"config_algorithm": dict(self.config.algorithm), "policy": {k: v.cpu() for k, v in pol.items()},
                    "critic": {k: v.cpu() for k, v in cri.items()},
                    "optimizer": {"policy_mu": self.policy_mu.cpu(), "policy_nu": self.policy_nu.cpu(), "critic_mu": self.critic_mu.cpu(),
                                  "critic_nu": self.critic_nu.cpu(), "count": self.opt_count}},
                   os.path.join(self.save_path, self.best_model_file_name))

    @classmethod
    def load(cls, config, train_env, eval_env, run_path, writer, explicitly_set_algorithm_params):
        ck = torch.load(config.runner.load_model, weights_only=False)
        for key, value in ck["config_algorithm"].items():
            if f"algorithm.{key}" not in explicitly_set_algorithm_params and key in config.algorithm and key not in ("name", "device"):
                config.algorithm[key] = value
        model = cls(config, train_env, eval_env, run_path, writer)
        model.load_named(ck["policy"], ck["critic"])
        o = ck["optimizer"]
        model.policy_mu.copy_(o["policy_mu"]); model.policy_nu.copy_(o["policy_nu"])
        model.critic_mu.copy_(o["critic_mu"]); model.critic_nu.copy_(o["critic_nu"])
        model.opt_count = int(o["count"])
        model.policy_step.fill_(model.opt_count)
        model.critic_step.fill_(model.opt_count)
        return model

    # ----------------------------------------------------------------------------------------------------- logging
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
        from rl_x_b200.algorithms.ppo_lstm.b200.general_properties import GeneralProperties
        return GeneralProperties
