#!/usr/bin/env python
"""Golden vectors of the FastTD3 update, made by EXECUTING the unmodified reference (rl_x/algorithms/fasttd3/pytorch/fasttd3.py) on CPU,
fp32 (bf16 autocast off).  Build container only:

    TORCHDYNAMO_DISABLE=1 python tests/golden/make_golden_fasttd3.py

Captured: the sampled batches (ReplayBuffer.sample is wrapped), every torch.randn_like draw (acting noise [nr_envs, act], target-policy
smoothing noise [batch, act] per critic update) and every torch.rand draw (the per-environment exploration scales), the
observation-normaliser statistics before each optimising step, the logged metrics (logging_frequency = nr_envs: every logged value is the
mean over that step's policy updates) and, at the end, all small parameter tensors plus every 61st element of the large matrices.
Initial parameters are NOT stored: the tests rebuild them by constructing the same torch modules in the same order under
torch.manual_seed(seed), as FastTD3.__init__ does (fasttd3.py:80-85).  Output: tests/golden/fasttd3_update.npz, fasttd3_update_variant.npz
"""
import os
import sys

os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_ppo import ConfigDict  # noqa: E402  (installs the ml_collections stub, adds the reference to sys.path)

import rl_x.algorithms.fasttd3.pytorch.fasttd3 as ref  # noqa: E402
import rl_x.algorithms.fasttd3.pytorch.replay_buffer as refrb  # noqa: E402
from rl_x.algorithms.fasttd3.pytorch.default_config import get_config  # noqa: E402
from make_golden_fastsac import SyntheticTorchEnv  # noqa: E402

STRIDE = 61


def run(tag="update", N=4, obs=7, act=3, batch=16, n_steps=1, steps=9, seed=4, ncu=2, npu=2, clipped=True, max_grad_norm=-1.0, clip_rescale=False,
        anneal=False, smoothing_epsilon=None):
    torch.set_num_threads(1)
    batches, randn_draws, rand_draws, norm_states = [], [], [], []

    class SpyRB(refrb.ReplayBuffer):
        def sample(self, n):
            out = super().sample(n)
            batches.append([t.numpy().copy() for t in out])
            return out

    ref.ReplayBuffer = SpyRB
    orig_randn_like, orig_rand = torch.randn_like, torch.rand

    def spy_randn_like(x, *a, **k):
        y = orig_randn_like(x, *a, **k)
        randn_draws.append(y.numpy().copy())
        return y

    def spy_rand(*a, **k):
        y = orig_rand(*a, **k)
        if k.get("generator") is None:   # the environment's own generator is not the reference's
            rand_draws.append(y.numpy().copy())
        return y

    torch.randn_like, torch.rand = spy_randn_like, spy_rand
    cfg = ConfigDict(algorithm=get_config("fasttd3.pytorch"), environment=ConfigDict(seed=seed, nr_envs=N),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False))
    a = cfg.algorithm
    a.device, a.bf16_mixed_precision_training, a.compile_mode = "cpu", False, "default"
    a.batch_size, a.buffer_size_per_env, a.learning_starts, a.total_timesteps, a.n_steps = batch, 8, 3, N * steps, n_steps
    a.nr_critic_updates_per_policy_update, a.nr_policy_updates_per_step, a.logging_frequency, a.save_frequency = ncu, npu, N, -1
    a.learning_rate, a.clipped_double_q_learning, a.max_grad_norm = 1e-3, clipped, max_grad_norm
    a.action_clipping_and_rescaling, a.anneal_learning_rate = clip_rescale, anneal
    if smoothing_epsilon is not None:
        a.smoothing_epsilon = smoothing_epsilon
    env = SyntheticTorchEnv(N, obs, act, seed + 100)
    try:
        model = ref.FastTD3(cfg, env, env, "/tmp/golden_fasttd3", None)
        nrm = model.observation_normalizer
        orig_normalize = nrm.normalize

        def normalize(observations, update=True):
            if update:
                norm_states.append([nrm.running_mean.numpy().copy(), nrm.running_var.numpy().copy(), int(nrm.count)])
            return orig_normalize(observations, update=update)

        nrm.normalize = normalize
        metrics = []
        model.log = lambda name, value, step: metrics.append((name, float(value), int(step)))
        model.train()
    finally:
        torch.randn_like, torch.rand = orig_randn_like, orig_rand
    out = {}
    nopt = len(batches)
    for u, b in enumerate(batches):
        for name, arr in zip(["states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps"], b):
            out[f"step{u}/{name}"] = arr
        out[f"step{u}/norm_mean"], out[f"step{u}/norm_var"], out[f"step{u}/norm_count"] = norm_states[2 * u][0], norm_states[2 * u][1], np.array(norm_states[2 * u][2])
    smooth = [x for x in randn_draws if x.shape == (batch, act)]
    acting = [x for x in randn_draws if x.shape == (N, act)]
    assert len(smooth) == nopt * npu * ncu and len(acting) == steps, (len(smooth), len(acting), nopt)
    for u in range(nopt):
        out[f"step{u}/smoothing_noise"] = np.stack(smooth[u * npu * ncu:(u + 1) * npu * ncu])   # order of use: critic updates (i, j)
    out["acting_noise"] = np.stack(acting)                  # [steps, N, act]
    out["noise_scale_draws"] = np.stack(rand_draws)         # [steps + 1, N, 1]: the initial scales, then one redraw per step
    for n in sorted({m[0] for m in metrics}):
        if not n.startswith("time/"):
            out[f"metric/{n}"] = np.array([m[1] for m in metrics if m[0] == n])

    def put(prefix, sd):
        for k, v in sd.items():
            v = v.detach().numpy().reshape(-1)
            out[f"{prefix}/{k.replace('_orig_mod.', '')}"] = v.copy() if v.size <= 2048 else v[::STRIDE].copy()

    for name, mod in [("policy", model.policy), ("q1", model.critic.q1), ("q2", model.critic.q2), ("q1_target", model.critic.q1_target),
                      ("q2_target", model.critic.q2_target)]:
        put(f"final/{name}", mod.state_dict())
    out["final/norm_mean"], out["final/norm_var"], out["final/norm_count"] = nrm.running_mean.numpy().copy(), nrm.running_var.numpy().copy(), np.array(int(nrm.count))
    out["meta"] = np.array([N, obs, act, batch, n_steps, nopt, seed, ncu, npu, a.nr_atoms, STRIDE, steps], dtype=np.int64)
    out["meta_f"] = np.array([a.gamma, a.tau, a.learning_rate, a.v_min, a.v_max, a.weight_decay, 0.9, 0.999, a.noise_std_min, a.noise_std_max,
                              a.smoothing_epsilon, a.smoothing_clip_value, -1.5, 0.5, float(clipped), max_grad_norm, float(clip_rescale), float(anneal)],
                             dtype=np.float64)
    path = os.path.join(HERE, f"fasttd3_{tag}.npz")
    np.savez_compressed(path, **out)
    print("->", path, os.path.getsize(path) // 1024, "KiB; optimising steps:", nopt, "metrics:", sorted({m[0] for m in metrics if not m[0].startswith("time/")}))
    print({n: out[f"metric/{n}"][:3] for n in ["loss/q_loss", "loss/policy_loss", "gradients/critic_grad_norm"]})


if __name__ == "__main__":
    run()   # reference defaults: clipped double-Q, n_steps = 1, no gradient clipping
    # the non-default options: mean-of-two-critics targets / actor loss, n-step returns, clip_grad_norm_, clipped and rescaled env actions,
    # annealed learning rate, and a smoothing scale at which the smoothing clip (0.5) is reached by some draws
    run("update_variant", n_steps=3, seed=6, clipped=False, max_grad_norm=0.5, clip_rescale=True, anneal=True, smoothing_epsilon=0.3)
    # default config and model-class method signatures of the reference's FastTD3 (the five-algorithm reference_surface.json stays as it is)
    import json
    import runpy
    from make_golden_reference_surface import class_methods
    ref_root = "/root/reference"
    cfg = runpy.run_path(os.path.join(ref_root, "rl_x/algorithms/fasttd3/pytorch/default_config.py"))["get_config"]("x")
    surface = {"config": {k: cfg[k] for k in cfg}, "class": "FastTD3",
               "methods": class_methods(os.path.join(ref_root, "rl_x/algorithms/fasttd3/pytorch/fasttd3.py"), "FastTD3")}
    with open(os.path.join(HERE, "fasttd3_reference_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=1, sort_keys=True)
        fh.write("\n")
