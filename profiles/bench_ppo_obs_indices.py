#!/usr/bin/env python
"""What observation index sets cost the PPO iteration: BASELINE config 2 (4096 synthetic envs x 128 steps, obs 376, act 17, hidden 256,
minibatch 32768, 10 epochs) on the wgmma engine, once with both nets reading every column (identity: no embed, no fold) and once
locomotion-like (the policy reads 188 permuted columns, the critic all 376 in permuted order: every call that reads layer 1 embeds W1p / W1c
into the [2H, obs] matrix first, and the layer-1 gradient is folded back).  Prints one JSON line:

    python profiles/bench_ppo_obs_indices.py [--steps K] [--warmup W] [--rounds R]

The two models are timed in alternating rounds (CUDA events around K whole iterations); then one iteration of the asymmetric model runs
under torch.profiler to give the launches and summed kernel time of ppo_embed_w1_kernel.  Card name and power limit are read in the same
process.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OBS, ACT, HID, N_ENVS, T, MB = 376, 17, 256, 4096, 128, 32768


def build(epochs, asymmetric):
    from rl_x_b200.runner.runner import Runner
    import numpy as np
    argv = [f"--environment.nr_envs={N_ENVS}", f"--environment.obs_dim={OBS}", f"--environment.act_dim={ACT}", "--environment.seed=1",
            "--environment.data_interface=torch", "--environment.horizon=1000", "--environment.stream=fresh", f"--algorithm.nr_steps={T}",
            f"--algorithm.nr_epochs={epochs}", f"--algorithm.minibatch_size={MB}", f"--algorithm.nr_hidden_units={HID}", "--algorithm.gemm_engine=tcgen05",
            "--algorithm.total_timesteps=1e15"]
    r = Runner(argv=argv)
    env, eval_env = r._create_train_and_eval_env(r._config)
    if asymmetric:
        rng = np.random.default_rng(0)
        env.policy_observation_indices = rng.permutation(OBS)[:OBS // 2]
        env.critic_observation_indices = rng.permutation(OBS)
    model = r._model_class(r._config, env, eval_env, "/tmp/rlx_bench_obs_indices", None)
    model.log = lambda *a, **k: None
    model._begin_training()
    return model


def timed(model, steps):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        model._train_iteration()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def embed_profile(model):
    """(launches, summed device ms) of ppo_embed_w1_kernel and of all kernels in one iteration, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model._train_iteration()
        torch.cuda.synchronize()
    n = ms = total = 0.0
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        dt = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += dt
        if "ppo_embed_w1_kernel" in ev.name:
            n += 1
            ms += dt
    return int(n), ms / 1e3, total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--epochs", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ppo_obs_indices: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    models = {"identity": build(args.epochs, False), "asymmetric": build(args.epochs, True)}
    for m in models.values():
        for _ in range(args.warmup):
            m._train_iteration()
    ms = {k: [] for k in models}
    for _ in range(args.rounds):
        for k, m in models.items():
            ms[k].append(timed(m, args.steps))
    n, embed_ms, all_ms = embed_profile(models["asymmetric"])
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    print(json.dumps({
        "card": card, "config": f"{N_ENVS} envs x {T} steps, obs {OBS}, act {ACT}, hidden {HID}, minibatch {MB}, {args.epochs} epochs, wgmma engine",
        "asymmetric_sets": f"policy {OBS // 2} permuted columns, critic all {OBS} permuted",
        "ms_per_iteration": ms, "mean_ms": mean, "asymmetric_over_identity": mean["asymmetric"] / mean["identity"],
        "embed_launches_per_iteration": n, "embed_kernel_ms_per_iteration": embed_ms, "all_kernels_ms_per_iteration": all_ms,
        "embed_share_of_kernel_time": embed_ms / max(all_ms, 1e-9), "time": time.strftime("%Y-%m-%d %H:%M:%S")}))


if __name__ == "__main__":
    main()
