#!/usr/bin/env python
"""FastTD3 at the reference's defaults on one GPU: batch 32768, 2 critic updates + 1 policy update per environment step, 101 atoms, on the
synthetic Box (obs 376, act 17), 1024 envs x buffer_size_per_env 1024 (~3.2 GB of ring).  Prints one JSON line:

    python profiles/bench_fasttd3.py [--steps K] [--warmup W] [--rounds R] [--policy-cols P] [--critic-cols C]

Times the exact-fp32 SIMT engine and the wgmma 3xTF32 engine in alternating rounds; the tensor engine is timed only after an agreement
check in a subprocess (tests/test_gpu_zzzzz_fasttd3.py::test_fasttd3_engines_agree_at_batch_1024) has passed.  Reported per engine: ms per
environment step (the optimising step: acting + sampling + normalising + the three updates) and per update, kernel_ms per kernel class
(rlx_timing_begin / rlx_timing_end), the algorithmic FLOPs computed from the layer shapes, the fraction of the 3xTF32 ceiling they imply
(dense BF16 peak / 6, DESIGN.md 3) and the number of products that ran on the tensor engine.

--policy-cols / --critic-cols give the environment observation index sets (asymmetric actor-critic): each a seeded permutation of that
many of the 376 columns.  Then the rounds alternate the identity network and the one with the sets, both on the wgmma engine, and the
sets leg also reports gather_ms_per_env_step: the kernel time of the column-gather launches (gather_cols_kernel, concat_kernel) of two
critic updates, a policy update and an acting step, from torch.profiler.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OBS, ACT, ATOMS, N_ENVS, BATCH = 376, 17, 101, 1024, 32768
H100_DENSE_BF16_TFLOPS = 989.4   # H100 SXM dense BF16 peak


def algorithmic_flops(obs=OBS, act=ACT, atoms=ATOMS, batch=BATCH, ncu=2, policy_cols=None, critic_cols=None):
    """2 x multiply-adds per environment step from the layer shapes (forward 1x, input gradient 1x, weight gradient 1x).  policy_cols /
    critic_cols: the layer-1 observation widths P and C with index sets (None = obs)."""
    P = obs if policy_cols is None else policy_cols
    Cc = obs if critic_cols is None else critic_cols
    pol = P * 512 + 512 * 256 + 256 * 128 + 128 * act
    q = (Cc + act) * 1024 + 1024 * 512 + 512 * 256 + 256 * atoms
    q_dx = q - (Cc + act) * 1024 + 1024 * act      # input gradient: no dX of the first layer except its action columns
    critic = pol + 2 * q + 2 * q + 2 * (q - (Cc + act) * 1024)   # pi(s'), 2 target fwd, 2 online fwd, 2 bwd (dW all, dX all but layer 1)
    critic += 2 * q                                               # ... and the weight gradients
    policy = pol + 2 * q + 2 * q_dx + 2 * pol                     # pi(s), 2 Q fwd, Q bwd to the actions, policy bwd (dX + dW)
    return 2.0 * batch * (ncu * critic + policy), 2.0 * batch * critic, 2.0 * batch * policy


def index_sets(policy_cols, critic_cols, seed=0):
    """Seeded permutations of policy_cols / critic_cols of the OBS columns (None: no set)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    return tuple(None if k is None else rng.permutation(OBS)[:k].astype(np.int64) for k in (policy_cols, critic_cols))


def make_model(engine, sets=(None, None)):
    import torch
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    from rl_x_b200.algorithms.fasttd3.b200.fasttd3 import FastTD3
    from rl_x_b200.environments.synthetic.box.create_env import create_train_and_eval_env
    from rl_x_b200.environments.synthetic.box.default_config import get_config as env_config
    e = env_config("synthetic.box")
    e.nr_envs = N_ENVS
    a = get_config("fasttd3.b200")
    a.buffer_size_per_env, a.gemm_engine = 1024, engine
    cfg = ConfigDict(algorithm=a, environment=e, runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    train_env, eval_env = create_train_and_eval_env(cfg)
    for env in (train_env, eval_env):
        for attr, ind in zip(("policy_observation_indices", "critic_observation_indices"), sets):
            if ind is not None:
                setattr(env, attr, ind)
    model = FastTD3(cfg, train_env, eval_env, tempfile.mkdtemp(), None)
    model.log = lambda *a_, **k: None
    torch.cuda.synchronize()
    return model


def gather_ms(model, reps=3):
    """Kernel time (ms) of the column-gather launches per environment step: 2 critic updates, 1 policy update and 1 acting step on random
    batches of the bench's shape, under torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    g, dev, n, A = torch.Generator(device="cuda").manual_seed(0), model.device, model.batch_size, model.dims.act_dim
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    s, ns, a = r(n, OBS), r(n, OBS), torch.rand(n, A, device=dev, generator=g) * 2 - 1
    rew, z, eff, m = r(n), torch.zeros(n, device=dev), torch.ones(n, device=dev), torch.zeros(8, device=dev)
    obs = r(N_ENVS, OBS)
    scales = model.draw_noise_scales()

    def step():
        for _ in range(model.nr_critic_updates_per_policy_update):
            model.critic_update(s, ns, a, rew, z, z, eff, m)
        model.policy_update(s, m)
        model.get_action(obs, scales)

    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            step()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "gather_cols_kernel" in e.key or "concat_kernel" in e.key)
    return us / 1e3 / reps


def time_engine(engine, steps, warmup, sets=(None, None)):
    """A model trained for learning_starts + warmup + steps environment steps; the last `steps` optimising steps are timed with CUDA events."""
    import torch
    from rl_x_b200 import _native as nt
    model = make_model(engine, sets)
    marks, state = [], {}
    orig_critic, orig_policy = model.critic_update, model.policy_update
    per_update = {"critic": [], "policy": []}

    def timed(kind, fn):
        def run(*a, **k):
            if state.get("timing"):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn(*a, **k)
                e.record()
                per_update[kind].append((s, e))
            else:
                fn(*a, **k)
        return run

    model.critic_update, model.policy_update = timed("critic", orig_critic), timed("policy", orig_policy)
    starts = model.learning_starts
    model.total_timesteps = (starts + warmup + steps) * N_ENVS
    orig_normalize = model.normalize
    counter = {"step": 0}

    def normalize(x, update):   # called once per acting step with update=False: marks the environment steps
        if not update:
            counter["step"] += 1
            if counter["step"] == starts + warmup + 1:
                torch.cuda.synchronize()
                state["timing"] = True
                nt.timing_begin()
                state["tc0"] = int(model.lib.rlx_aux_tc_gemm_count())
                ev = torch.cuda.Event(enable_timing=True)
                ev.record()
                marks.append(ev)
        return orig_normalize(x, update)

    model.normalize = normalize
    model.train()
    end = torch.cuda.Event(enable_timing=True)
    end.record()
    torch.cuda.synchronize()
    kernels = nt.timing_end()
    total_ms = marks[0].elapsed_time(end)
    upd = {k: sum(s.elapsed_time(e) for s, e in v) / max(len(v), 1) for k, v in per_update.items()}
    out = dict(ms_per_env_step=total_ms / steps, ms_per_critic_update=upd["critic"], ms_per_policy_update=upd["policy"],
               kernel_ms={k: round(v["ms"] / steps, 4) for k, v in kernels.items() if v["launches"]},
               kernel_ms_total=sum(v["ms"] for v in kernels.values()) / steps, tensor_gemms=int(model.lib.rlx_aux_tc_gemm_count()) - state["tc0"])
    if any(x is not None for x in sets):
        model.critic_update, model.policy_update = orig_critic, orig_policy
        out["gather_ms_per_env_step"] = round(gather_ms(model), 4)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--policy-cols", type=int, help="policy observation index set: a seeded permutation of this many columns")
    p.add_argument("--critic-cols", type=int, help="critic observation index set: a seeded permutation of this many columns")
    p.add_argument("--engine", choices=["simt", "tcgen05"], help=argparse.SUPPRESS)   # one leg, in a child process
    p.add_argument("--with-sets", action="store_true", help=argparse.SUPPRESS)
    args = p.parse_args()
    with_cols = args.policy_cols is not None or args.critic_cols is not None
    if args.engine:
        sets = index_sets(args.policy_cols, args.critic_cols) if args.with_sets else (None, None)
        print(json.dumps(time_engine(args.engine, args.steps, args.warmup, sets)))
        return
    import torch
    props = torch.cuda.get_device_properties(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                               timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        power = f"unavailable ({exc})"
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    check = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_zzzzz_fasttd3.py"), "-q", "-p", "no:cacheprovider",
                            "-k", "engines_agree"], env=dict(env, RLX_AUX_GEMM_ENGINE="1"), cwd=ROOT, capture_output=True, text=True, timeout=900)
    tc_ok = check.returncode == 0
    if with_cols:   # identity and index-set networks alternate on one engine
        eng = "tcgen05" if tc_ok else "simt"
        legs = {f"{eng}_identity": (eng, False), f"{eng}_sets": (eng, True)}
    else:
        legs = {k: (k, False) for k in (["simt", "tcgen05"] if tc_ok else ["simt"])}
    cols = []
    for flag, v in (("--policy-cols", args.policy_cols), ("--critic-cols", args.critic_cols)):
        cols += [flag, str(v)] if v is not None else []
    runs = {k: [] for k in legs}
    for _ in range(args.rounds):
        for leg, (eng, sets) in legs.items():   # alternating, each leg in a fresh process
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--engine", eng, "--steps", str(args.steps), "--warmup", str(args.warmup)]
                                 + cols + (["--with-sets"] if sets else []), env=env, cwd=ROOT, capture_output=True, text=True, timeout=3000)
            if out.returncode != 0:
                raise RuntimeError(out.stdout[-2000:] + out.stderr[-4000:])
            runs[leg].append(json.loads(out.stdout.strip().splitlines()[-1]))
    flops, critic_flops, policy_flops = algorithmic_flops()
    ceiling_tflops = H100_DENSE_BF16_TFLOPS / 6
    result = dict(workload="fasttd3.b200 synthetic.box obs376 act17 atoms101 batch32768 2 critic + 1 policy updates/step, 1024 envs x 1024",
                  policy_cols=args.policy_cols, critic_cols=args.critic_cols,
                  gpu=props.name, power_limit_w=power, steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                  algorithmic_gflop_per_env_step=round(flops / 1e9, 1), critic_update_gflop=round(critic_flops / 1e9, 1),
                  policy_update_gflop=round(policy_flops / 1e9, 1), bound_ms_3xtf32=round(flops / (ceiling_tflops * 1e12) * 1e3, 2),
                  tensor_engine_agreement=tc_ok, tensor_engine_check_tail=None if tc_ok else (check.stdout + check.stderr)[-1500:])
    for leg, rs in runs.items():
        best = min(rs, key=lambda r: r["ms_per_env_step"])
        best["all_ms_per_env_step"] = [round(r["ms_per_env_step"], 3) for r in rs]
        leg_flops = algorithmic_flops(policy_cols=args.policy_cols, critic_cols=args.critic_cols)[0] if legs[leg][1] else flops
        best["algorithmic_gflop_per_env_step"] = round(leg_flops / 1e9, 1)
        best["fraction_of_3xtf32_ceiling"] = round(leg_flops / (best["kernel_ms_total"] * 1e-3) / (ceiling_tflops * 1e12), 4)
        result[leg] = best
    print(json.dumps(result))


if __name__ == "__main__":
    main()
