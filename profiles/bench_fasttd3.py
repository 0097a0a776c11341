#!/usr/bin/env python
"""FastTD3 at the reference's defaults on one GPU: batch 32768, 2 critic updates + 1 policy update per environment step, 101 atoms, on the
synthetic Box (obs 376, act 17), 1024 envs x buffer_size_per_env 1024 (~3.2 GB of ring).  Prints one JSON line:

    python profiles/bench_fasttd3.py [--steps K] [--warmup W] [--rounds R]

Times the exact-fp32 SIMT engine and the wgmma 3xTF32 engine in alternating rounds; the tensor engine is timed only after an agreement
check in a subprocess (tests/test_gpu_zzzzz_fasttd3.py::test_fasttd3_engines_agree_at_batch_1024) has passed.  Reported per engine: ms per
environment step (the optimising step: acting + sampling + normalising + the three updates) and per update, kernel_ms per kernel class
(rlx_timing_begin / rlx_timing_end), the algorithmic FLOPs computed from the layer shapes, the fraction of the 3xTF32 ceiling they imply
(dense BF16 peak / 6, DESIGN.md 3) and the number of products that ran on the tensor engine.  Writes nothing into the tree."""
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


def algorithmic_flops(obs=OBS, act=ACT, atoms=ATOMS, batch=BATCH, ncu=2):
    """2 x multiply-adds per environment step from the layer shapes (forward 1x, input gradient 1x, weight gradient 1x)."""
    pol = obs * 512 + 512 * 256 + 256 * 128 + 128 * act
    q = (obs + act) * 1024 + 1024 * 512 + 512 * 256 + 256 * atoms
    q_dx = q - (obs + act) * 1024 + 1024 * act      # input gradient: no dX of the first layer except its action columns
    critic = pol + 2 * q + 2 * q + 2 * (q - (obs + act) * 1024)   # pi(s'), 2 target fwd, 2 online fwd, 2 bwd (dW all, dX all but layer 1)
    critic += 2 * q                                               # ... and the weight gradients
    policy = pol + 2 * q + 2 * q_dx + 2 * pol                     # pi(s), 2 Q fwd, Q bwd to the actions, policy bwd (dX + dW)
    return 2.0 * batch * (ncu * critic + policy), 2.0 * batch * critic, 2.0 * batch * policy


def make_model(engine):
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
    model = FastTD3(cfg, train_env, eval_env, tempfile.mkdtemp(), None)
    model.log = lambda *a_, **k: None
    torch.cuda.synchronize()
    return model


def time_engine(engine, steps, warmup):
    """A model trained for learning_starts + warmup + steps environment steps; the last `steps` optimising steps are timed with CUDA events."""
    import torch
    from rl_x_b200 import _native as nt
    model = make_model(engine)
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
    return dict(ms_per_env_step=total_ms / steps, ms_per_critic_update=upd["critic"], ms_per_policy_update=upd["policy"],
                kernel_ms={k: round(v["ms"] / steps, 4) for k, v in kernels.items() if v["launches"]},
                kernel_ms_total=sum(v["ms"] for v in kernels.values()) / steps, tensor_gemms=int(model.lib.rlx_aux_tc_gemm_count()) - state["tc0"])


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--engine", choices=["simt", "tcgen05"], help=argparse.SUPPRESS)   # one leg, in a child process
    args = p.parse_args()
    if args.engine:
        print(json.dumps(time_engine(args.engine, args.steps, args.warmup)))
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
    legs = ["simt", "tcgen05"] if tc_ok else ["simt"]
    runs = {k: [] for k in legs}
    for _ in range(args.rounds):
        for leg in legs:   # alternating, each leg in a fresh process
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--engine", leg, "--steps", str(args.steps), "--warmup", str(args.warmup)],
                                 env=env, cwd=ROOT, capture_output=True, text=True, timeout=3000)
            if out.returncode != 0:
                raise RuntimeError(out.stdout[-2000:] + out.stderr[-4000:])
            runs[leg].append(json.loads(out.stdout.strip().splitlines()[-1]))
    flops, critic_flops, policy_flops = algorithmic_flops()
    ceiling_tflops = H100_DENSE_BF16_TFLOPS / 6
    result = dict(workload="fasttd3.b200 synthetic.box obs376 act17 atoms101 batch32768 2 critic + 1 policy updates/step, 1024 envs x 1024",
                  gpu=props.name, power_limit_w=power, steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                  algorithmic_gflop_per_env_step=round(flops / 1e9, 1), critic_update_gflop=round(critic_flops / 1e9, 1),
                  policy_update_gflop=round(policy_flops / 1e9, 1), bound_ms_3xtf32=round(flops / (ceiling_tflops * 1e12) * 1e3, 2),
                  tensor_engine_agreement=tc_ok, tensor_engine_check_tail=None if tc_ok else (check.stdout + check.stderr)[-1500:])
    for leg, rs in runs.items():
        best = min(rs, key=lambda r: r["ms_per_env_step"])
        best["all_ms_per_env_step"] = [round(r["ms_per_env_step"], 3) for r in rs]
        best["fraction_of_3xtf32_ceiling"] = round(flops / (best["kernel_ms_total"] * 1e-3) / (ceiling_tflops * 1e12), 4)
        result[leg] = best
    print(json.dumps(result))


if __name__ == "__main__":
    main()
