"""FastTD3 (rl_x_b200/csrc/fasttd3.cu, rl_x_b200/algorithms/fasttd3/b200) checked WITHOUT a GPU.

The oracle (oracle/fasttd3_oracle.py) is replayed through the batches and normal draws of the executed reference run
(tests/golden/fasttd3_update*.npz) and must reproduce what the reference logged and its final parameters; the kernel source, compiled with
g++ -DRLX_EMU (csrc/dual_build.cuh), runs side by side and must track the oracle after every update.  The plugin class itself is then run on
CPU against the same emulation builds and must reproduce the reference's logged metrics."""
import ctypes as C
import json
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from conftest import emu_build_cmd

from oracle import fasttd3_oracle as TD
from rl_x_b200 import _native as nt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAGS = ["update", "update_variant"]
METRIC_NAMES_CRITIC = ["loss/q_loss", "q/q_min", "q/q_max", "gradients/critic_grad_norm"]
METRIC_NAMES_POLICY = ["loss/policy_loss", "gradients/policy_grad_norm"]


def golden(tag):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"fasttd3_{tag}.npz"))
    N, obs, act, batch, n_steps, nopt, seed, ncu, npu, atoms, stride, steps = (int(x) for x in z["meta"])
    f = [float(x) for x in z["meta_f"]]
    meta = dict(N=N, obs=obs, act=act, batch=batch, n_steps=n_steps, nopt=nopt, seed=seed, ncu=ncu, npu=npu, atoms=atoms, stride=stride, steps=steps,
                gamma=f[0], tau=f[1], lr=f[2], v_min=f[3], v_max=f[4], wd=f[5], nsmin=f[8], nsmax=f[9], se=f[10], sclip=f[11], low=f[12], high=f[13],
                clipped=bool(f[14]), max_gn=f[15], clip_rescale=bool(f[16]), anneal=bool(f[17]))
    return z, meta


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = tmp_path_factory.mktemp("fasttd3_emu") / "libfasttd3_emu.so"
    subprocess.run(emu_build_cmd(out, os.path.join(ROOT, "rl_x_b200", "csrc", "fasttd3.cu")), check=True)
    lib = C.CDLL(str(out))
    lib.rlx_fasttd3_workspace_bytes.restype = C.c_size_t
    lib.rlx_fasttd3_workspace_bytes.argtypes = [C.POINTER(nt.FastTd3Dims), C.c_int64]
    lib.rlx_fasttd3_act_f32.argtypes = nt._SIGNATURES["rlx_fasttd3_act_f32"][1]
    return lib


def flat(net):
    return np.concatenate([t.detach().numpy().reshape(-1) for t in TD.leaves(net)]).astype(np.float32)


def lr_at(m, step):
    if not m["anneal"]:
        return m["lr"]
    total = m["steps"] - 3   # (total_timesteps // nr_envs) - learning_starts of the golden runs
    return m["lr"] * (1.0 - min(step, total) / total)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_and_emulated_kernels_reproduce_the_reference_run(emu, tag):
    """The oracle replays the golden run and matches the reference's logged metrics and final parameters; the emulated library, fed the same
    batches and draws, tracks the oracle after every critic / policy update (workspace of exactly the requested size, NaN-filled; the
    first optimising step is repeated with the emulated threads in descending order and must give the same bits)."""
    z, m = golden(tag)
    torch.set_num_threads(1)
    obs, act, atoms, batch, ncu, npu = m["obs"], m["act"], m["atoms"], m["batch"], m["ncu"], m["npu"]
    pol, q1, q2 = TD.reference_init(obs, act, atoms, m["seed"])
    L = TD.Learner(pol, q1, q2, m["lr"], m["wd"], m["gamma"], m["tau"], m["v_min"], m["v_max"], atoms, m["se"], m["sclip"], m["clipped"], m["max_gn"])
    nrm = TD.Normalizer(obs)
    d = nt.FastTd3Dims(obs, act, atoms)
    poff, qoff = (C.c_int64 * 9)(), (C.c_int64 * 9)()
    assert emu.rlx_fasttd3_param_layout(C.byref(d), poff, qoff) == 0
    P, Q = flat(L.pol), np.concatenate([flat(L.q1), flat(L.q2)])
    assert poff[8] == P.size and 2 * qoff[8] == Q.size
    QT = Q.copy()
    gP, mP, vP, gQ, mQ, vQ = (np.zeros_like(x) for x in (P, P, P, Q, Q, Q))
    lr_a, steps = np.array([m["lr"]], np.float32), np.zeros(2, np.int64)
    nbytes = emu.rlx_fasttd3_workspace_bytes(C.byref(d), batch)
    ws = np.full(nbytes // 4, np.nan, np.float32)
    hp = nt.FastTd3Hparams(m["gamma"], m["tau"], m["v_min"], m["v_max"], m["se"], m["sclip"], m["wd"], 0.9, 0.999, 1e-8, m["max_gn"], float(m["clipped"]))
    state = dict(P=P, gP=gP, mP=mP, vP=vP, Q=Q, gQ=gQ, mQ=mQ, vQ=vQ, QT=QT, steps=steps)

    def call(fn, metrics, race_check, **tensors):
        keep = {k: np.ascontiguousarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32) for k, v in tensors.items()}
        a = nt.FastTd3UpdateArgs()
        a.dims, a.n = d, batch
        for k, v in keep.items():
            setattr(a, k, v.ctypes.data)
        a.policy_params, a.policy_grads, a.policy_m, a.policy_v = P.ctypes.data, gP.ctypes.data, mP.ctypes.data, vP.ctypes.data
        a.q_params, a.q_grads, a.q_m, a.q_v, a.q_target_params = Q.ctypes.data, gQ.ctypes.data, mQ.ctypes.data, vQ.ctypes.data, QT.ctypes.data
        a.lr, a.steps, a.hp, a.metrics, a.workspace, a.workspace_bytes = lr_a.ctypes.data, steps.ctypes.data, hp, metrics.ctypes.data, ws.ctypes.data, nbytes
        before = {k: v.copy() for k, v in state.items()}
        assert fn(C.byref(a), None) == 0
        if race_check:
            first = {k: v.copy() for k, v in state.items()}
            first_metrics = metrics.copy()
            for k, v in state.items():
                v[...] = before[k]
            ws[:] = np.nan
            emu.rlx_emu_set_thread_order(1)
            try:
                assert fn(C.byref(a), None) == 0
            finally:
                emu.rlx_emu_set_thread_order(0)
            for k, v in state.items():
                assert np.array_equal(v, first[k]), f"{k} depends on the thread order"
            assert np.array_equal(metrics, first_metrics)

    # Adam divides by sqrt(v): fp32 rounding of a near-zero gradient entry becomes a difference of a fraction of lr in that entry, and
    # clip_grad_norm_ scaling the gradient down puts more entries in that regime - entries are bound by one step (lr), the tensor by its norm
    # (the two runs evolve independently for six optimising steps, so under clipping the metrics drift apart as well: 1e-3 there, 3e-4 otherwise)
    rel_bar, metric_bar = (2e-5, 3e-4) if m["max_gn"] == -1.0 else (1e-4, 1e-3)

    def close_params(ours, ref, what, lr):
        # one AdamW step moves an entry by at most ~lr; with an annealed rate the earlier, larger steps bound it: the initial rate
        np.testing.assert_allclose(ours, ref, rtol=3e-4, atol=m["lr"], err_msg=what)
        rel = float(np.linalg.norm(ours - ref) / np.linalg.norm(ref))
        assert rel <= rel_bar, (what, rel)

    logged = {}
    for u in range(m["nopt"]):
        lr = lr_at(m, u)
        L.set_lr(lr)
        lr_a[0] = lr
        b = {k: torch.from_numpy(z[f"step{u}/{k}"]) for k in ["states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps"]}
        np.testing.assert_allclose(nrm.mean.numpy().reshape(-1), z[f"step{u}/norm_mean"].reshape(-1), rtol=1e-5, atol=1e-6)
        s, ns = nrm.normalize(b["states"], update=True), nrm.normalize(b["next_states"], update=True)
        view = lambda t: t.reshape(npu, ncu, batch, *t.shape[1:])
        s, ns, a_, r, dn, tr, eff = (view(t) for t in (s, ns, b["actions"], b["rewards"], b["dones"], b["truncations"], b["effective_n_steps"]))
        smooth = torch.from_numpy(z[f"step{u}/smoothing_noise"])
        k, step_metrics = 0, []
        for i in range(npu):
            for j in range(ncu):
                mo = L.critic_step(s[i, j], ns[i, j], a_[i, j], r[i, j], dn[i, j], tr[i, j], eff[i, j], smooth[k])
                mc = np.zeros(8, np.float32)
                call(emu.rlx_fasttd3_critic_update_f32, mc, u == 0 and i == 0 and j == 0, states=s[i, j], next_states=ns[i, j], actions=a_[i, j],
                     rewards=r[i, j], dones=dn[i, j], truncations=tr[i, j], effective_n_steps=eff[i, j], smoothing_noise=smooth[k])
                k += 1
                for idx, name in enumerate(METRIC_NAMES_CRITIC):
                    assert abs(float(mc[idx]) - mo[name]) <= metric_bar * max(1.0, abs(mo[name])), (u, i, j, name, mc[idx], mo[name])
                close_params(Q, np.concatenate([flat(L.q1), flat(L.q2)]), f"q params after critic update {u}.{i}.{j}", lr)
                close_params(QT, np.concatenate([flat(L.q1t), flat(L.q2t)]), "target params", lr)
            mp_ = L.policy_step(s[i, -1])
            mp = np.zeros(8, np.float32)
            call(emu.rlx_fasttd3_policy_update_f32, mp, u == 0 and i == 0, states=s[i, -1])
            for idx, name in enumerate(METRIC_NAMES_POLICY):
                assert abs(float(mp[idx]) - mp_[name]) <= metric_bar * max(1.0, abs(mp_[name])), (u, i, name, mp[idx], mp_[name])
            close_params(P, flat(L.pol), f"policy params after policy update {u}.{i}", lr)
            step_metrics.append({**mo, **mp_})
        for name in METRIC_NAMES_CRITIC + METRIC_NAMES_POLICY:
            logged.setdefault(name, []).append(float(np.mean([sm[name] for sm in step_metrics])))
    # the oracle against what the executed reference logged, and its final parameters against the reference's
    for name, vals in logged.items():
        np.testing.assert_allclose(vals, z[f"metric/{name}"], rtol=2e-4, atol=2e-6, err_msg=name)
    stride = m["stride"]
    for prefix, net in (("policy", L.pol), ("q1", L.q1), ("q2", L.q2), ("q1_target", L.q1t), ("q2_target", L.q2t)):
        key = "policy" if prefix == "policy" else "critic"
        for idx, t in enumerate(TD.leaves(net)):
            ref = z[f"final/{prefix}/{key}.{2 * (idx // 2)}.{'weight' if idx % 2 == 0 else 'bias'}"]
            ours = t.detach().numpy().reshape(-1)
            ours = ours if ours.size <= 2048 else ours[::stride]
            np.testing.assert_allclose(ours, ref, rtol=1e-4, atol=m["lr"], err_msg=f"{prefix} {idx}")
    assert list(steps) == [m["nopt"] * npu * ncu, m["nopt"] * npu]
    np.testing.assert_allclose(Q, np.concatenate([flat(L.q1), flat(L.q2)]), rtol=1e-3, atol=m["lr"])


@pytest.mark.parametrize("mode", ["noisy", "deterministic", "clip_rescale"])
def test_emulated_acting_matches_the_oracle(emu, mode):
    obs, act, atoms, n = 11, 5, 21, 37
    pol, _, _ = TD.reference_init(obs, act, atoms, 3)
    g = torch.Generator().manual_seed(1)
    pol = [(w + 0.05 * torch.randn(w.shape, generator=g), b + 0.05 * torch.randn(b.shape, generator=g)) for w, b in pol]   # a non-trivial head
    P = np.concatenate([t.numpy().reshape(-1) for t in TD.leaves(pol)]).astype(np.float32)
    x = torch.randn(n, obs, generator=g) * 2
    noise = torch.randn(n, act, generator=g) if mode != "deterministic" else None
    scales = torch.rand(n, 1, generator=g) * 0.4 + 0.001 if noise is not None else None
    low, high = torch.linspace(-2.0, -0.5, act), torch.linspace(0.5, 3.0, act)
    clip = mode == "clip_rescale"
    ref_a, ref_env = TD.act(pol, x, noise, scales, low, high, clip)
    d = nt.FastTd3Dims(obs, act, atoms)
    nbytes = emu.rlx_fasttd3_workspace_bytes(C.byref(d), n)
    ws = np.full(nbytes // 4, np.nan, np.float32)
    keep = [np.ascontiguousarray(t.numpy(), dtype=np.float32) if t is not None else None for t in (x, noise, scales, low, high)]
    action, env_action = np.zeros((n, act), np.float32), np.zeros((n, act), np.float32)
    p = lambda arr: arr.ctypes.data if arr is not None else None
    assert emu.rlx_fasttd3_act_f32(C.byref(d), P.ctypes.data, p(keep[0]), p(keep[1]), p(keep[2]), p(keep[3]), p(keep[4]), int(clip), n,
                                   action.ctypes.data, env_action.ctypes.data, ws.ctypes.data, nbytes, None) == 0
    np.testing.assert_allclose(action, ref_a.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(env_action, ref_env.numpy(), rtol=1e-5, atol=1e-6)
    if clip:
        assert (env_action >= low.numpy() - 1e-6).all() and (env_action <= high.numpy() + 1e-6).all()


# --------------------------------------------------------------------------------------------------- the plugin class on CPU
class _Sp:
    def __init__(self, shape, **kw):
        self.shape = shape
        self.__dict__.update(kw)


def _props():
    from rl_x_b200.environments.types import ActionSpaceType, ObservationSpaceType, DataInterfaceType

    class Props:
        observation_space_type, action_space_type, data_interface_type = ObservationSpaceType.FLAT_VALUES, ActionSpaceType.CONTINUOUS, DataInterfaceType.TORCH
    return Props


def _load_plugin(modname, lib=None, replay=None):
    """rl_x_b200/algorithms/fasttd3/b200/fasttd3.py with its device hooks rewritten (device -> cpu, stream -> NULL, library -> `lib`; the shipped
    module raises without CUDA)."""
    src = open(os.path.join(ROOT, "rl_x_b200", "algorithms", "fasttd3", "b200", "fasttd3.py")).read()
    imp = "from rl_x_b200.algorithms.fastsac.b200.replay_buffer import ReplayBuffer"
    assert imp in src
    src = src.replace(imp, "")
    for old, new in [('torch.device("cuda", torch.cuda.current_device())', 'torch.device("cpu")'),
                     ('if a.device != "gpu" or not torch.cuda.is_available():', 'if False:'),
                     ("return C.c_void_p(torch.cuda.current_stream().cuda_stream)", "return None")] + ([("self.lib = nt.load()", "self.lib = LIB")] if lib else []):
        assert old in src
        src = src.replace(old, new)
    mod = types.ModuleType(modname)
    mod.LIB, mod.ReplayBuffer = lib, replay
    exec(compile(src, modname, "exec"), mod.__dict__)
    return mod


@pytest.mark.parametrize("tag", TAGS)
def test_plugin_class_reproduces_the_reference_run_under_emulation(tmp_path, tag):
    """The whole plugin (FastTD3 class + FastSAC's n-step ReplayBuffer) on CPU against host emulation builds of fasttd3.cu, fastsac.cu (the
    normaliser) and replay_nstep.cu.  With the golden run's seed and environment the torch generator is consumed in the reference's order
    (module init, exploration scales, acting noise, torch.randint sampling, smoothing noise), so the run must reproduce the metrics the
    executed reference logged at every step."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    emus = []
    for name in ("fasttd3", "fastsac", "replay_nstep"):
        out = tmp_path / f"lib{name}_emu.so"
        subprocess.run(emu_build_cmd(out, os.path.join(ROOT, "rl_x_b200", "csrc", f"{name}.cu")), check=True)
        emus.append(C.CDLL(str(out)))

    class Lib:
        def __getattr__(self, name):
            for e in emus:
                try:
                    f = getattr(e, name)
                except AttributeError:
                    continue
                res, args = nt._SIGNATURES[name]
                f.argtypes, f.restype = args, res
                return f
            raise AttributeError(name)

    lib = Lib()
    rsrc = open(os.path.join(ROOT, "rl_x_b200", "algorithms", "fastsac", "b200", "replay_buffer.py")).read()
    for old, new in [("C.c_void_p(torch.cuda.current_stream().cuda_stream)", "None"), ("self.lib = nt.load()", "self.lib = LIB"),
                     ("if not torch.cuda.is_available():", "if False:")]:
        rsrc = rsrc.replace(old, new)
    rb = types.ModuleType("fasttd3_replay_emulated")
    rb.LIB = lib
    exec(compile(rsrc, "fasttd3_replay_emulated", "exec"), rb.__dict__)
    mod = _load_plugin("fasttd3_emulated", lib, rb.ReplayBuffer)
    z, m = golden(tag)
    N, obs, act = m["N"], m["obs"], m["act"]
    Props = _props()

    class Env:  # the environment of tests/golden/make_golden_fastsac.py
        general_properties, horizon = Props, 5

        def __init__(self):
            self.g = torch.Generator().manual_seed(m["seed"] + 100)
            self.single_observation_space = _Sp((obs,))
            low, high = np.full(act, -1.5, np.float32), np.full(act, 0.5, np.float32)
            self.single_action_space = _Sp((act,), low=low, high=high, center=(low + high) / 2, scale=np.full(act, 0.8, np.float32))
            self.t = 0

        def reset(self):
            return torch.randn(N, obs, generator=self.g) * 2 + 1, {}

        def step(self, action):
            self.t += 1
            return (torch.randn(N, obs, generator=self.g) * 2 + 1, torch.randn(N, generator=self.g), torch.rand(N, generator=self.g) < 0.2,
                    torch.full((N,), self.t % 4 == 0), {})

        def get_logging_info_dict(self, info):
            return {}

    a = get_config("fasttd3.b200")
    a.batch_size, a.buffer_size_per_env, a.learning_starts, a.total_timesteps, a.n_steps = m["batch"], 8, 3, N * m["steps"], m["n_steps"]
    a.nr_critic_updates_per_policy_update, a.nr_policy_updates_per_step, a.logging_frequency, a.save_frequency = m["ncu"], m["npu"], N, -1
    a.learning_rate, a.clipped_double_q_learning, a.max_grad_norm = m["lr"], m["clipped"], m["max_gn"]
    a.action_clipping_and_rescaling, a.anneal_learning_rate, a.smoothing_epsilon = m["clip_rescale"], m["anneal"], m["se"]
    cfg = ConfigDict(algorithm=a, environment=ConfigDict(seed=m["seed"], nr_envs=N),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    torch.set_num_threads(1)
    env = Env()
    model = mod.FastTD3(cfg, env, env, str(tmp_path), None)
    logged = []
    model.log = lambda name, value, step: logged.append((name, float(value)))
    model.train()
    checked = 0
    for key in z.files:
        if key.startswith("metric/"):
            name = key[len("metric/"):]
            np.testing.assert_allclose([v for nme, v in logged if nme == name], z[key], rtol=5e-4, atol=5e-6, err_msg=name)
            checked += 1
    assert checked >= 11


def _ckpt_env(obs, act, Props):
    class Env:
        general_properties, horizon = Props, 3
        single_observation_space = _Sp((obs,))
        single_action_space = _Sp((act,), low=np.full(act, -1.0, np.float32), high=np.full(act, 1.0, np.float32))
    return Env


def test_plugin_checkpoint_has_the_reference_layout(tmp_path):
    """FastTD3.save() writes the reference's file (fasttd3.py:449-462): the state dicts load with strict=True into torch modules shaped like the
    reference's Policy / QNetwork, both AdamW optimisers accept their states (q1's parameters numbered before q2's), and load() restores the
    flat buffers exactly."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    mod = _load_plugin("fasttd3_ckpt")   # only the layout query of the real library (a host function) is used here
    obs, act, atoms = 9, 4, 21
    Env = _ckpt_env(obs, act, _props())
    a = get_config("fasttd3.b200")
    a.nr_atoms = atoms
    cfg = ConfigDict(algorithm=a, environment=ConfigDict(seed=8, nr_envs=4),
                     runner=ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    model = mod.FastTD3(cfg, Env(), Env(), str(tmp_path / "run"), None)
    pol0, q10, q20 = TD.reference_init(obs, act, atoms, 8)   # bit-identical initial parameters
    assert torch.equal(model.policy_params, torch.cat([t.reshape(-1) for t in TD.leaves(pol0)]))
    assert torch.equal(model.q_params, torch.cat([t.reshape(-1) for t in TD.leaves(q10) + TD.leaves(q20)]))
    g = torch.Generator().manual_seed(0)
    for t in (model.policy_m, model.policy_v, model.q_m, model.q_v, model.q_target_params, model.norm_mean):
        t.copy_(torch.rand(t.shape, generator=g))
    model.steps.copy_(torch.tensor([12, 6]))
    model.norm_count.fill_(77)
    model.save()
    path = tmp_path / "run" / "models" / "latest.model"
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {"config_algorithm", "policy_state_dict", "q1_state_dict", "q2_state_dict", "q1_target_state_dict", "q2_target_state_dict",
                       "policy_optimizer_state_dict", "q_optimizer_state_dict", "observation_normalizer_state_dict"}

    def seq(inp, widths, out, tanh):
        layers, last = [], inp
        for w in widths:
            layers += [torch.nn.Linear(last, w), torch.nn.ReLU()]
            last = w
        return torch.nn.Sequential(*layers, torch.nn.Linear(last, out), *([torch.nn.Tanh()] if tanh else []))

    class Policy(torch.nn.Module):       # module structure of rl_x/algorithms/fasttd3/pytorch/policy.py:33-42
        def __init__(self):
            super().__init__()
            self.policy = seq(obs, (512, 256, 128), act, True)

    class QNetwork(torch.nn.Module):     # q_network.py:27-35
        def __init__(self):
            super().__init__()
            self.critic = seq(obs + act, (1024, 512, 256), atoms, False)

    pol, q1, q2 = Policy(), QNetwork(), QNetwork()
    pol.load_state_dict(ck["policy_state_dict"], strict=True)
    q1.load_state_dict(ck["q1_state_dict"], strict=True)
    q2.load_state_dict(ck["q2_state_dict"], strict=True)
    QNetwork().load_state_dict(ck["q2_target_state_dict"], strict=True)
    popt, qopt = torch.optim.AdamW(pol.parameters(), lr=1e-3), torch.optim.AdamW(list(q1.parameters()) + list(q2.parameters()), lr=1e-3)
    popt.load_state_dict(ck["policy_optimizer_state_dict"])
    qopt.load_state_dict(ck["q_optimizer_state_dict"])
    nq = model.q_offsets[-1]
    assert torch.equal(qopt.state[q2.critic[0].weight]["exp_avg"].reshape(-1), model.q_m[nq:nq + q2.critic[0].weight.numel()])
    x = torch.randn(5, obs)
    with torch.no_grad():
        opol = [(pol.policy[i].weight, pol.policy[i].bias) for i in (0, 2, 4, 6)]
        assert torch.allclose(pol.policy(x), TD.policy_forward(opol, x), atol=1e-6)
    cfg.runner.load_model = str(path)
    cfg.runner.save_model = False
    again = mod.FastTD3.load(cfg, Env(), Env(), str(tmp_path / "run2"), None, [])
    for name in ("policy_params", "q_params", "q_target_params", "policy_m", "policy_v", "q_m", "q_v", "norm_mean", "norm_var", "norm_std", "norm_count",
                 "steps"):
        assert torch.equal(getattr(model, name), getattr(again, name)), name


def test_checkpoints_move_between_the_plugin_and_the_reference_classes(tmp_path):
    """With the reference's OWN classes (staged into oracle/_ref by oracle/make_ref_fasttd3.py): a `latest.model` written by the reference's FastTD3.save() after AdamW steps
    is read by the plugin's load() tensor for tensor, and the file the plugin's save() writes goes through the reference's FastTD3.load()."""
    from oracle import make_ref_fasttd3
    if not make_ref_fasttd3.available():
        pytest.skip("oracle/_ref (with the FastTD3 modules) not staged: python oracle/make_ref_fasttd3.py")
    make_ref_fasttd3.verify()
    from oracle import ref_arm
    os.environ["TORCHDYNAMO_DISABLE"] = "1"
    ref_arm.import_reference()
    import rl_x.algorithms.fasttd3.pytorch.fasttd3 as reftd
    from rl_x.algorithms.fasttd3.pytorch.default_config import get_config as ref_config
    from rl_x.environments.action_space_type import ActionSpaceType as RA
    from rl_x.environments.data_interface_type import DataInterfaceType as RD
    from rl_x.environments.observation_space_type import ObservationSpaceType as RO
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    obs, act, atoms, N = 9, 4, 21, 4

    class Props:
        observation_space_type, action_space_type, data_interface_type = RO.FLAT_VALUES, RA.CONTINUOUS, RD.TORCH

    Env = _ckpt_env(obs, act, Props)
    ra = ref_config("fasttd3.pytorch")
    ra.device, ra.bf16_mixed_precision_training, ra.compile_mode, ra.nr_atoms = "cpu", False, "default", atoms
    rcfg = ref_arm._ConfigDict(algorithm=ra, environment=ref_arm._ConfigDict(seed=8, nr_envs=N),
                               runner=ref_arm._ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False))
    ref = reftd.FastTD3(rcfg, Env(), Env(), str(tmp_path / "ref_run"), None)
    g = torch.Generator().manual_seed(0)
    for opt in (ref.policy_optimizer, ref.q_optimizer):
        for _ in range(3):
            for group in opt.param_groups:
                for p in group["params"]:
                    p.grad = torch.randn(p.shape, generator=g) * 0.1
            opt.step()
    ref.observation_normalizer.train()
    ref.observation_normalizer.normalize(torch.randn(32, obs, generator=g) * 2 + 1, update=True)
    ref.save()
    mod = _load_plugin("fasttd3_interop")
    cfg = ConfigDict(algorithm=get_config("fasttd3.b200"), environment=ConfigDict(seed=8, nr_envs=N),
                     runner=ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False,
                                       load_model=str(tmp_path / "ref_run" / "models" / "latest.model")))
    ours = mod.FastTD3.load(cfg, Env(), Env(), str(tmp_path / "our_run"), None, [])
    assert int(ours.dims.nr_atoms) == atoms
    nq = ours.q_offsets[-1]

    def check(module, opt, flat_, m_, v_, net, step_index):
        named = ours._named(flat_, net)
        nm, nv = (ours._named(m_, net), ours._named(v_, net)) if m_ is not None else (None, None)
        for name, p in module.named_parameters():
            name = name.replace("_orig_mod.", "")
            assert torch.equal(named[name], p.detach()), (net, name)
            if opt is not None:
                st = opt.state[p]
                assert torch.equal(nm[name], st["exp_avg"]) and torch.equal(nv[name], st["exp_avg_sq"]), (net, name)
                assert int(ours.steps[step_index]) == int(float(st["step"])) == 3

    def check_all(r):
        check(r.policy, r.policy_optimizer, ours.policy_params, ours.policy_m, ours.policy_v, "policy", 1)
        check(r.critic.q1, r.q_optimizer, ours.q_params[:nq], ours.q_m[:nq], ours.q_v[:nq], "q", 0)
        check(r.critic.q2, r.q_optimizer, ours.q_params[nq:], ours.q_m[nq:], ours.q_v[nq:], "q", 0)
        check(r.critic.q1_target, None, ours.q_target_params[:nq], None, None, "q", 0)
        check(r.critic.q2_target, None, ours.q_target_params[nq:], None, None, "q", 0)
        nsd = r.observation_normalizer.state_dict()
        assert torch.equal(ours.norm_mean.reshape(-1), nsd["running_mean"].reshape(-1)) and int(ours.norm_count[0]) == int(nsd["count"])

    check_all(ref)
    for t in (ours.policy_params, ours.q_params, ours.q_target_params, ours.policy_m, ours.q_m):
        t.add_(torch.randn(t.shape, generator=g) * 0.01)
    ours.save()
    rcfg2 = ref_arm._ConfigDict(algorithm=ref_config("fasttd3.pytorch"), environment=ref_arm._ConfigDict(seed=8, nr_envs=N),
                                runner=ref_arm._ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False,
                                                           load_model=str(tmp_path / "our_run" / "models" / "latest.model")))
    rcfg2.algorithm.device, rcfg2.algorithm.bf16_mixed_precision_training, rcfg2.algorithm.compile_mode = "cpu", False, "default"
    back = reftd.FastTD3.load(rcfg2, Env(), Env(), str(tmp_path / "ref_run2"), None, ["algorithm.device", "algorithm.bf16_mixed_precision_training",
                                                                                     "algorithm.compile_mode"])
    check_all(back)


def test_default_config_and_registration_match_the_reference_surface():
    """Every key of the reference's fasttd3 default_config.py with its value (bf16_mixed_precision_training: False here, True raises), every
    method of the reference's FastTD3 class with the same parameter names, and the plugin registered under `fasttd3.b200` with the
    reference's general properties (FLAT_VALUES x CONTINUOUS x TORCH)."""
    import ast
    import importlib
    with open(os.path.join(ROOT, "tests", "golden", "fasttd3_reference_surface.json")) as fh:
        surface = json.load(fh)
    cfg = importlib.import_module("rl_x_b200.algorithms.fasttd3.b200.default_config").get_config("fasttd3.b200")
    ours = {k: json.loads(json.dumps(cfg[k])) for k in cfg}
    ref = surface["config"]
    assert [k for k in ref if k not in ours] == []
    assert {k for k in ref if k != "name" and ref[k] != ours[k]} == {"bf16_mixed_precision_training"}
    assert set(ours) - set(ref) == {"gemm_engine"}
    path = os.path.join(ROOT, "rl_x_b200", "algorithms", "fasttd3", "b200", "fasttd3.py")
    for node in ast.walk(ast.parse(open(path).read())):
        if isinstance(node, ast.ClassDef) and node.name == "FastTD3":
            methods = {f.name: [a.arg for a in f.args.args if a.arg != "cls"] for f in node.body if isinstance(f, ast.FunctionDef)}
    for name, args in surface["methods"].items():
        assert methods.get(name) == args, name
    importlib.import_module("rl_x_b200.algorithms.fasttd3.b200")
    from rl_x_b200.algorithms import algorithm_manager as am
    from rl_x_b200.environments.types import ActionSpaceType, ObservationSpaceType, DataInterfaceType
    props = am.get_algorithm_general_properties("fasttd3.b200")
    assert am.get_algorithm_model_class("fasttd3.b200").__name__ == "FastTD3"
    assert list(props.observation_space_types) == [ObservationSpaceType.FLAT_VALUES] and list(props.action_space_types) == [ActionSpaceType.CONTINUOUS]
    assert list(props.data_interface_types) == [DataInterfaceType.TORCH]
    # the reference runner's compatibility check (runner.py:86-101) with the reference's own enums, where the staged copy is available
    from oracle import make_ref
    if make_ref.available():
        from oracle import ref_arm
        ref_arm.import_reference()
        from rl_x.algorithms import algorithm_manager as ref_manager
        ref_manager._algorithms.pop("fasttd3.b200", None)
        importlib.reload(importlib.import_module("rl_x_b200.algorithms.fasttd3.b200"))   # what the reference runner's import does, rl_x importable
        from rl_x.environments.action_space_type import ActionSpaceType as RA
        from rl_x.environments.observation_space_type import ObservationSpaceType as RO
        from rl_x.environments.data_interface_type import DataInterfaceType as RD
        from rl_x.algorithms.deep_learning_framework_type import DeepLearningFrameworkType as RF
        p = ref_manager.get_algorithm_general_properties("fasttd3.b200")
        assert RA.CONTINUOUS in p.action_space_types and RO.FLAT_VALUES in p.observation_space_types and RD.TORCH in p.data_interface_types
        assert RA.DISCRETE not in p.action_space_types and RF.TORCH == p.deep_learning_framework_type
