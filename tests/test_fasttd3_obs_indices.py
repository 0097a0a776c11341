"""FastTD3 with observation index sets (asymmetric actor-critic) checked WITHOUT a GPU.

The env's `policy_observation_indices` / `critic_observation_indices` select the columns each network reads (rl_x/algorithms/fasttd3/
pytorch/policy.py:52, q_network.py:39).  tests/golden/fasttd3_obs_indices.npz is a run of the executed reference on such an env
(obs 12, policy on 7 shuffled columns, critic on 10).  The index-selecting layer over the oracle (tests/fasttd3_obs_indices_oracle.py)
must reproduce it; the host emulation of csrc/fasttd3.cu must track that oracle at index sets on and off the 4-float grid, in
NaN-filled workspaces of exactly the requested size and with its threads run in both orders; explicit `arange` sets must give the bits
of the NULL (identity) sets; and the plugin class under emulation must reproduce the reference's logged metrics."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import emu_build_cmd
from test_fasttd3_emulation import _ckpt_env, _load_plugin, _props, _Sp, emu, flat, golden  # noqa: F401  (emu: fixture)

import fasttd3_obs_indices_oracle as X
from oracle import fasttd3_oracle as TD
from rl_x_b200 import _native as nt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRIC_NAMES_CRITIC = ["loss/q_loss", "q/q_min", "q/q_max", "gradients/critic_grad_norm"]
METRIC_NAMES_POLICY = ["loss/policy_loss", "gradients/policy_grad_norm"]
BATCH_KEYS = ["states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps"]


def _golden():
    z, m = golden("obs_indices")
    return z, m, z["policy_idx"].astype(np.int64), z["critic_idx"].astype(np.int64)


def _dims(obs, act, atoms, pidx, cidx):
    """FastTd3Dims with host int32 copies of the sets (the emulation's device memory is host memory); keep the returned arrays alive."""
    d = nt.FastTd3Dims(obs, act, atoms)
    keep = []
    for k, ind in (("policy", pidx), ("critic", cidx)):
        if ind is not None:
            arr = np.ascontiguousarray(ind, dtype=np.int32)
            keep.append(arr)
            setattr(d, f"{k}_in_dim", arr.size)
            setattr(d, f"{k}_idx", arr.ctypes.data)
    return d, keep


class _Emu:
    """The flat buffers of one learner and the emulated update / acting calls (NaN-filled workspace of exactly the requested size)."""

    def __init__(self, lib, obs, act, atoms, n, nets, hp, pidx, cidx, lr):
        self.lib, self.n, self.act = lib, n, act
        self.d, self._keep = _dims(obs, act, atoms, pidx, cidx)
        self.P = flat(nets[0])
        self.Q = np.concatenate([flat(nets[1]), flat(nets[2])])
        self.QT = self.Q.copy()
        self.gP, self.mP, self.vP, self.gQ, self.mQ, self.vQ = (np.zeros_like(x) for x in (self.P, self.P, self.P, self.Q, self.Q, self.Q))
        self.lr, self.steps, self.hp = np.array([lr], np.float32), np.zeros(2, np.int64), hp
        self.nbytes = lib.rlx_fasttd3_workspace_bytes(C.byref(self.d), n)
        assert self.nbytes > 0
        self.ws = np.full(self.nbytes // 4, np.nan, np.float32)
        poff, qoff = (C.c_int64 * 9)(), (C.c_int64 * 9)()
        assert lib.rlx_fasttd3_param_layout(C.byref(self.d), poff, qoff) == 0
        assert poff[8] == self.P.size and 2 * qoff[8] == self.Q.size

    def state(self):
        return dict(P=self.P, gP=self.gP, mP=self.mP, vP=self.vP, Q=self.Q, gQ=self.gQ, mQ=self.mQ, vQ=self.vQ, QT=self.QT, steps=self.steps)

    def update(self, which, race_check=False, **tensors):
        keep = {k: np.ascontiguousarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32) for k, v in tensors.items()}
        a = nt.FastTd3UpdateArgs()
        a.dims, a.n = self.d, self.n
        for k, v in keep.items():
            setattr(a, k, v.ctypes.data)
        a.policy_params, a.policy_grads, a.policy_m, a.policy_v = self.P.ctypes.data, self.gP.ctypes.data, self.mP.ctypes.data, self.vP.ctypes.data
        a.q_params, a.q_grads, a.q_m, a.q_v, a.q_target_params = self.Q.ctypes.data, self.gQ.ctypes.data, self.mQ.ctypes.data, self.vQ.ctypes.data, self.QT.ctypes.data
        metrics = np.full(8, np.nan, np.float32)
        a.lr, a.steps, a.hp, a.metrics, a.workspace, a.workspace_bytes = (self.lr.ctypes.data, self.steps.ctypes.data, self.hp, metrics.ctypes.data,
                                                                          self.ws.ctypes.data, self.nbytes)
        fn = self.lib.rlx_fasttd3_critic_update_f32 if which == "critic" else self.lib.rlx_fasttd3_policy_update_f32
        before = {k: v.copy() for k, v in self.state().items()}
        self.ws[:] = np.nan
        assert fn(C.byref(a), None) == 0
        if race_check:   # the same call with the emulated threads in descending order: the same bits
            first, first_metrics = {k: v.copy() for k, v in self.state().items()}, metrics.copy()
            for k, v in self.state().items():
                v[...] = before[k]
            self.ws[:] = np.nan
            self.lib.rlx_emu_set_thread_order(1)
            try:
                assert fn(C.byref(a), None) == 0
            finally:
                self.lib.rlx_emu_set_thread_order(0)
            for k, v in self.state().items():
                assert np.array_equal(v, first[k]), f"{k} depends on the thread order"
            assert np.array_equal(metrics, first_metrics, equal_nan=True)
        return metrics

    def act_(self, x, noise, scales, low, high, clip):
        n = x.shape[0]
        nbytes = self.lib.rlx_fasttd3_workspace_bytes(C.byref(self.d), n)
        ws = np.full(nbytes // 4, np.nan, np.float32)
        keep = [np.ascontiguousarray(t.numpy(), dtype=np.float32) if t is not None else None for t in (x, noise, scales, low, high)]
        action, env_action = np.full((n, self.act), np.nan, np.float32), np.full((n, self.act), np.nan, np.float32)
        p = lambda arr: arr.ctypes.data if arr is not None else None
        assert self.lib.rlx_fasttd3_act_f32(C.byref(self.d), self.P.ctypes.data, p(keep[0]), p(keep[1]), p(keep[2]), p(keep[3]), p(keep[4]), int(clip), n,
                                            action.ctypes.data, env_action.ctypes.data, ws.ctypes.data, nbytes, None) == 0
        return action, env_action


# ------------------------------------------------------------------------------------------------------------ the golden run
def test_golden_index_sets_are_asymmetric():
    z, m, pidx, cidx = _golden()
    assert (m["obs"], len(pidx), len(cidx)) == (12, 7, 10)
    assert len(set(pidx) & set(cidx)) > 0 and len(set(cidx) - set(pidx)) > 0 and len(set(range(m["obs"])) - set(pidx) - set(cidx)) > 0
    assert z["final/policy/policy.0.weight"].size == -(-512 * 7 // m["stride"]) and z["final/q1/critic.0.weight"].size == -(-1024 * 13 // m["stride"])


def test_initial_parameters_are_the_reference_modules_with_the_selected_fan_ins():
    """The plugin's reference_init and the oracle layer's build the reference's modules (fan-ins P and C + act) in its order under its seed."""
    from rl_x_b200.algorithms.fasttd3.b200.fasttd3 import reference_init
    _, m, pidx, cidx = _golden()
    pol, q1, q2 = X.reference_init(m["obs"], m["act"], m["atoms"], m["seed"], pidx, cidx)
    assert pol[0][0].shape == (512, 7) and q1[0][0].shape == (1024, 13)
    P, Q = reference_init(m["obs"], m["act"], m["atoms"], m["seed"], len(pidx), len(cidx))
    assert torch.equal(P, torch.from_numpy(flat(pol))) and torch.equal(Q, torch.from_numpy(np.concatenate([flat(q1), flat(q2)])))
    P0, Q0 = reference_init(m["obs"], m["act"], m["atoms"], m["seed"])   # no sets: the network of before, unchanged
    pol0, q10, q20 = TD.reference_init(m["obs"], m["act"], m["atoms"], m["seed"])
    assert torch.equal(P0, torch.from_numpy(flat(pol0))) and torch.equal(Q0, torch.from_numpy(np.concatenate([flat(q10), flat(q20)])))


def test_oracle_layer_and_emulated_kernels_reproduce_the_reference_run(emu):
    """The oracle layer replays the golden run and matches the reference's logged metrics and final parameters; the emulated library with
    the two index sets, fed the same batches and draws, tracks it after every critic / policy update (the first ones also with the threads
    in descending order)."""
    z, m, pidx, cidx = _golden()
    torch.set_num_threads(1)
    obs, act, atoms, batch, ncu, npu = m["obs"], m["act"], m["atoms"], m["batch"], m["ncu"], m["npu"]
    nets = X.reference_init(obs, act, atoms, m["seed"], pidx, cidx)
    L = X.Learner(*nets, m["lr"], m["wd"], m["gamma"], m["tau"], m["v_min"], m["v_max"], atoms, m["se"], m["sclip"], m["clipped"], m["max_gn"],
                  policy_idx=pidx, critic_idx=cidx)
    nrm = TD.Normalizer(obs)
    hp = nt.FastTd3Hparams(m["gamma"], m["tau"], m["v_min"], m["v_max"], m["se"], m["sclip"], m["wd"], 0.9, 0.999, 1e-8, m["max_gn"], float(m["clipped"]))
    E = _Emu(emu, obs, act, atoms, batch, nets, hp, pidx, cidx, m["lr"])

    # an Adam entry whose gradient is within rounding of zero moves by up to lr in either run: the per-entry bar is lr
    def close_params(ours, ref, what):
        np.testing.assert_allclose(ours, ref, rtol=3e-4, atol=m["lr"], err_msg=what)
        assert float(np.linalg.norm(ours - ref) / np.linalg.norm(ref)) <= 2e-5, what

    logged = {}
    for u in range(m["nopt"]):
        b = {k: torch.from_numpy(z[f"step{u}/{k}"]) for k in BATCH_KEYS}
        np.testing.assert_allclose(nrm.mean.numpy().reshape(-1), z[f"step{u}/norm_mean"].reshape(-1), rtol=1e-5, atol=1e-6)
        s, ns = nrm.normalize(b["states"], update=True), nrm.normalize(b["next_states"], update=True)   # full rows, as the reference
        view = lambda t: t.reshape(npu, ncu, batch, *t.shape[1:])
        s, ns, a_, r, dn, tr, eff = (view(t) for t in (s, ns, b["actions"], b["rewards"], b["dones"], b["truncations"], b["effective_n_steps"]))
        smooth = torch.from_numpy(z[f"step{u}/smoothing_noise"])
        k, step_metrics = 0, []
        for i in range(npu):
            for j in range(ncu):
                mo = L.critic_step(s[i, j], ns[i, j], a_[i, j], r[i, j], dn[i, j], tr[i, j], eff[i, j], smooth[k])
                mc = E.update("critic", u == 0 and i == 0 and j == 0, states=s[i, j], next_states=ns[i, j], actions=a_[i, j], rewards=r[i, j],
                              dones=dn[i, j], truncations=tr[i, j], effective_n_steps=eff[i, j], smoothing_noise=smooth[k])
                k += 1
                for idx, name in enumerate(METRIC_NAMES_CRITIC):
                    assert abs(float(mc[idx]) - mo[name]) <= 3e-4 * max(1.0, abs(mo[name])), (u, i, j, name, mc[idx], mo[name])
                close_params(E.Q, np.concatenate([flat(L.q1), flat(L.q2)]), f"q params after critic update {u}.{i}.{j}")
                close_params(E.QT, np.concatenate([flat(L.q1t), flat(L.q2t)]), "target params")
            mp_ = L.policy_step(s[i, -1])
            mp = E.update("policy", u == 0 and i == 0, states=s[i, -1])
            for idx, name in enumerate(METRIC_NAMES_POLICY):
                assert abs(float(mp[idx]) - mp_[name]) <= 3e-4 * max(1.0, abs(mp_[name])), (u, i, name, mp[idx], mp_[name])
            close_params(E.P, flat(L.pol), f"policy params after policy update {u}.{i}")
            step_metrics.append({**mo, **mp_})
        for name in METRIC_NAMES_CRITIC + METRIC_NAMES_POLICY:
            logged.setdefault(name, []).append(float(np.mean([sm[name] for sm in step_metrics])))
    for name, vals in logged.items():
        np.testing.assert_allclose(vals, z[f"metric/{name}"], rtol=2e-4, atol=2e-6, err_msg=name)
    for prefix, net in (("policy", L.pol), ("q1", L.q1), ("q2", L.q2), ("q1_target", L.q1t), ("q2_target", L.q2t)):
        key = "policy" if prefix == "policy" else "critic"
        for idx, t in enumerate(TD.leaves(net)):
            ref = z[f"final/{prefix}/{key}.{2 * (idx // 2)}.{'weight' if idx % 2 == 0 else 'bias'}"]
            ours = t.detach().numpy().reshape(-1)
            ours = ours if ours.size <= 2048 else ours[::m["stride"]]
            np.testing.assert_allclose(ours, ref, rtol=1e-4, atol=m["lr"], err_msg=f"{prefix} {idx}")
    assert list(E.steps) == [m["nopt"] * npu * ncu, m["nopt"] * npu]


# ------------------------------------------------------------------------------------------------------------ kernel shapes
HP = dict(gamma=0.97, tau=0.1, v_min=-10.0, v_max=10.0, se=0.2, sclip=0.5, wd=0.1, lr=1e-3)
SHAPES = [
    # obs, act, P, C, n
    (20, 4, 8, 12, 24),    # P and C + act = 16 on the 4-float grid, P < 32
    (40, 3, 33, 29, 24),   # P = 33 off the grid, C + act = 32 on it
    (12, 3, 7, 10, 16),    # the golden's sets: both off the grid
    (9, 5, 9, 3, 20),      # P = obs (a full permutation), C + act = 8 on the grid
]


def _batch(obs, act, n, seed):
    g = torch.Generator().manual_seed(seed)
    r, u = (lambda *s: torch.randn(*s, generator=g)), (lambda *s: torch.rand(*s, generator=g))
    return {"states": r(n, obs), "next_states": r(n, obs), "actions": u(n, act) * 2 - 1, "rewards": r(n), "dones": (u(n) < 0.1).float(),
            "truncations": (u(n) < 0.05).float(), "effective_n_steps": torch.randint(1, 4, (n,), generator=g).float(), "smoothing_noise": r(n, act)}


def _hp(clipped=True):
    h = HP
    return nt.FastTd3Hparams(h["gamma"], h["tau"], h["v_min"], h["v_max"], h["se"], h["sclip"], h["wd"], 0.9, 0.999, 1e-8, -1.0, float(clipped))


def _sets(obs, P, C, seed):
    rng = np.random.default_rng(seed)
    return rng.permutation(obs)[:P].astype(np.int64), rng.permutation(obs)[:C].astype(np.int64)


@pytest.mark.parametrize("obs,act,P,C,n", SHAPES)
def test_emulated_updates_and_acting_track_the_oracle_layer(emu, obs, act, P, C, n):
    """Two critic updates and a policy update, then acting (noisy, clipped and rescaled), against the oracle layer in float32."""
    torch.set_num_threads(1)
    atoms = 21
    pidx, cidx = _sets(obs, P, C, obs + P + C)
    nets = X.reference_init(obs, act, atoms, 3, pidx, cidx)
    L = X.Learner(*nets, HP["lr"], HP["wd"], HP["gamma"], HP["tau"], HP["v_min"], HP["v_max"], atoms, HP["se"], HP["sclip"], True, -1.0,
                  policy_idx=pidx, critic_idx=cidx)
    E = _Emu(emu, obs, act, atoms, n, nets, _hp(), pidx, cidx, HP["lr"])
    for step, which in enumerate(("critic", "critic", "policy")):
        b = _batch(obs, act, n, 10 + step)
        if which == "critic":
            mo = L.critic_step(*(b[k] for k in BATCH_KEYS), b["smoothing_noise"])
            mc = E.update("critic", step == 0, **b)
            names, ours, ref = METRIC_NAMES_CRITIC, E.Q, np.concatenate([flat(L.q1), flat(L.q2)])
            np.testing.assert_allclose(E.QT, np.concatenate([flat(L.q1t), flat(L.q2t)]), rtol=3e-4, atol=HP["lr"])
        else:
            mo = L.policy_step(b["states"])
            mc = E.update("policy", True, states=b["states"])
            names, ours, ref = METRIC_NAMES_POLICY, E.P, flat(L.pol)
        for i, name in enumerate(names):
            assert abs(float(mc[i]) - mo[name]) <= 3e-4 * max(1.0, abs(mo[name])), (which, name, mc[i], mo[name])
        np.testing.assert_allclose(ours, ref, rtol=3e-4, atol=HP["lr"], err_msg=which)
        assert float(np.linalg.norm(ours - ref) / np.linalg.norm(ref)) <= 2e-5, which
    g = torch.Generator().manual_seed(5)
    x, noise, scales = torch.randn(37, obs, generator=g) * 2, torch.randn(37, act, generator=g), torch.rand(37, 1, generator=g) * 0.4 + 0.001
    low, high = torch.linspace(-2.0, -0.5, act), torch.linspace(0.5, 3.0, act)
    pol = [(torch.from_numpy(w.detach().numpy().copy()), torch.from_numpy(bb.detach().numpy().copy())) for w, bb in L.pol]
    ref_a, ref_env = X.act(pol, x, noise, scales, low, high, True, policy_idx=pidx)
    action, env_action = E.act_(x, noise, scales, low, high, True)
    np.testing.assert_allclose(action, ref_a.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(env_action, ref_env.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("obs", [12, 11])
def test_arange_sets_give_the_bits_of_null_sets(emu, obs):
    """Explicit arange(obs) sets (gathered input, staged policy weight) against NULL ones (states read in place): the same bits in every
    buffer and metric after critic and policy updates, and in acting."""
    act, atoms, n = 3, 21, 24
    nets = TD.reference_init(obs, act, atoms, 2)
    ar = np.arange(obs)
    runs = []
    for sets in ((None, None), (ar, ar)):
        E = _Emu(emu, obs, act, atoms, n, nets, _hp(), *sets, HP["lr"])
        metrics = []
        for step, which in enumerate(("critic", "policy", "critic", "policy")):
            b = _batch(obs, act, n, 20 + step)
            metrics.append(E.update(which, **(b if which == "critic" else {"states": b["states"]})))
        g = torch.Generator().manual_seed(1)
        acting = E.act_(torch.randn(9, obs, generator=g), torch.randn(9, act, generator=g), torch.rand(9, 1, generator=g), torch.full((act,), -1.0),
                        torch.full((act,), 2.0), True)
        runs.append(({k: v.copy() for k, v in E.state().items()}, metrics, acting))
        if sets[0] is not None:
            assert E.nbytes > _Emu(emu, obs, act, atoms, n, nets, _hp(), None, None, HP["lr"]).nbytes   # the gathered input has its own rows
    (s0, m0, a0), (s1, m1, a1) = runs
    for k in s0:
        assert np.array_equal(s0[k], s1[k]), k
    assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(m0, m1))
    assert all(np.array_equal(x, y) for x, y in zip(a0, a1))


def test_null_tail_is_the_network_of_before(emu):
    """A zero / NULL tail: the layout and workspace of the three-field dims every existing caller passes; inconsistent fields are refused."""
    obs, act, atoms = 376, 17, 101
    base = nt.FastTd3Dims(obs, act, atoms)
    explicit = nt.FastTd3Dims(obs, act, atoms, obs, obs, None, None)
    for n in (1, 1000, 32768):
        assert emu.rlx_fasttd3_workspace_bytes(C.byref(base), n) == emu.rlx_fasttd3_workspace_bytes(C.byref(explicit), n)
    off = [(C.c_int64 * 9)() for _ in range(4)]
    assert emu.rlx_fasttd3_param_layout(C.byref(base), off[0], off[1]) == 0 and emu.rlx_fasttd3_param_layout(C.byref(explicit), off[2], off[3]) == 0
    assert list(off[0]) == list(off[2]) and list(off[1]) == list(off[3])
    assert off[0][1] == 512 * obs and off[1][1] == 1024 * (obs + act)
    d, keep = _dims(obs, act, atoms, np.arange(188), np.arange(300))
    assert emu.rlx_fasttd3_param_layout(C.byref(d), off[0], off[1]) == 0
    assert off[0][1] == 512 * 188 and off[1][1] == 1024 * (300 + act)
    idx = np.arange(5, dtype=np.int32)
    for bad in [(obs, act, atoms, 0, 0, idx.ctypes.data, None), (obs, act, atoms, 0, obs + 1, None, idx.ctypes.data),
                (obs, act, atoms, 5, 0, None, None), (obs, act, atoms, 0, obs - 1, None, None)]:
        dd = nt.FastTd3Dims(*bad)
        assert emu.rlx_fasttd3_param_layout(C.byref(dd), off[0], off[1]) != 0
        assert emu.rlx_fasttd3_workspace_bytes(C.byref(dd), 16) == 0


def test_emulation_under_address_sanitizer():
    """The kernel-shape tests again with the emulation built under AddressSanitizer: a gather or a GEMM operand that reads past its buffer
    (aux_gemm's emulation touches the last element each operand extent declares) fails here."""
    if os.environ.get("RLX_EMU_CXXFLAGS"):
        pytest.skip("already running under custom emulation flags")
    libasan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan) or not os.path.exists(libasan):
        pytest.skip("no libasan")
    env = dict(os.environ, RLX_EMU_CXXFLAGS="-g -fsanitize=address", LD_PRELOAD=libasan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "emulated_updates_and_acting or arange_sets"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout.splitlines()[-1], r.stdout[-2000:]


# ------------------------------------------------------------------------------------------------------- the plugin class
def _emulated_plugin(tmp_path, modname):
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

    import types
    lib = Lib()
    rsrc = open(os.path.join(ROOT, "rl_x_b200", "algorithms", "fastsac", "b200", "replay_buffer.py")).read()
    for old, new in [("C.c_void_p(torch.cuda.current_stream().cuda_stream)", "None"), ("self.lib = nt.load()", "self.lib = LIB"),
                     ("if not torch.cuda.is_available():", "if False:")]:
        rsrc = rsrc.replace(old, new)
    rb = types.ModuleType(modname + "_replay")
    rb.LIB = lib
    exec(compile(rsrc, modname + "_replay", "exec"), rb.__dict__)
    return _load_plugin(modname, lib, rb.ReplayBuffer)


def test_plugin_class_reproduces_the_reference_run_under_emulation(tmp_path):
    """The whole plugin on CPU against host emulation builds, on the golden's env with its two index sets: the metrics the executed
    reference logged at every step."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    mod = _emulated_plugin(tmp_path, "fasttd3_obs_indices_emulated")
    z, m, pidx, cidx = _golden()
    N, obs, act = m["N"], m["obs"], m["act"]
    Props = _props()

    class Env:  # tests/golden/make_golden_fastsac.py's SyntheticTorchEnv with the golden's sets
        general_properties, horizon = Props, 5

        def __init__(self):
            self.g = torch.Generator().manual_seed(m["seed"] + 100)
            self.single_observation_space = _Sp((obs,))
            low, high = np.full(act, -1.5, np.float32), np.full(act, 0.5, np.float32)
            self.single_action_space = _Sp((act,), low=low, high=high, center=(low + high) / 2, scale=np.full(act, 0.8, np.float32))
            self.policy_observation_indices, self.critic_observation_indices = pidx.copy(), cidx.copy()
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
    assert (model.dims.policy_in_dim, model.dims.critic_in_dim) == (len(pidx), len(cidx)) and model.dims.policy_idx and model.dims.critic_idx
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


def test_checkpoints_move_between_the_plugin_and_the_reference_classes_with_index_sets(tmp_path):
    """With the reference's OWN classes (staged into oracle/_ref by oracle/make_ref_fasttd3.py) on an env with index sets: the reference's
    initial weights are the plugin's bit for bit; its `latest.model` after AdamW steps is read by the plugin's load() tensor for tensor
    (both optimisers' parameter numbering included); the file the plugin writes loads strictly into the reference's Policy / QNetwork
    through the reference's FastTD3.load()."""
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
    from rl_x_b200.algorithms.fasttd3.b200.fasttd3 import reference_init
    obs, act, atoms, N = 11, 4, 21, 4
    pidx, cidx = np.array([9, 2, 5, 0, 7]), np.array([3, 10, 2, 8, 6, 1, 9])

    class Props:
        observation_space_type, action_space_type, data_interface_type = RO.FLAT_VALUES, RA.CONTINUOUS, RD.TORCH

    Base = _ckpt_env(obs, act, Props)

    class Env(Base):
        policy_observation_indices, critic_observation_indices = pidx, cidx

    ra = ref_config("fasttd3.pytorch")
    ra.device, ra.bf16_mixed_precision_training, ra.compile_mode, ra.nr_atoms = "cpu", False, "default", atoms
    rcfg = ref_arm._ConfigDict(algorithm=ra, environment=ref_arm._ConfigDict(seed=8, nr_envs=N),
                               runner=ref_arm._ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False))
    ref = reftd.FastTD3(rcfg, Env(), Env(), str(tmp_path / "ref_run"), None)
    P0, Q0 = reference_init(obs, act, atoms, 8, len(pidx), len(cidx))
    assert torch.equal(P0, torch.cat([p.detach().reshape(-1) for p in ref.policy.parameters()]))
    assert torch.equal(Q0, torch.cat([p.detach().reshape(-1) for q in (ref.critic.q1, ref.critic.q2) for p in q.parameters()]))
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
    mod = _load_plugin("fasttd3_obs_indices_interop")
    cfg = ConfigDict(algorithm=get_config("fasttd3.b200"), environment=ConfigDict(seed=8, nr_envs=N),
                     runner=ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False,
                                       load_model=str(tmp_path / "ref_run" / "models" / "latest.model")))
    ours = mod.FastTD3.load(cfg, Env(), Env(), str(tmp_path / "our_run"), None, [])
    nq = ours.q_offsets[-1]
    assert ours.policy_offsets[1] == 512 * len(pidx) and ours.q_offsets[1] == 1024 * (len(cidx) + act)

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

    check_all(ref)
    for t in (ours.policy_params, ours.q_params, ours.q_target_params, ours.policy_m, ours.q_m):
        t.add_(torch.randn(t.shape, generator=g) * 0.01)
    ours.save()
    ck = torch.load(tmp_path / "our_run" / "models" / "latest.model", weights_only=False)
    ref.policy.load_state_dict(ck["policy_state_dict"], strict=True)
    ref.critic.q2.load_state_dict(ck["q2_state_dict"], strict=True)
    rcfg2 = ref_arm._ConfigDict(algorithm=ref_config("fasttd3.pytorch"), environment=ref_arm._ConfigDict(seed=8, nr_envs=N),
                                runner=ref_arm._ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False,
                                                           load_model=str(tmp_path / "our_run" / "models" / "latest.model")))
    rcfg2.algorithm.device, rcfg2.algorithm.bf16_mixed_precision_training, rcfg2.algorithm.compile_mode = "cpu", False, "default"
    back = reftd.FastTD3.load(rcfg2, Env(), Env(), str(tmp_path / "ref_run2"), None, ["algorithm.device", "algorithm.bf16_mixed_precision_training",
                                                                                     "algorithm.compile_mode"])
    check_all(back)
    x = torch.randn(6, obs, generator=g)
    with torch.no_grad():
        pol = [(back.policy.policy[i].weight, back.policy.policy[i].bias) for i in (0, 2, 4, 6)]
        assert torch.allclose(back.policy(x), X.policy_forward(pol, x, pidx), atol=1e-6)


# ------------------------------------------------------------------------------------------------------- validation
BAD_SETS = [
    ("out of range", lambda obs: np.array([0, 1, obs])),
    ("negative", lambda obs: np.array([0, -1, 2])),
    ("duplicate", lambda obs: np.array([0, 3, 3])),
    ("empty", lambda obs: np.array([], dtype=np.int64)),
    ("2-D", lambda obs: np.arange(4).reshape(2, 2)),
    ("float dtype", lambda obs: np.array([0.0, 1.0, 2.0])),
]


@pytest.mark.parametrize("attr", ["policy_observation_indices", "critic_observation_indices"])
@pytest.mark.parametrize("case", [c[0] for c in BAD_SETS])
def test_bad_index_sets_are_refused_before_any_device_work(attr, case, monkeypatch, tmp_path):
    """The shipped plugin module: a malformed set raises ValueError naming its attribute before the device check, the library or CUDA."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200 import fasttd3 as td3_mod
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    obs, act = 9, 4
    Env = _ckpt_env(obs, act, _props())
    env = Env()
    setattr(env, attr, dict(BAD_SETS)[case](obs))

    def no_device(*a, **k):
        raise AssertionError("device work before the index sets were validated")
    monkeypatch.setattr(td3_mod.nt, "load", no_device)
    monkeypatch.setattr(torch.cuda, "current_device", no_device)
    monkeypatch.setattr(torch.cuda, "is_available", no_device)
    cfg = ConfigDict(algorithm=get_config("fasttd3.b200"), environment=ConfigDict(seed=0, nr_envs=4),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    with pytest.raises(ValueError, match=attr):
        td3_mod.FastTD3(cfg, env, env, str(tmp_path), None)


def test_identity_sets_take_the_existing_path(tmp_path):
    """arange sets validate to None: the plugin's dims carry a NULL tail, the network of an env without sets."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    mod = _load_plugin("fasttd3_identity_sets")
    obs, act = 9, 4
    Base = _ckpt_env(obs, act, _props())

    class Env(Base):
        policy_observation_indices, critic_observation_indices = np.arange(obs), list(range(obs))

    cfg = ConfigDict(algorithm=get_config("fasttd3.b200"), environment=ConfigDict(seed=0, nr_envs=4),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    model = mod.FastTD3(cfg, Env(), Env(), str(tmp_path), None)
    assert model.policy_observation_indices is None and model.critic_observation_indices is None
    assert (model.dims.policy_in_dim, model.dims.critic_in_dim, model.dims.policy_idx, model.dims.critic_idx) == (0, 0, None, None)
    assert model.policy_offsets[1] == 512 * obs and model.q_offsets[1] == 1024 * (obs + act)
