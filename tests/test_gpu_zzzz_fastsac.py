"""FastSAC update path on the GPU (rl_x_b200/csrc/fastsac.cu through librlx_b200.so) against oracle/fastsac_oracle.py, and a short run of
the fastsac.b200 plugin.  The same sources are also validated in host emulation against the executed reference
(tests/test_fastsac_emulation.py)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import fastsac_oracle as FS

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fastsac_updates_match_oracle_on_golden_batches():
    from rl_x_b200 import _native as nt
    from test_fastsac_emulation import flat
    lib = nt.load()
    z = np.load(os.path.join(ROOT, "tests", "golden", "fastsac_update.npz"))
    N, obs, act, batch, n_steps, nopt, seed, ncu, npu, atoms, stride = (int(x) for x in z["meta"])
    gamma, tau, lr, lsmin, lsmax, tgt_ent, vmin, vmax, wd, b1, b2, alpha0, low, high, scale = (float(x) for x in z["meta_f"][:15])
    torch.set_num_threads(1)
    pol, q1, q2 = FS.reference_init(obs, act, atoms, seed)
    center = (low + high) / 2
    action_scale = torch.full((act,), max(abs(low - center), abs(high - center)) / scale)
    L = FS.Learner(pol, q1, q2, action_scale, lr, wd, (b1, b2), gamma, tau, vmin, vmax, atoms, tgt_ent, alpha0, lsmin, lsmax)
    d = nt.FastSacDims(obs, act, atoms)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).to(DEV).contiguous()
    P, Q = t(flat(L.pol)), t(np.concatenate([flat(L.q1), flat(L.q2)]))
    QT = Q.clone()
    zl = torch.zeros_like
    gP, mP, vP, gQ, mQ, vQ = zl(P), zl(P), zl(P), zl(Q), zl(Q), zl(Q)
    la, astate, lr_d = t([np.log(alpha0)]), torch.zeros(3, device=DEV), t([lr])
    steps = torch.zeros(3, dtype=torch.int64, device=DEV)
    sc = action_scale.to(DEV)
    nbytes = lib.rlx_fastsac_workspace_bytes(C.byref(d), batch)
    ws = torch.zeros(nbytes // 4 + 64, device=DEV)
    hp = nt.FastSacHparams(gamma, tau, vmin, vmax, tgt_ent, lsmin, lsmax, wd, b1, b2, 1e-8, -1.0, 0.0)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(fn, metrics, **tensors):
        a = nt.FastSacUpdateArgs()
        a.dims, a.n = d, batch
        keep = []
        for name, v in tensors.items():
            v = t(v.numpy() if torch.is_tensor(v) else v)
            keep.append(v)
            setattr(a, name, v.data_ptr())
        a.action_scale = sc.data_ptr()
        a.policy_params, a.policy_grads, a.policy_m, a.policy_v = P.data_ptr(), gP.data_ptr(), mP.data_ptr(), vP.data_ptr()
        a.q_params, a.q_grads, a.q_m, a.q_v, a.q_target_params = Q.data_ptr(), gQ.data_ptr(), mQ.data_ptr(), vQ.data_ptr(), QT.data_ptr()
        a.log_alpha, a.alpha_state, a.lr, a.steps = la.data_ptr(), astate.data_ptr(), lr_d.data_ptr(), steps.data_ptr()
        a.hp, a.metrics, a.workspace, a.workspace_bytes = hp, metrics.data_ptr(), ws.data_ptr(), nbytes
        nt.check(fn(C.byref(a), st), "fastsac update")
        torch.cuda.synchronize()

    nrm = FS.Normalizer(obs)
    for u in range(2):
        b = {k: torch.from_numpy(z[f"step{u}/{k}"]) for k in ["states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps"]}
        s = nrm.normalize(b["states"], update=True).view(npu, ncu, batch, obs)
        ns = nrm.normalize(b["next_states"], update=True).view(npu, ncu, batch, obs)
        view = lambda x: x.view(npu, ncu, batch, *x.shape[1:])
        a_, r, dn, tr, eff = (view(b[k]) for k in ["actions", "rewards", "dones", "truncations", "effective_n_steps"])
        normals = torch.from_numpy(z[f"step{u}/normals"])
        k = 0
        for i in range(npu):
            for j in range(ncu):
                m = L.critic_and_entropy_step(s[i, j], ns[i, j], a_[i, j], r[i, j], dn[i, j], tr[i, j], eff[i, j], normals[k])
                mc = torch.zeros(8, device=DEV)
                call(lib.rlx_fastsac_critic_update_f32, mc, states=s[i, j], next_states=ns[i, j], actions=a_[i, j], rewards=r[i, j], dones=dn[i, j],
                     truncations=tr[i, j], effective_n_steps=eff[i, j], noise=normals[k])
                k += 1
                assert abs(float(mc[0]) - m["loss/q_loss"]) <= 3e-4 * abs(m["loss/q_loss"])
                ref = np.concatenate([flat(L.q1), flat(L.q2)])
                assert float(np.linalg.norm(Q.cpu().numpy() - ref) / np.linalg.norm(ref)) <= 3e-5
            mo = L.policy_step(s[i, -1], normals[k])
            mp = torch.zeros(8, device=DEV)
            call(lib.rlx_fastsac_policy_update_f32, mp, states=s[i, -1], noise=normals[k])
            k += 1
            assert abs(float(mp[0]) - mo["loss/policy_loss"]) <= 3e-4 * max(1.0, abs(mo["loss/policy_loss"]))
            ref = flat(L.pol)
            assert float(np.linalg.norm(P.cpu().numpy() - ref) / np.linalg.norm(ref)) <= 3e-5


@pytest.mark.skipif(os.environ.get("RLX_AUX_GEMM_ENGINE") != "1", reason="runs inside the tensor-engine subprocess (next test)")
def test_fastsac_engines_agree_at_batch_1024():
    """The golden batches above have 16 rows, too few for a tensor-core tile, so they exercise the SIMT engine whatever the switch says.
    Here: one critic and one policy update at the bench's layer shapes (obs 48, act 12, 101 atoms) on 1024 random rows, once per engine from
    the same state.  The SIMT engine is the one pinned to the oracle; the 3xTF32 engine is fp32-equivalent (6e-7 + 3.2e-9 K relative per
    product, tests/test_gpu_tc_engine.py; PPO's three-layer update lands at 1.5e-6 - 3.1e-6 of the gradient norm with it, DESIGN.md 4a), so
    through these four-layer LayerNorm torsos the gradients must agree to 3e-5 of their norm and the losses to 2e-5 - a wrong tile, a wrong
    extent or a missed epilogue is off by orders of magnitude more."""
    from rl_x_b200 import _native as nt
    from test_fastsac_emulation import flat
    lib = nt.load()
    obs, act, atoms, n = 48, 12, 101, 1024
    torch.manual_seed(11)
    pol, q1, q2 = FS.reference_init(obs, act, atoms, 3)
    d = nt.FastSacDims(obs, act, atoms)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float32).to(DEV).contiguous()
    P0, Q0 = t(flat(pol)), t(np.concatenate([flat(q1), flat(q2)]))
    batch = dict(states=torch.randn(n, obs), next_states=torch.randn(n, obs), actions=torch.rand(n, act) * 2 - 1, rewards=torch.randn(n),
                 dones=(torch.rand(n) < 0.05).float(), truncations=(torch.rand(n) < 0.02).float(), effective_n_steps=torch.randint(1, 4, (n,)).float(),
                 noise=torch.randn(n, act))
    dev = {k: t(v) for k, v in batch.items()}
    sc = torch.ones(act, device=DEV)
    nbytes = lib.rlx_fastsac_workspace_bytes(C.byref(d), n)
    hp = nt.FastSacHparams(0.99, 0.005, -10.0, 10.0, -float(act), -5.0, 0.0, 0.1, 0.9, 0.95, 1e-8, -1.0, 0.0)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = {}
    for engine in (0, 1):
        assert lib.rlx_set_aux_gemm_engine(engine) == engine
        before = int(lib.rlx_aux_tc_gemm_count())
        P, Q, QT = P0.clone(), Q0.clone(), Q0.clone()
        zl = torch.zeros_like
        gP, mP, vP, gQ, mQ, vQ = zl(P), zl(P), zl(P), zl(Q), zl(Q), zl(Q)
        la, astate, lr_d = t([np.log(0.001)]), torch.zeros(3, device=DEV), t([3e-4])
        steps, ws = torch.zeros(3, dtype=torch.int64, device=DEV), torch.zeros(nbytes // 4 + 64, device=DEV)
        res = {}
        for fn, names, key in ((lib.rlx_fastsac_critic_update_f32, list(dev), "critic"), (lib.rlx_fastsac_policy_update_f32, ["states", "noise"], "policy")):
            a = nt.FastSacUpdateArgs()
            a.dims, a.n = d, n
            for name in names:
                setattr(a, name, dev[name].data_ptr())
            a.action_scale = sc.data_ptr()
            a.policy_params, a.policy_grads, a.policy_m, a.policy_v = P.data_ptr(), gP.data_ptr(), mP.data_ptr(), vP.data_ptr()
            a.q_params, a.q_grads, a.q_m, a.q_v, a.q_target_params = Q.data_ptr(), gQ.data_ptr(), mQ.data_ptr(), vQ.data_ptr(), QT.data_ptr()
            a.log_alpha, a.alpha_state, a.lr, a.steps = la.data_ptr(), astate.data_ptr(), lr_d.data_ptr(), steps.data_ptr()
            metrics = torch.zeros(8, device=DEV)
            a.hp, a.metrics, a.workspace, a.workspace_bytes = hp, metrics.data_ptr(), ws.data_ptr(), nbytes
            nt.check(fn(C.byref(a), st), f"fastsac {key} update, engine {engine}")
            torch.cuda.synchronize()
            res[key] = (metrics.cpu().numpy().copy(), (gQ if key == "critic" else gP).cpu().numpy().copy())
        out[engine] = (res, int(lib.rlx_aux_tc_gemm_count()) - before)
    lib.rlx_set_aux_gemm_engine(1)   # the subprocess's setting
    assert out[0][1] == 0 and out[1][1] > 0, "engine 1 must have put GEMMs on the tensor engine, engine 0 none"
    for key in ("critic", "policy"):
        (m0, g0), (m1, g1) = out[0][0][key], out[1][0][key]
        assert np.isfinite(g1).all() and float(np.linalg.norm(g1 - g0) / np.linalg.norm(g0)) <= 3e-5, key
        assert abs(float(m1[0]) - float(m0[0])) <= 2e-5 * max(1.0, abs(float(m0[0]))), (key, m0[0], m1[0])


def test_fastsac_suite_in_a_subprocess_with_dense_layers_on_the_tensor_engine(tmp_path):
    """rlx_set_aux_gemm_engine(1): the torso layers of the policy and of both C51 critics (forward, input and weight gradients) run on the
    wgmma 3xTF32 engine; the 101-column logits layer (row pitch not a multiple of 16 bytes) and the skinny heads stay on the SIMT engine.
    The whole file - the golden-batch parity against the pinned oracle included - must pass that way and must have used the tensor engine."""
    from conftest import run_suite_with_switches
    rc, tail, tc, _ = run_suite_with_switches(__file__, tmp_path, tensor_engine=True)
    assert rc == 0, tail
    assert tc > 0, f"the tensor engine was never used ({tc})"


def test_fastsac_plugin_runs_on_device_env():
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fastsac.b200.default_config import get_config
    from rl_x_b200.algorithms.fastsac.b200.fastsac import FastSAC
    from test_gpu_train import _props
    N, obs, act = 16, 10, 4

    class Sp:
        def __init__(self, shape, **kw):
            self.shape = shape
            self.__dict__.update(kw)

    class Env:
        general_properties, horizon = _props("TORCH"), 4
        single_observation_space = Sp((obs,))
        single_action_space = Sp((act,), low=np.full(act, -1.0, np.float32), high=np.full(act, 1.0, np.float32), center=np.zeros(act, np.float32),
                                 scale=np.ones(act, np.float32))
        g = torch.Generator(device=DEV).manual_seed(1)

        def reset(self):
            return torch.randn(N, obs, device=DEV, generator=self.g), {}

        def step(self, action):
            assert tuple(action.shape) == (N, act) and float(action.abs().max()) <= 1.0 + 1e-6
            return (torch.randn(N, obs, device=DEV, generator=self.g), torch.randn(N, device=DEV, generator=self.g),
                    torch.rand(N, device=DEV, generator=self.g) < 0.1, torch.zeros(N, dtype=torch.bool, device=DEV), {})

        def get_logging_info_dict(self, info):
            return {}

        def close(self):
            pass

    a = get_config("fastsac.b200")
    a.batch_size, a.buffer_size_per_env, a.learning_starts, a.total_timesteps, a.n_steps = 64, 16, 2, N * 6, 3
    a.nr_critic_updates_per_policy_update, a.nr_policy_updates_per_step, a.logging_frequency, a.save_frequency = 2, 1, N, -1
    cfg = ConfigDict(algorithm=a, environment=ConfigDict(seed=3, nr_envs=N),
                     runner=ConfigDict(save_model=False, track_console=False, track_tb=False, track_wandb=False, load_model=""))
    env = Env()
    model = FastSAC(cfg, env, env, "/tmp/rlx_test_fastsac", None)
    logged = []
    model.log = lambda name, value, step: logged.append((name, float(value)))
    model.train()
    q = [v for n_, v in logged if n_ == "loss/q_loss"]
    assert len(q) == 4 and all(np.isfinite(q))
    assert all(np.isfinite(v) for n_, v in logged if not n_.startswith("time/"))
