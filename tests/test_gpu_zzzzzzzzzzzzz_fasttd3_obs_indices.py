"""FastTD3 with observation index sets on the GPU: the critic and policy updates and the acting kernel on both engines of `aux_gemm` against
the index-selecting oracle layer (tests/fasttd3_obs_indices_oracle.py) run in float64, with a count of the GEMM launches of every call.

The machinery is test_gpu_zzzzzzz_aux_tc_float64.py's: NaN-filled workspaces of exactly rlx_fasttd3_workspace_bytes and NaN-filled gradient
buffers, rows near a ReLU kink or a clipped-double-Q tie filtered out at float64, per parameter tensor bounds (BAR = 2e-5 on both engines,
and the tensor engine within twice the SIMT engine's distance plus the 3xTF32 floor F), and the launch counters compared with a table
derived from the gate.  `td3_gemms_idx` lists the GEMMs each entry point issues with index sets (fasttd3.cu): the policy's layer 1 on the
gathered input s[:, policy_idx] and its staged weight, both at pitch align4(P); the Q networks' layer 1 on [s[:, critic_idx] | a] at pitch
align4(C + act); the actor's gradient through a critic from the action block at column C of its [1024, C + act] weight.  So a gathered
layer-1 product that the gate admits but that ran on the SIMT engine fails the count.

Sorted after the other GPU files: a kernel fault on a new shape takes the CUDA context with it, and then costs only this file."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fasttd3_obs_indices_oracle as X
import test_gpu_zzzzzzz_aux_tc_float64 as A
from oracle import fasttd3_oracle as TD

gpu = pytest.mark.gpu
DEV = "cuda"
TC_NONE, TC_BIAS_TANH, TC_BIAS_RELU, TC_DRELU, TC_BIAS = A.TC_NONE, A.TC_BIAS_TANH, A.TC_BIAS_RELU, A.TC_DRELU, A.TC_BIAS
_fwd, _dx, _dw = A._fwd, A._dx, A._dw


def _a4(x):
    return -(-x // 4) * 4


def td3_gemms_idx(obs, act, atoms, n, entry, pidx=None, cidx=None):
    """The GEMMs of rlx_fasttd3_{critic_update,policy_update,act}_f32 in issue order with index sets (None = identity, states in place)."""
    PW, QW = TD.POLICY_WIDTHS, TD.Q_WIDTHS
    P = obs if pidx is None else len(pidx)
    Cc = obs if cidx is None else len(cidx)
    po, qo = A.mlp_offsets(P, PW, act), A.mlp_offsets(Cc + act, QW, atoms)
    pitch = _a4(Cc + act)
    # policy layer 1: the parameter block at pitch obs, or the staged copy (an aligned workspace segment) at the gathered input's pitch
    ldp, w1p = (obs, po[0]) if pidx is None else (_a4(P), 0)

    def mlp_fwd(tag, off, widths, inp, out, head_epi, base, ldx, w1, ldw1):
        dims = (inp,) + tuple(widths)
        g = [_fwd(f"{tag}.fwd0", n, inp, widths[0], TC_BIAS_RELU, w1, ldx, ldw1)]
        g += [_fwd(f"{tag}.fwd{k}", n, dims[k], widths[k], TC_BIAS_RELU, base + off[2 * k]) for k in (1, 2)]
        return g + [_fwd(f"{tag}.fwd3", n, widths[2], out, head_epi, base + off[6])]

    def mlp_bwd(tag, off, widths, inp, out, base, ldx):
        g = [_dw(f"{tag}.dw3", n, widths[2], out), _dx(f"{tag}.dx3", n, widths[2], out, TC_DRELU, base + off[6])]
        for k in (2, 1, 0):
            if k > 0:
                g += [_dw(f"{tag}.dw{k}", n, widths[k - 1], widths[k]), _dx(f"{tag}.dx{k}", n, widths[k - 1], widths[k], TC_DRELU, base + off[2 * k])]
            else:
                g.append(_dw(f"{tag}.dw0", n, inp, widths[0], ldx, ldx))
        return g

    pol_fwd = mlp_fwd("pol", po, PW, P, act, TC_BIAS_TANH, 0, ldp, w1p, ldp)
    q_fwd = lambda q, tag: mlp_fwd(f"{tag}{q + 1}", qo, QW, Cc + act, atoms, TC_BIAS, 0, pitch, 0, pitch)
    if entry == "act":
        return pol_fwd
    if entry == "critic":
        g = pol_fwd + q_fwd(0, "qt") + q_fwd(1, "qt")
        for q in (0, 1):
            g += q_fwd(q, "q") + mlp_bwd(f"q{q + 1}", qo, QW, Cc + act, atoms, 0, pitch)
        return g
    g = pol_fwd + q_fwd(0, "q") + q_fwd(1, "q")
    for q in (0, 1):
        g.append(_dx(f"q{q + 1}.dx3", n, QW[2], atoms, TC_DRELU, qo[6]))
        g += [_dx(f"q{q + 1}.dx{k}", n, QW[k - 1], QW[k], TC_DRELU, qo[2 * k]) for k in (2, 1)]
        g.append(_dx(f"q{q + 1}.dx0_actions", n, act, QW[0], TC_NONE, qo[0] + Cc, Cc + act))   # the action block at column C
    return g + mlp_bwd("pol", po, PW, P, act, 0, ldp)


def algo_with(pidx, cidx):
    """test_gpu_zzzzzzz_aux_tc_float64.Td3 with the index sets: the oracle layer's learner and the GEMM table above."""

    class Td3Idx(A.Td3):
        sets = (pidx, cidx)

        @classmethod
        def learner(cls, nets, clipped, dtype, **_):
            h = cls.hp
            return X.Learner(*nets, A.LR, h["wd"], h["gamma"], h["tau"], h["v_min"], h["v_max"], nets[1][-1][0].shape[0], h["se"], h["sclip"],
                             bool(clipped), -1.0, dtype=dtype, policy_idx=pidx, critic_idx=cidx)

        @staticmethod
        def gemms(obs, act, atoms, n, entry):
            return td3_gemms_idx(obs, act, atoms, n, entry, pidx, cidx)

    return Td3Idx


def margins(algo, nets, b, clipped, device):
    """test_gpu_zzzzzzz_aux_tc_float64.td3_margins on the selected columns."""
    pidx, cidx = algo.sets
    pol, q1, q2 = (A._to(algo, net, device, torch.float64) for net in nets)
    b = {k: v.to(device, torch.float64) for k, v in b.items()}
    inf = torch.full_like(b["rewards"], float("inf"))
    sc, sp = X.select(b["states"], cidx), X.select(b["states"], pidx)
    with torch.no_grad():
        xa = torch.cat([sc, b["actions"]], 1)
        relu_c = torch.minimum(A._relu_margin(q1, xa)[0], A._relu_margin(q2, xa)[0])
        L = algo.learner((pol, q1, q2), clipped, torch.float64)
    algo.critic_step(L, b)
    with torch.no_grad():
        val_c = (L.next_values[0] - L.next_values[1]).abs() if clipped else inf
        mp, pre = A._relu_margin(pol, sp)
        xp = torch.cat([sc, torch.tanh(pre)], 1)
        (m1, l1), (m2, l2) = A._relu_margin(q1, xp), A._relu_margin(q2, xp)
        support = torch.linspace(algo.hp["v_min"], algo.hp["v_max"], l1.shape[1], dtype=torch.float64, device=device)
        v1, v2 = (F.softmax(l1, 1) * support).sum(1), (F.softmax(l2, 1) * support).sum(1)
        relu_p, val_p = torch.minimum(mp, torch.minimum(m1, m2)), (v1 - v2).abs() if clipped else inf
    return (relu_c, val_c), (relu_p, val_p)


def make_batches(algo, nets, obs, act, n, seed, clipped, device):
    out = []
    for which, s in ((0, seed), (1, seed + 1)):
        cand = A._draw(algo, obs, act, 2 * n + 64, s)
        kept = A._keep(cand, margins(algo, nets, cand, clipped, device)[which], n)
        relu, val = margins(algo, nets, kept, clipped, device)[which]
        assert float(relu.min()) > A.RELU_MARGIN and float(val.min()) > A.VALUE_MARGIN, (float(relu.min()), float(val.min()))
        out.append(kept)
    return tuple(out)


def _sets(obs, P, Cc, seed):
    if P is None:
        return None, None
    rng = np.random.default_rng(seed)
    return rng.permutation(obs)[:P].astype(np.int64), rng.permutation(obs)[:Cc].astype(np.int64)


def _dims(nt, obs, act, atoms, pidx, cidx):
    """FastTd3Dims with device int32 copies of the sets; keep the returned tensors alive."""
    d, keep = nt.FastTd3Dims(obs, act, atoms), []
    for k, ind in (("policy", pidx), ("critic", cidx)):
        if ind is not None:
            t = torch.as_tensor(np.asarray(ind), dtype=torch.int32).to(DEV).contiguous()
            keep.append(t)
            setattr(d, f"{k}_in_dim", int(t.numel()))
            setattr(d, f"{k}_idx", t.data_ptr())
    return d, keep


class _Device(A._Device):
    """test_gpu_zzzzzzz_aux_tc_float64._Device (its FastTD3 branch) with the index sets in the dims."""

    def __init__(self, algo, lib, obs, act, atoms, n, nets, clipped):
        from rl_x_b200 import _native as nt
        self.algo, self.lib, self.nt, self.n, self.dims, self.like = algo, lib, nt, n, (obs, act, atoms), nets
        self.P, self.Q = A._t(A._flat(algo, nets[0])), A._t(np.concatenate([A._flat(algo, nets[1]), A._flat(algo, nets[2])]))
        self.QT = self.Q.clone()
        zl = torch.zeros_like
        self.gP, self.mP, self.vP, self.gQ, self.mQ, self.vQ = zl(self.P), zl(self.P), zl(self.P), zl(self.Q), zl(self.Q), zl(self.Q)
        self.lr, self.steps = A._t([A.LR]), torch.zeros(3, dtype=torch.int64, device=DEV)
        h = algo.hp
        self.d, self._keep = _dims(nt, obs, act, atoms, *algo.sets)
        self.Args = nt.FastTd3UpdateArgs
        self.hp = nt.FastTd3Hparams(h["gamma"], h["tau"], h["v_min"], h["v_max"], h["se"], h["sclip"], h["wd"], 0.9, 0.999, 1e-8, -1.0, float(clipped))
        self.nbytes = lib.rlx_fasttd3_workspace_bytes(C.byref(self.d), n)
        self.fns = dict(critic=lib.rlx_fasttd3_critic_update_f32, policy=lib.rlx_fasttd3_policy_update_f32)
        assert self.nbytes > 0 and self.nbytes % 4 == 0
        self.ws = torch.empty(self.nbytes // 4, device=DEV)   # exactly the size the library asks for


# ------------------------------------------------------------------------------------------------------------ host-only
@pytest.mark.parametrize("obs,act,atoms,n", [(376, 17, 101, 8192), (375, 18, 100, 1024), (64, 64, 101, 40)])
def test_identity_table_is_the_existing_table(obs, act, atoms, n):
    """With no sets the table is test_gpu_zzzzzzz_aux_tc_float64.td3_gemms, GEMM for GEMM."""
    for entry in ("act", "critic", "policy"):
        assert td3_gemms_idx(obs, act, atoms, n, entry) == A.td3_gemms(obs, act, atoms, n, entry)


def test_table_puts_the_gathered_layer_1_products_where_the_gate_says():
    """The bench shape (policy on 188 of 376 columns, critic on all 376 permuted): every layer-1 product on the tensor engine except the
    action-block input gradient (its B starts at column C of rows C + act wide: both multiples of 4 only when act is); P < 32 sends the
    policy's layer-1 forward and weight gradient to SIMT."""
    pidx, cidx = _sets(376, 188, 376, 0)
    on = {g.name: A.on_tensor_engine(g) for e in ("critic", "policy") for g in td3_gemms_idx(376, 17, 101, 8192, e, pidx, cidx)}
    assert on["pol.fwd0"] and on["pol.dw0"] and on["q1.fwd0"] and on["q1.dw0"] and not on["q1.dx0_actions"]
    on = {g.name: A.on_tensor_engine(g) for g in td3_gemms_idx(376, 17, 101, 8192, "policy", *_sets(376, 24, 300, 0))}
    assert not on["pol.fwd0"] and not on["pol.dw0"] and on["q1.fwd0"]
    on = {g.name: A.on_tensor_engine(g) for g in td3_gemms_idx(64, 64, 101, 1024, "policy", *_sets(64, 48, 60, 0))}
    assert on["q1.dx0_actions"] and on["pol.fwd0"] and not on["pol.dw0"]   # N = P = 48 < 64


# ------------------------------------------------------------------------------------------------------------ device side
@pytest.fixture
def lib():
    from rl_x_b200 import _native as nt
    lib = nt.load()
    try:
        yield lib
    finally:
        lib.rlx_set_aux_gemm_engine(0)


CASES = [
    # obs, act, atoms, n, clipped, P, C
    (376, 17, 101, 8192, 1, 188, 376),   # the bench shape: P on the grid, C + act = 393 off it; eight weight-gradient splits
    (376, 17, 101, 2500, 1, 190, 303),   # ragged last split; P off the grid (pitch 192), C + act = 320 on it (action block at column 303)
    (376, 17, 101, 1024, 0, 188, 300),   # one split; the mean of the two values
    (376, 17, 101, 1024, 1, 24, 200),    # P < 32: the policy's layer 1 on SIMT
    (64, 64, 101, 4099, 1, 48, 60),      # act 64, C + act = 124, last split of 3 rows
]


@gpu
@pytest.mark.parametrize("obs,act,atoms,n,clipped,P,Cc", CASES)
def test_updates_vs_float64_on_both_engines(lib, obs, act, atoms, n, clipped, P, Cc):
    pidx, cidx = _sets(obs, P, Cc, obs + n)
    algo = algo_with(pidx, cidx)
    nets = X.reference_init(obs, act, atoms, 3, pidx, cidx)
    cb, pb = make_batches(algo, nets, obs, act, n, 11, clipped, DEV)
    refs = {w: A.oracle_update(algo, nets, w, b, clipped, DEV) for w, b in (("critic", cb), ("policy", pb))}
    report, simt = [], {}
    for engine in (0, 1):
        for which, b in (("critic", cb), ("policy", pb)):
            dev = _Device(algo, lib, obs, act, atoms, n, nets, clipped)
            metrics, _ = A._counted(lib, engine, algo.gemms(obs, act, atoms, n, which), lambda: dev.update(which, b))
            floor = A._floor(algo.gemms, obs, act, atoms, n, which)
            label = f"fasttd3 sets ({obs}, {act}, {atoms}, {n}, P {P}, C {Cc}) {which} engine {engine}"
            d = A._check_update(algo, dev, refs[which], which, metrics, label, report, simt.get(which) if engine else None, floor)
            if engine == 0:
                simt[which] = d
    print("\n" + "\n".join(report))


@gpu
@pytest.mark.parametrize("n", [63, 64, 4097])
def test_acting_vs_float64_on_both_engines(lib, n):
    from rl_x_b200 import _native as nt
    obs, act, atoms = 376, 17, 101
    pidx, cidx = _sets(obs, 188, 376, 1)
    pol = X.reference_init(obs, act, atoms, 6, pidx, cidx)[0]
    g = torch.Generator().manual_seed(n)
    pol = [(w + 0.05 * torch.randn(w.shape, generator=g), b + 0.05 * torch.randn(b.shape, generator=g)) for w, b in pol]
    x, noise, scales = torch.randn(n, obs, generator=g), torch.randn(n, act, generator=g), torch.rand(n, 1, generator=g) * 0.4 + 0.001
    dd = lambda t: t.to(DEV, torch.float64)
    with torch.no_grad():
        ref = X.act([(dd(w), dd(b)) for w, b in pol], dd(x), dd(noise), dd(scales), policy_idx=pidx)[0].cpu()
    P = A._t(np.concatenate([t.numpy().reshape(-1) for t in TD.leaves(pol)]))
    dx, dn, ds = A._t(x), A._t(noise), A._t(scales)
    d, keep = _dims(nt, obs, act, atoms, pidx, cidx)
    nbytes = lib.rlx_fasttd3_workspace_bytes(C.byref(d), n)
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for engine in (0, 1):
        action = torch.full((n, act), float("nan"), device=DEV)
        ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
        run = lambda: nt.check(lib.rlx_fasttd3_act_f32(C.byref(d), P.data_ptr(), dx.data_ptr(), dn.data_ptr(), ds.data_ptr(), None, None, 0, n,
                                                       action.data_ptr(), None, ws.data_ptr(), nbytes, st()), "rlx_fasttd3_act_f32")
        A._counted(lib, engine, td3_gemms_idx(obs, act, atoms, n, "act", pidx, cidx), run)
        got = action.cpu().double()
        assert torch.isfinite(got).all()
        np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=1e-5, atol=1e-5, err_msg=f"engine {engine}")
        assert float((got - ref).norm() / ref.norm()) <= 5e-6, (engine, float((got - ref).norm() / ref.norm()))


@gpu
@pytest.mark.parametrize("obs,engine", [(376, 0), (375, 0), (376, 1)])
def test_arange_sets_give_the_bits_of_null_sets(lib, obs, engine):
    """Explicit arange(obs) sets against NULL ones: critic, policy, critic updates and acting leave the same bits in every buffer."""
    from rl_x_b200 import _native as nt
    act, atoms, n = 17, 101, 2048
    nets = TD.reference_init(obs, act, atoms, 2)
    ar = np.arange(obs)
    b = A._draw(A.Td3, obs, act, n, 7)
    runs = []
    assert lib.rlx_set_aux_gemm_engine(engine) == engine
    for sets in ((None, None), (ar, ar)):
        dev = _Device(algo_with(*sets), lib, obs, act, atoms, n, nets, True)
        ms = [dev.update(w, b) for w in ("critic", "policy", "critic")]
        d, keep = _dims(nt, obs, act, atoms, *sets)
        action = torch.full((n, act), float("nan"), device=DEV)
        nt.check(lib.rlx_fasttd3_act_f32(C.byref(d), dev.P.data_ptr(), A._t(b["states"]).data_ptr(), None, None, None, None, 0, n, action.data_ptr(),
                                         None, dev.ws.data_ptr(), dev.nbytes, C.c_void_p(torch.cuda.current_stream().cuda_stream)), "act")
        torch.cuda.synchronize()
        runs.append([t.cpu() for t in (dev.P, dev.Q, dev.QT, dev.mP, dev.vP, dev.mQ, dev.vQ, action)] + [torch.from_numpy(m) for m in ms])
    for i, (x, y) in enumerate(zip(*runs)):
        assert torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0)), i


@gpu
@pytest.mark.parametrize("engine", ["simt", "tcgen05"])
def test_plugin_trains_with_index_sets_saves_loads_and_continues(tmp_path, engine):
    """fasttd3.b200 on synthetic.box with an asymmetric pair of sets: a few environment steps, save, load, and a few more."""
    from rl_x_b200.config_dict import ConfigDict
    from rl_x_b200.algorithms.fasttd3.b200.default_config import get_config
    from rl_x_b200.algorithms.fasttd3.b200.fasttd3 import FastTD3
    from rl_x_b200.environments.synthetic.box.create_env import create_train_and_eval_env
    from rl_x_b200.environments.synthetic.box.default_config import get_config as env_config
    N, obs, act = 32, 24, 6
    pidx, cidx = _sets(obs, 13, 20, 3)
    e = env_config("synthetic.box")
    e.nr_envs, e.obs_dim, e.act_dim, e.horizon, e.seed = N, obs, act, 8, 5
    a = get_config("fasttd3.b200")
    a.batch_size, a.buffer_size_per_env, a.learning_starts, a.total_timesteps, a.n_steps = 128, 16, 2, N * 6, 3
    a.logging_frequency, a.save_frequency, a.action_clipping_and_rescaling, a.gemm_engine = N, N, True, engine
    cfg = ConfigDict(algorithm=a, environment=e, runner=ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False, load_model=""))

    def envs():
        tr, ev = create_train_and_eval_env(cfg)
        for env in (tr, ev):
            env.policy_observation_indices, env.critic_observation_indices = pidx, cidx
        return tr, ev

    try:
        model = FastTD3(cfg, *envs(), str(tmp_path / "run"), None)
        assert model.dims.policy_in_dim == 13 and model.dims.critic_in_dim == 20
        logged = []
        model.log = lambda name, value, step: logged.append((name, float(value)))
        model.train()
        q = [v for n_, v in logged if n_ == "loss/q_loss"]
        assert len(q) == 4 and all(np.isfinite(q))
        assert all(np.isfinite(v) for n_, v in logged if not n_.startswith("time/"))
        model.save()
        path = tmp_path / "run" / "models" / "latest.model"
        ck = torch.load(path, weights_only=False)
        assert ck["policy_state_dict"]["policy.0.weight"].shape == (512, 13) and ck["q1_state_dict"]["critic.0.weight"].shape == (1024, 26)
        cfg.runner.load_model, cfg.runner.save_model = str(path), False
        again = FastTD3.load(cfg, *envs(), str(tmp_path / "run2"), None, [])
        for name in ("policy_params", "q_params", "q_target_params", "policy_m", "q_v", "steps", "norm_mean"):
            assert torch.equal(getattr(model, name), getattr(again, name)), name
        logged2 = []
        again.log = lambda name, value, step: logged2.append((name, float(value)))
        again.train()
        assert all(np.isfinite(v) for n_, v in logged2 if not n_.startswith("time/"))
        assert int(again.steps[0]) > int(model.steps[0])
    finally:
        from rl_x_b200 import _native as nt
        nt.load().rlx_set_aux_gemm_engine(0)
