"""FastSAC n-step replay sampling kernel (rlx_replay_sample_nstep_f32) against the executed reference (tests/golden/fastsac_replay.npz)
and against oracle/fastsac_replay_oracle.py on a large random ring."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAMES = ["states", "next_states", "actions", "rewards", "dones", "truncations", "effective_n_steps"]


def _buffer(ring, cap, nr_envs, obs, act, n_steps, gamma, size, pos):
    from rl_x_b200.algorithms.fastsac.b200.replay_buffer import ReplayBuffer
    buf = ReplayBuffer(cap, nr_envs, (obs,), (act,), n_steps, gamma, DEV)
    for k in ["states", "next_states", "actions", "rewards", "dones", "truncations"]:
        getattr(buf, k).copy_(torch.from_numpy(np.ascontiguousarray(ring[k])))
    buf.size, buf.pos = size, pos
    return buf


def test_nstep_sample_matches_reference_golden():
    import os
    from conftest import GOLDEN_DIR
    z = np.load(os.path.join(GOLDEN_DIR, "fastsac_replay.npz"))
    for tag in [str(c) for c in z["cases"]]:
        cap, nr_envs, obs, act, n_steps, size, pos, ns = (int(x) for x in z[f"{tag}/meta"])
        ring = {k: z[f"{tag}/ring/{k}"] for k in NAMES[:6]}
        buf = _buffer(ring, cap, nr_envs, obs, act, n_steps, 0.0, size, pos)
        buf.discounts.copy_(torch.from_numpy(z[f"{tag}/discounts"]))
        got = buf.gather(torch.from_numpy(z[f"{tag}/idx_t"]).to(DEV), torch.from_numpy(z[f"{tag}/idx_e"]).to(DEV))
        for name, v in zip(NAMES, got):
            ref = z[f"{tag}/out/{name}"]
            if name == "rewards":
                np.testing.assert_allclose(v.cpu().numpy(), ref, rtol=3e-7, atol=3e-7, err_msg=f"{tag}/{name}")
            else:
                assert np.array_equal(v.cpu().numpy(), ref), f"{tag}/{name}"


@pytest.mark.parametrize("n_steps", [1, 3, 8, 32])
def test_nstep_sample_matches_oracle_large_ring(n_steps):
    """BASELINE-sized observation rows (obs 48, act 12), 1024 x 256 ring, full and wrapped: bit-exact against the oracle's explicit loops
    (same (r * mask) * discount products, summed in step order)."""
    from oracle import fastsac_replay_oracle as F
    cap, nr_envs, obs, act, gamma = 1024, 256, 48, 12, 0.97
    g = np.random.default_rng(n_steps)
    ring = {"states": g.standard_normal((cap, nr_envs, obs), dtype=np.float32), "next_states": g.standard_normal((cap, nr_envs, obs), dtype=np.float32),
            "actions": g.standard_normal((cap, nr_envs, act), dtype=np.float32), "rewards": g.standard_normal((cap, nr_envs), dtype=np.float32),
            "dones": (g.random((cap, nr_envs)) < 0.05).astype(np.float32), "truncations": (g.random((cap, nr_envs)) < 0.03).astype(np.float32)}
    size, pos = cap, 700
    buf = _buffer(ring, cap, nr_envs, obs, act, n_steps, gamma, size, pos)
    n = 4096
    idx_t = np.concatenate([g.integers(0, cap, n - 64), np.arange(pos - 32, pos + 32) % cap]).astype(np.int64)  # incl. windows over the newest row
    idx_e = g.integers(0, nr_envs, n).astype(np.int64)
    got = buf.gather(torch.from_numpy(idx_t).to(DEV), torch.from_numpy(idx_e).to(DEV))
    want = F.sample(ring, idx_t, idx_e, n_steps, buf.discounts.cpu().numpy(), size, pos)
    for name, v, w in zip(NAMES, got, want):
        assert np.array_equal(v.cpu().numpy(), w), name
    # the public call draws its own indices: shapes, ranges and the effective-n identity
    s, ns, a, r, d, t, eff = buf.sample(512)
    assert s.shape == (512, obs) and a.shape == (512, act) and r.shape == (512,)
    assert float(eff.min()) >= 1.0 and float(eff.max()) <= n_steps
