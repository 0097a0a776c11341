#!/usr/bin/env python
"""Generate the PPO golden vectors of an env with observation index sets by EXECUTING the unmodified reference (RL-X @ /root/reference).

The reference's PPO index-selects its networks' inputs with the env's `policy_observation_indices` / `critic_observation_indices`
(rl_x/algorithms/ppo/pytorch/policy.py:14,36-37,62, critic.py:10,26-27,45): layer 1 of the policy has len(policy indices) inputs, the
critic's len(critic indices).  This run gives the synthetic TORCH env of make_golden_ppo.py an asymmetric pair of index sets, the shape
of the reference's robot environments: the policy reads 23 shuffled columns of a 40-wide observation, the critic 33 shuffled columns
that overlap the policy's and include columns the policy never sees.  Build container only:

    python tests/golden/make_golden_ppo_obs_indices.py

Outputs:
  * tests/golden/ppo_obs_indices.npz: the `ppo_<tag>.npz` layout of make_golden_ppo.py (read by tests/conftest.py's Golden) plus the
    two index arrays `policy_idx` / `critic_idx`; one iteration (8 Adam steps: 2 epochs x 4 minibatches) and no Adam moments, which keeps
    the fixture small (hidden 128, the smallest width the wgmma engine takes, makes every weight snapshot ~150 KB compressed),
  * tests/golden/ppo_obs_indices_ref_checkpoint.model: the `best.model` the reference's own PPO.save() (ppo.py:426-436) writes at the end
    of the same run: the final weights AND both Adam states, so the moments are pinned by this file.  Its pickled config tree is
    rl_x_b200.config_dict.ConfigDict, so the file unpickles wherever this repository is importable.
"""
import os
import shutil
import sys

os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_ppo as G  # noqa: E402  (installs the ml_collections stub and imports the reference)
from rl_x_b200.config_dict import ConfigDict  # noqa: E402

# config trees the reference builds (get_config looks the class up on the stub module at call time) are this repository's class
sys.modules["ml_collections.config_dict"].ConfigDict = ConfigDict
G.ConfigDict = ConfigDict

OBS, ACT, HID = 40, 4, 128
N, T, MB, E, ITERS, SEED = 16, 16, 64, 2, 1, 5
ACT_LOW, ACT_HIGH, STD_DEV, ENTROPY_COEF = -1.5, 1.0, 0.8, 0.005
_perm = np.random.default_rng(2024)
POLICY_IDX = _perm.permutation(OBS)[:23].astype(np.int64)
CRITIC_IDX = _perm.permutation(OBS)[:33].astype(np.int64)
assert len(set(POLICY_IDX) & set(CRITIC_IDX)) > 0 and len(set(CRITIC_IDX) - set(POLICY_IDX)) > 0


class IndexedSyntheticTorchEnv(G.SyntheticTorchEnv):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.policy_observation_indices = POLICY_IDX.copy()
        self.critic_observation_indices = CRITIC_IDX.copy()


def save_reference_checkpoint():
    """The same run again with save_model=True, then the reference's own save()."""
    torch.set_num_threads(1)
    a = G.get_config("ppo.pytorch")
    a.device, a.bf16_mixed_precision_training = "cpu", False
    a.nr_steps, a.minibatch_size, a.nr_epochs, a.nr_hidden_units = T, MB, E, HID
    a.total_timesteps = N * T * ITERS
    a.std_dev, a.entropy_coef = STD_DEV, ENTROPY_COEF
    cfg = ConfigDict(algorithm=a, environment=ConfigDict(seed=SEED, nr_envs=N),
                     runner=ConfigDict(save_model=True, track_console=False, track_tb=False, track_wandb=False))
    env = IndexedSyntheticTorchEnv(N, OBS, ACT, seed=SEED + 1000, act_low=ACT_LOW, act_high=ACT_HIGH)
    run_path = "/tmp/rlx_golden_obs_indices_ckpt"
    shutil.rmtree(run_path, ignore_errors=True)
    model = G.refppo.PPO(cfg, env, env, run_path, None)
    model.log = lambda *a_, **k_: None
    model.start_logging = model.end_logging = lambda *a_, **k_: None
    model.train()
    model.save()
    dst = os.path.join(HERE, "ppo_obs_indices_ref_checkpoint.model")
    shutil.copyfile(os.path.join(run_path, "models", "best.model"), dst)
    ck = torch.load(dst, weights_only=False)
    print("wrote", dst, os.path.getsize(dst), "bytes; policy.0.weight", tuple(ck["policy_state_dict"]["policy_mean.0.weight"].shape),
          "critic.0.weight", tuple(ck["critic_state_dict"]["critic.0.weight"].shape))


def main():
    G.SyntheticTorchEnv = IndexedSyntheticTorchEnv  # run() builds its env from this name
    G.run("obs_indices", N=N, T=T, obs_dim=OBS, act_dim=ACT, hidden=HID, mb=MB, epochs=E, iterations=ITERS, seed=SEED,
          act_low=ACT_LOW, act_high=ACT_HIGH, std_dev=STD_DEV, entropy_coef=ENTROPY_COEF, keep_moments=False)
    path = os.path.join(HERE, "ppo_obs_indices.npz")
    z = dict(np.load(path))
    z["policy_idx"], z["critic_idx"] = POLICY_IDX, CRITIC_IDX
    np.savez_compressed(path, **z)
    save_reference_checkpoint()


if __name__ == "__main__":
    main()
