#!/usr/bin/env python
"""Golden vectors of the FastTD3 update on an env with observation index sets, made by EXECUTING the unmodified reference
(rl_x/algorithms/fasttd3/pytorch) on CPU, fp32.

The reference's FastTD3 index-selects its networks' inputs with the env's `policy_observation_indices` / `critic_observation_indices`
(policy.py:12,26,30,52, q_network.py:10,22,24,39): the policy's layer 1 has len(policy indices) inputs, the Q networks' len(critic
indices) + act.  This run gives the synthetic TORCH env of make_golden_fasttd3.py an asymmetric pair of sets, the shape of the reference's
robot environments: the policy reads 7 shuffled columns of a 12-wide observation, the critic 10 shuffled columns that overlap the policy's
and include columns the policy never sees.  The replay buffer and the observation normaliser stay full-width, as in the reference.
Build container only:

    TORCHDYNAMO_DISABLE=1 python tests/golden/make_golden_fasttd3_obs_indices.py

Output: tests/golden/fasttd3_obs_indices.npz, in the capture format of make_golden_fasttd3.py (fasttd3_update.npz) plus the two index
arrays `policy_idx` / `critic_idx`.
"""
import os
import sys

os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402

import make_golden_fasttd3 as G  # noqa: E402  (imports the reference)

OBS, ACT = 12, 3
_perm = np.random.default_rng(77)
POLICY_IDX = _perm.permutation(OBS)[:7].astype(np.int64)
CRITIC_IDX = _perm.permutation(OBS)[:10].astype(np.int64)
assert len(set(POLICY_IDX) & set(CRITIC_IDX)) > 0 and len(set(CRITIC_IDX) - set(POLICY_IDX)) > 0


class IndexedSyntheticTorchEnv(G.SyntheticTorchEnv):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.policy_observation_indices = POLICY_IDX.copy()
        self.critic_observation_indices = CRITIC_IDX.copy()


def main():
    G.SyntheticTorchEnv = IndexedSyntheticTorchEnv   # run() builds its env from this name
    G.run("obs_indices", obs=OBS, act=ACT, seed=9, steps=7)   # 4 optimising steps
    path = os.path.join(HERE, "fasttd3_obs_indices.npz")
    z = dict(np.load(path))
    assert z["final/policy/policy.0.weight"].size == 512 * len(POLICY_IDX) // G.STRIDE + 1
    z["policy_idx"], z["critic_idx"] = POLICY_IDX, CRITIC_IDX
    np.savez_compressed(path, **z)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
